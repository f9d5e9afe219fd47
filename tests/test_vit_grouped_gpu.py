"""Packed ViterbiFilter on the survivor list grouped by (class, model) (launch_vit_group + vitp_kernel, kernels_vitp.cu):
scores bit-identical to the int32 kernels (CKM_VITP=0 / int32_only) and to the oracle's orc_vitfilter, for a model whose
pairs span many chunks, one model of every class, a model without a class, pairs the redo list must take (int16 ceiling,
outside C1'), per-bin query subsets and a search whose queues overflow and are re-run."""
import numpy as np
import pytest

from tools import synth
from conftest import CPR_HMM

pytestmark = pytest.mark.gpu

CHUNK = 64                     # VITP_CHUNK (stages.hpp)
# one model per class W = 1, 2, 3, 4, 6, 8, 10, 12, 14, 16, and one beyond the classes (M > 1024)
CLASS_M = [40, 100, 150, 200, 300, 450, 600, 700, 850, 1000, 1100]


def _same(a, b):
    return a == b or (np.isinf(a) and np.isinf(b) and np.sign(a) == np.sign(b))


def _pack(seqs):
    off = np.zeros(len(seqs) + 1, np.int64)
    off[1:] = np.cumsum([len(s) for s in seqs])
    return np.concatenate(seqs).astype(np.uint8), off


def _packed_vs_int32(engine, models, res, off, model_idx=None):
    db = engine.seqdb(res, off)
    vp = engine.viterbi_scores(models, db, model_idx=model_idx)
    n_redo = engine.stats().n_vit_redo
    v32 = engine.viterbi_scores(models, db, model_idx=model_idx, int32_only=True)
    db.close()
    assert vp.tobytes() == v32.tobytes(), np.argwhere(vp != v32)[:5]
    return vp, n_redo


@pytest.fixture(scope='module')
def class_db(engine, oracle, tmp_path_factory):
    p = str(tmp_path_factory.mktemp('vitgrp') / 'classes.hmm')
    hm = synth.make_model_db(p, CPR_HMM, CLASS_M, seed=13)
    models = engine.load_models(p)
    yield hm, models, oracle.HmmFile(p)
    models.close()


def test_every_class_and_model_without_class(engine, class_db, oracle):
    hm, models, ohf = class_db
    rng = np.random.default_rng(31)
    seqs = [rng.choice(20, size=int(L), p=synth.BG) for L in synth.random_lengths(rng, 120, hi=1500)]
    seqs += [rng.choice(20, size=L, p=synth.BG) for L in (0, 1, 5, 17, 64)]
    for h in hm:                                               # full homologs reach the int16 ceiling; partial ones do not
        seqs.append(synth.emit_homolog(h, rng))
        k0 = int(rng.integers(1, h.M // 2))
        seqs.append(synth.emit_homolog(h, rng, k_from=k0, k_to=min(h.M, k0 + h.M // 3)))
    seqs.append(rng.choice(20, size=20000, p=synth.BG))       # outside C1' for the long models: the int32 kernels take it
    res, off = _pack([np.asarray(s, np.uint8) for s in seqs])
    vp, n_redo = _packed_vs_int32(engine, models, res, off)
    assert (vp == np.inf).any()
    assert n_redo >= len(seqs)                                 # at least every pair of the model without a class
    pairs = [(a, s) for a in range(models.n) for s in range(len(seqs))]
    pick = np.random.default_rng(3).choice(len(pairs), size=min(len(pairs), 2500), replace=False)
    for a, s in [pairs[i] for i in pick] + [(models.n - 1, len(seqs) - 1), (9, len(seqs) - 1)]:
        exp = np.float32(oracle.vitfilter(ohf, a, res[off[s]:off[s + 1]]))
        assert _same(vp[a, s], exp), (CLASS_M[a], s, off[s + 1] - off[s], vp[a, s], exp)


def test_model_with_many_chunks(engine, cpr_models, cpr_oracle, oracle):
    """One model against 11 chunks' worth of ORFs (the last one partial), alone and in a reversed query list with two
    other models; every pair against the oracle."""
    hm = synth.read_hmms(CPR_HMM)
    m = 7
    rng = np.random.default_rng(32)
    n = 10 * CHUNK + 17
    seqs = [synth.emit_homolog(hm[m], rng) if i % 9 == 0 else rng.choice(20, size=int(rng.integers(1, 900)), p=synth.BG)
            for i in range(n)]
    res, off = _pack([np.asarray(s, np.uint8) for s in seqs])
    vp, _ = _packed_vs_int32(engine, cpr_models, res, off, model_idx=[m])
    for s in range(n):
        exp = np.float32(oracle.vitfilter(cpr_oracle, m, res[off[s]:off[s + 1]]))
        assert _same(vp[0, s], exp), (s, vp[0, s], exp)
    vr, _ = _packed_vs_int32(engine, cpr_models, res, off, model_idx=[30, m, 2])
    assert vr[1].tobytes() == vp[0].tobytes()


def _search(engine, models, res, off, monkeypatch, vitp, **kw):
    monkeypatch.setenv('CKM_VITP', vitp)
    binof, nbins, dense = kw.pop('binof', None), kw.pop('nbins', 1), kw.pop('dense', False)
    db = engine.seqdb(res, off, binof, nbins)
    hits = engine.search(models, db, **kw)
    st = engine.stats()
    fs = engine.filter_scores(models, db) if dense else None
    db.close()
    return hits, st, fs


def test_search_dense_scores_and_per_bin_subsets(engine, cpr_models, monkeypatch):
    """Dense Viterbi scores and pass bits of ckm_filter_scores and the rows of ckm_search_per_bin: packed kernels against
    CKM_VITP=0."""
    hm = synth.read_hmms(CPR_HMM)
    parts = [synth.make_bin('vg%d' % i, hm, seed=800 + i, n_orfs=150, max_len=1200, tandem_prob=0.1) for i in range(3)]
    res = np.concatenate([b.residues for b in parts])
    off = np.concatenate([[0]] + [b.offsets[1:] + sum(len(q.residues) for q in parts[:i]) for i, b in enumerate(parts)]).astype(np.int64)
    binof = np.concatenate([np.full(b.nseq, i, np.int32) for i, b in enumerate(parts)])
    h1, st1, fs1 = _search(engine, cpr_models, res, off, monkeypatch, '1', dense=True)
    h0, st0, fs0 = _search(engine, cpr_models, res, off, monkeypatch, '0', dense=True)
    assert st1.n_vit_redo > 0 and st0.n_vit_redo == 0
    assert st1.n_past_vit == st0.n_past_vit
    assert h1.tobytes() == h0.tobytes()
    for a, b in zip(fs1, fs0):
        assert a.tobytes() == b.tobytes()
    lists = [[7, 0, 42, 13], list(range(43))[::-1], [5]]
    midx = np.concatenate([np.asarray(l, np.int32) for l in lists])
    boff = np.concatenate([[0], np.cumsum([len(l) for l in lists])]).astype(np.int64)
    kw = dict(binof=binof, nbins=3, model_idx=midx, bin_model_offsets=boff)
    p1, _, _ = _search(engine, cpr_models, res, off, monkeypatch, '1', **dict(kw))
    p0, _, _ = _search(engine, cpr_models, res, off, monkeypatch, '0', **dict(kw))
    assert len(p1) > 0 and p1.tobytes() == p0.tobytes()


def test_queue_overflow_retry(engine, cpr_models, monkeypatch):
    """Every ORF carries homologs of the three queried models: the queues overflow, the cascade is re-run with larger ones,
    and the grouped work list is rebuilt for the larger survivor list."""
    hm = synth.read_hmms(CPR_HMM)
    rng = np.random.default_rng(33)
    idx = [0, 1, 2]
    distinct = [np.concatenate(sum([[synth.emit_homolog(hm[m], rng, sharpen=0.6), rng.choice(20, size=12, p=synth.BG).astype(np.uint8)]
                                    for m in idx], []) + [np.array([27], np.uint8)]) for _ in range(200)]
    n = 40000
    res, off = _pack([distinct[i % 200] for i in range(n)])
    h1, st1, _ = _search(engine, cpr_models, res, off, monkeypatch, '1', model_idx=idx)
    h0, st0, _ = _search(engine, cpr_models, res, off, monkeypatch, '0', model_idx=idx)
    assert st1.n_queue_retries >= 1 and st1.n_past_fwd == 3 * n
    assert h1.tobytes() == h0.tobytes()
