"""The search as production runs it, against the oracle and against itself.

  * per-bin model subsets (ckm_search_per_bin, CheckM's lineage_wf): every bin of one batch has its own query list --
    overlapping, disjoint, unsorted, all models, only the long ones, none, a one-ORF bin -- over a database that mixes
    the 43 CPR models with models of M = 1,100 (chunked kernels), 2,500 (a chained SSV tile) and 3,300 (no SSV tile: the
    bypass kernel).  Each bin's rows must be the oracle's rows of that bin searched alone with its own list (Z = its ORFs),
    and the bytes of that bin searched alone on the device;
  * envelope rescoring in many waves: a scratch budget of 1 MiB (CKM_ENV_SCRATCH_MB) cuts the envelopes into about one
    wave each -- offsets reset per wave, device arrays addressed at the wave's start, the scratch buffer regrown between
    waves, the last wave handed to the trace ensemble, both orders of ensemble and envelopes (CKM_ENS_FIRST).  The rows
    must be the bytes of the single-wave run;
  * two engines in flight on one device, sharing one model database, as MarkerGeneFinder and bench.py run them: every
    result must be the bytes the session engine returns for the same batch searched alone."""
import os
import threading

import numpy as np
import pytest

import bench
from conftest import CPR_HMM
from test_search_gpu import compare
from test_text_parity_gpu import CASES, _both_tables, _compare
from tools import synth

pytestmark = pytest.mark.gpu

NCPR = 43
LONG_M = (1100, 2500, 3300)        # database indices 43, 44, 45
CKM_EINVAL = 1


def _keys(rows, hits):
    ko = [(r['model'], r['seqidx'], r['dom'], r['ndom'], r['hmm_from'], r['hmm_to'], r['ali_from'], r['ali_to'], r['env_from'], r['env_to'])
          for r in rows]
    kg = [tuple(int(h[f]) for f in ('model', 'seq', 'dom', 'ndom', 'hmm_from', 'hmm_to', 'ali_from', 'ali_to', 'env_from', 'env_to'))
          for h in hits]
    return ko, kg


def _compare_long(rows, hits):
    """The chunked kernels (M > 1024) against the oracle: the tolerance of test_search_gpu.compare plus 2e-5 bits per
    residue of the target.  The null2 bias correction is a sum over every residue of the envelope of a score derived from
    fp32 posteriors; its rounding grows with the envelope's length, which 1e-4 * |bias| does not follow.  Measured: a
    3,300-position model on a 3,613-residue target (envelope of 3,399 residues) -- Forward score equal to 2e-4 bits, bias
    66.138 (oracle) vs 66.172 bits (device)."""
    worst = 0.0
    for r, h in zip(rows, hits):
        slack = 1e-3 + 1e-5 * abs(float(r['full_score'])) + 1e-4 * abs(float(r['full_bias'])) + 2e-5 * int(r['tlen'])
        for a, b in ((r['full_score'], h['full_score']), (r['dom_score'], h['dom_score']), (r['full_bias'], h['full_bias']), (r['dom_bias'], h['dom_bias'])):
            d = abs(float(np.float32(a)) - float(b))
            worst = max(worst, d / slack)
            assert d <= slack, (r, h)
        assert abs(float(np.float32(r['acc'])) - float(h['acc'])) <= 1e-3
        for a, b in ((r['full_E'], h['full_evalue']), (r['c_E'], h['c_evalue']), (r['i_E'], h['i_evalue'])):
            assert abs(np.log(max(a, 1e-300)) - np.log(max(float(b), 1e-300))) <= 1e-12 + slack * 1.5, (a, b)
    return worst


def _compare_mixed(rows, hits):
    """Row order and coordinates exactly; floats bit for bit for the CPR models (M <= 1024), within the chunked kernels'
    tolerance for the long ones.  Returns (exact rows, chunked rows, worst chunked difference as a fraction of its slack)."""
    ko, kg = _keys(rows, hits)
    assert ko == kg, [(a, b) for a, b in zip(ko, kg) if a != b][:10] or (len(ko), len(kg))
    parts = {True: [], False: []}
    for r, h in zip(rows, hits):
        parts[r['model'] < NCPR].append((r, h))
    worst = 0.0
    if parts[True]:
        compare([r for r, _ in parts[True]], np.array([h for _, h in parts[True]], dtype=hits.dtype), exact=True)
    if parts[False]:
        worst = _compare_long([r for r, _ in parts[False]], [h for _, h in parts[False]])
    return len(parts[True]), len(parts[False]), worst


def _batch(parts):
    """(residues, offsets) of every bin -> one batch: residues, offsets, bin of every ORF, first ORF of every bin."""
    res = np.concatenate([r for r, _ in parts])
    lens = np.concatenate([np.diff(o) for _, o in parts])
    off = np.zeros(len(lens) + 1, np.int64)
    off[1:] = np.cumsum(lens)
    nseq = [len(o) - 1 for _, o in parts]
    binof = np.repeat(np.arange(len(parts), dtype=np.int32), nseq)
    first = np.concatenate([[0], np.cumsum(nseq)]).astype(np.int64)
    return res, off, binof, first


def _bin_rows(hits, b, first):
    sub = hits[hits['bin'] == b].copy()
    sub['seq'] -= int(first[b])
    sub['bin'] = 0
    return sub


@pytest.fixture(scope='module')
def mixed(engine, oracle, tmp_path_factory):
    """The 43 CPR models followed by synthetic models of M = 1,100, 2,500 and 3,300, as one file."""
    d = tmp_path_factory.mktemp('mixed')
    syn, path = str(d / 'long.hmm'), str(d / 'mixed.hmm')
    synth.make_model_db(syn, CPR_HMM, LONG_M, seed=51)
    with open(path, 'w') as out:
        out.write(open(CPR_HMM).read().rstrip('\n') + '\n')
        out.write(open(syn).read())
    models = engine.load_models(path)
    assert models.n == NCPR + len(LONG_M)
    assert [mi.M for mi in models.info()[NCPR:]] == list(LONG_M)
    yield models, oracle.HmmFile(path), synth.read_hmms(path)
    models.close()


@pytest.fixture(scope='module')
def engine2():
    """A second engine on the same device, alive for this module (CKM_PIPELINE=2 runs two)."""
    from checkm_b200.engine import Engine
    e = Engine(0)
    yield e
    e.close()


# ---------------------------------------------------------------------------------------------------------------------
# 1. per-bin model subsets

def _per_bin_inputs(hm):
    rng = np.random.default_rng(61)
    lists = [[44, 5, 17, 0, 43, 30, 12],                        # unsorted; chained SSV tile and chunked model
             [17, 45, 3, 5, 22, 41, 44, 36],                    # overlaps the first on 5, 17, 44; bypass-kernel model
             [40, 1, 2, 4, 6, 7, 8, 9, 10, 11],                 # disjoint from both
             [int(i) for i in rng.permutation(len(hm))],        # every model, shuffled
             [45, 43, 44],                                      # only the long models
             [],                                                # none: the bin must return no rows
             [44, 5, 0, 12]]                                    # a one-ORF bin
    parts = []
    for i in range(len(lists) - 1):
        # every bin carries homologs of every model, so a model left out of a bin's list would show up in its rows
        b = synth.make_bin('pb%d' % i, hm, seed=600 + i, n_orfs=120, copies=(0, 1, 1), max_len=1200, split_prob=0.0, tandem_prob=0.1)
        parts.append((b.residues, b.offsets))
    one = synth.make_bin('pb1orf', [hm[5]], seed=700, n_orfs=8, copies=(1,), split_prob=0.0)
    o = one.planted[0][1]
    parts.append((one.residues[one.offsets[o]:one.offsets[o + 1]], np.array([0, one.offsets[o + 1] - one.offsets[o]], np.int64)))
    return lists, parts


def test_per_bin_subsets_match_oracle_and_solo(engine, mixed, oracle):
    models, ohf, hm = mixed
    lists, parts = _per_bin_inputs(hm)
    res, off, binof, first = _batch(parts)
    db = engine.seqdb(res, off, binof, len(parts))
    midx = np.concatenate([np.asarray(l, np.int32) for l in lists])
    boff = np.concatenate([[0], np.cumsum([len(l) for l in lists])]).astype(np.int64)
    hits = engine.search(models, db, model_idx=midx, bin_model_offsets=boff)
    st = engine.stats()
    db.close()
    assert st.n_pairs == sum((len(o) - 1) * len(l) for (_, o), l in zip(parts, lists))
    assert np.all(np.diff(hits['bin']) >= 0)
    report = []
    for b, (idx, (r_b, o_b)) in enumerate(zip(lists, parts)):
        sub = _bin_rows(hits, b, first)
        if not idx:
            assert len(sub) == 0
            report.append((b, 0, 0, 0.0))
            continue
        assert set(int(m) for m in sub['model']) <= set(idx)
        # the oracle: this bin alone, its own list (rows in list order, Z = its ORFs, domZ per model)
        rp = oracle.search(ohf, r_b, o_b, nthreads=os.cpu_count() or 8, models=idx)
        rows = oracle.hits_table(rp)
        oracle.free_results(rp)
        for r in rows:
            r['model'] = idx[r['model']]
        report.append((b,) + _compare_mixed(rows, sub))
        # the device: this bin alone through ckm_search with the same list
        sdb = engine.seqdb(r_b, o_b)
        solo = engine.search(models, sdb, model_idx=idx)
        sdb.close()
        assert solo.tobytes() == sub.tobytes(), b
    print('per-bin subsets: (bin, exact rows, chunked rows, worst chunked difference / slack) =', report)
    assert sum(x[1] for x in report) >= 100
    assert sum(x[2] for x in report) >= 5
    assert report[-1][1] + report[-1][2] >= 1            # the one-ORF bin has its planted homolog


def test_per_bin_duplicate_model_is_refused(engine, mixed):
    """A model listed twice in one bin's list is refused like a duplicate in ckm_search's list (CKM_EINVAL); the engine
    keeps working."""
    from checkm_b200._lib import CkmError
    models, _, hm = mixed
    b = synth.make_bin('dup', hm[:8], seed=71, n_orfs=30)
    res, off, binof, _ = _batch([(b.residues, b.offsets), (b.residues, b.offsets)])
    db = engine.seqdb(res, off, binof, 2)
    with pytest.raises(CkmError, match='duplicate model index in the query list of bin 1') as ex:
        engine.search(models, db, model_idx=np.array([3, 7, 1, 2, 1], np.int32), bin_model_offsets=np.array([0, 2, 5], np.int64))
    assert ex.value.code == CKM_EINVAL
    with pytest.raises(CkmError, match='duplicate') as ex:
        engine.search(models, db, model_idx=[3, 7, 3])
    assert ex.value.code == CKM_EINVAL
    hits = engine.search(models, db, model_idx=np.array([3, 7, 1, 2], np.int32), bin_model_offsets=np.array([0, 2, 4], np.int64))
    db.close()
    assert len(hits) > 0


# ---------------------------------------------------------------------------------------------------------------------
# 2. envelope rescoring in waves

def _vq(M):
    for q, lim in zip((2, 4, 6, 8, 12, 16, 20, 24, 28, 32), (64, 128, 192, 256, 384, 512, 640, 768, 896, 1024)):
        if M <= lim:
            return q
    return 0


def _env_need(M, Ld, blk):
    """Floats of rescoring scratch one envelope of Ld residues needs (search.cu envelope_need): one matrix of 32*Q columns
    for the lane-blocked kernels, two of the padded model width for the chunked ones, plus the special states."""
    vq = _vq(M) if blk else 0
    width = 32 * vq if vq else ((M + 1) + 31) // 32 * 32 + 32
    return (1 if vq else 2) * (Ld + 1) * 3 * width + (Ld + 1) * 15 + 64


def _repeat_bin(hm):
    """The repeat protein of test_search_gpu.test_region_with_more_domains_than_slots (150 domains, domain phase repeated)."""
    fam = min(hm, key=lambda h: h.M)
    rng = np.random.default_rng(103)
    repeats = np.concatenate([synth.emit_homolog(fam, rng, k_from=int(rng.integers(20, 25)), k_to=int(rng.integers(45, 50)), sharpen=0.6)
                              for _ in range(150)])
    b = synth.make_bin('r', hm, seed=78, n_orfs=120, max_len=900)
    order = list(range(15)) + [None] + list(range(15, 30))
    seqs = [repeats if i is None else b.seq(i) for i in order]
    offsets = np.concatenate([[0], np.cumsum([len(s) for s in seqs])]).astype(np.int64)
    names = ['r_%d' % k for k in range(len(seqs))]
    return synth.Bin('repeat', np.concatenate(seqs), offsets, names, ['# 1 # 3 # 1 # ID=%d_1' % k for k in range(len(seqs))], [])


def _wave_inputs(hm):
    cases = {tag: (seed, kw) for tag, seed, kw in CASES}
    out = [synth.make_bin(tag, hm, seed=cases[tag][0], **cases[tag][1]) for tag in ('tandem', 'sharp')]
    return out + [_repeat_bin(hm)]


def _search_bytes(engine, models, b, **kw):
    db = engine.seqdb(b.residues, b.offsets)
    hits = engine.search(models, db, **kw)
    st = engine.stats()
    db.close()
    return hits, st


@pytest.mark.parametrize('which', ['tandem', 'sharp', 'repeat'])
def test_envelope_waves_equal_single_wave_and_oracle(engine, cpr_models, cpr_oracle, oracle, tmp_path, monkeypatch, which):
    hm = synth.read_hmms(CPR_HMM)
    b = {x.bin_id: x for x in _wave_inputs(hm)}[which]
    monkeypatch.delenv('CKM_ENV_SCRATCH_MB', raising=False)
    monkeypatch.delenv('CKM_ENS_FIRST', raising=False)
    g, o, ref, rows = _both_tables(engine, cpr_models, cpr_oracle, oracle, b, tmp_path, which)
    assert len(g) >= 20
    assert not _compare(g, o, ref, rows, which, [])
    st0 = engine.stats()
    launches = {}
    for mb in (None, '1', '64'):
        for ens in (None, '0', '1'):
            for k, v in (('CKM_ENV_SCRATCH_MB', mb), ('CKM_ENS_FIRST', ens)):
                if v is None:
                    monkeypatch.delenv(k, raising=False)
                else:
                    monkeypatch.setenv(k, v)
            hits, st = _search_bytes(engine, cpr_models, b)
            assert hits.tobytes() == ref.tobytes(), (which, mb, ens)
            assert st.n_queue_retries == st0.n_queue_retries and st.n_domains == st0.n_domains
            launches[(mb, ens)] = st.kernel_launches
    # the chunked kernels (two matrices per envelope): 1 MiB against their own single-wave run
    monkeypatch.delenv('CKM_ENS_FIRST', raising=False)
    monkeypatch.setenv('CKM_BLK', '0')
    monkeypatch.delenv('CKM_ENV_SCRATCH_MB', raising=False)
    blk0, _ = _search_bytes(engine, cpr_models, b)
    monkeypatch.setenv('CKM_ENV_SCRATCH_MB', '1')
    blk0_waves, st = _search_bytes(engine, cpr_models, b)
    assert blk0_waves.tobytes() == blk0.tobytes()
    print('%s: %d rows; %d domains, domain phase repeated %d times; kernel launches by (MiB, CKM_ENS_FIRST): %s; CKM_BLK=0 at 1 MiB: %d'
          % (which, len(ref), st0.n_domains, st0.n_queue_retries, launches, st.kernel_launches))


@pytest.mark.parametrize('blk', ['1', '0'])
def test_envelope_waves_are_really_split(engine, cpr_models, monkeypatch, blk):
    """40 ORFs, each one full homolog of the longest CPR model (one class of envelope kernel), searched with that model
    alone.  At 1 MiB every wave holds at most max(1 MiB, the largest envelope) of scratch, which the longest ORF bounds;
    so the envelopes the rows report need at least ceil(sum of their needs / that bound) waves, each with its own launch,
    where the single-wave run launches that class at most twice (single-domain and multi-domain envelopes)."""
    hm = synth.read_hmms(CPR_HMM)
    m = int(np.argmax([h.M for h in hm]))
    M = hm[m].M
    rng = np.random.default_rng(91)
    seqs = [np.concatenate([rng.choice(20, size=int(rng.integers(0, 20)), p=synth.BG), synth.emit_homolog(hm[m], rng, sharpen=0.5),
                            rng.choice(20, size=int(rng.integers(0, 20)), p=synth.BG)]).astype(np.uint8) for _ in range(40)]
    res = np.concatenate(seqs)
    off = np.concatenate([[0], np.cumsum([len(s) for s in seqs])]).astype(np.int64)
    b = synth.Bin('fam', res, off, [], [], [])
    monkeypatch.setenv('CKM_BLK', blk)
    monkeypatch.delenv('CKM_ENV_SCRATCH_MB', raising=False)
    one, st1 = _search_bytes(engine, cpr_models, b, model_idx=[m])
    monkeypatch.setenv('CKM_ENV_SCRATCH_MB', '1')
    many, stn = _search_bytes(engine, cpr_models, b, model_idx=[m])
    assert many.tobytes() == one.tobytes()
    assert len(one) >= 35
    use_blk = blk == '1'
    bound = max((1 << 20) // 4, _env_need(M, int(np.diff(off).max()), use_blk))
    need = sum(_env_need(M, int(h['env_to']) - int(h['env_from']) + 1, use_blk) for h in one)
    waves = -(-need // bound)
    extra = stn.kernel_launches - st1.kernel_launches
    print('CKM_BLK=%s, M=%d: %d rows need %d floats of scratch; wave bound %d floats -> at least %d waves; kernel launches %d '
          '(unset) vs %d (1 MiB): %d extra' % (blk, M, len(one), need, bound, waves, st1.kernel_launches, stn.kernel_launches, extra))
    assert waves >= 20
    assert extra >= waves - 2


# ---------------------------------------------------------------------------------------------------------------------
# 3. two engines in flight

def _concurrently(jobs):
    """Runs the callables on their own threads, released together by a barrier; returns their results in order."""
    barrier = threading.Barrier(len(jobs))
    out, errs = [None] * len(jobs), []

    def run(i, fn):
        try:
            barrier.wait(timeout=120)
            out[i] = fn()
        except BaseException as ex:          # noqa: B902 -- re-raised on the calling thread
            errs.append(ex)
    ts = [threading.Thread(target=run, args=(i, fn), daemon=True) for i, fn in enumerate(jobs)]
    for t in ts:
        t.start()
    for t in ts:
        t.join(timeout=900)
    assert not any(t.is_alive() for t in ts), 'a search thread did not finish'
    if errs:
        raise errs[0]
    return out


class _Batch(object):
    def __init__(self, bins, lists=None):
        self.res, self.off, self.binof, self.first = _batch([(b.residues, b.offsets) for b in bins])
        self.nbins = len(bins)
        self.lists = lists

    def seqdb(self, eng):
        return eng.seqdb(self.res, self.off, self.binof, self.nbins)

    def per_bin(self):
        return (np.concatenate([np.asarray(l, np.int32) for l in self.lists]),
                np.concatenate([[0], np.cumsum([len(l) for l in self.lists])]).astype(np.int64))


def test_two_engines_concurrently_equal_one_serially(engine, engine2, cpr_models, mixed, monkeypatch):
    mixed_models = mixed[0]
    hm = synth.read_hmms(CPR_HMM)
    bins = {tag: synth.make_bin(tag, hm, seed=seed, **kw) for tag, seed, kw in CASES}
    X = _Batch([bins['single'], bins['tandem']], lists=[[44, 5, 17, 0, 43, 30], [45, 3, 22, 44]])
    Y = _Batch([bins['split'], bins['sharp'], bins['degenerate']], lists=[[1, 2, 44], [], [40, 41, 42, 43, 36, 12]])
    dbs = {(id(eng), id(bt)): bt.seqdb(eng) for eng in (engine, engine2) for bt in (X, Y)}
    calls = {'whole database': lambda eng, bt, db: eng.search(cpr_models, db),
             'model_idx': lambda eng, bt, db: eng.search(cpr_models, db, model_idx=[5, 0, 17, 42, 9, 30, 21, 2]),
             'per-bin lists': lambda eng, bt, db: eng.search(mixed_models, db, model_idx=bt.per_bin()[0], bin_model_offsets=bt.per_bin()[1])}
    monkeypatch.delenv('CKM_ENV_SCRATCH_MB', raising=False)
    monkeypatch.delenv('CKM_ENS_FIRST', raising=False)
    serial = {(kind, id(bt)): fn(engine, bt, dbs[(id(engine), id(bt))]) for kind, fn in calls.items() for bt in (X, Y)}
    for (kind, _), h in serial.items():
        assert len(h) > 0, kind
    rounds = [('whole database', None), ('model_idx', None), ('per-bin lists', None), ('whole database', '1'), ('per-bin lists', '1'),
              ('model_idx', None)]
    compared = 0
    for r, (kind, mb) in enumerate(rounds):
        if mb is None:
            monkeypatch.delenv('CKM_ENV_SCRATCH_MB', raising=False)
        else:
            monkeypatch.setenv('CKM_ENV_SCRATCH_MB', mb)           # set before the threads start: both engines run in waves
        a, b = (X, Y) if r % 2 == 0 else (Y, X)                    # the session engine takes X in even rounds, Y in odd ones
        fn = calls[kind]
        got = _concurrently([lambda: fn(engine, a, dbs[(id(engine), id(a))]), lambda: fn(engine2, b, dbs[(id(engine2), id(b))])])
        for bt, h in zip((a, b), got):
            want = serial[(kind, id(bt))]
            assert h.tobytes() == want.tobytes(), (r, kind, mb, len(h), len(want))
            compared += len(h)
    monkeypatch.delenv('CKM_ENV_SCRATCH_MB', raising=False)
    for db in dbs.values():
        db.close()
    print('two engines: %d rounds, %d rows compared byte for byte with the serial searches' % (len(rounds), compared))


def test_two_engines_production_shape(engine, engine2, monkeypatch):
    """bench.py's shape: the 5,000-model database (the 43 CPR models repeated under new names), 2 bins of 2,900 ORFs per
    engine, the default scratch budget.  Also the replica invariant of test_fullsize_gpu: every replica of a base model
    reports the rows of the original."""
    monkeypatch.delenv('CKM_ENV_SCRATCH_MB', raising=False)
    monkeypatch.delenv('CKM_ENS_FIRST', raising=False)
    models = engine.load_models(bench.model_db(bench.N_MODELS))
    hm = synth.read_hmms(bench.CPR)
    A = _Batch([synth.make_bin('pa%d' % i, hm, seed=4300 + i, n_orfs=bench.CFG[3]['orfs']) for i in range(2)])
    B = _Batch([synth.make_bin('pb%d' % i, hm, seed=4310 + i, n_orfs=bench.CFG[3]['orfs']) for i in range(2)])
    try:
        serial = []
        for bt in (A, B):
            db = bt.seqdb(engine)
            serial.append(engine.search(models, db))
            db.close()
        da, db_ = A.seqdb(engine), B.seqdb(engine2)
        got = _concurrently([lambda: engine.search(models, da), lambda: engine2.search(models, db_)])
        da.close()
        db_.close()
        fields = [f for f in serial[0].dtype.names if f != 'model']
        for h, want in zip(got, serial):
            assert len(h) > 2000
            assert h.tobytes() == want.tobytes()
            # model index = replica * 43 + base model (bench.model_db writes the 43 models round after round)
            per = {}
            for row in h:
                per.setdefault((int(row['bin']), int(row['model'])), []).append(tuple(row[f].item() for f in fields))
            groups = 0
            for bi in range(2):
                for mb in range(NCPR):
                    for mi in range(mb + NCPR, models.n, NCPR):
                        assert per.get((bi, mi), []) == per.get((bi, mb), []), (bi, mb, mi)
                        groups += 1
            assert groups > 9000
        print('production shape: %d + %d rows compared byte for byte; replica groups identical' % (len(got[0]), len(got[1])))
    finally:
        models.close()
