"""Strain heterogeneity on the GPU: ckm_align_groups behind HmmerAligner, ckm_aai_pairs behind AminoAcidIdentity.

Bars: every group's states and scores equal the oracle's and `Engine.align` on that group alone; the files of each
HmmerAligner method, the -a file, the AAI scores and the QA tables equal what the REFERENCE's own code made of the same
fixture (tests/golden/make_aai_goldens.py, tests/golden/aai/expected.json); aai() equals the reference's bit for bit."""
import io
import json
import os
import shutil
from contextlib import redirect_stdout

import numpy as np
import pytest

from conftest import CPR_HMM, GOLDEN
from tools import synth

pytestmark = pytest.mark.gpu
AAI = os.path.join(GOLDEN, 'aai')
BIN_IDS = ['strainA', 'strainB', 'strainC']


@pytest.fixture(scope='module')
def expected():
    with open(os.path.join(AAI, 'expected.json')) as f:
        return json.load(f)


@pytest.fixture()
def sorted_listdir(monkeypatch):
    """Bins and files in sorted order, as the goldens were recorded (the reference takes os.listdir's order)."""
    real = os.listdir
    monkeypatch.setattr(os, 'listdir', lambda p='.': sorted(real(p)))


@pytest.fixture()
def dataroot():
    from checkm_b200.defaultValues import DefaultValues
    saved = DefaultValues.CHECKM_DATA_DIR
    DefaultValues.set_data_root(os.path.join(GOLDEN, 'reduction', 'data'))
    yield
    DefaultValues.set_data_root(saved)


def _tree(root):
    out = {}
    for d, _, files in os.walk(root):
        for f in files:
            out[os.path.relpath(os.path.join(d, f), root)] = open(os.path.join(d, f)).read()
    return out


def _setup(tmp_path, with_tables=True):
    out = str(tmp_path / 'out')
    os.makedirs(os.path.join(out, 'storage', 'aai_qa'))
    if with_tables:
        for b in BIN_IDS:
            bdir = os.path.join(out, 'bins', b)
            os.makedirs(bdir)
            shutil.copyfile(os.path.join(AAI, 'bins', b + '.faa'), os.path.join(bdir, 'genes.faa'))
            shutil.copyfile(os.path.join(AAI, 'bins', b + '.hmmer.analyze.txt'), os.path.join(bdir, 'hmmer.analyze.txt'))
    return out


def _models_and_sets(out):
    from checkm_b200.hmmerModelParser import HmmModelParser
    from checkm_b200.markerSets import MarkerSetParser
    models = HmmModelParser(CPR_HMM).models()
    return {b: models for b in BIN_IDS}, MarkerSetParser(1).getMarkerSets(out, BIN_IDS, CPR_HMM)


def test_align_groups_match_oracle_and_align(engine, cpr_models, cpr_oracle, oracle):
    hm = synth.read_hmms(CPR_HMM)
    rng = np.random.default_rng(31)
    bg = lambda n: rng.choice(20, size=n, p=synth.BG).astype(np.uint8)      # noqa: E731
    group_model, groups = [], []
    for m in (0, 6, 17, 18, 30, 2):                 # M = 86 ... 863: several lane-block classes
        h = hm[m]
        seqs = [synth.emit_homolog(h, rng), np.concatenate([bg(33), synth.emit_homolog(h, rng), [27]]),
                synth.emit_homolog(h, rng, k_from=h.M // 3, k_to=2 * h.M // 3), bg(90),
                np.concatenate([synth.emit_homolog(h, rng), synth.emit_homolog(h, rng)]), np.zeros(0, np.uint8)]
        group_model.append(m)
        groups.append([np.asarray(s, np.uint8) for s in seqs])
    group_model.insert(3, 5)
    groups.insert(3, [])                              # a group without sequences
    seqs = [s for g in groups for s in g]
    off = np.zeros(len(seqs) + 1, np.int64)
    off[1:] = np.cumsum([len(s) for s in seqs])
    goff = np.zeros(len(groups) + 1, np.int64)
    goff[1:] = np.cumsum([len(g) for g in groups])
    db = engine.seqdb(np.concatenate(seqs), off)
    state, oasc = engine.align_groups(cpr_models, db, group_model, goff)
    db.close()
    for g, m in enumerate(group_model):
        gs = groups[g]
        if not gs:
            continue
        o = np.zeros(len(gs) + 1, np.int64)
        o[1:] = np.cumsum([len(s) for s in gs])
        gdb = engine.seqdb(np.concatenate(gs), o)
        st1, sc1 = engine.align(cpr_models, gdb, m)
        gdb.close()
        r0, r1 = off[goff[g]], off[goff[g + 1]]
        assert np.array_equal(state[r0:r1], st1), (g, m)
        assert np.array_equal(oasc[goff[g]:goff[g + 1]].view(np.int32), sc1.view(np.int32)), (g, m)
        for i, s in enumerate(gs):
            exp, sc, rc = oracle.align(cpr_oracle, m, s)
            k = goff[g] + i
            assert np.array_equal(state[off[k]:off[k + 1]], exp), (m, i)
            assert np.float32(sc) == oasc[k], (m, i, sc, oasc[k])


def test_align_groups_refusals(engine, cpr_models):
    from checkm_b200._lib import CkmError
    db = engine.seqdb(np.zeros(10, np.uint8), np.array([0, 4, 10], np.int64))
    try:
        for gm, go in (([0], [0, 3]), ([0, 1], [0, 2, 1]), ([99], [0, 2]), ([-1], [0, 1])):
            with pytest.raises(CkmError) as e:
                engine.align_groups(cpr_models, db, gm, go)
            assert e.value.code == 1
    finally:
        db.close()


@pytest.mark.parametrize('method', ['multi', 'tophit', 'phylo'])
def test_hmmer_aligner_files(method, expected, tmp_path, sorted_listdir, dataroot):
    from checkm_b200.defaultValues import DefaultValues
    from checkm_b200.hmmerAligner import HmmerAligner
    out = _setup(tmp_path)
    binIdToModels, bms = _models_and_sets(out)
    HA = HmmerAligner(4)
    dest = str(tmp_path / method)
    if method == 'multi':
        HA.makeAlignmentsOfMultipleHits(out, CPR_HMM, 'hmmer.analyze.txt', binIdToModels, bms, False, DefaultValues.E_VAL,
                                        DefaultValues.LENGTH, dest)
    elif method == 'tophit':
        rp = HA.makeAlignmentTopHit(out, CPR_HMM, 'hmmer.analyze.txt', binIdToModels, False, DefaultValues.E_VAL,
                                    DefaultValues.LENGTH, True, dest, True)
        assert {b: [[m, [h.target_name for h in hits]] for m, hits in rp.results[b].markerHits.items()] for b in BIN_IDS} \
            == expected['extract']['tophit_sorted']
    else:
        HA.makeAlignmentToPhyloMarkers(out, CPR_HMM, 'hmmer.analyze.txt', binIdToModels, False, DefaultValues.E_VAL,
                                       DefaultValues.LENGTH, True, dest)
    got, want = _tree(dest), expected[method + '_files']
    assert sorted(got) == sorted(want)
    for k in want:
        assert got[k] == want[k], (method, k)


def test_analyze_then_qa_in_one_process(expected, tmp_path, monkeypatch, sorted_listdir, dataroot):
    """find -> multi-copy alignments -> AAI -> QA tables, in one process that has CUDA initialised: nothing may fork."""
    import multiprocessing
    from checkm_b200.aminoAcidIdentity import AminoAcidIdentity
    from checkm_b200.defaultValues import DefaultValues
    from checkm_b200.hmmerAligner import HmmerAligner
    from checkm_b200.markerGeneFinder import MarkerGeneFinder
    from checkm_b200.resultsParser import ResultsParser

    def no_fork(*a, **k):
        raise AssertionError('a process was started after CUDA was initialised')
    monkeypatch.setattr(multiprocessing, 'Process', no_fork)
    out = _setup(tmp_path, with_tables=False)
    binFiles = [os.path.join(AAI, 'bins', b + '.faa') for b in BIN_IDS]
    binIdToModels = MarkerGeneFinder(1).find(binFiles, out, 'hmmer.analyze.txt', 'hmmer.analyze.ali.txt', CPR_HMM, False, False, True)
    from checkm_b200.markerSets import MarkerSetParser
    bms = MarkerSetParser(1).getMarkerSets(out, BIN_IDS, CPR_HMM)
    HmmerAligner(8).makeAlignmentsOfMultipleHits(out, CPR_HMM, 'hmmer.analyze.txt', binIdToModels, bms, False,
                                                 DefaultValues.E_VAL, DefaultValues.LENGTH, os.path.join(out, 'storage', 'aai_qa'))
    assert _tree(os.path.join(out, 'storage', 'aai_qa')) == expected['multi_files']
    with open(os.path.join(out, 'storage', 'bin_stats.analyze.tsv'), 'w') as f:
        f.write(''.join(l + '\n' for l in expected['bin_stats']))
    RP = ResultsParser(binIdToModels)
    RP.analyseResults(out, 'bin_stats.analyze.tsv', 'hmmer.analyze.txt')
    for thr, e in expected['aai'].items():
        aai = AminoAcidIdentity()
        afile = str(tmp_path / ('aai_%s.txt' % thr))
        aai.run(float(thr), out, afile)
        assert open(afile).read() == e['alignment_file']
        assert {b: {m: [repr(v) for v in vs] for m, vs in ms.items()} for b, ms in aai.aaiRawScores.items()} == e['raw']
        assert {b: {m: repr(v) for m, v in ms.items()} for b, ms in aai.aaiHetero.items()} == e['hetero']
        assert {b: repr(v) for b, v in aai.aaiMeanBinHetero.items()} == e['mean']
        assert any(float(v) > 0 for v in e['mean'].values())
        for key, want in e['tables'].items():
            buf = io.StringIO()
            with redirect_stdout(buf):
                RP.printSummary(int(key[0]), aai, bms, False, None, key[1] == 't', '', out)
            assert buf.getvalue() == want, (thr, key)


def test_aai_known_answers(expected, engine):
    from checkm_b200.aminoAcidIdentity import AminoAcidIdentity
    aai = AminoAcidIdentity()
    for a, b, want in expected['aai_vectors']:
        assert repr(aai.aai(a, b)) == want, (a, b)
    # all vectors in one call, rows in mixed order and offsets that are not multiples of 16
    rows = [r for a, b, _ in expected['aai_vectors'] for r in (b, a)]
    off = np.zeros(len(rows) + 1, np.int64)
    off[1:] = np.cumsum([len(r) for r in rows])
    pairs = np.array([(2 * i + 1, 2 * i) for i in range(len(rows) // 2)], np.int32)
    mis, ln = engine.aai_pairs(''.join(rows).encode(), off, pairs)
    for (a, b, want), m, n in zip(expected['aai_vectors'], mis.tolist(), ln.tolist()):
        assert repr(0.0 if n == 0 else 1.0 - (float(m) / n)) == want, (a, b)


def test_aai_pairs_random_rows(engine):
    """Wide rows with gap runs at both ends against a restatement of the reference's loop."""
    rng = np.random.default_rng(7)
    rows, pairs = [], []
    for w in (1, 2, 15, 16, 17, 511, 512, 513, 1500):
        for _ in range(6):
            r = np.frombuffer(rng.choice(list(b'ACDE-'), size=w, p=[0.2, 0.2, 0.2, 0.1, 0.3]).astype(np.uint8).tobytes(), np.uint8).copy()
            r[:int(rng.integers(0, w + 1)) // 3] = ord('-')
            rows.append(r.tobytes().decode())
        pairs += [(len(rows) - 6 + i, len(rows) - 6 + j) for i in range(6) for j in range(i + 1, 6)]
    off = np.zeros(len(rows) + 1, np.int64)
    off[1:] = np.cumsum([len(r) for r in rows])
    mis, ln = engine.aai_pairs(''.join(rows).encode(), off, np.array(pairs, np.int32))
    for (i, j), m, n in zip(pairs, mis.tolist(), ln.tolist()):
        a, b = rows[i], rows[j]
        s = 0
        for c in range(len(a)):
            if a[c] == '-' or b[c] == '-':
                s = c + 1
            else:
                break
        e = len(a)
        for c in range(len(a) - 1, 0, -1):
            if a[c] == '-' or b[c] == '-':
                e = c
            else:
                break
        wm = sum(1 for c in range(s, e) if a[c] != b[c])
        wl = wm + sum(1 for c in range(s, e) if a[c] == b[c] and a[c] != '-')
        assert (m, n) == (wm, wl), (i, j)


def test_aai_unequal_widths_refused(engine):
    from checkm_b200._lib import CkmError
    with pytest.raises(CkmError) as e:
        engine.aai_pairs(b'ACGTACG', np.array([0, 4, 7], np.int64), np.array([[0, 1]], np.int32))
    assert e.value.code == 1 and 'unequal width' in str(e.value)
