"""`checkm merge` on the device (checkm_b200.merger.Merger over ckm_merge_pairs, csrc/merge.cu):
merger.tsv byte for byte against the reference's own Merger (tests/golden/merge/, made by
tests/golden/make_merge_goldens.py, whose inputs are laid out as a CheckM output directory here), the production path from gene calls to merger.tsv, and the pair records against a
numpy restatement at scale, at the capacity limit and at the edges."""
import ctypes as C
import json
import os
import shutil

import numpy as np
import pytest

from conftest import CPR_HMM, GOLDEN

pytestmark = pytest.mark.gpu
MG = os.path.join(GOLDEN, 'merge')
E2E = os.path.join(GOLDEN, 'e2e')
BINFILES = [os.path.join(E2E, 'bins', f) for f in ('binA.faa', 'binB.faa.gz', 'binC.faa')]
TABLE = 'merger.table.txt'
DEFAULT = (5.0, 10.0, 50.0, 20.0)
PERMISSIVE = (-1e9, 1e9, -1e9, 1e9)


@pytest.fixture(scope='module')
def golden():
    with open(os.path.join(MG, 'merge_goldens.json')) as f:
        return json.load(f)


@pytest.fixture(scope='module')
def dataroot(tmp_path_factory, engine):
    """A CheckM data root in miniature: the e2e Pfam clan file and hmms/checkm.hmm = the CPR fixture."""
    from checkm_b200.defaultValues import DefaultValues
    root = str(tmp_path_factory.mktemp('checkm_data'))
    shutil.copytree(os.path.join(E2E, 'data'), root, dirs_exist_ok=True)
    os.makedirs(os.path.join(root, 'hmms'))
    shutil.copyfile(CPR_HMM, os.path.join(root, 'hmms', 'checkm.hmm'))
    saved = DefaultValues.CHECKM_DATA_DIR
    DefaultValues.set_data_root(root)
    yield root
    DefaultValues.set_data_root(saved)


def _marker_file(which):
    return {'hmm': CPR_HMM, 'taxon': os.path.join(E2E, 'markers', 'taxon.ms'), 'twosets': os.path.join(MG, 'twosets.ms')}[which]


def _e2e():
    with open(os.path.join(E2E, 'expected.json')) as f:
        return json.load(f)


def _layout(golden, case, out, bins=None):
    """<out>/bins/<id>/merger.table.txt for the case's bins; returns the bins' model dicts."""
    from checkm_b200.hmmerModelParser import HmmModelParser
    models = HmmModelParser(CPR_HMM).models()
    if case.startswith('e2e_'):
        e2e = _e2e()[case[4:]]
        tables = {b: ''.join(l + '\n' for l in lines) for b, lines in e2e['domtblout'].items()}
        subset = e2e['subset']
    else:
        tables, subset = golden['inputs'], None
    binIds = sorted(tables) if bins is None else bins
    for b in binIds:
        os.makedirs(os.path.join(out, 'bins', b))
        with open(os.path.join(out, 'bins', b, TABLE), 'w') as f:
            f.write(tables[b])
    os.makedirs(os.path.join(out, 'storage'), exist_ok=True)
    return {b: ({a: models[a] for a in subset[b]} if subset else models) for b in binIds}


def _run(golden, case, which, thr, tmp_path, bins=None):
    from checkm_b200.markerSets import MarkerSetParser
    from checkm_b200.merger import Merger
    out = str(tmp_path / ('%s_%s_%d' % (case, which, len(os.listdir(str(tmp_path))))))
    binIdToModels = _layout(golden, case, out, bins)
    ms = MarkerSetParser().getMarkerSets(out, list(binIdToModels), _marker_file(which))
    path = Merger().run([], out, TABLE, binIdToModels, ms, *thr)
    assert path == os.path.join(out, 'merger.tsv')
    return open(path).read()


def test_every_golden_byte_for_byte(golden, dataroot, tmp_path):
    n = 0
    for case, g in golden['cases'].items():
        for which, entry in g.items():
            for label, tsv in entry['tsv'].items():
                assert _run(golden, case, which, entry['thresholds'][label], tmp_path) == tsv, (case, which, label)
                n += 1
    assert n == 16


@pytest.mark.parametrize('mode', ['hmm', 'taxon'])
def test_production_path(mode, golden, dataroot, tmp_path):
    """Gene calls -> MarkerGeneFinder.find -> getMarkerSets -> Merger.run, as `checkm merge` runs it (main.py:805-841)."""
    from checkm_b200.markerGeneFinder import MarkerGeneFinder
    from checkm_b200.markerSets import MarkerSetParser
    from checkm_b200.merger import Merger
    out = str(tmp_path / 'out')
    for d in ('bins', 'storage', os.path.join('storage', 'hmms')):
        os.makedirs(os.path.join(out, d), exist_ok=True)
    mfile = _marker_file(mode)
    binIdToModels = MarkerGeneFinder(1).find(BINFILES, out, TABLE, 'merger.hmmer3', mfile, False, False, True)
    ms = MarkerSetParser().getMarkerSets(out, ['binA', 'binB', 'binC'], mfile)
    entry = golden['cases']['e2e_' + mode][mode]
    for label in ('default', 'permissive'):
        path = Merger().run(BINFILES, out, TABLE, binIdToModels, ms, *entry['thresholds'][label])
        assert open(path).read() == entry['tsv'][label], label


def restate(counts, n_markers, thr):
    """numpy restatement of the pair filter: (i, j, p, s) of every kept pair, i ascending then j."""
    pres = (counts > 0).astype(np.float64)
    x = pres @ pres.T
    p1 = pres.sum(1)
    s1 = counts.sum(1, dtype=np.int64).astype(np.float64)
    n = n_markers.astype(np.float64)
    comp1 = 100 * p1 / n
    cont1 = 100 * (s1 - p1) / n
    i, j = np.triu_indices(len(counts), 1)
    p = p1[i] + p1[j] - x[i, j]
    s = s1[i] + s1[j]
    comp = 100 * p / n[j]
    cont = 100 * (s - p) / n[j]
    dcomp = comp - np.maximum(comp1[i], comp1[j])
    dcont = cont - np.maximum(cont1[i], cont1[j])
    mdc, mxc, mmc, mxm = thr
    keep = (comp >= mmc) & (cont < mxm) & (dcomp >= mdc) & (dcont < mxc)
    return np.stack([i[keep], j[keep], p[keep].astype(np.int64), s[keep].astype(np.int64)], axis=1)


def _random_bins(rng, nb, ng):
    """Copy numbers: mostly 0 and 1, some small multi-copy counts, a few above 2^16; 2 % all-zero bins; each bin's
    completeness around a bin-specific level so that some pairs are complementary."""
    level = rng.random(nb)[:, None]
    counts = (rng.random((nb, ng)) < level).astype(np.int32)
    counts += (rng.random((nb, ng)) < 0.02).astype(np.int32) * rng.integers(1, 4, size=(nb, ng), dtype=np.int32)
    big = rng.random((nb, ng)) < 2e-5
    counts[big] = rng.integers(1 << 16, 1 << 17, size=int(big.sum()), dtype=np.int32)
    counts[rng.random(nb) < 0.02] = 0
    n_markers = ng + rng.integers(0, 4, size=nb).astype(np.int32)
    return counts, n_markers


def _records(pairs):
    return np.stack([pairs['i'], pairs['j'], pairs['p'], pairs['s']], axis=1).astype(np.int64)


@pytest.mark.parametrize('ng', [104, 1001, 5000])
def test_scale_against_numpy(ng, engine):
    rng = np.random.default_rng(ng)
    nb = 3000
    counts, n_markers = _random_bins(rng, nb, ng)
    for thr in ((5.0, 10.0, 50.0, 20.0), (-5.0, 3.0, 60.0, 8.0)):
        pairs, ms = engine.merge_pairs(counts, n_markers, *thr)
        want = restate(counts, n_markers, thr)
        assert len(want) > 0
        np.testing.assert_array_equal(_records(pairs), want)
    pairs, _ = engine.merge_pairs(counts, n_markers, *PERMISSIVE)
    assert len(pairs) == nb * (nb - 1) // 2 == 4_498_500
    np.testing.assert_array_equal(_records(pairs), restate(counts, n_markers, PERMISSIVE))


def test_capacity(engine):
    from checkm_b200 import _lib
    from checkm_b200.engine import MERGE_PAIR_DTYPE
    rng = np.random.default_rng(5)
    counts, n_markers = _random_bins(rng, 700, 300)
    thr = (-5.0, 3.0, 60.0, 8.0)
    want = restate(counts, n_markers, thr)
    assert len(want) > 100
    out = np.zeros(100, dtype=MERGE_PAIR_DTYPE)
    need, ms = C.c_int64(), C.c_float()
    rc = _lib.lib().ckm_merge_pairs(engine._h, counts.ctypes.data, 700, 300, n_markers.ctypes.data, *thr, out.ctypes.data,
                                    100, C.byref(need), C.byref(ms))
    assert rc == 8 and need.value == len(want)                    # CKM_ECAPACITY with the count needed
    assert not out.view(np.int32).any()
    pairs, _ = engine.merge_pairs(counts, n_markers, *thr, capacity=100)
    np.testing.assert_array_equal(_records(pairs), want)


def test_bad_input_is_refused(engine):
    from checkm_b200._lib import CkmError
    counts = np.ones((4, 40), dtype=np.int32)
    with pytest.raises(CkmError):
        engine.merge_pairs(counts, np.array([40, 40, 0, 40]), *DEFAULT)        # a marker set without markers
    counts[2, 3] = -1
    with pytest.raises(CkmError):
        engine.merge_pairs(counts, np.full(4, 40), *DEFAULT)                  # a negative copy number


@pytest.mark.parametrize('nb,ng', [(1, 50), (2, 50), (2, 1), (65, 33), (130, 257), (191, 4097)])
def test_shapes_off_the_tile_grid(nb, ng, engine):
    rng = np.random.default_rng(nb * 10007 + ng)
    counts, n_markers = _random_bins(rng, nb, ng)
    for thr in (DEFAULT, (-5.0, 3.0, 60.0, 8.0), PERMISSIVE):
        pairs, _ = engine.merge_pairs(counts, n_markers, *thr)
        want = restate(counts, n_markers, thr) if nb > 1 else np.zeros((0, 4), np.int64)
        np.testing.assert_array_equal(_records(pairs), want)


def test_identical_bins(engine):
    counts = np.tile(np.random.default_rng(1).integers(0, 3, size=(1, 600), dtype=np.int32), (200, 1))
    n_markers = np.full(200, 600, dtype=np.int32)
    for thr in (PERMISSIVE, (0.0, 1e9, -1.0, 1e9), (0.1, 1e9, -1.0, 1e9)):
        pairs, _ = engine.merge_pairs(counts, n_markers, *thr)
        np.testing.assert_array_equal(_records(pairs), restate(counts, n_markers, thr))
    assert len(engine.merge_pairs(counts, n_markers, 0.0, 1e9, -1.0, 1e9)[0]) == 200 * 199 // 2   # delta 0 >= 0
    assert len(engine.merge_pairs(counts, n_markers, 0.1, 1e9, -1.0, 1e9)[0]) == 0


def test_one_and_two_bins_write_the_reference_rows(golden, dataroot, tmp_path):
    from checkm_b200.merger import HEADER
    assert _run(golden, 'synth', 'hmm', PERMISSIVE, tmp_path, bins=['half0']) == HEADER
    two = _run(golden, 'synth', 'hmm', PERMISSIVE, tmp_path, bins=['half0', 'half1']).splitlines(keepends=True)
    rows = [l for l in golden['cases']['synth']['hmm']['tsv']['permissive'].splitlines(keepends=True) if l.startswith('half0\thalf1\t')]
    assert two == [HEADER] + rows and len(rows) == 1


def test_marker_set_mismatch_exits_before_writing(golden, dataroot, tmp_path):
    from checkm_b200.markerSets import MarkerSetParser
    from checkm_b200.merger import Merger
    out = str(tmp_path / 'synth')
    binIdToModels = _layout(golden, 'synth', out, bins=['half0', 'half1'])
    ms = MarkerSetParser().getMarkerSets(out, ['half0'], _marker_file('hmm'))
    ms.update(MarkerSetParser().getMarkerSets(out, ['half1'], _marker_file('taxon')))
    with pytest.raises(SystemExit) as exc:
        Merger().run([], out, TABLE, binIdToModels, ms, *DEFAULT)
    assert exc.value.code == 1
    assert not os.path.exists(os.path.join(out, 'merger.tsv'))
