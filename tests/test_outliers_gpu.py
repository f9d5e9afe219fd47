"""`checkm outliers` on the device (checkm_b200.binTools.BinTools over ckm_outlier_scores, csrc/outliers.cu): the outlier
file byte for byte against the reference's own BinTools (tests/golden/outliers/, made by
tests/golden/make_outlier_goldens.py), every value of the device call bit for bit against the reference's numpy
arithmetic at scale and under more than one batch split, the dictionary-taking methods against the reference's arrays,
tetra -> outliers -> modify in miniature, and the inputs the reference crashes on."""
import gzip
import hashlib
import json
import logging
import os
import shutil

import numpy as np
import pytest

from conftest import GOLDEN

pytestmark = pytest.mark.gpu
OG = os.path.join(GOLDEN, 'outliers')
OUTDIR = os.path.join(OG, 'out')
PROFILE = None


@pytest.fixture(scope='module', autouse=True)
def profile_file(tmp_path_factory, expected):
    """The fixture's profile file, written from its FASTA files as the golden generator wrote it."""
    from oracle.outliers_oracle import profile_text
    global PROFILE
    PROFILE = str(tmp_path_factory.mktemp('outliers') / 'tetra.tsv')
    with open(PROFILE, 'w') as f:
        f.write(profile_text([os.path.join(OG, 'extra.fna')] + _bin_files(expected)))


@pytest.fixture(scope='module')
def expected():
    with open(os.path.join(OG, 'expected.json')) as f:
        return json.load(f)


@pytest.fixture(scope='module')
def dataroot(engine):
    """The synthetic distribution files as the data root's distributions/ directory."""
    from checkm_b200.defaultValues import DefaultValues
    saved = DefaultValues.CHECKM_DATA_DIR
    DefaultValues.set_data_root(os.path.join(OG, 'data'))
    yield os.path.join(OG, 'data')
    DefaultValues.set_data_root(saved)


def _bin_files(expected):
    return [os.path.join(OG, 'bins', f) for f in expected['bins']]


def _u64(a):
    return np.ascontiguousarray(a, dtype=np.float64).view(np.uint64)


@pytest.mark.parametrize('report', ['any', 'all'])
@pytest.mark.parametrize('distribution', [90, 95, 99, 85])
def test_outlier_file_is_the_references(expected, dataroot, tmp_path, report, distribution):
    from checkm_b200.binTools import BinTools
    out = str(tmp_path / 'outliers.tsv')
    BinTools(threads=2).identifyOutliers(OUTDIR, _bin_files(expected), PROFILE, distribution, report, out)
    assert open(out).read() == expected['outliers']['%s_%d' % (report, distribution)]


def test_outlier_file_does_not_depend_on_the_batching(expected, dataroot, tmp_path, monkeypatch):
    from checkm_b200 import binTools
    monkeypatch.setattr(binTools, 'BATCH_BYTES', 4096)                   # a device call every bin or two
    out = str(tmp_path / 'outliers.tsv')
    binTools.BinTools().identifyOutliers(OUTDIR, _bin_files(expected), PROFILE, 95, 'any', out)
    assert open(out).read() == expected['outliers']['any_95']


def test_dictionary_methods_return_the_references_arrays(expected, dataroot):
    from checkm_b200.binStatistics import _GeneFeatures
    from checkm_b200.binTools import BinTools, readFasta
    from checkm_b200.genomicSignatures import GenomicSignatures
    bt = BinTools()
    gs = GenomicSignatures(4, 1)
    tetraSigs = gs.read(PROFILE)
    for path in _bin_files(expected):
        binId = os.path.basename(path).split('.')[0]
        if binId not in expected['helpers']:
            continue
        want = expected['helpers'][binId]
        seqs = readFasta(path)
        meanGC, deltaGCs, GCs = bt.gcDist(seqs)
        assert type(meanGC) is float and type(GCs) is list and deltaGCs.dtype == np.float64
        assert meanGC == want['meanGC'] and GCs == want['GCs'] and np.array_equal(_u64(deltaGCs), _u64(want['deltaGCs'])), binId
        meanCD, deltaCDs, CDs = bt.codingDensityDist(seqs, _GeneFeatures(os.path.join(OUTDIR, 'bins', binId, 'genes.gff')))
        assert meanCD == want['meanCD'] and CDs == want['CDs'] and np.array_equal(_u64(deltaCDs), _u64(want['deltaCDs'])), binId
        binSig = bt.binTetraSig(seqs, tetraSigs)
        assert binSig.shape == (136,) and np.array_equal(_u64(binSig), _u64(want['binSig'])), binId
        meanTD, deltaTDs = bt.tetraDiffDist(seqs, gs, tetraSigs, binSig)
        assert np.array_equal(_u64(deltaTDs), _u64(want['deltaTDs'])) and _u64([meanTD])[0] == _u64([want['meanTD']])[0], binId
    # the bin signature handed in is the one the distances are measured against
    seqs = readFasta(_bin_files(expected)[0])
    other = np.full(136, 1.0 / 136)
    _, deltaTDs = bt.tetraDiffDist(seqs, gs, tetraSigs, other)
    assert np.array_equal(_u64(deltaTDs), _u64([gs.distance(tetraSigs[s], other) for s in seqs]))


def _reference_scores(bin_off, lens, acgt, coding, rows, matrix):
    """binTools.py:148-209 with the reference's own numpy expressions, per bin."""
    means, sigs, vals = [], [], []
    for b in range(len(bin_off) - 1):
        lo, hi = int(bin_off[b]), int(bin_off[b + 1])
        gc = [float(int(c[1] + c[2])) / int(c.sum()) for c in acgt[lo:hi]]
        meanGC = float(int(acgt[lo:hi, 1:3].sum())) / int(acgt[lo:hi].sum())
        cd = [float(int(c)) / int(n) for c, n in zip(coding[lo:hi], lens[lo:hi])]
        meanCD = float(int(coding[lo:hi].sum())) / int(lens[lo:hi].sum())
        binSize = int(lens[lo:hi].sum())
        binSig = None
        for s in range(lo, hi):
            weighted = matrix[rows[s]] * (float(int(lens[s])) / binSize)
            if binSig is None:
                binSig = weighted
            else:
                binSig += weighted
        td = np.zeros(hi - lo)
        for i, s in enumerate(range(lo, hi)):
            td[i] = np.sum(np.abs(matrix[rows[s]] - binSig))
        means.append((meanGC, meanCD, np.mean(td)))
        sigs.append(binSig)
        vals.append(np.stack([gc, np.array(gc) - meanGC, cd, np.array(cd) - meanCD, td], axis=1))
    return np.array(means), np.array(sigs), np.concatenate(vals)


def test_scores_equal_numpys_bit_for_bit_at_scale(engine):
    """300 bins of 50,000 sequences plus one bin of 100,000, rows scattered over a larger profile matrix; one call, and the
    same bins in three calls."""
    rng = np.random.default_rng(2025)
    sizes = np.maximum(1, rng.multinomial(50000 - 300, rng.dirichlet(np.full(300, 0.7))) + 1)
    sizes[:4] = [1, 7, 128, 129]
    sizes = np.concatenate([sizes[:150], [100000], sizes[150:]])
    bin_off = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
    ns = int(bin_off[-1])
    lens = np.maximum(4, rng.lognormal(8.0, 1.2, ns)).astype(np.int64)
    frac = rng.dirichlet([3, 2, 2, 3], ns)
    acgt = np.floor(frac * (lens * 0.98)[:, None]).astype(np.int64)
    acgt[:, 0] += 1
    coding = (lens * rng.random(ns)).astype(np.int64)
    matrix = rng.dirichlet(np.full(136, 0.5), ns + 5000)
    matrix[rng.random(matrix.shape) < 0.05] = 0.0
    rows = rng.permutation(ns + 5000)[:ns].astype(np.int64)
    table_off = [0, 3, 5, 9]
    key = [1000, 500, 5000, 2000.5, 800, 500, 1000, 2000, 10000]
    tlo = [-0.05, -0.08, -0.02, -0.3, -0.4, 0, 0, 0, 0]
    thi = [0.05, 0.08, 0.02, 0, 0, 1.0, 0.9, 0.8, 0.7]
    nb = len(sizes)
    bin_gc, bin_cd = np.zeros(nb, dtype=np.int32), np.ones(nb, dtype=np.int32)
    sigs = engine.signatures(matrix)
    try:
        means, binsig, values, mask, ms = engine.outlier_scores(sigs, bin_off, lens, acgt, coding, rows, bin_gc, bin_cd, 2, table_off,
                                                                key, tlo, thi, want_binsig=True)
        pieces = []
        for lo, hi in ((0, 100), (100, 151), (151, nb)):
            a, z = int(bin_off[lo]), int(bin_off[hi])
            pieces.append(engine.outlier_scores(sigs, bin_off[lo:hi + 1] - a, lens[a:z], acgt[a:z], coding[a:z], rows[a:z],
                                                bin_gc[lo:hi], bin_cd[lo:hi], 2, table_off, key, tlo, thi, want_binsig=True))
    finally:
        sigs.close()
    for k, whole in enumerate((means, binsig, values, mask)):
        assert np.array_equal(np.concatenate([p[k] for p in pieces]).view(np.uint8), whole.view(np.uint8)), k
    wmeans, wsigs, wvals = _reference_scores(bin_off, lens, acgt, coding, rows, matrix)
    assert np.array_equal(_u64(binsig), _u64(wsigs))
    assert np.array_equal(_u64(values[:, :5]), _u64(wvals))
    assert np.array_equal(_u64(means), _u64(wmeans))
    # bounds and mask: the nearest length key, the first of two equally near ones
    karr, lo_arr, hi_arr = np.array(key, dtype=float), np.array(tlo, dtype=float), np.array(thi, dtype=float)

    def at(t, arr):
        sl = slice(table_off[t], table_off[t + 1])
        return arr[sl][np.argmin(np.abs(karr[sl][None, :] - lens[:, None]), axis=1)]
    want_bounds = np.stack([at(0, lo_arr), at(0, hi_arr), at(1, lo_arr), at(2, hi_arr)], axis=1)
    assert np.array_equal(values[:, 5:], want_bounds)
    want_mask = (((wvals[:, 1] < want_bounds[:, 0]) | (wvals[:, 1] > want_bounds[:, 1])) * 1 + (wvals[:, 3] < want_bounds[:, 2]) * 2 +
                 (wvals[:, 4] > want_bounds[:, 3]) * 4)
    assert np.array_equal(mask, want_mask.astype(np.uint8)) and len(set(mask.tolist())) > 4
    assert all(m > 0 for m in ms)


def test_scores_equal_the_oracle_on_the_golden_bins(expected, engine):
    """The pure-Python oracle (every sum written out) and the device agree bit for bit, the nan bin included."""
    from checkm_b200.genomicSignatures import parse_profiles
    from oracle import outliers_oracle as oo
    from oracle.binstats_oracle import base_counts, coding_bases
    with open(PROFILE, 'rb') as f:
        ids, matrix = parse_profiles(f.read())
    rowOf = {i: r for r, i in enumerate(ids)}
    sigs = oo.read_profile(PROFILE)
    sg = engine.signatures(matrix)
    try:
        for path in _bin_files(expected):
            seqs = oo.read_fasta(path)
            _, covered = coding_bases(os.path.join(OUTDIR, 'bins', oo.bin_id(path), 'genes.gff'))
            want = oo.bin_scores(seqs, sigs, covered)
            n = len(seqs)
            means, binsig, values, _, _ = engine.outlier_scores(
                sg, [0, n], [len(s) for s in seqs.values()], [base_counts(s) for s in seqs.values()],
                [int(covered.get(i, 0)) for i in seqs], [rowOf[i] for i in seqs], [0], [0], 0, [0, 1], [0.0], [0.0], [0.0],
                want_binsig=True)
            assert np.array_equal(_u64(means[0]), _u64([want['meanGC'], want['meanCD'], want['meanTD']])), path
            assert np.array_equal(_u64(binsig[0]), _u64(want['binSig'])), path
            for col, name in enumerate(('GC', 'deltaGC', 'CD', 'deltaCD', 'TD')):
                assert np.array_equal(_u64(values[:, col]), _u64(want[name])), (path, name)
    finally:
        sg.close()


def test_tetra_outliers_modify_in_miniature(expected, dataroot, tmp_path):
    """The profile written by this package's GenomicSignatures from all bins' sequences, the outlier file from it equal to
    the oracle's and to the reference's, the cleaned bin equal to the reference's."""
    from checkm_b200.binTools import BinTools
    from checkm_b200.genomicSignatures import GenomicSignatures
    from oracle import outliers_oracle as oo
    assembly = str(tmp_path / 'assembly.fna')
    with open(assembly, 'wb') as f:
        for path in _bin_files(expected):
            f.write((gzip.open if path.endswith('.gz') else open)(path, 'rb').read())
    profile = str(tmp_path / 'tetra.tsv')
    GenomicSignatures(4, 2).calculate(assembly, profile)
    out = str(tmp_path / 'outliers.tsv')
    bt = BinTools()
    bt.identifyOutliers(OUTDIR, _bin_files(expected), profile, 95, 'any', out)
    text = open(out).read()
    assert text == oo.identify_outliers(OUTDIR, _bin_files(expected), profile, 95, 'any', dataroot)
    assert text == expected['outliers']['any_95']
    cleaned = str(tmp_path / 'b1_plain.cleaned.fna')
    bt.removeOutliers(os.path.join(OG, 'bins', 'b1_plain.fna'), out, cleaned)
    assert hashlib.sha256(open(cleaned, 'rb').read()).hexdigest() == expected['removeOutliers']['b1_plain.fna']['sha256']


def _layout(tmp_path, records, gff=True):
    root = str(tmp_path)
    binFile = os.path.join(root, 'odd.fna')
    with open(binFile, 'w') as f:
        f.write(''.join('>%s\n%s\n' % r for r in records))
    if gff:
        os.makedirs(os.path.join(root, 'bins', 'odd'))
        shutil.copyfile(os.path.join(OUTDIR, 'bins', 'b2_one', 'genes.gff'), os.path.join(root, 'bins', 'odd', 'genes.gff'))
    return root, binFile


@pytest.mark.parametrize('records,gff,message', [
    ([('solo', 'ACGTACGTAC'), ('blank', 'NNNNNNNN')], True, 'Sequence blank of bin odd has no A, C, G or T'),
    ([('solo', 'ACGTACGTAC'), ('stranger', 'ACGTTTGA')], True, 'Sequence stranger of bin odd is not in the tetranucleotide profile file'),
    ([], True, 'Bin odd has no sequences'),
    ([('solo', 'ACGTACGTAC')], False, 'Missing gene feature file (genes.gff). This plot if not compatible with the --genes option.'),
])
def test_inputs_the_reference_crashes_on_exit_with_a_message(dataroot, tmp_path, caplog, records, gff, message):
    from checkm_b200.binTools import BinTools
    root, binFile = _layout(tmp_path, records, gff)
    with caplog.at_level(logging.ERROR, logger='timestamp'):
        with pytest.raises(SystemExit) as err:
            BinTools().identifyOutliers(root, [binFile], PROFILE, 95, 'any', os.path.join(root, 'o.tsv'))
    assert err.value.code == 1
    assert message in caplog.text


def test_the_library_refuses_what_it_cannot_score(engine):
    from checkm_b200._lib import CkmError
    sigs = engine.signatures(np.full((2, 136), 1.0 / 136))
    ok = dict(bin_off=[0, 1], lens=[10], acgt=[[3, 2, 2, 3]], coding=[0], sig_row=[0], bin_gc_table=[0], bin_cd_table=[0], td_table=0,
              table_off=[0, 1], table_key=[0.0], table_lo=[0.0], table_hi=[0.0])
    try:
        engine.outlier_scores(sigs, **ok)
        for change, what in ((dict(acgt=[[0, 0, 0, 0]]), 'has no A, C, G or T'), (dict(lens=[0]), 'is empty'),
                             (dict(sig_row=[2]), 'has no row in the signature matrix'),
                             (dict(bin_off=[0, 0, 1], bin_gc_table=[0, 0], bin_cd_table=[0, 0]), 'bin 0 has no sequences')):
            with pytest.raises(CkmError) as err:
                engine.outlier_scores(sigs, **dict(ok, **change))
            assert err.value.code == 1 and what in str(err.value)
    finally:
        sigs.close()
