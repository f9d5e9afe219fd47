"""The plot windows on the device (checkm_b200.plot over ckm_window_stats, csrc/windows.cu): every recorded plot call
equal to the reference's (tests/golden/plots/, made by tests/golden/make_plot_goldens.py) with every float bit-equal, the
window statistics bit-equal to a CPU restatement at scale, the refusals, and tetra -> profile -> dist_plot end to end."""
import gzip
import hashlib
import json
import os
import types

import numpy as np
import pytest

from conftest import GOLDEN

pytestmark = pytest.mark.gpu
PG = os.path.join(GOLDEN, 'plots')
OG = os.path.join(GOLDEN, 'outliers')


@pytest.fixture(scope='module')
def rec():
    """The stand-in matplotlib, installed for this module only."""
    from tools import axes_recorder
    axes_recorder.install()
    yield axes_recorder
    axes_recorder.uninstall()


@pytest.fixture(scope='module')
def expected():
    with gzip.open(os.path.join(PG, 'expected.json.gz'), 'rt') as f:
        return json.load(f)


@pytest.fixture(scope='module')
def dataroot(engine):
    from checkm_b200.defaultValues import DefaultValues
    saved = DefaultValues.CHECKM_DATA_DIR
    DefaultValues.set_data_root(os.path.join(OG, 'data'))
    yield
    DefaultValues.set_data_root(saved)


def bin_files():
    out = [(os.path.join(OG, 'bins', f), os.path.join(OG, 'out')) for f in sorted(os.listdir(os.path.join(OG, 'bins')))]
    return out + [(os.path.join(PG, 'bins', 'p1_edges.fna'), os.path.join(PG, 'out'))]


@pytest.fixture(scope='module')
def tetra_sigs(tmp_path_factory):
    from oracle.outliers_oracle import profile_text
    from checkm_b200.genomicSignatures import GenomicSignatures
    path = str(tmp_path_factory.mktemp('plots') / 'tetra.tsv')
    with open(path, 'w') as f:
        f.write(profile_text([os.path.join(OG, 'extra.fna')] + [b for b, _ in bin_files()]))
    return GenomicSignatures(4, 1).read(path)


def options(results_dir, gc=5000, td=5000, cd=10000, window=5000):
    return types.SimpleNamespace(font_size=8, dpi=600, width=6.5, height=8, gc_window_size=gc, td_window_size=td,
                                 cd_window_size=cd, window_size=window, gc_bin_width=0.01, cd_bin_width=0.01,
                                 td_bin_width=0.01, results_dir=results_dir)


def run_case(rec, key, case, tetraSigs, files):
    from checkm_b200.plot.codingDensityPlots import CodingDensityPlots
    from checkm_b200.plot.distributionPlots import DistributionPlots
    from checkm_b200.plot.gcBiasPlots import GcBiasPlot
    from checkm_b200.plot.gcPlots import GcPlots
    from checkm_b200.plot.tetraDistPlots import TetraDistPlots
    parts = key.split('|')
    binFile, resultsDir = files[parts[1]]
    rec.reset()
    if parts[0] == 'dist':
        gc, td, cd = (int(x) for x in parts[2].split('_'))
        fn = lambda: DistributionPlots(options(resultsDir, gc=gc, td=td, cd=cd)).plot(binFile, tetraSigs, [95, 85])  # noqa: E731
    elif parts[0] == 'bias':
        from oracle.binstats_oracle import read_fasta
        from oracle.plot_windows_oracle import synthetic_coverage
        W = int(parts[2])
        cov = synthetic_coverage({i: len(q) for i, q in read_fasta(binFile).items()}, W)
        fn = lambda: GcBiasPlot(options(resultsDir, window=W)).plot(binFile, cov)  # noqa: E731
    else:
        W, dist = int(parts[2]), [int(x) for x in parts[3].split('_')]
        o = options(resultsDir, gc=W, td=W, cd=W, window=W)
        fn = {'gc': lambda: GcPlots(o).plot(binFile, dist), 'cd': lambda: CodingDensityPlots(o).plot(binFile, dist),
              'td': lambda: TetraDistPlots(o).plot(binFile, tetraSigs, dist)}[parts[0]]
    if 'raises' in case:
        with pytest.raises(SystemExit) as e:        # the reference divides by zero there: an error and exit status 1
            fn()
        assert e.value.code == 1, key
    elif 'log' in case:
        fn()
        assert json.loads(json.dumps(rec.LOG)) == case['log'], key
    else:                                           # small window sizes: the log's SHA-256 (make_plot_goldens.log_digest)
        fn()
        got = hashlib.sha256(json.dumps(rec.LOG, sort_keys=True, separators=(',', ':')).encode()).hexdigest()
        assert got == case['sha256'], key


def test_every_plot_call_is_the_references(rec, expected, dataroot, tetra_sigs):
    from oracle.outliers_oracle import bin_id
    files = {bin_id(b): (b, r) for b, r in bin_files()}
    for key in sorted(expected['runs']):
        run_case(rec, key, expected['runs'][key], tetra_sigs, files)
    assert sum('raises' in c for c in expected['runs'].values()) >= 10


def _layout(seqs):
    lens = np.array([len(s) for s in seqs], dtype=np.int64)
    starts = np.concatenate([[0], np.cumsum((lens + 63) // 64 * 64)[:-1]]).astype(np.int64)
    data = np.zeros(int(((lens + 63) // 64 * 64).sum()) + 64, dtype=np.uint8)
    for s, a in zip(seqs, starts):
        data[a:a + len(s)] = s
    return data, starts, lens


def _numpy_windows(seqs, W, binSig):
    """The window statistics restated with numpy, for sizes where the oracle's Python loops are too slow; sums of the
    distance in numpy's pairwise order by oracle.outliers_oracle.pairwise_sum."""
    from oracle.outliers_oracle import pairwise_sum
    from oracle.plot_windows_oracle import _COLUMN
    col = np.array([_COLUMN[x] for x in range(256)], dtype=np.int64)
    acgt, td = [], []
    for s in seqs:
        nwin = max(len(s) - 1, 0) // W
        if nwin == 0:
            continue
        u = s[:nwin * W] & 0xDF
        cls = np.full(len(u), 4, dtype=np.int64)
        for k, ch in enumerate(b'ACGT'):
            cls[u == ch] = k
        cls[u == ord('U')] = 3
        win = np.arange(len(u)) // W
        acgt.append(np.bincount(win * 5 + cls, minlength=nwin * 5).reshape(nwin, 5)[:, :4])
        if binSig is None:
            continue
        code = np.full(len(u), 4, dtype=np.int64)
        for k, ch in enumerate(b'ACGT'):
            code[u == ch] = k
        p = np.arange(len(u) - 3)
        ok = (code[p] < 4) & (code[p + 1] < 4) & (code[p + 2] < 4) & (code[p + 3] < 4) & ((p % W) + 3 < W)
        p = p[ok]
        raw = (code[p] << 6) | (code[p + 1] << 4) | (code[p + 2] << 2) | code[p + 3]
        counts = np.bincount(win[p] * 136 + col[raw], minlength=nwin * 136).reshape(nwin, 136)
        with np.errstate(invalid='ignore'):
            sig = counts.astype(np.float64) / counts.sum(axis=1, keepdims=True).astype(np.float64)
        d = np.abs(sig - binSig)
        td.extend(pairwise_sum(row.tolist()) for row in d)
    return (np.concatenate(acgt) if acgt else np.zeros((0, 4), dtype=np.int64)), np.array(td)


def _random_bin(rng, total, short=False):
    seqs, n = [], 0
    while n < total:
        L = int(rng.integers(1, 2000)) if short else int(rng.integers(1, 400000))
        g = rng.uniform(0.2, 0.8)
        s = rng.choice(np.frombuffer(b'ACGT', dtype=np.uint8), size=L, p=[(1 - g) / 2, g / 2, g / 2, (1 - g) / 2])
        for _ in range(int(rng.integers(0, 4))):                 # N runs, lower case, U and IUPAC codes
            a = int(rng.integers(0, L))
            b = min(L, a + int(rng.integers(1, 3000)))
            s[a:b] = rng.choice(np.frombuffer(b'NNNNacgtuURYKM', dtype=np.uint8)) if rng.random() < 0.5 else s[a:b] | 0x20
        seqs.append(s)
        n += L
    return seqs


def _same(a, b):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    return a.shape == b.shape and bool(np.all((a.view(np.uint64) == b.view(np.uint64)) | (np.isnan(a) & np.isnan(b))))


@pytest.mark.parametrize('W', [1, 3, 63, 64, 65, 2047, 2048, 2049, 5000, 10000])
def test_window_stats_bit_equal_to_the_cpu_restatement(engine, W):
    from checkm_b200.coverageWindows import window_offsets
    rng = np.random.default_rng(W)
    total = 300000 if W < 64 else 24000000
    seqs = _random_bin(rng, total // 2, short=True) + _random_bin(rng, total // 2)
    binSig = rng.dirichlet(np.ones(136))
    data, starts, lens = _layout(seqs)
    off = window_offsets(lens, W)
    for sig in (binSig, None):
        acgt, td, ms = engine.window_stats(data, starts, lens, W, off, sig)
        want_acgt, want_td = _numpy_windows(seqs, W, sig)
        assert np.array_equal(acgt, want_acgt), W
        if sig is None:
            assert td is None
        else:
            assert _same(td, want_td), (W, np.flatnonzero(td != want_td)[:5])


def test_window_stats_match_the_oracle_on_small_bins(engine):
    from checkm_b200.coverageWindows import window_offsets
    from oracle.plot_windows_oracle import window_stats
    rng = np.random.default_rng(11)
    seqs = _random_bin(rng, 40000, short=True)
    binSig = rng.dirichlet(np.ones(136))
    data, starts, lens = _layout(seqs)
    for W in (1, 7, 100, 2048):
        acgt, td, _ = engine.window_stats(data, starts, lens, W, window_offsets(lens, W), binSig)
        want = [w for s in seqs for w in window_stats(bytes(s).decode('latin-1'), W, binSig.tolist())]
        assert acgt.tolist() == [list(w[:4]) for w in want]
        assert _same(td, [w[4] for w in want])


def test_refusals(engine, rec, dataroot, tmp_path, tetra_sigs):
    from checkm_b200._lib import CkmError
    from checkm_b200.coverageWindows import window_offsets
    from checkm_b200.plot.codingDensityPlots import CodingDensityPlots
    from checkm_b200.plot.gcPlots import GcPlots
    data, starts, lens = _layout([np.frombuffer(b'ACGT' * 100, dtype=np.uint8)])
    with pytest.raises(CkmError):
        engine.window_stats(data, starts, lens, 0, np.zeros(2, dtype=np.int64))
    with pytest.raises(CkmError):
        engine.window_stats(data, starts, lens, 7, window_offsets(lens, 7) + np.array([0, 1]))
    binFile = os.path.join(OG, 'bins', 'b1_plain.fna')
    with pytest.raises(SystemExit) as e:
        GcPlots(options(os.path.join(OG, 'out'), gc=0)).plot(binFile, [95])
    assert e.value.code == 1
    with pytest.raises(SystemExit) as e:                     # no genes.gff under this results directory
        CodingDensityPlots(options(str(tmp_path), cd=100)).plot(binFile, [95])
    assert e.value.code == 1


def test_dist_plot_end_to_end_from_tetra(rec, expected, dataroot, tmp_path):
    """checkm tetra writes the profile, the plots read it: the dist_plot calls are the reference's."""
    from checkm_b200.genomicSignatures import GenomicSignatures
    from oracle.outliers_oracle import bin_id
    files = dict((bin_id(b), (b, r)) for b, r in bin_files())
    assembly = str(tmp_path / 'assembly.fna')
    with open(assembly, 'w') as f:
        for b in ('extra.fna', 'bins/b1_plain.fna', 'bins/b8_edge.fna'):
            f.write(open(os.path.join(OG, b)).read())
    profile = str(tmp_path / 'tetra.tsv')
    gs = GenomicSignatures(4, 1)
    gs.calculate(assembly, profile)
    sigs = gs.read(profile)
    for binId in ('b1_plain', 'b8_edge'):
        for sizes in ('5000_5000_10000', '100_100_100', '7_100_7'):
            key = 'dist|%s|%s' % (binId, sizes)
            run_case(rec, key, expected['runs'][key], sigs, files)
