"""The length plots on the device (checkm_b200.plot.nxPlot / lengthHistogram / markerGenePosPlot over
ckm_length_profile, csrc/lengths.cu): every recorded call equal to the reference's (tests/golden/length_plots/, made by
tests/golden/make_length_plot_goldens.py) at every Nx step, every reference exception an exit status 1 naming the bin, the
device call equal to a numpy restatement on 1,000 bins, one-bin and many-bin calls equal, the refusals, and
find -> qa -> marker_plot in one process."""
import gzip
import hashlib
import json
import logging
import os
import shutil
import types

import numpy as np
import pytest

from conftest import CPR_HMM, GOLDEN

pytestmark = pytest.mark.gpu
LG = os.path.join(GOLDEN, 'length_plots')
AAI = os.path.join(GOLDEN, 'aai')
MARKER_BINS = ['strainA', 'strainB', 'strainC']


@pytest.fixture(scope='module')
def rec():
    from tools import axes_recorder
    axes_recorder.install()
    yield axes_recorder
    axes_recorder.uninstall()


@pytest.fixture(scope='module')
def expected():
    with gzip.open(os.path.join(LG, 'expected.json.gz'), 'rt') as f:
        return json.load(f)


class _Messages(logging.Handler):
    def __init__(self):
        logging.Handler.__init__(self)
        self.records = []

    def emit(self, record):
        self.records.append(record)


@pytest.fixture()
def messages():
    h = _Messages()
    logger = logging.getLogger('timestamp')
    saved = logger.level
    logger.addHandler(h)
    logger.setLevel(logging.INFO)
    yield h
    logger.removeHandler(h)
    logger.setLevel(saved)


def bin_files():
    og = os.path.join(GOLDEN, 'outliers', 'bins')
    out = [os.path.join(og, f) for f in sorted(os.listdir(og))] + [os.path.join(GOLDEN, 'plots', 'bins', 'p1_edges.fna')]
    return out + [os.path.join(LG, 'bins', f) for f in sorted(os.listdir(os.path.join(LG, 'bins')))]


def options(results_dir='', step=0.05):
    return types.SimpleNamespace(font_size=8, dpi=600, width=6.5, height=6.5, fig_padding=0.2, step_size=step,
                                 results_dir=results_dir, image_type='png')


def check_run(rec, messages, key, case, fn, binId):
    rec.reset()
    del messages.records[:]
    if 'raises' in case:
        with pytest.raises(SystemExit) as e:
            fn()
        assert e.value.code == 1, key
        errors = [r.getMessage() for r in messages.records if r.levelno >= logging.ERROR]
        assert errors and binId in errors[-1], (key, errors)
        return
    got = fn()
    if 'log' in case:
        assert json.loads(json.dumps(rec.LOG)) == case['log'], key
    else:
        assert hashlib.sha256(json.dumps(rec.LOG, sort_keys=True, separators=(',', ':')).encode()).hexdigest() == case['sha256'], key
    if 'returns' in case and key.startswith('marker|'):
        assert got == case['returns'], key
    assert [r.getMessage() for r in messages.records if r.levelno == logging.INFO] == case['info'], key


def test_every_nx_and_len_hist_call_is_the_references(engine, rec, expected, messages):
    from checkm_b200.plot.lengthHistogram import LengthHistogram
    from checkm_b200.plot.nxPlot import NxPlot
    n = 0
    for binFile in bin_files():
        binId = os.path.basename(binFile).split('.')[0]
        for step in expected['steps']:
            key = 'nx|%s|%r' % (binId, step)
            check_run(rec, messages, key, expected['runs'][key], lambda: NxPlot(options(step=step)).plot(binFile), binId)
            n += 1
        key = 'len|' + binId
        check_run(rec, messages, key, expected['runs'][key], lambda: LengthHistogram(options()).plot(binFile), binId)
    assert n == 8 * len(bin_files())


def test_calculate_nx_is_the_references(engine, expected):
    from checkm_b200.plot.nxPlot import NxPlot
    from oracle.binstats_oracle import read_fasta
    for binFile in bin_files():
        binId = os.path.basename(binFile).split('.')[0]
        seqs = read_fasta(binFile)
        for step in expected['steps']:
            want = expected['values'][binId][str(step)]
            x = np.arange(0, 1.0 + 0.5 * step, step)
            if 'raises' in want:
                with pytest.raises(IndexError):
                    NxPlot(options(step=step)).calculateNx(x, seqs)
            else:
                assert NxPlot(options(step=step)).calculateNx(x, seqs) == want['nx'], (binId, step)


def _marker_cases(expected):
    return {k: {g: dict(m) for g, m in c} for k, c in expected['marker_cases'].items()}


def test_every_marker_plot_call_is_the_references(engine, rec, expected, messages, tmp_path):
    from checkm_b200.plot.markerGenePosPlot import MarkerGenePosPlot
    out = str(tmp_path)
    for b in MARKER_BINS:
        os.makedirs(os.path.join(out, 'bins', b))
        shutil.copyfile(os.path.join(AAI, 'bins', b + '.faa'), os.path.join(out, 'bins', b, 'genes.faa'))
    for key, mgs in sorted(_marker_cases(expected).items()):
        binId = key.split('|')[1]
        fn = lambda: MarkerGenePosPlot(options(out)).plot(os.path.join(LG, 'markers', binId + '.fna'), mgs,  # noqa: E731
                                                          expected['bin_stats'][binId])
        check_run(rec, messages, 'marker|' + key, expected['runs']['marker|' + key], fn, binId)
    assert sum('raises' in r for k, r in expected['runs'].items() if k.startswith('marker|')) == 2


def _numpy_profile(lens, off, x):
    """The device's outputs restated with numpy: stable descending order, exact prefix sums, the first prefix reaching
    each threshold by the same ceil rule the CPU tests hold to Python's exact comparison, np.histogram's classes."""
    nb, m = len(off) - 1, len(x)
    total = np.zeros(nb, np.int64)
    nx = np.full((nb, m), -1, np.int64)
    status = np.zeros(nb, np.int32)
    fail = np.full(nb, -1, np.int64)
    classes = np.zeros((nb, 10), np.int64)
    rank = np.zeros(len(lens), np.int32)
    for b in range(nb):
        L = lens[off[b]:off[b + 1]]
        order = np.argsort(-L, kind='stable')
        rank[off[b] + order] = np.arange(len(L))
        s = L[order]
        c = np.cumsum(s)
        t = int(L.sum())
        total[b] = t
        need = np.ceil(x * float(t))
        ks = [int(np.searchsorted(c, int(v), side='left')) for v in need]
        reached = [k for k in ks if k < len(L)]
        nx[b, :len(reached)] = s[reached]
        if len(reached) < m:
            status[b], fail[b] = 2, len(reached)
        elif ks[-1] < len(L) - 1:
            status[b], fail[b] = 1, ks[-1] + 1
        classes[b] = np.histogram(L.astype(np.float64) / 1e3, bins=[0, 1, 2, 5, 10, 20, 50, 100, 200, 500, 1e12])[0]
    return total, nx, status, fail, classes, rank


def _random_bins(rng, nbins):
    sizes = np.exp(rng.uniform(np.log(100), np.log(20000), nbins)).astype(np.int64)
    sizes[:20] = 1                                                       # single-record bins
    sizes[20:25] = 0                                                     # empty bins
    bins = []
    for b, n in enumerate(sizes):
        kind = b % 4
        if kind == 0:
            L = rng.integers(0, 6, n)                                    # heavy ties, zero lengths
        elif kind == 1:
            L = rng.choice([999, 1000, 1001, 2000, 500000, 500001, 10 ** 12 // 1000 * 1000], n)
        elif kind == 2:
            L = rng.integers(1, 3 * 10 ** 6, n)                          # totals above 2^32
        else:                                                            # totals past 2^53; len / 1e3 at and past 1e12
            L = rng.integers(10 ** 15 - 2, 10 ** 15 + 3, min(n, 4000))
        bins.append(L.astype(np.int64))
    return bins


def test_device_equals_the_numpy_restatement_on_1000_bins(engine):
    rng = np.random.default_rng(2026)
    bins = _random_bins(rng, 1000)
    lens = np.concatenate(bins)
    off = np.zeros(len(bins) + 1, np.int64)
    off[1:] = np.cumsum([len(b) for b in bins])
    assert max(int(b.sum()) for b in bins) > 1 << 53 and sum(int(b.sum()) > 1 << 32 for b in bins) > 100
    for step in (0.01, 0.05, 0.07, 0.3, 1.0):
        x = np.arange(0, 1.0 + 0.5 * step, step)
        got = engine.length_profile(lens, off, x)[:6]
        want = _numpy_profile(lens, off, x)
        for name, g, w in zip(('total', 'nx', 'status', 'fail', 'classes', 'rank'), got, want):
            assert np.array_equal(g, w), (step, name, np.argwhere(np.asarray(g) != np.asarray(w))[:5])
        assert {0, 1, 2} <= set(got[2].tolist()), step


def test_device_equals_the_oracle_on_small_bins(engine):
    from oracle import length_plots_oracle as lo
    rng = np.random.default_rng(7)
    bins = [rng.integers(0, 50, int(rng.integers(0, 40))) for _ in range(300)]
    bins += [np.array([(1 << 52) + 1, (1 << 52) - 1, 3, 1]), np.array([(1 << 53) - 1, 1, 1]), np.array([5, 4, 3, 2, 1]),
             np.array([100, 1, 1, 1]), np.array([5, 0]), np.array([0]), np.array([0, 0])]
    lens = np.concatenate(bins).astype(np.int64)
    off = np.zeros(len(bins) + 1, np.int64)
    off[1:] = np.cumsum([len(b) for b in bins])
    for step in (0.01, 0.05, 0.07, 0.1, 0.25, 0.3, 0.5, 1.0, 0.33):
        x = np.arange(0, 1.0 + 0.5 * step, step)
        total, nx, status, fail, classes, _, _ = engine.length_profile(lens, off, x)
        for b, L in enumerate(bins):
            want, exc = lo.nx(x.tolist(), [int(v) for v in L])
            assert status[b] == {None: 0 if len(want) == len(x) else 2, 'IndexError': 1}[exc], (step, b)
            k = len(x) if status[b] != 2 else fail[b]
            assert nx[b][:k].tolist() == want[:k], (step, b)
            assert classes[b].tolist() == lo.length_classes([int(v) for v in L])
            assert total[b] == sum(int(v) for v in L)


def test_one_bin_and_many_bin_calls_agree(engine):
    rng = np.random.default_rng(3)
    bins = _random_bins(rng, 60)
    lens = np.concatenate(bins)
    off = np.zeros(len(bins) + 1, np.int64)
    off[1:] = np.cumsum([len(b) for b in bins])
    x = np.arange(0, 1.025, 0.05)
    many = engine.length_profile(lens, off, x)
    for b, L in enumerate(bins):
        one = engine.length_profile(L, np.array([0, len(L)], np.int64), x)
        assert one[0][0] == many[0][b] and np.array_equal(one[1][0], many[1][b]) and one[2][0] == many[2][b]
        assert one[3][0] == many[3][b] and np.array_equal(one[4][0], many[4][b])
        assert np.array_equal(one[5], many[5][off[b]:off[b + 1]])


def test_length_profiles_of_many_files_equal_one_by_one(engine):
    from checkm_b200.plot.AbstractPlot import length_profiles
    files = bin_files()
    many = length_profiles(files, 0.07)
    for f, p in zip(files, many):
        q = length_profiles([f], 0.07)[0]
        assert (p.ids, p.total, p.status, p.fail) == (q.ids, q.total, q.status, q.fail)
        assert np.array_equal(p.nx, q.nx) and np.array_equal(p.classes, q.classes) and np.array_equal(p.rank, q.rank)


def test_refusals(engine):
    from checkm_b200._lib import CkmError
    x = np.arange(0, 1.05, 0.1)
    for lens, off, xx in ((np.array([3, -1]), [0, 2], x), (np.array([3, 1]), [0, 2], x[::-1]),
                          (np.array([3, 1]), [0, 2], np.array([0.0, np.nan])), (np.array([3, 1]), [0, 2], np.zeros(0)),
                          (np.array([(1 << 62), (1 << 62)]), [0, 2], x), (np.array([3]), [0, 2, 1], x)):
        with pytest.raises((CkmError, ValueError)) as e:
            engine.length_profile(lens, np.array(off, np.int64), xx)
        assert not isinstance(e.value, CkmError) or e.value.code == 1


def test_find_qa_marker_plot_in_one_process(engine, rec, expected, messages, tmp_path, monkeypatch):
    """find -> qa's cached files -> marker_plot, in one process with CUDA initialised: the reference's calls and INFO."""
    import multiprocessing
    from checkm_b200.defaultValues import DefaultValues
    from checkm_b200.markerGeneFinder import MarkerGeneFinder
    from checkm_b200.markerSets import MarkerSetParser
    from checkm_b200.plot.markerGenePosPlot import MarkerGenePosPlot
    from checkm_b200.resultsParser import ResultsParser

    def no_fork(*a, **k):
        raise AssertionError('a process was started after CUDA was initialised')
    monkeypatch.setattr(multiprocessing, 'Process', no_fork)
    real = os.listdir
    monkeypatch.setattr(os, 'listdir', lambda p='.': sorted(real(p)))
    saved = DefaultValues.CHECKM_DATA_DIR
    DefaultValues.set_data_root(os.path.join(GOLDEN, 'reduction', 'data'))
    try:
        out = str(tmp_path / 'out')
        os.makedirs(os.path.join(out, 'storage'))
        binFiles = [os.path.join(AAI, 'bins', b + '.faa') for b in MARKER_BINS]
        binIdToModels = MarkerGeneFinder(1).find(binFiles, out, 'hmmer.analyze.txt', 'hmmer.analyze.ali.txt', CPR_HMM,
                                                 False, False, True)
        with open(os.path.join(AAI, 'expected.json')) as f:
            stats = json.load(f)['bin_stats']
        with open(os.path.join(out, 'storage', 'bin_stats.analyze.tsv'), 'w') as f:
            f.write(''.join(l + '\n' for l in stats))
        RP = ResultsParser(binIdToModels)
        RP.analyseResults(out, 'bin_stats.analyze.tsv', 'hmmer.analyze.txt')
        RP.cacheResults(out, MarkerSetParser(1).getMarkerSets(out, MARKER_BINS, CPR_HMM), False)
        for name in ('marker_gene_stats.tsv',):
            assert open(os.path.join(out, 'storage', name)).read() == open(os.path.join(LG, 'markers', 'storage', name)).read()
        parser = ResultsParser(None)
        mgs, bs = parser.parseMarkerGeneStats(out), parser.parseBinStatsExt(out)
        for binId in MARKER_BINS:
            key = 'marker|files|' + binId
            fn = lambda: MarkerGenePosPlot(options(out)).plot(os.path.join(LG, 'markers', binId + '.fna'), mgs[binId],  # noqa: E731
                                                              bs[binId])
            check_run(rec, messages, key, expected['runs'][key], fn, binId)
    finally:
        DefaultValues.set_data_root(saved)
