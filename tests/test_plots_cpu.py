"""The plot windows without a device: the oracle (oracle/plot_windows_oracle.py) against every window value the
reference computed (tests/golden/plots/, made by tests/golden/make_plot_goldens.py), the stand-in matplotlib, the host's
coding-interval arithmetic against the literal numpy mask, and that checkm_b200 imports without matplotlib."""
import gzip
import json
import os
import subprocess
import sys

import numpy as np
import pytest

from conftest import GOLDEN, ROOT

PG = os.path.join(GOLDEN, 'plots')
OG = os.path.join(GOLDEN, 'outliers')


@pytest.fixture(scope='module')
def expected():
    with gzip.open(os.path.join(PG, 'expected.json.gz'), 'rt') as f:
        return json.load(f)


def bin_files():
    out = [(os.path.join(OG, 'bins', f), os.path.join(OG, 'out')) for f in sorted(os.listdir(os.path.join(OG, 'bins')))]
    return out + [(os.path.join(PG, 'bins', 'p1_edges.fna'), os.path.join(PG, 'out'))]


def reference_genes(path):
    """prodigal.py:215-248 as it parses: genes per sequence (a repeated gene number overwrites) and the largest end."""
    genes, last, counter = {}, {}, 0
    for line in open(path):
        if line[0] == '#' or line.strip() == '"':
            continue
        f = line.split('\t')
        if f[0] not in genes:
            counter, genes[f[0]], last[f[0]] = 0, {}, 0
        genes[f[0]][counter] = (int(f[3]), int(f[4]))
        counter += 1
        last[f[0]] = max(last[f[0]], int(f[4]))
    return genes, last


def test_oracle_matches_every_reference_window_value(expected):
    from oracle import outliers_oracle as oo, plot_windows_oracle as pw
    from oracle.binstats_oracle import read_fasta
    profile = oo.profile_text([os.path.join(OG, 'extra.fna')] + [b for b, _ in bin_files()])
    sigs = {}
    for line in profile.split('\n')[1:]:
        if line:
            parts = line.split('\t')
            sigs[parts[0]] = [float(x) for x in parts[1:]]
    checked = 0
    for binFile, resultsDir in bin_files():
        binId = oo.bin_id(binFile)
        seqs = read_fasta(binFile)
        binSig = oo.bin_tetra_sig(seqs, sigs)
        genes, last = reference_genes(os.path.join(resultsDir, 'bins', binId, 'genes.gff'))
        masks = {s: pw.coding_mask(g.values(), last[s]) for s, g in genes.items()}
        for W in expected['windows']:
            want = expected['values'][binId][str(W)]
            acgt, coding, td = [], [], []
            for seqId, seq in seqs.items():
                for (lo, hi), (a, c, g, t, d) in zip(pw.windows(len(seq), W), pw.window_stats(seq, W, binSig)):
                    acgt.append([a, c, g, t])
                    coding.append(float.hex(float(np.sum(masks[seqId][lo:hi])) if seqId in masks else 0.0))
                    td.append(float.hex(d))
            assert acgt == want['acgt'], (binId, W)
            assert coding == want['coding'], (binId, W)
            assert td == want['td'], (binId, W)
            checked += len(acgt)
    assert checked > 10000


def test_recorder_logs_calls_attributes_and_exact_floats():
    from tools import axes_recorder as rec
    before = sys.modules.get('matplotlib')
    rec.install()
    try:
        import matplotlib
        from matplotlib.figure import Figure
        from matplotlib.backends.backend_agg import FigureCanvasAgg
        matplotlib.rcParams['font.size'] = 8
        fig = Figure(dpi=600)
        FigureCanvasAgg(fig)
        ax = fig.add_subplot(121)
        ax.hist([0.1, np.float64(0.2)], bins=np.array([0.0, 0.5]), density=True)
        ax.yaxis.majorTicks[0].tick1On = True
        ax.xaxis.get_ticklines()[1].set_color((0.5, 0.5, 0.5))
        [s for _, s in ax.spines.items()][1].set_color('none')
        assert ax.get_xlim() == rec.XLIM and list(ax.get_yticks()) == list(rec.YTICKS)
        assert rec.LOG == [
            ['rcParams', '=font.size', float.hex(8.0)],
            ['fig0', 'Figure', [], {'dpi': float.hex(600.0)}],
            ['fig0', 'FigureCanvasAgg', [], {}],
            ['fig0', 'add_subplot', [float.hex(121.0)], {}],
            ['fig0.ax121', 'hist', [[float.hex(0.1), float.hex(0.2)]], {'bins': ['0x0.0p+0', '0x1.0000000000000p-1'],
                                                                        'density': True}],
            ['fig0.ax121.yaxis.tick0', '=tick1On', True],
            ['fig0.ax121.xaxis', 'get_ticklines', [], {}],
            ['fig0.ax121.xaxis.line1', 'set_color', [[float.hex(0.5)] * 3], {}],
            ['fig0.ax121.spine.right', 'set_color', ['none'], {}],
            ['fig0.ax121', 'get_xlim', [], {}],
            ['fig0.ax121', 'get_yticks', [], {}]]
    finally:
        rec.uninstall()
    assert sys.modules.get('matplotlib') is before


def test_window_coding_bases_match_the_literal_mask():
    from checkm_b200.binStatistics import _GeneFeatures
    from oracle.plot_windows_oracle import coding_mask
    rng = np.random.default_rng(7)
    for trial in range(10000):
        L = int(rng.integers(1, 400))
        genes = []
        for _ in range(int(rng.integers(1, 6))):
            s = int(rng.choice([0, int(rng.integers(-3, L + 20))]))
            genes.append((s, int(rng.integers(max(s, 1), L + 30))))
        last = max([0] + [e for _, e in genes])
        mask = coding_mask(genes, last)
        f = _GeneFeatures.__new__(_GeneFeatures)
        f.intervals = {'s': _GeneFeatures._mask_intervals(genes, last)}
        W = int(rng.integers(1, 60))
        starts = np.arange(0, last + 2 * W, W, dtype=np.int64)
        got = f.windowCodingBases('s', starts, starts + W)
        want = [int(np.sum(mask[a:a + W])) for a in starts]
        assert got.tolist() == want, (genes, W)
        assert f.windowCodingBases('absent', starts, starts + W).tolist() == [0] * len(starts)


def test_package_imports_without_matplotlib():
    code = ('import sys, importlib, pkgutil, checkm_b200\n'
            'for m in pkgutil.iter_modules(checkm_b200.__path__):\n'
            '    if m.name not in ("plot", "libckm"): importlib.import_module("checkm_b200." + m.name)\n'
            'assert "matplotlib" not in sys.modules and "checkm_b200.plot" not in sys.modules\n')
    subprocess.check_call([sys.executable, '-c', code], cwd=ROOT)
    for dirpath, _, files in os.walk(os.path.join(ROOT, 'checkm_b200')):
        if os.path.basename(dirpath) == 'plot':
            continue
        for name in files:
            if name.endswith('.py'):
                text = open(os.path.join(dirpath, name)).read()
                assert 'checkm_b200.plot' not in text and 'from .plot' not in text and 'from . import plot' not in text, name
