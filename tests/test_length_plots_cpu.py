"""The length plots without a device: the oracle (oracle/length_plots_oracle.py) against every value the reference's
NxPlot, LengthHistogram and MarkerGenePosPlot recorded (tests/golden/length_plots/, made by
tests/golden/make_length_plot_goldens.py), the stand-in matplotlib's extension against the existing plot logs, the exact
int-against-float threshold comparison near 2^53, and the three classes importing over the stand-in alone."""
import ast
import gzip
import json
import math
import os
import subprocess
import sys
from fractions import Fraction

import numpy as np
import pytest

from conftest import GOLDEN, ROOT

LG = os.path.join(GOLDEN, 'length_plots')


@pytest.fixture(scope='module')
def expected():
    with gzip.open(os.path.join(LG, 'expected.json.gz'), 'rt') as f:
        return json.load(f)


def bin_files():
    og = os.path.join(GOLDEN, 'outliers', 'bins')
    out = [os.path.join(og, f) for f in sorted(os.listdir(og))] + [os.path.join(GOLDEN, 'plots', 'bins', 'p1_edges.fna')]
    return out + [os.path.join(LG, 'bins', f) for f in sorted(os.listdir(os.path.join(LG, 'bins')))]


def bin_id(path):
    return os.path.basename(path).split('.')[0]


def test_oracle_matches_every_reference_value(expected):
    from oracle import length_plots_oracle as lo
    from oracle.binstats_oracle import read_fasta
    nraise = 0
    for binFile in bin_files():
        binId = bin_id(binFile)
        lens = [len(s) for s in read_fasta(binFile).values()]
        for step in expected['steps']:
            x = np.arange(0, 1.0 + 0.5 * step, step).tolist()
            nx, exc = lo.nx(x, lens)
            want = expected['values'][binId][str(step)]
            assert (exc is None and nx == want.get('nx')) or (exc is not None and exc == want.get('raises')), (binId, step)
            _, pexc = lo.plot_nx(x, lens)
            run = expected['runs']['nx|%s|%r' % (binId, step)]
            assert pexc == run.get('raises'), (binId, step)
            nraise += pexc is not None
        bar = [e for e in expected['runs']['len|' + binId]['log'] if e[1] == 'bar']
        assert [float.hex(float(c)) for c in lo.length_classes(lens)] == bar[0][3]['height'], binId
    assert nraise >= 20


def _storage(name):
    out = {}
    for line in open(os.path.join(LG, 'markers', 'storage', name)):
        f = line.split('\t')
        out[f[0]] = ast.literal_eval(f[1])
    return out


def test_oracle_marker_rows_match_the_reference(expected):
    from oracle import length_plots_oracle as lo
    from oracle.binstats_oracle import read_fasta
    from tools.axes_recorder import canon
    files = _storage('marker_gene_stats.tsv')
    cases = {k: {g: dict(m) for g, m in c} for k, c in expected['marker_cases'].items()}
    for key, case in cases.items():
        binId = key.split('|')[1]
        if key.startswith('files|'):
            assert case == files[binId], key
        seqs = read_fasta(os.path.join(LG, 'markers', binId + '.fna'))
        genePos = {}
        for line in open(os.path.join(GOLDEN, 'aai', 'bins', binId + '.faa')):
            if line.startswith('>'):
                f = line[1:].split()
                genePos[f[0]] = [int(f[2]), int(f[4])]
        order, size, rows, exc = lo.marker_rows(case, {s: len(q) for s, q in seqs.items()}, genePos)
        run = expected['runs']['marker|' + key]
        if order is None:
            assert run['returns'] is False and run['info'] == []
            continue
        assert exc == run.get('raises'), key
        if exc is not None or 'log' not in run:          # a large log is kept as its digest: held on the device
            continue
        log = run['log']
        colours = [(1.0, 1.0, 1.0), (127 / 255.0, 201 / 255.0, 127 / 255.0), (255 / 255.0, 192 / 255.0, 134 / 255.0),
                   (190 / 255.0, 174 / 255.0, 212 / 255.0), (0.0, 0.0, 0.0)]
        want = [canon(colours[min(n, 4)]) for row in rows for n in row]
        assert [e[3]['facecolor'] for e in log if e[1] == 'Rectangle'] == want, key
        assert [e for e in log if e[1] == 'set_yticklabels'][-1][2] == [[s for s, _ in order]], key
        assert ['set_xlabel', ['Position ({:,} bp/bin)'.format(size)]] in [e[1:3] for e in log], key
    assert sum('raises' in r for k, r in expected['runs'].items() if k.startswith('marker|')) == 2


def _replay(log):
    """Issues every call of a recorded log again through the stand-in's objects, with the logged values."""
    import matplotlib
    from matplotlib.backends.backend_agg import FigureCanvasAgg
    from matplotlib.figure import Figure

    def val(v):
        if isinstance(v, str) and v.startswith(('0x', '-0x')) and 'p' in v:
            f = float.fromhex(v)
            return int(f) if f.is_integer() else f
        if isinstance(v, list):
            return [val(x) for x in v]
        if isinstance(v, dict):
            return {k: val(x) for k, x in v.items()}
        return v
    objs, canvases = {}, {}

    def obj(name):
        if name not in objs:
            head, _, tail = name.rpartition('.')
            if head.endswith('.spine'):
                objs[name] = dict(obj(head[:-len('.spine')]).spines.items())[tail]
            elif tail.startswith('tick'):
                objs[name] = obj(head).majorTicks[int(tail[4:])]
            else:
                objs[name] = getattr(obj(head), tail)
        return objs[name]
    for entry in log:
        name, what = entry[0], entry[1]
        if name == 'rcParams':
            matplotlib.rcParams[what[1:]] = val(entry[2])
        elif what.startswith('='):
            setattr(obj(name), what[1:], val(entry[2]))
        elif what == 'Figure':
            objs[name] = Figure(*val(entry[2]), **val(entry[3]))
        elif what == 'FigureCanvasAgg':
            canvases[name] = FigureCanvasAgg(objs[name])
        elif what == 'draw':
            canvases[name].draw()
        elif what == 'get_ticklines':
            for i, line in enumerate(obj(name).get_ticklines()):
                objs['%s.line%d' % (name, i)] = line
        else:
            got = getattr(obj(name), what)(*val(entry[2]), **val(entry[3]))
            if what == 'add_subplot':
                objs[object.__getattribute__(got, '_name')] = got


def test_recorder_extension_leaves_the_plot_logs_unchanged():
    from tools import axes_recorder as rec
    with gzip.open(os.path.join(GOLDEN, 'plots', 'expected.json.gz'), 'rt') as f:
        runs = json.load(f)['runs']
    rec.install()
    try:
        replayed = 0
        for key in sorted(runs):
            if 'log' not in runs[key]:
                continue
            rec.reset()
            _replay(runs[key]['log'])
            assert json.loads(json.dumps(rec.LOG)) == runs[key]['log'], key
            replayed += 1
    finally:
        rec.uninstall()
    assert replayed >= 100


def _ge_like_the_device(c, t):
    """csrc/lengths.cu's int_ge: c >= t through ceil(t) as a 64-bit integer."""
    if not t > -9223372036854775808.0:
        return True
    if t >= 9223372036854775808.0:
        return False
    return c >= int(math.ceil(t))


def test_threshold_comparison_is_exact_near_2_53():
    from oracle import length_plots_oracle as lo
    rng = np.random.default_rng(53)
    checked = 0
    for _ in range(2000):
        total = (1 << 53) + int(rng.integers(-4096, 4096))
        t = float(rng.choice([0.05, 0.1, 0.3, 0.7, 0.9, 0.95, 1.0, 1.0 - 2 ** -53])) * total
        for c in (int(math.floor(t)) + d for d in range(-3, 4)):
            assert _ge_like_the_device(c, t) == (Fraction(c) >= Fraction(t)) == (c >= t)
            checked += 1
    assert checked == 14000
    # 2^53 + 1 has no double (float() rounds it to 2^53); the exact rule still orders it between 2^53 and 2^53 + 2
    assert _ge_like_the_device((1 << 53) + 1, float(1 << 53)) and not _ge_like_the_device((1 << 53) + 1, float((1 << 53) + 2))
    for lens in ([(1 << 52) + 1, (1 << 52) - 1, 3, 1], [(1 << 52) + 1, (1 << 52), 1], [(1 << 53) - 1, 1, 1]):
        x = np.arange(0, 1.0 + 0.5 * 0.05, 0.05).tolist()
        total = sum(lens)
        got, exc = lo.nx(x, lens)
        want, run = [], 0
        order = sorted(lens, reverse=True)
        prefix = [sum(order[:k + 1]) for k in range(len(order))]
        for v in x:
            k = next((k for k, s in enumerate(prefix) if Fraction(s) >= Fraction(v * total)), None)
            if k is not None:
                want.append(order[k])
        assert got[:len(want)] == want


def test_classes_import_over_the_stand_in_alone():
    code = ('import sys\n'
            'sys.modules["matplotlib"] = None\n'
            'import checkm_b200\n'
            'from tools import axes_recorder as rec\n'
            'rec.install()\n'
            'from checkm_b200.plot.nxPlot import NxPlot\n'
            'from checkm_b200.plot.lengthHistogram import LengthHistogram\n'
            'from checkm_b200.plot.markerGenePosPlot import MarkerGenePosPlot\n'
            'from checkm_b200.plot.AbstractPlot import length_profiles\n'
            'import types\n'
            'm = MarkerGenePosPlot(types.SimpleNamespace(font_size=8, dpi=600))\n'
            'assert m.roundUpToNearest100(101.0) == 200 and m.roundUpToNearest100(0.0) == 0\n'
            'pos, num = m.getMarkerGenesPerSeq({"s_1_3": {"M1": [[1, 9], [20, 30]], "M2": [[5, 6]]}, "s_1_4": {"M1": [[2, 3]]}})\n'
            'assert pos == {"s_1": [["s_1_3", "M1", 20, 30], ["s_1_3", "M2", 5, 6], ["s_1_4", "M1", 2, 3]]}, pos\n'
            'assert num == {"M1": 1, "M2": 1}\n'
            'assert type(sys.modules["matplotlib"]).__name__ == "module" and not hasattr(sys.modules["matplotlib"], "__file__")\n')
    subprocess.check_call([sys.executable, '-c', code], cwd=ROOT)
