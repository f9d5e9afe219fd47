"""Read depth per window (`checkm gc_bias_plot`'s coverage profile) without a GPU: the oracle against every value the
reference's own CoverageWindows computed (tests/golden/coverage_windows/), the window layout, and the refusals that
happen before any device work."""
import gzip
import json
import logging
import os
import re
import shutil

import numpy as np
import pytest

from conftest import GOLDEN, ROOT

CW = os.path.join(GOLDEN, 'coverage_windows')
BAMS = {'windows': os.path.join(CW, 'windows.bam'), 'sample1': os.path.join(GOLDEN, 'coverage', 'sample1.bam'),
        'sample2': os.path.join(GOLDEN, 'coverage', 'sample2.bam')}


@pytest.fixture(scope='module')
def expected():
    with gzip.open(os.path.join(CW, 'expected.json.gz'), 'rt') as f:
        return json.load(f)


def unrle(runs):
    return [float(v) for v, n in runs for _ in range(n)]


def test_oracle_matches_every_golden(expected):
    from oracle import coverage_windows_oracle as cwo
    assert expected['windows'] == [1, 7, 100, 5000] and set(expected['values']) == set(BAMS)
    for bam_label, path in BAMS.items():
        for label, o in expected['options'].items():
            names, lens, cnt, deps = cwo.depths(path, o['bAllReads'], o['minAlignPer'], o['maxEditDistPer'])
            assert [int(d.sum()) for d in deps] == cnt[:, 8].tolist()
            for W in expected['windows']:
                want = expected['values'][bam_label][label][str(W)]
                assert list(want) == names
                for name, L, c, d in zip(names, lens, cnt, deps):
                    wins = [float(int(v)) / W for v in cwo.window_sums(d, W)]
                    assert len(wins) == max(0, (L - 1) // W)
                    assert repr(float(int(c[8])) / L) == want[name][0], (bam_label, label, W, name)
                    assert wins == unrle(want[name][1]), (bam_label, label, W, name)


def test_fixture_covers_the_cases_it_names(expected):
    from oracle import coverage_windows_oracle as cwo
    names, lens, cnt, deps = cwo.depths(BAMS['windows'])
    by = dict(zip(names, zip(lens, cnt.tolist(), deps)))
    assert by['w4'][1][0] == 0                                     # a reference without reads
    assert by['w8'][0] == 1 and by['w8'][1][8] == 1               # length 1, a read clipped to one base
    assert by['w1'][2][-1] > 0                                    # reads run up to the reference end
    assert by['w3'][1][0] == 2                                    # the two reads past its end are not fetched
    assert cnt[:, 1:8].sum(axis=0).min() > 0                    # every filter branch fires


def test_window_offsets():
    from checkm_b200.coverageWindows import window_offsets
    assert window_offsets([15000, 10001, 5000, 1, 5001], 5000).tolist() == [0, 2, 4, 4, 4, 5]
    assert window_offsets([7, 8, 1], 1).tolist() == [0, 6, 13, 13]
    assert window_offsets([], 100).tolist() == [0]


@pytest.mark.parametrize('W', [0, -5, 2.5])
def test_window_size_below_one_is_refused(tmp_path, caplog, W):
    from checkm_b200.coverageWindows import CoverageWindows
    caplog.set_level(logging.ERROR, logger='timestamp')
    with pytest.raises(SystemExit) as e:
        CoverageWindows(1).run([], BAMS['windows'], False, 0.98, 0.02, W)
    assert e.value.code == 1
    assert any('Window size must be a positive integer' in r.getMessage() for r in caplog.records)


def test_missing_index_exits_with_the_reference_message(tmp_path, caplog):
    from checkm_b200.coverageWindows import CoverageWindows
    noindex = str(tmp_path / 'noindex.bam')
    shutil.copyfile(BAMS['windows'], noindex)
    caplog.set_level(logging.ERROR, logger='timestamp')
    with pytest.raises(SystemExit) as e:
        CoverageWindows(1).run([], noindex, False, 0.98, 0.02, 5000)
    assert e.value.code == 1
    assert any(r.getMessage() == 'BAM file is not sorted: ' + noindex + '\n' for r in caplog.records)


def test_oracle_refuses_what_the_reference_raises_on(tmp_path):
    from oracle import coverage_windows_oracle as cwo
    from tools import bamsynth as bs
    rng = np.random.default_rng(5)
    for name, kw in (('nonm', dict(nm=None)), ('znm', dict(nm=None, aux=b'NMZ1\x00')), ('nocigar', dict(cigar=(), l_seq=100))):
        b, e = bs.record(rng, 0, 10, name, **kw)
        path = str(tmp_path / (name + '.bam'))
        bs.write_bam(path, [('chr', 5000)], [b], [0], [10], [e])
        with pytest.raises(ValueError, match=name):
            cwo.depths(path)


def test_package_never_imports_pysam():
    pkg = os.path.join(ROOT, 'checkm_b200')
    pat = re.compile(r'^\s*(import\s+pysam|from\s+pysam\s+import)|\bcheckm\.coverageWindows\b', re.M)
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith('.py'):
                with open(os.path.join(dirpath, f)) as fh:
                    assert not pat.search(fh.read()), f
