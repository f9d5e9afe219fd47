"""`checkm coverage`, CPU side: the host BGZF block walker (`ckm_bgzf_blocks`), the header, BAI and anchor readers against
the values the writer (tools/bamsynth.py) knows, the oracle against every coverage file the reference's own Coverage wrote
(tests/golden/coverage/, made by tests/golden/make_coverage_goldens.py), parseCoverage and binProfiles against the
reference's dicts, and the package's independence from pysam."""
import json
import os
import re
import shutil

import numpy as np
import pytest

from conftest import GOLDEN, ROOT

CV = os.path.join(GOLDEN, 'coverage')
BINS = [os.path.join(CV, 'bin1.fna'), os.path.join(CV, 'bin2.fna')]
BAMS = [os.path.join(CV, 'sample1.bam'), os.path.join(CV, 'sample2.bam')]


@pytest.fixture(scope='module')
def expected():
    with open(os.path.join(CV, 'expected.json')) as f:
        return json.load(f)


def _raw(name):
    with open(os.path.join(CV, name), 'rb') as f:
        return f.read()


@pytest.mark.parametrize('sample', ['sample1', 'sample2'])
def test_block_walker_matches_the_writer(expected, sample):
    from checkm_b200 import bam
    raw = _raw(sample + '.bam')
    blocks, used = bam.bgzf_blocks(raw)
    assert used == len(raw)
    assert [list(map(int, b)) for b in blocks.tolist()] == expected['known'][sample]['blocks']
    assert blocks['isize'][-1] == 0 and blocks['clen'][-1] == 28            # the EOF block


def test_block_walker_stops_at_the_last_whole_block(expected):
    from checkm_b200 import bam
    raw = _raw('sample1.bam')
    known = expected['known']['sample1']['blocks']
    for k, (c, n, _) in enumerate(known):
        for cut in (c + 1, c + 11, c + 17, c + n // 2, c + n - 1):
            blocks, used = bam.bgzf_blocks(np.frombuffer(raw[:cut], dtype=np.uint8))
            assert len(blocks) == k and used == c
        blocks, used = bam.bgzf_blocks(np.frombuffer(raw[:c + n], dtype=np.uint8))
        assert len(blocks) == k + 1 and used == c + n
    # a range that starts mid-file reports file offsets; cap limits the count
    c0 = known[5][0]
    blocks, used = bam.bgzf_blocks(np.frombuffer(raw[c0:], dtype=np.uint8), base=c0, cap=3)
    assert [list(map(int, b)) for b in blocks.tolist()] == known[5:8]
    assert used == known[8][0] - c0


def test_block_walker_refuses_a_header_that_is_not_bgzf(expected):
    from checkm_b200 import bam
    from checkm_b200._lib import CkmError
    raw = bytearray(_raw('sample1.bam'))
    c = expected['known']['sample1']['blocks'][7][0]
    for at, val in ((0, 0x1e), (3, 0x00), (12, ord('X'))):
        bad = bytearray(raw)
        bad[c + at] = val
        with pytest.raises(CkmError) as e:
            bam.bgzf_blocks(bad)
        assert e.value.code == 3 and 'file offset %d' % c in str(e.value)
    with pytest.raises(CkmError) as e:
        bam.bgzf_blocks(raw[:c] + b'plain text, not BGZF' * 2)
    assert e.value.code == 3


@pytest.mark.parametrize('sample', ['sample1', 'sample2'])
def test_header_index_and_anchors(expected, sample):
    from checkm_b200 import bam
    k = expected['known'][sample]
    lay = bam.Layout(os.path.join(CV, sample + '.bam'))
    try:
        assert lay.header.names == k['names'] and lay.header.lengths == k['lengths']
        assert lay.header.end == k['header_end']
        starts = set(k['record_starts'])
        assert lay.anchors[0] == k['header_end'] and set(lay.anchors[1:].tolist()) <= starts
        assert np.all(np.diff(lay.anchors) > 0)
        assert len(lay.anchors) > len(k['names'])                    # more than one window on the long contigs
        # the placed reads end where the unplaced tail begins: the index's pseudo-bins
        from oracle import coverage_oracle as co
        stream = co.inflate(os.path.join(CV, sample + '.bam'))
        p = lay.seg_end[-1]
        assert int.from_bytes(stream[p + 4:p + 8], 'little', signed=True) == -1
        assert lay.U[-1] == len(stream)
        # every segment starts on a record start and batches cut only at anchors
        for budget in (1 << 30, 20000, 1):
            segs = [(b0, b1, s, e) for b0, b1, s, e in lay.batches(budget)]
            got = np.concatenate([s + lay.U[b0] for b0, _, s, _ in segs])
            assert np.array_equal(got, lay.seg_start)
            for b0, b1, s, e in segs:
                assert e[-1] + lay.U[b0] <= lay.U[b1]
    finally:
        lay.close()


def test_index_of_another_file_is_refused(tmp_path):
    from checkm_b200 import bam
    from checkm_b200._lib import CkmError
    shutil.copyfile(BAMS[0], str(tmp_path / 'a.bam'))
    shutil.copyfile(BAMS[1] + '.bai', str(tmp_path / 'a.bam.bai'))
    with pytest.raises(CkmError) as e:
        bam.Layout(str(tmp_path / 'a.bam'))
    assert e.value.code == 3 and 'does not belong' in str(e.value)
    raw = _raw('sample1.bam')
    with open(str(tmp_path / 't.bam'), 'wb') as f:
        f.write(raw[:len(raw) // 2])
    shutil.copyfile(BAMS[0] + '.bai', str(tmp_path / 't.bam.bai'))
    with pytest.raises(CkmError) as e:
        bam.Layout(str(tmp_path / 't.bam'))
    assert e.value.code == 3


def test_oracle_matches_every_golden(expected):
    from oracle import coverage_oracle as co
    for label, o in expected['options'].items():
        got = co.coverage_tsv(BINS, BAMS, o['bAllReads'], o['minAlignPer'], o['maxEditDistPer'], o['minQC'])
        with open(os.path.join(CV, 'coverage_%s.tsv' % label)) as f:
            assert got == f.read(), label


def test_parse_coverage_and_bin_profiles(expected):
    from checkm_b200.coverage import Coverage
    cov = Coverage(1)
    assert cov.parseCoverage(os.path.join(CV, 'coverage_defaults.tsv')) == expected['parseCoverage']
    for label, want in expected['profiles'].items():
        prof = cov.binProfiles(os.path.join(CV, 'coverage_%s.tsv' % label))
        got = {b: {k: [repr(float(v[0])), repr(float(v[1]))] for k, v in d.items()} for b, d in prof.items()}
        assert got == want, label
        assert [[b, list(d.keys())] for b, d in prof.items()] == expected['profile_order'][label]


def test_package_never_imports_pysam():
    pkg = os.path.join(ROOT, 'checkm_b200')
    pat = re.compile(r'^\s*(import\s+pysam|from\s+pysam\s+import)|\bcheckm\.coverage\b', re.M)
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith('.py'):
                with open(os.path.join(dirpath, f)) as fh:
                    assert not pat.search(fh.read()), f
