"""Read depth per window on the device (checkm_b200.coverageWindows.CoverageWindows over ckm_bam_windows, csrc/bam.cu):
every value the reference's own CoverageWindows returned (tests/golden/coverage_windows/) bit for bit, the INFO summary,
batching, the integer window sums against the oracle on about a million seeded records, and the refusals."""
import gzip
import json
import logging
import os
import shutil

import numpy as np
import pytest

from conftest import GOLDEN

pytestmark = pytest.mark.gpu
CW = os.path.join(GOLDEN, 'coverage_windows')
BAMS = {'windows': os.path.join(CW, 'windows.bam'), 'sample1': os.path.join(GOLDEN, 'coverage', 'sample1.bam'),
        'sample2': os.path.join(GOLDEN, 'coverage', 'sample2.bam')}


@pytest.fixture(scope='module')
def expected():
    with gzip.open(os.path.join(CW, 'expected.json.gz'), 'rt') as f:
        return json.load(f)


def unrle(runs):
    return [float(v) for v, n in runs for _ in range(n)]


def _run(path, o, W):
    from checkm_b200.coverageWindows import CoverageWindows
    cw = CoverageWindows(1)
    return cw.run([], path, o['bAllReads'], o['minAlignPer'], o['maxEditDistPer'], W), cw


def _assert_equal(got, want):
    assert list(got) == list(want)
    for name, (cov, wins) in got.items():
        assert type(cov) is float and cov == float(want[name][0]), name
        ref = unrle(want[name][1])
        assert len(wins) == len(ref), name
        assert all(type(v) is float for v in wins)
        assert wins == ref, name


@pytest.mark.parametrize('bam_label', sorted(BAMS))
def test_values_equal_the_reference_bit_for_bit(expected, bam_label):
    for label, o in expected['options'].items():
        for W in expected['windows']:
            got, cw = _run(BAMS[bam_label], o, W)
            _assert_equal(got, expected['values'][bam_label][label][str(W)])
            assert cw.timing['batches'] == 1


def test_info_summary_matches_the_reference(expected, capsys):
    logger = logging.getLogger('timestamp')
    saved = logger.level
    logger.setLevel(logging.INFO)
    try:
        capsys.readouterr()
        _run(BAMS['windows'], expected['options']['defaults'], 5000)
        assert capsys.readouterr().out == expected['summary']
    finally:
        logger.setLevel(saved)


@pytest.mark.parametrize('mb', ['1', '0.01'])
def test_small_batches_give_the_same_values(expected, monkeypatch, mb):
    monkeypatch.setenv('CKM_BAM_BATCH_MB', mb)
    for bam_label in ('windows', 'sample1'):
        for W in (1, 100):
            got, cw = _run(BAMS[bam_label], expected['options']['loose'], W)
            _assert_equal(got, expected['values'][bam_label]['loose'][str(W)])
            if mb == '0.01':
                assert cw.timing['batches'] > 3


# ---- about a million seeded records against the oracle ----
def _write(d, name, lens, reads, seed):
    from tools import bamsynth as bs
    rng = np.random.default_rng(seed)
    body, ref, pos, end = bs.bulk_records(rng, lens, reads)
    tail = b''.join(bs.record(rng, -1, -1, 'tail%d' % i, flag=0x4, cigar=(), l_seq=150, nm=None)[0] for i in range(50))
    refs = [('ctg%d' % i, int(n)) for i, n in enumerate(lens)]
    path = str(d / name)
    bs.write_bam(path, refs, body, ref, pos, end, np.zeros(len(ref), bool), n_unplaced=50, unplaced=tail, levels=(6,),
                 threads=os.cpu_count() or 1)
    return path, len(ref)


@pytest.fixture(scope='module')
def big_bams(tmp_path_factory):
    """Short contigs (40,000 of 300-3,000 bp, ~1x) and long contigs (4, 6 Mbp in all, ~12x): ~0.94 M records."""
    d = tmp_path_factory.mktemp('cwbig')
    rng = np.random.default_rng(2027)
    short = rng.integers(300, 3000, size=40000)
    long_ = np.array([2_000_000, 1_500_000, 1_600_000, 900_000])
    return {'short': _write(d, 'short.bam', short, short // 150, 11),
            'long': _write(d, 'long.bam', long_, long_ // 12, 12)}


@pytest.mark.parametrize('shape', ['short', 'long'])
def test_window_sums_equal_the_oracle_at_scale(engine, big_bams, shape):
    from checkm_b200 import bam
    from checkm_b200.coverageWindows import window_offsets
    from oracle import coverage_windows_oracle as cwo
    path, nrec = big_bams[shape]
    names, lens, want_cnt, deps = cwo.depths(path)
    assert 0 < want_cnt[:, 0].sum() <= nrec and want_cnt[:, 7].sum() > 0
    for W in (1, 100, 5000):
        want = np.concatenate([cwo.window_sums(dp, W) for dp in deps] + [np.zeros(0, np.int64)])
        off = window_offsets(lens, W)
        lay = bam.Layout(path)
        cnt = np.zeros((len(names), 9), dtype=np.int64)
        win = np.zeros(int(off[-1]), dtype=np.int64)
        for b0, b1, s, e in lay.batches(64 << 20):
            comp, base = lay.comp(b0, b1)
            engine.bam_windows(comp, lay.blocks[b0:b1], s, e, lens, W, off, cnt, win, comp_base=base)
        lay.close()
        assert np.array_equal(cnt, want_cnt), W
        assert np.array_equal(win, want), W


# ---- refusals ----
def _one_batch(path):
    from checkm_b200 import bam
    lay = bam.Layout(path)
    (b0, b1, s, e), = list(lay.batches(1 << 30))
    comp, base = lay.comp(b0, b1)
    out = (comp.copy(), lay.blocks[b0:b1].copy(), s, e, base, list(lay.header.lengths))
    lay.close()
    return out


def _refused(engine, path, W=100, lens=None):
    from checkm_b200._lib import CkmError
    from checkm_b200.coverageWindows import window_offsets
    comp, blocks, s, e, base, hl = _one_batch(path)
    lens = hl if lens is None else lens
    off = window_offsets(lens, max(W, 1))
    cnt = np.zeros((len(lens), 9), dtype=np.int64)
    win = np.zeros(max(int(off[-1]), 1), dtype=np.int64)
    with pytest.raises(CkmError) as x:
        engine.bam_windows(comp, blocks, s, e, lens, W, off, cnt, win, comp_base=base)
    return x.value


def _bam_with(tmp_path, name, target, **kw):
    """chr (5,000 bp): reads read0..read5 at 100, 200, ... with `target` at position kw.pop('pos', 300)."""
    from tools import bamsynth as bs
    rng = np.random.default_rng(9)
    at = kw.pop('pos', 300)
    recs = [bs.record(rng, 0, p, 'read%d' % p) for p in (100, 200, 400, 500)] + [bs.record(rng, 0, at, target, **kw)]
    pos = [100, 200, 400, 500, at]
    order = np.argsort(pos, kind='stable')
    path = str(tmp_path / (name + '.bam'))
    bs.write_bam(path, [('chr', 5000)], [recs[i][0] for i in order], [0] * 5, [pos[i] for i in order],
                 [recs[i][1] for i in order])
    return path


@pytest.mark.parametrize('case,kw', [
    ('absent', dict(nm=None)),
    ('type_A', dict(nm=None, aux=b'NMAx')),
    ('type_Z', dict(nm=None, aux=b'NMZ1\x00')),
    ('type_H', dict(nm=None, aux=b'NMH0A\x00')),
    ('type_B', dict(nm=None, aux=b'NMBC\x01\x00\x00\x00\x01')),
])
def test_a_read_without_a_numeric_nm_is_refused(engine, tmp_path, case, kw):
    err = _refused(engine, _bam_with(tmp_path, case, 'bad_' + case, **kw))
    assert err.code == 3 and 'no numeric NM tag' in str(err) and 'in read bad_' + case in str(err)


def test_a_read_without_a_cigar_and_a_negative_position_are_refused(engine, tmp_path):
    err = _refused(engine, _bam_with(tmp_path, 'nocig', 'no_cigar', cigar=(), l_seq=100))
    assert err.code == 3 and 'no CIGAR' in str(err) and 'in read no_cigar' in str(err)
    err = _refused(engine, _bam_with(tmp_path, 'neg', 'negative', pos=-5))
    assert err.code == 3 and 'negative position' in str(err) and 'in read negative' in str(err)


def test_bad_window_size_zero_length_and_an_array_too_large_are_refused(engine, tmp_path):
    path = _bam_with(tmp_path, 'ok', 'fine')
    err = _refused(engine, path, W=0)
    assert err.code == 1 and 'window size 0' in str(err)
    err = _refused(engine, path, lens=[0])
    assert err.code == 1 and 'length 0' in str(err)
    # 400 references of 2^31 - 1 bp at W = 1: 6.4 TiB of windows.  The array is refused before it is allocated, so the
    # call goes to the library directly with a one-element host array.
    import ctypes as C
    from checkm_b200 import _lib
    from checkm_b200.coverageWindows import window_offsets
    comp, blocks, s, e, base, _ = _one_batch(path)
    lens = np.full(400, (1 << 31) - 1, dtype=np.int64)
    off = window_offsets(lens, 1)
    cnt = np.zeros((400, 9), dtype=np.int64)
    win = np.zeros(1, dtype=np.int64)
    s, e = np.ascontiguousarray(s, dtype=np.int64), np.ascontiguousarray(e, dtype=np.int64)
    filt = _lib.BamFilter(0, 0, 0.98, 0.02)
    rc = _lib.lib().ckm_bam_windows(engine._h, comp.ctypes.data, int(base), comp.size, blocks.ctypes.data, len(blocks),
                                    s.ctypes.data, e.ctypes.data, len(s), 400, C.byref(filt), lens.ctypes.data, 1,
                                    off.ctypes.data, cnt.ctypes.data, win.ctypes.data, None, None)
    msg = _lib.lib().ckm_last_error().decode()
    assert rc == 6 and 'the smallest window size that fits is' in msg, msg
    smallest = int(msg.rsplit(' ', 1)[1])
    assert 2 <= smallest and 400 * (((1 << 31) - 2) // smallest) * 8 <= 80 << 30
    assert not cnt.any() and not win.any()


def test_foreign_index_and_truncated_file_are_format_errors(tmp_path, caplog):
    from checkm_b200.coverageWindows import CoverageWindows
    caplog.set_level(logging.ERROR, logger='timestamp')
    shutil.copyfile(BAMS['sample1'], str(tmp_path / 'a.bam'))
    shutil.copyfile(BAMS['sample2'] + '.bai', str(tmp_path / 'a.bam.bai'))
    with open(BAMS['sample1'], 'rb') as f:
        raw = f.read()
    with open(str(tmp_path / 't.bam'), 'wb') as f:
        f.write(raw[:len(raw) * 2 // 3])
    shutil.copyfile(BAMS['sample1'] + '.bai', str(tmp_path / 't.bam.bai'))
    for name in ('a.bam', 't.bam'):
        caplog.clear()
        with pytest.raises(SystemExit) as e:
            CoverageWindows(1).run([], str(tmp_path / name), False, 0.98, 0.02, 5000)
        assert e.value.code == 1
        assert any('libckm error 3' in r.getMessage() for r in caplog.records), name
