"""`checkm coverage` on the device (checkm_b200.coverage.Coverage over ckm_bam_coverage, csrc/bam.cu): every coverage
file the reference's own Coverage wrote (tests/golden/coverage/) byte for byte, the inflate kernel against zlib over every
block type and strategy, the counters against the oracle on a seeded BAM of a few hundred MB, batching, and the error
returns for input that does not fit together."""
import logging
import os
import shutil
import zlib

import numpy as np
import pytest

from conftest import GOLDEN

pytestmark = pytest.mark.gpu
CV = os.path.join(GOLDEN, 'coverage')
BINS = [os.path.join(CV, 'bin1.fna'), os.path.join(CV, 'bin2.fna')]
BAMS = [os.path.join(CV, 'sample1.bam'), os.path.join(CV, 'sample2.bam')]
OPTS = {'defaults': (False, 0.98, 0.02, 15), 'all_reads': (True, 0.98, 0.02, 15), 'loose': (False, 0.5, 0.1, 0),
        'strict': (True, 0.99, 0.0, 30)}


def _run(tmp_path, label, threads=1, bams=BAMS):
    from checkm_b200.coverage import Coverage
    out = str(tmp_path / ('%s_%d.tsv' % (label, threads)))
    cov = Coverage(threads)
    cov.run(BINS, bams, out, *OPTS[label])
    with open(out) as f:
        return f.read(), cov


@pytest.mark.parametrize('threads', [1, 8])
@pytest.mark.parametrize('label', sorted(OPTS))
def test_coverage_file_matches_golden(tmp_path, label, threads):
    got, cov = _run(tmp_path, label, threads)
    with open(os.path.join(CV, 'coverage_%s.tsv' % label)) as f:
        assert got == f.read()
    assert cov.timing['batches'] == 2


def test_info_summary_matches_the_reference(tmp_path, capsys):
    import json
    with open(os.path.join(CV, 'expected.json')) as f:
        want = json.load(f)['summary']
    logger = logging.getLogger('timestamp')
    saved = logger.level
    logger.setLevel(logging.INFO)
    try:
        capsys.readouterr()
        _run(tmp_path, 'defaults')
        assert capsys.readouterr().out == want
    finally:
        logger.setLevel(saved)


def test_small_batches_give_the_same_bytes(tmp_path, monkeypatch):
    with open(os.path.join(CV, 'coverage_defaults.tsv')) as f:
        want = f.read()
    monkeypatch.setenv('CKM_BAM_BATCH_MB', '0.01')          # 10 kB: many cuts, and segments larger than the budget
    got, cov = _run(tmp_path, 'defaults')
    assert got == want
    assert cov.timing['batches'] > 10


def _blocks_of(payloads, level, strategy):
    """BGZF blocks of the payloads; one that does not fit a block at this level (65,536 stored bytes) is cut to 65,280."""
    from checkm_b200 import bam
    from tools import bamsynth as bs
    parts, used_payloads = [], []
    for p in payloads:
        try:
            parts.append(bs.bgzf_block(p, level, strategy))
        except ValueError:
            p = p[:bs.BLOCK_PAYLOAD]
            parts.append(bs.bgzf_block(p, level, strategy))
        used_payloads.append(p)
    raw = b''.join(parts)
    blocks, used = bam.bgzf_blocks(raw)
    assert used == len(raw)
    return raw, blocks, used_payloads


def _payloads(rng):
    out = [rng.integers(0, 256, size=65280, dtype=np.uint8).tobytes(),        # incompressible
           rng.choice(np.frombuffer(b'ACGT', dtype=np.uint8), size=65536).tobytes(),   # the largest ISIZE
           rng.choice(np.frombuffer(b'ACGT', dtype=np.uint8), size=60000).tobytes(),
           b'A' * 65280, b'', b'x',
           bytes(range(256)) * 255]
    half = rng.integers(0, 256, size=32768, dtype=np.uint8).tobytes()
    out.append(half + half[:32512])                                            # matches at the maximum distance 32768
    words = [rng.integers(97, 123, size=int(rng.integers(2, 12)), dtype=np.uint8).tobytes() for _ in range(200)]
    out.append(b' '.join(words[int(i)] for i in rng.integers(0, 200, size=9000))[:65000])
    out.append(np.repeat(rng.integers(0, 4, size=3000, dtype=np.uint8), rng.integers(1, 40, size=3000)).tobytes()[:65000])
    return out


def test_inflate_equals_zlib_on_every_level_and_strategy(engine):
    rng = np.random.default_rng(5)
    payloads = _payloads(rng)
    n = 0
    for level in range(10):
        for strategy in ('default', 'filtered', 'huffman', 'rle', 'fixed'):
            raw, blocks, used = _blocks_of(payloads, level, strategy)
            out, _ = engine.bgzf_inflate(raw, blocks)
            assert out.tobytes() == b''.join(used), (level, strategy)
            assert level == 0 or used == payloads
            n += 1
    assert n == 50


def test_inflate_equals_zlib_on_every_fixture_block(engine):
    from checkm_b200 import bam
    for path in BAMS:
        with open(path, 'rb') as f:
            raw = f.read()
        blocks, _ = bam.bgzf_blocks(raw)
        out, _ = engine.bgzf_inflate(raw, blocks)
        want = b''.join(zlib.decompress(raw[c + 18:c + n - 8], -15) for c, n, _ in blocks.tolist())
        assert out.tobytes() == want


def test_inflate_refuses_damaged_blocks(engine):
    from checkm_b200._lib import CkmError
    rng = np.random.default_rng(9)
    payloads = _payloads(rng)
    raw, blocks, _ = _blocks_of(payloads, 6, 'default')
    for k in (0, 3, 8):
        c, n, _ = blocks[k].tolist()
        for at in (n - 8, n - 5, 18, 18 + (n - 26) // 2, n - 9):
            bad = bytearray(raw)
            bad[c + at] ^= 0x5A
            with pytest.raises(CkmError) as e:
                engine.bgzf_inflate(bytes(bad), blocks)
            assert e.value.code == 3 and 'file offset %d' % c in str(e.value)


@pytest.fixture(scope='module')
def big_bam(tmp_path_factory):
    """~380 MB of records (1.3 M): 20,000 short contigs and 4 long contigs at high coverage, level-6 blocks, an unplaced tail."""
    from tools import bamsynth as bs
    rng = np.random.default_rng(2026)
    d = tmp_path_factory.mktemp('bigbam')
    short = rng.integers(1000, 20000, size=20000)
    long_ = np.array([2_000_000, 1_500_000, 3_000_000, 900_000])
    lens = np.concatenate([short[:10000], long_[:2], short[10000:], long_[2:]])
    reads = np.where(lens > 100000, lens // 12, lens // 300)            # ~12x and ~0.5x coverage of 150 bp reads
    body, ref, pos, end = bs.bulk_records(rng, lens, reads)
    tail = b''.join(bs.record(rng, -1, -1, 'tail%d' % i, flag=0x4, cigar=(), l_seq=150, nm=None)[0] for i in range(500))
    refs = [('ctg%d' % i, int(n)) for i, n in enumerate(lens)]
    path = str(d / 'big.bam')
    bs.write_bam(path, refs, body, ref, pos, end, np.zeros(len(ref), bool), n_unplaced=500, unplaced=tail, levels=(6,),
                 threads=os.cpu_count() or 1)
    return path, len(ref)


def test_counters_equal_the_oracle_at_scale(engine, big_bam):
    from checkm_b200 import bam
    from oracle import coverage_oracle as co
    path, nrec = big_bam
    names, lens, want = co.counters(path, False, 0.98, 0.02, 15)
    assert want[:, 0].sum() == nrec and want[:, 7].sum() > 0 and want[:, 1:7].min(axis=0).sum() >= 0
    for budget_mb in (None, 1):
        lay = bam.Layout(path)
        budget = (256 if budget_mb is None else budget_mb) << 20
        cnt = np.zeros((len(names), 9), dtype=np.int64)
        nb = 0
        for b0, b1, s, e in lay.batches(budget):
            comp, base = lay.comp(b0, b1)
            engine.bam_coverage(comp, lay.blocks[b0:b1], s, e, len(names), cnt, comp_base=base)
            nb += 1
        csize = int(lay.blocks['coffset'][-1])
        lay.close()
        assert np.array_equal(cnt, want), budget_mb
        if budget_mb == 1:
            assert nb >= csize // (1 << 20)
    for opts in ((True, 0.5, 0.1, 0), (False, 0.99, 0.0, 30)):
        names, lens, want = co.counters(path, *opts)
        lay = bam.Layout(path)
        cnt = np.zeros((len(names), 9), dtype=np.int64)
        for b0, b1, s, e in lay.batches(256 << 20):
            comp, base = lay.comp(b0, b1)
            engine.bam_coverage(comp, lay.blocks[b0:b1], s, e, len(names), cnt, comp_base=base, all_reads=opts[0],
                                min_align=opts[1], max_edit=opts[2], min_qc=opts[3])
        lay.close()
        assert np.array_equal(cnt, want), opts


def test_one_mib_batches_give_the_default_bytes(big_bam, tmp_path, monkeypatch):
    from checkm_b200.coverage import Coverage
    path, _ = big_bam
    outs, batches = [], []
    for mb in (None, '1'):
        if mb is None:
            monkeypatch.delenv('CKM_BAM_BATCH_MB', raising=False)
        else:
            monkeypatch.setenv('CKM_BAM_BATCH_MB', mb)
        cov = Coverage(1)
        out = str(tmp_path / ('cov_%s.tsv' % mb))
        cov.run([], [path], out, False, 0.98, 0.02, 15)
        with open(out, 'rb') as f:
            outs.append(f.read())
        batches.append((cov.timing['batches'], cov.timing['compressed_bytes']))
    assert outs[0] == outs[1]
    assert batches[0][0] == 1
    assert batches[1][0] >= os.path.getsize(path) // (1 << 20)


def _exit_with(tmp_path, caplog, bams, text):
    from checkm_b200.coverage import Coverage
    caplog.set_level(logging.ERROR, logger='timestamp')
    with pytest.raises(SystemExit) as e:
        Coverage(1).run(BINS, bams, str(tmp_path / 'out.tsv'), False, 0.98, 0.02, 15)
    assert e.value.code == 1
    assert any(text in r.getMessage() for r in caplog.records), [r.getMessage() for r in caplog.records]


def test_missing_index_exits_with_the_reference_message(tmp_path, caplog):
    noindex = str(tmp_path / 'noindex.bam')
    shutil.copyfile(BAMS[1], noindex)
    _exit_with(tmp_path, caplog, [BAMS[0], noindex], 'BAM file is either unsorted or not indexed: ' + noindex)


def test_foreign_index_truncated_file_and_bad_crc_are_format_errors(tmp_path, caplog):
    from checkm_b200 import bam
    shutil.copyfile(BAMS[0], str(tmp_path / 'a.bam'))
    shutil.copyfile(BAMS[1] + '.bai', str(tmp_path / 'a.bam.bai'))
    _exit_with(tmp_path, caplog, [str(tmp_path / 'a.bam')], 'libckm error 3')
    caplog.clear()
    with open(BAMS[0], 'rb') as f:
        raw = f.read()
    with open(str(tmp_path / 't.bam'), 'wb') as f:
        f.write(raw[:len(raw) * 2 // 3])
    shutil.copyfile(BAMS[0] + '.bai', str(tmp_path / 't.bam.bai'))
    _exit_with(tmp_path, caplog, [str(tmp_path / 't.bam')], 'libckm error 3')
    caplog.clear()
    blocks, _ = bam.bgzf_blocks(raw)
    c, n, _ = blocks[len(blocks) // 2].tolist()
    bad = bytearray(raw)
    bad[c + n - 7] ^= 0x01                                              # one CRC byte
    with open(str(tmp_path / 'c.bam'), 'wb') as f:
        f.write(bytes(bad))
    shutil.copyfile(BAMS[0] + '.bai', str(tmp_path / 'c.bam.bai'))
    _exit_with(tmp_path, caplog, [str(tmp_path / 'c.bam')], 'BGZF block at file offset %d: CRC32 mismatch' % c)


def test_a_walk_that_misses_an_anchor_and_a_read_without_nm_are_refused(engine, tmp_path):
    from checkm_b200 import bam
    from checkm_b200._lib import CkmError
    from tools import bamsynth as bs
    lay = bam.Layout(BAMS[0])
    (b0, b1, s, e), = list(lay.batches(1 << 30))
    comp, base = lay.comp(b0, b1)
    cnt = np.zeros((len(lay.header.names), 9), dtype=np.int64)
    with pytest.raises(CkmError) as x:                                  # a segment that starts one byte late
        engine.bam_coverage(comp, lay.blocks[b0:b1], s[:1] + 1, e[:1], len(cnt), cnt, comp_base=base)
    assert x.value.code == 3
    lay.close()
    rng = np.random.default_rng(3)
    recs = [bs.record(rng, 0, 10 * i, 'read%d' % i, nm=(0, 'C') if i != 7 else None) for i in range(20)]
    path = str(tmp_path / 'nonm.bam')
    bs.write_bam(path, [('chr', 5000)], [r[0] for r in recs], [0] * 20, [10 * i for i in range(20)], [r[1] for r in recs])
    lay = bam.Layout(path)
    (b0, b1, s, e), = list(lay.batches(1 << 30))
    comp, base = lay.comp(b0, b1)
    cnt = np.zeros((1, 9), dtype=np.int64)
    with pytest.raises(CkmError) as x:
        engine.bam_coverage(comp, lay.blocks[b0:b1], s, e, 1, cnt, comp_base=base)
    assert x.value.code == 3 and 'no integer NM tag in read read7' in str(x.value)
    lay.close()
