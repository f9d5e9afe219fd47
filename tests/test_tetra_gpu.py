"""Genomic signatures on the device (`checkm tetra`): `GenomicSignatures.calculate` writes, byte for byte, the profile files
the reference wrote for the fixtures; `ckm_kmer_counts` is held to a numpy sliding-window restatement on adversarial
layouts, at 48 MB, and on low-complexity sequence."""
import ctypes as C
import json
import os

import numpy as np
import pytest

from conftest import GOLDEN

pytestmark = pytest.mark.gpu

TT = os.path.join(GOLDEN, 'tetra')
FILES = {'fixture.fna': os.path.join(TT, 'fixture.fna')}
FILES.update({f: os.path.join(GOLDEN, 'binstats', 'bins', f) for f in ('bin1.fna', 'bin2.fna.gz', 'bin3.fna')})
NCOLS = {1: 2, 2: 10, 3: 32, 4: 136}


def _layout(seqs, pad_byte=0):
    lens = np.array([len(s) for s in seqs], dtype=np.int64)
    padded = (lens + 63) // 64 * 64
    starts = np.concatenate([[0], np.cumsum(padded)[:-1]]).astype(np.int64) if len(seqs) else np.zeros(0, dtype=np.int64)
    data = np.full(int(padded.sum()) + 64, pad_byte, dtype=np.uint8)
    for s, at in zip(seqs, starts):
        data[at:at + len(s)] = np.frombuffer(bytes(s), dtype=np.uint8)
    return data, starts, lens


def _numpy_counts(seqs, K):
    """Sliding windows over all sequences at once: a window counts if its K bytes are ACGT (either case) and lie in one
    sequence; its column is the rank of min(code, reverse-complement code) among the canonical codes."""
    code = np.full(256, 4, dtype=np.int64)
    for i, ch in enumerate(b'ACGT'):
        code[ch] = code[ch + 32] = i
    joined = np.frombuffer(b'\x00'.join(bytes(s) for s in seqs) + b'\x00' * K, dtype=np.uint8)
    seq_of = np.repeat(np.arange(len(seqs)), [len(s) + 1 for s in seqs])
    c = code[joined]
    n = len(seq_of)
    win = np.zeros(n, dtype=np.int64)
    ok = np.ones(n, dtype=bool)
    for j in range(K):
        win = win * 4 + c[j:j + n].clip(0, 3)
        ok &= c[j:j + n] < 4
    rc = np.zeros(1 << (2 * K), dtype=np.int64)
    for x in range(1 << (2 * K)):
        r, y = 0, x
        for _ in range(K):
            r = r * 4 + (3 - (y & 3))
            y >>= 2
        rc[x] = r
    canon = np.minimum(np.arange(1 << (2 * K)), rc)
    cols = np.unique(canon)
    col_of = np.searchsorted(cols, canon)
    out = np.bincount(seq_of[ok] * len(cols) + col_of[win[ok]], minlength=len(seqs) * len(cols))
    return out.reshape(len(seqs), len(cols))


def _check(engine, seqs, K=4, pad_byte=0):
    data, starts, lens = _layout(seqs, pad_byte)
    got, ms = engine.kmer_counts(data, starts, lens, K)
    want = _numpy_counts(seqs, K)
    bad = np.flatnonzero((got != want).any(axis=1))
    assert len(bad) == 0, ('sequences differ', bad[:10], [len(seqs[i]) for i in bad[:10]])
    return got, ms


def test_calculate_writes_the_reference_profiles(engine, tmp_path):
    from checkm_b200.genomicSignatures import GenomicSignatures
    for threads in (1, 8):
        for name, path in FILES.items():
            out = str(tmp_path / ('%s.%d.tsv' % (name, threads)))
            GenomicSignatures(4, threads).calculate(path, out)
            want = open(os.path.join(TT, name.replace('.gz', '') + '.tetra.tsv'), 'rb').read()
            assert open(out, 'rb').read() == want, (name, threads)
    # read() and distance() work on what calculate() wrote
    gs = GenomicSignatures(4, 1)
    sig = gs.read(str(tmp_path / 'bin1.fna.1.tsv'))
    assert len(sig) == 6 and gs.distance(sig['scaf_a'], sig['scaf_a']) == 0.0


def test_calculate_exits_on_an_unreadable_file(engine, tmp_path):
    from checkm_b200.genomicSignatures import GenomicSignatures
    with pytest.raises(SystemExit) as e:
        GenomicSignatures(4, 1).calculate(str(tmp_path / 'missing.fna'), str(tmp_path / 'out.tsv'))
    assert e.value.code == 1


def test_seq_signature_equals_the_reference(engine):
    from checkm_b200.genomicSignatures import GenomicSignatures
    want = json.load(open(os.path.join(TT, 'signatures.json')))['seqSignature']
    for K, cases in want.items():
        gs = GenomicSignatures(int(K), 1)
        for seq, values in cases:
            sig = gs.seqSignature(seq)
            assert sig.dtype == np.float64
            assert [repr(float(v)) for v in sig] == values, (K, seq)


def test_every_length_and_invalid_byte_offset(engine):
    rng = np.random.default_rng(1)
    for K in (1, 2, 3, 4):
        seqs = [rng.choice(np.frombuffer(b'ACGTacgt', dtype=np.uint8), size=n).tobytes() for n in range(301)]
        _check(engine, seqs, K)
        _check(engine, seqs, K, pad_byte=ord('A'))               # whatever the padding holds is not sequence
    # one invalid byte at every offset of a 64-byte chunk, of the 512-byte block around it, and of a 2 KB row edge
    seqs = []
    base = rng.choice(np.frombuffer(b'ACGT', dtype=np.uint8), size=6200)
    for at in list(range(0, 600)) + list(range(2030, 2070)) + list(range(4090, 4100)):
        for bad in b'NU*n':
            s = base.copy()
            s[at] = bad
            seqs.append(s.tobytes())
    for K in (1, 4):
        _check(engine, seqs, K)
        _check(engine, seqs[::5], K, pad_byte=ord('A'))


def test_200k_short_contigs(engine):
    rng = np.random.default_rng(2)
    lens = rng.integers(0, 400, size=200_000)
    pool = rng.choice(np.frombuffer(b'ACGTN', dtype=np.uint8), size=1 << 22, p=[0.249, 0.25, 0.25, 0.249, 0.002])
    offs = rng.integers(0, (1 << 22) - 400, size=len(lens))
    seqs = [pool[o:o + n].tobytes() for o, n in zip(offs, lens)]
    _check(engine, seqs, 4)
    _check(engine, seqs[::3], 3, pad_byte=ord('A'))


def test_48mb_sequence_across_many_warps(engine):
    rng = np.random.default_rng(3)
    big = rng.choice(np.frombuffer(b'ACGT', dtype=np.uint8), size=48 << 20).tobytes()
    seqs = [big] + [rng.choice(np.frombuffer(b'ACGT', dtype=np.uint8), size=int(n)).tobytes() for n in rng.integers(1, 30000, size=200)]
    for K in (1, 4):
        got, ms = _check(engine, seqs, K)
        assert int(got[0].sum()) == len(big) - K + 1
        print('K=%d: %.1f MB in %.3f ms = %.0f GB/s' % (K, sum(map(len, seqs)) / 1e6, ms, sum(map(len, seqs)) / ms / 1e6))


def test_low_complexity_16mb(engine):
    seqs = [b'A' * (8 << 20), b'AC' * (2 << 20), b'c' * 3_000_000, b'GATC' * 100_000] + [b'T' * 5000] * 200
    for K in (1, 2, 3, 4):
        got, ms = _check(engine, seqs, K)
        print('K=%d low complexity: %.3f ms' % (K, ms))


def test_bad_arguments_are_refused(engine):
    from checkm_b200 import _lib
    data, starts, lens = _layout([b'ACGT' * 100, b'ACGT'])
    out = np.zeros((2, 136), dtype=np.uint32)
    ms = C.c_float()
    L = _lib.lib()

    def call(st, k, nbytes=None):
        st = np.ascontiguousarray(st, dtype=np.int64)
        return L.ckm_kmer_counts(engine._h, data.ctypes.data, data.size if nbytes is None else nbytes, st.ctypes.data,
                                 lens.ctypes.data, 2, k, out.ctypes.data, C.byref(ms))
    assert call(starts, 4) == 0
    for k in (0, 5, -1):
        assert call(starts, k) == 1
        assert b'1..4' in L.ckm_last_error()
    assert call([0, 417], 4) == 1                                 # not a multiple of 64
    assert call([0, -64], 4) == 1
    assert call(starts, 4, nbytes=400) == 1                       # the second sequence lies outside the buffer
    with pytest.raises(ValueError):
        from checkm_b200.genomicSignatures import GenomicSignatures
        GenomicSignatures(5, 1)
