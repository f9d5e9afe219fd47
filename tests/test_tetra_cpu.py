"""Genomic signatures (`checkm tetra`), CPU side: the library's profile writer (host code, no device) against numpy's own
`str(np.float64)` and against the profile files the reference's GenomicSignatures wrote; the oracle port and the column
order against the goldens (tests/golden/tetra/, made by tests/golden/make_tetra_goldens.py)."""
import json
import os

import numpy as np

from conftest import GOLDEN

TT = os.path.join(GOLDEN, 'tetra')
FILES = {'fixture.fna': os.path.join(TT, 'fixture.fna')}
FILES.update({f: os.path.join(GOLDEN, 'binstats', 'bins', f) for f in ('bin1.fna', 'bin2.fna.gz', 'bin3.fna')})


def _golden(name):
    return open(os.path.join(TT, name.replace('.gz', '') + '.tetra.tsv')).read()


def _format_pairs(c, t):
    """The writer at K = 1 (two columns) with counts (c, t - c): its first column is c / t."""
    from checkm_b200.genomicSignatures import format_profiles
    counts = np.stack([c, t - c], axis=1).astype(np.uint32)
    text = format_profiles(counts, ['s'] * len(c), 1).decode()
    return [line.split('\t')[1] for line in text.splitlines()]


def test_writer_prints_values_as_numpy_does():
    t = np.concatenate([np.full(k + 1, k, dtype=np.int64) for k in range(2001)])
    c = np.concatenate([np.arange(k + 1, dtype=np.int64) for k in range(2001)])
    got = _format_pairs(c, t)
    with np.errstate(invalid='ignore'):
        want = [str(v) for v in np.float64(c) / np.float64(t)]          # t = 0: 0/0 -> nan
    assert got == want
    rng = np.random.default_rng(99)
    t = rng.integers(1, 1 << 32, size=1_000_000, dtype=np.int64)
    c = (rng.random(1_000_000) * (t + 1)).astype(np.int64).clip(0, t)
    c[:1000] = rng.integers(0, 4, size=1000)                            # tiny ratios: the 1e-05 layout
    got = _format_pairs(c, t)
    want = [str(v) for v in np.float64(c) / np.float64(t)]
    assert got == want


def test_writer_reproduces_the_golden_profiles():
    from oracle import tetra_oracle as to
    from checkm_b200.genomicSignatures import format_profiles, kmer_columns
    index = to.kmer_index(4)
    for name, path in FILES.items():
        seqs = to.read_fasta(path)
        counts = np.array([to.kmer_counts(s, 4, index) for s in seqs.values()], dtype=np.uint32).reshape(len(seqs), 136)
        text = 'Sequence Id' + ''.join('\t' + k for k in kmer_columns(4)) + '\n'
        text += format_profiles(counts, list(seqs.keys()), 4).decode()
        assert text == _golden(name), name


def test_oracle_reproduces_the_goldens():
    from oracle import tetra_oracle as to
    for name, path in FILES.items():
        assert to.profile_text(to.read_fasta(path), 4) == _golden(name), name
    want = json.load(open(os.path.join(TT, 'signatures.json')))['seqSignature']
    for K, cases in want.items():
        for seq, values in cases:
            assert [repr(float(v)) for v in to.seq_signature(seq, int(K))] == values, (K, seq)


def test_canonical_orders():
    from oracle import tetra_oracle as to
    from checkm_b200.genomicSignatures import kmer_columns
    want = json.load(open(os.path.join(TT, 'signatures.json')))['order']
    for K in (1, 2, 3, 4):
        assert kmer_columns(K) == want[str(K)] == to.kmer_columns(K) == sorted(want[str(K)])
        assert len(want[str(K)]) == (2, 10, 32, 136)[K - 1]


def test_writer_and_columns_refuse_bad_arguments():
    import ctypes as C
    import pytest
    from checkm_b200 import _lib
    from checkm_b200.genomicSignatures import kmer_columns
    for K in (0, 5):
        with pytest.raises(ValueError):
            kmer_columns(K)
        assert _lib.lib().ckm_kmer_columns(K, C.create_string_buffer(1024)) == 1          # CKM_EINVAL
    counts = np.array([[1, 2]], dtype=np.uint32)
    offsets = np.array([0, 1], dtype=np.int64)
    used = C.c_int64()
    out = C.create_string_buffer(4)
    rc = _lib.lib().ckm_format_kmer_profiles(counts.ctypes.data, 1, 1, b's', offsets.ctypes.data, out, 4, C.byref(used))
    assert rc == 8 and used.value == len('s\t0.3333333333333333\t0.6666666666666666\n')       # CKM_ECAPACITY, size needed
    assert _lib.lib().ckm_format_kmer_profiles(counts.ctypes.data, 1, 5, b's', offsets.ctypes.data, out, 4, C.byref(used)) == 1
