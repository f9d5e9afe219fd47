"""The layout check that the three nucleotide scans share (csrc/ntrows.cuh, nt_check_layout): ckm_scaffold_stats,
ckm_kmer_counts and ckm_window_stats each refuse a sequence the row list cannot describe, with CKM_EINVAL and a message
that names the call."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def _layout(seqs):
    lens = np.array([len(s) for s in seqs], dtype=np.int64)
    padded = (lens + 63) // 64 * 64
    starts = np.concatenate([[0], np.cumsum(padded)[:-1]]).astype(np.int64)
    data = np.zeros(int(padded.sum()) + 64, dtype=np.uint8)
    for s, at in zip(seqs, starts):
        data[at:at + len(s)] = np.frombuffer(s, dtype=np.uint8)
    return data, starts, lens


@pytest.mark.parametrize('scan, noun', [('scaffold_stats', 'scaffold'), ('kmer_counts', 'sequence'), ('window_stats', 'sequence')])
def test_every_scan_refuses_a_bad_layout(engine, scan, noun):
    """A start that is not a multiple of 64, a negative start and a sequence past the end of the buffer."""
    from checkm_b200._lib import CkmError
    from checkm_b200.coverageWindows import window_offsets
    data, starts, lens = _layout([b'ACGT' * 100, b'ACGT'])

    def call(st, nbytes):
        if scan == 'window_stats':
            return engine.window_stats(data[:nbytes], st, lens, 7, window_offsets(lens, 7))
        return getattr(engine, scan)(data[:nbytes], st, lens)
    call(starts, data.size)
    for st, nbytes in (([0, 417], data.size), ([0, -64], data.size), (starts, 400)):
        with pytest.raises(CkmError) as e:
            call(np.array(st, dtype=np.int64), nbytes)
        assert e.value.code == 1
        assert 'ckm_%s: every %s must start at a multiple of 64 bytes' % (scan, noun) in str(e.value), str(e.value)
