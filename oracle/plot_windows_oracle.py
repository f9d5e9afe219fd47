"""CPU restatement of the plots' window statistics (checkm/plot/*.py) -- TEST INFRASTRUCTURE ONLY; the product computes
them with ckm_window_stats (checkm_b200/csrc/windows.cu) and never comes here.

Per window [kW, (k+1)W) of a sequence, for k while (k+1)W < len: the A, C, G, T(+U) counts of the upper-cased bytes; the
canonical 4-mer counts of the 4-mers wholly inside it (A/C/G/T only, U not T), their frequencies and the distance to a bin
signature summed in numpy's pairwise order; and the coding bases as the sum of a literal numpy mask built as prodigal.py
builds it.  Plain Python loops, so every count and the order of every sum is written out here."""
import numpy as np

from oracle.outliers_oracle import pairwise_sum

_CODE = {'A': 0, 'C': 1, 'G': 2, 'T': 3}


def _revcomp(x):
    r = 0
    for _ in range(4):
        r = (r << 2) | ((x & 3) ^ 3)
        x >>= 2
    return r


_CANON = sorted(x for x in range(256) if x <= _revcomp(x))
_COLUMN = {x: _CANON.index(min(x, _revcomp(x))) for x in range(256)}


def windows(length, W):
    return [(k * W, (k + 1) * W) for k in range(max(length - 1, 0) // W)]


def base_counts(window):
    up = window.upper()
    return up.count('A'), up.count('C'), up.count('G'), up.count('T') + up.count('U')


def kmer_counts(window):
    counts = [0] * 136
    up = window.upper()
    for i in range(len(up) - 3):
        code = 0
        for ch in up[i:i + 4]:
            if ch not in _CODE:
                code = None
                break
            code = (code << 2) | _CODE[ch]
        if code is not None:
            counts[_COLUMN[code]] += 1
    return counts


def distance(counts, bin_sig):
    total = float(sum(counts))
    sig = [c / total if total else float('nan') for c in counts]
    return pairwise_sum([abs(s - b) for s, b in zip(sig, bin_sig)])


def coding_mask(genes, last):
    """prodigal.py:250-261: zeros of length `last`, mask[start-1:end] = 1 per (start, end)."""
    mask = np.zeros(last)
    for start, end in genes:
        mask[start - 1:end] = 1
    return mask


def window_stats(seq, W, bin_sig=None):
    """[(a, c, g, t, distance or None)] for every window of seq."""
    out = []
    for lo, hi in windows(len(seq), W):
        w = seq[lo:hi]
        out.append(base_counts(w) + ((distance(kmer_counts(w), bin_sig) if bin_sig is not None else None),))
    return out


def synthetic_coverage(seq_lens, W):
    """A coverage profile for gc_bias_plot's goldens, {seqId: [coverage, window coverages]} with (L - 1) // W windows per
    sequence of `seq_lens` ({seqId: length}, in the bin's order).  The values are a few exact binary fractions, so the tests
    make the same profile again and the recorded call logs stay small."""
    out = {}
    for i, (seq_id, length) in enumerate(seq_lens.items()):
        out[seq_id] = [1.0 + (i * 7 % 23) / 4.0, [((i * 13 + k * 5) % 61) / 8.0 for k in range(max(length - 1, 0) // W)]]
    return out
