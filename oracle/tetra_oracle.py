"""CPU restatement of CheckM's genomic signatures (checkm/genomicSignatures.py:44-84,97-149) -- TEST INFRASTRUCTURE ONLY.

Only tests/ and bench legs that time a CPU baseline may import this; the product (checkm_b200/genomicSignatures.py) counts
on the device and never comes here.  Pinned: tests/test_tetra_cpu.py holds it to the profiles the reference's own
GenomicSignatures wrote for the fixtures (tests/golden/tetra/, made by tests/golden/make_tetra_goldens.py).

Plain string operations, one dict look-up per window, as in the reference."""
import numpy as np

from oracle.binstats_oracle import read_fasta  # noqa: F401  (util/seqUtils.py:180-211, shared with the bin statistics)

_COMPL = str.maketrans('ACGT', 'TGCA')


def rev_comp(seq):
    return seq.translate(_COMPL)[::-1]


def kmer_columns(K):
    """_makeKmerColNames: every K-mer in A<C<G<T order, each replaced by the smaller of it and its reverse complement, first
    occurrences kept."""
    mers = ['']
    for _ in range(K):
        mers = [m + c for m in mers for c in 'ACGT']
    cols = []
    for m in mers:
        c = min(m, rev_comp(m))
        if c not in cols:
            cols.append(c)
    return cols


def kmer_index(K):
    index = {}
    for i, c in enumerate(kmer_columns(K)):
        index[c] = i
        index[rev_comp(c)] = i
    return index


def kmer_counts(seq, K, index=None):
    """The integer half of seqSignature: counts of the canonical k-mers of seq.upper(); windows with other letters skipped."""
    index = index or kmer_index(K)
    sig = [0] * (max(index.values()) + 1)
    s = seq.upper()
    for i in range(len(s) - K + 1):
        j = index.get(s[i:i + K])
        if j is not None:
            sig[j] += 1
    return sig


def seq_signature(seq, K, index=None):
    """seqSignature: the counts divided by their sum (NaN where the sum is 0)."""
    sig = np.array(kmer_counts(seq, K, index), dtype=float)
    with np.errstate(invalid='ignore'):
        sig /= np.sum(sig)
    return sig


def profile_text(seqs, K):
    """_storeResults at threads=1: the header, then `id\\tv1\\t...` per sequence in the dict's order."""
    index = kmer_index(K)
    out = ['Sequence Id' + ''.join('\t' + c for c in kmer_columns(K)) + '\n']
    for seqId, seq in seqs.items():
        out.append(seqId + '\t' + '\t'.join(map(str, seq_signature(seq, K, index))) + '\n')
    return ''.join(out)
