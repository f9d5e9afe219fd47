"""Genomic signatures (tetranucleotide profiles, `checkm tetra`) behind the reference's GenomicSignatures interface
(checkm/genomicSignatures.py:34-200).  The profile file feeds `checkm outliers` (binTools.py:186-239) and the plots.

The per-base work -- the canonical k-mer counts of every sequence -- is one scan on the device per batch of about 512 MiB
of sequence (`ckm_kmer_counts`); the profile lines are written from the counts by the library's host formatter
(`ckm_format_kmer_profiles`), which prints each ratio exactly as the reference's `str(np.float64)` does, in up to `threads`
host threads.  There is no CPU path for the scan; K is limited to 1..4.

Sequences are written in file order.  The reference writes them in the order its worker processes finish, which is file
order only at threads=1; the lines themselves are the same."""
import ctypes as C
import logging
import sys
import threading
import time

import numpy as np

from . import _lib, runtime, seqio

BATCH_BYTES = 1 << 29           # sequence bytes scanned by one device call
_COLS = {1: 2, 2: 10, 3: 32, 4: 136}
_VALUE_BYTES = 24               # the longest value str(np.float64) prints for a ratio in [0, 1] is 23 characters, plus a tab


def kmer_columns(K):
    """The canonical k-mers of K in the reference's column order (ascending lexicographic)."""
    if K not in _COLS:
        raise ValueError('GenomicSignatures: K must lie in 1..4 (got %r)' % (K,))
    buf = C.create_string_buffer(K * _COLS[K])
    _lib.check(_lib.lib().ckm_kmer_columns(K, buf))
    raw = buf.raw.decode('ascii')
    return [raw[i:i + K] for i in range(0, len(raw), K)]


def format_profiles(counts, ids, K):
    """counts (n x C uint32) and the n ids -> the profile lines as bytes, one `id\\tv1\\t...\\tvC\\n` per sequence."""
    counts = np.ascontiguousarray(counts, dtype=np.uint32)
    n = len(ids)
    enc = [i.encode('utf-8') for i in ids]
    offsets = np.zeros(n + 1, dtype=np.int64)
    if n:
        offsets[1:] = np.cumsum([len(b) for b in enc])
    blob = b''.join(enc)
    cap = int(offsets[-1]) + n * (_COLS[K] * _VALUE_BYTES + 1)
    out = C.create_string_buffer(max(cap, 1))
    used = C.c_int64()
    _lib.check(_lib.lib().ckm_format_kmer_profiles(counts.ctypes.data if n else None, n, K, blob, offsets.ctypes.data, out,
                                                   cap, C.byref(used)))
    return out.raw[:used.value]


def parse_profiles(raw, ncols=136, threads=1):
    """The profile file's bytes -> the ids of its lines (in file order, repeats included) and their values as an
    n x ncols float64 matrix, each value what float() makes of its text (ckm_parse_kmer_profiles, up to `threads` host
    threads)."""
    cap = raw.count(b'\n') + 1
    starts = np.empty(cap, dtype=np.int64)
    id_lens = np.empty(cap, dtype=np.int32)
    values = np.empty((cap, ncols), dtype=np.float64)
    found = C.c_int64()
    _lib.check(_lib.lib().ckm_parse_kmer_profiles(raw, len(raw), ncols, max(1, int(threads or 1)), starts.ctypes.data,
                                                  id_lens.ctypes.data, values.ctypes.data, cap, C.byref(found)))
    n = found.value
    ids = [raw[a:a + k].decode('utf-8', 'replace') for a, k in zip(starts[:n].tolist(), id_lens[:n].tolist())]
    return ids, values[:n]


def _monotonic(data, starts, lens):
    """The layout with starts in increasing order (scan_nt_fasta keeps a repeated id in its first place but with its last
    record's bytes, so starts can go backwards)."""
    if len(starts) < 2 or np.all(np.diff(starts) > 0):
        return data, starts
    padded = (lens + 63) // 64 * 64
    new = np.concatenate([[0], np.cumsum(padded)[:-1]]).astype(np.int64)
    out = np.zeros(int(padded.sum()), dtype=np.uint8)
    for a, b, n in zip(starts, new, lens):
        out[b:b + n] = data[a:a + n]
    return out, new


class GenomicSignatures(object):
    """Canonical k-mer signatures of sequences (name, arguments and results of checkm.genomicSignatures.GenomicSignatures)."""

    def __init__(self, K, threads):
        self.logger = logging.getLogger('timestamp')
        self.K = K
        self.compl = str.maketrans('ACGT', 'TGCA')
        self.kmerCols = kmer_columns(K)
        self.kmerToCanonicalIndex = {}
        for index, kmer in enumerate(self.kmerCols):
            self.kmerToCanonicalIndex[kmer] = index
            self.kmerToCanonicalIndex[self._revComp(kmer)] = index
        self.totalThreads = threads
        self.timings = {}           # seconds of the last calculate(): read and layout, device calls, kernels, format and write

    def _revComp(self, seq):
        return seq.translate(self.compl)[::-1]

    def canonicalKmerOrder(self):
        return self.kmerCols

    def seqSignature(self, seq):
        """Frequencies of the canonical k-mers of one sequence (float64; NaN everywhere if no window counts)."""
        raw = seq.encode('latin-1', 'replace')
        n = len(raw)
        data = np.zeros((n + 63) // 64 * 64 + 64, dtype=np.uint8)
        data[:n] = np.frombuffer(raw, dtype=np.uint8)
        counts, _ = runtime.engine().kmer_counts(data, np.zeros(1, dtype=np.int64), np.array([n], dtype=np.int64), self.K)
        sig = np.array(counts[0], dtype=float)
        with np.errstate(invalid='ignore'):
            sig /= np.sum(sig)
        return sig

    def calculate(self, seqFile, outputFile):
        """Genomic signature of each sequence of seqFile -> outputFile (header `Sequence Id<TAB>kmers`, one line per sequence)."""
        self.logger.info('Determining tetranucleotide signature of each sequence.')
        t0 = time.perf_counter()
        try:
            ids, data, starts, lens = seqio.scan_nt_fasta(seqio.read_bytes(seqFile))
        except Exception as e:                        # util/seqUtils.py:205-209
            print(e)
            self.logger.error("Failed to process sequence file: {}".format(seqFile))
            sys.exit(1)
        data, starts = _monotonic(data, starts, lens)
        t_read = time.perf_counter() - t0
        t_dev = t_kernel = t_write = 0.0
        show = self.logger.getEffectiveLevel() <= logging.INFO
        total = len(ids)
        eng = runtime.engine()
        with open(outputFile, 'wb') as fout:
            fout.write(('Sequence Id' + ''.join('\t' + k for k in self.canonicalKmerOrder()) + '\n').encode())
            i0 = 0
            ends = starts + (lens + 63) // 64 * 64
            while i0 < total:
                i1 = int(np.searchsorted(ends, starts[i0] + BATCH_BYTES, side='right'))
                i1 = max(i1, i0 + 1)
                base = int(starts[i0])
                t1 = time.perf_counter()
                counts, ms = eng.kmer_counts(data[base:int(ends[i1 - 1])], starts[i0:i1] - base, lens[i0:i1], self.K)
                t2 = time.perf_counter()
                t_dev += t2 - t1
                t_kernel += ms / 1e3
                for chunk in self._format(counts, ids[i0:i1]):
                    fout.write(chunk)
                t_write += time.perf_counter() - t2
                i0 = i1
                if show:
                    sys.stderr.write('    Finished processing %d of %d (%.2f%%) sequences.\r' % (i0, total, float(i0) * 100 / total))
                    sys.stderr.flush()
        if show:
            sys.stderr.write('\n')
        self.timings = {'read_and_layout': t_read, 'device_calls': t_dev, 'kernels': t_kernel, 'format_and_write': t_write}

    def _format(self, counts, ids):
        """The lines of one batch, formatted in up to totalThreads host threads (the formatter releases the GIL)."""
        parts = max(1, min(int(self.totalThreads or 1), len(ids) // 256 or 1))
        cuts = [len(ids) * p // parts for p in range(parts + 1)]
        out = [None] * parts

        def work(p):
            out[p] = format_profiles(counts[cuts[p]:cuts[p + 1]], ids[cuts[p]:cuts[p + 1]], self.K)
        if parts == 1:
            work(0)
        else:
            threads = [threading.Thread(target=work, args=(p,)) for p in range(parts)]
            for t in threads:
                t.start()
            for t in threads:
                t.join()
        return out

    # ---- restated on the host, so that binTools and the plots work with this module ----
    def distance(self, sig1, sig2):
        return np.sum(np.abs(sig1 - sig2))

    def read(self, tetraProfileFile):
        sig = {}
        with open(tetraProfileFile) as f:
            next(f)
            for line in f:
                lineSplit = line.split('\t')
                sig[lineSplit[0]] = np.array([float(x) for x in lineSplit[1:]])
        return sig
