"""Unbinned sequences (`checkm unbinned`) behind the reference's Unbinned interface (checkm/unbinned.py:29-85).

The reference reads every bin and the assembly into dicts and tests each assembly id against the binned ones, then counts
the bases of every unbinned sequence with str.count.  Here each file is cut into records by the library's line scan
(`ckm_fasta_scan_nt`), the ids of all records of all files are joined in one device call (`ckm_id_join`, csrc/idjoin.cu),
the bases of the kept sequences are counted by the scaffold scan (`ckm_scaffold_stats`) in batches of device memory, and
both output files are written by the library's host formatter (`ckm_format_unbinned`, the reference's '%.2f').  No step
loops over records in Python.

Where the reference stops with an uncaught exception, an error naming the file or the sequence is logged and the run
exits with status 1: a kept sequence without A/C/G/T/U (ZeroDivisionError), an assembly without records, an assembly
without bases.  Files the reference's readFasta cannot read (not UTF-8, sequence before the first header, a header
without an id) exit 1 with its own message.  One deliberate difference: a file with non-ASCII bytes in a sequence line is
refused the same way, because the reference measures such a sequence in characters and the scan in bytes."""
import ctypes as C
import logging
import sys
import time

import numpy as np

from . import _lib, runtime, seqio
from .binStatistics import BATCH_BYTES
from .common import checkFileExists

STATS_HEADER = 'Sequence Id\tLength\tGC\n'


def format_records(text, id_start, id_len, data, starts, lens, acgt):
    """The FASTA and the stats rows of records (ids in `text`, sequences in `data`) as two bytes objects."""
    id_start, id_len, starts, lens = (np.ascontiguousarray(a, dtype=np.int64) for a in (id_start, id_len, starts, lens))
    acgt = np.ascontiguousarray(acgt, dtype=np.int64)
    data = np.ascontiguousarray(data, dtype=np.uint8)
    n = len(lens)
    fcap = int(id_len.sum() + lens.sum()) + 3 * n
    scap = int(id_len.sum()) + 48 * n
    fout, sout = np.empty(max(fcap, 1), dtype=np.uint8), np.empty(max(scap, 1), dtype=np.uint8)
    fw, sw = C.c_int64(), C.c_int64()
    _lib.check(_lib.lib().ckm_format_unbinned(text, id_start.ctypes.data, id_len.ctypes.data,
                                              data.ctypes.data if data.size else None, starts.ctypes.data, lens.ctypes.data,
                                              acgt.ctypes.data, n, fout.ctypes.data, fcap, sout.ctypes.data, scap,
                                              C.byref(fw), C.byref(sw)))
    return fout[:fw.value].tobytes(), sout[:sw.value].tobytes()


class Unbinned():
    def __init__(self):
        self.logger = logging.getLogger('timestamp')
        self.timing = {}                  # seconds per phase of the last run, and the kernels' milliseconds

    def _fail(self, message):
        self.logger.error(message)
        sys.exit(1)

    def _read(self, fastaFile):
        """One file's bytes, or the reference's readFasta failure (seqUtils.py:205-209)."""
        try:
            raw = seqio.read_bytes(fastaFile)
            if not raw.isascii():
                raw.decode('utf-8')
            return raw
        except Exception as e:
            print(e)
            self._fail("Failed to process sequence file: {}".format(fastaFile))

    def _scan(self, fastaFile, raw):
        """One file as seqio.scan_nt_raw lays it out, or the reference's readFasta failure."""
        try:
            scan = seqio.scan_nt_raw(raw)
            if not raw.isascii() and not scan[1].tobytes().isascii():
                raise ValueError('non-ASCII bytes in a sequence line')
            return scan
        except Exception as e:
            print(e)
            self._fail("Failed to process sequence file: {}".format(fastaFile))

    def _count(self, data, starts, lens):
        """A, C, G, T+U of the sequences data[starts:starts+lens] (n x 4), in device calls of at most BATCH_BYTES."""
        n = len(lens)
        acgt = np.zeros((n, 4), dtype=np.int64)
        order = np.argsort(starts, kind='stable')
        s, ln = starts[order], lens[order]
        ends = s + ln
        eng = runtime.engine()
        i0 = 0
        while i0 < n:
            i1 = max(i0 + 1, int(np.searchsorted(ends, s[i0] + BATCH_BYTES, side='right')))
            lo, hi = int(s[i0]), int((ends[i1 - 1] + 63) // 64 * 64)
            stats, _, _, ms = eng.scaffold_stats(data[lo:hi], s[i0:i1] - lo, ln[i0:i1])
            acgt[order[i0:i1]] = stats[:, :4]
            self.timing['count_ms'] += ms
            self.timing['count_calls'] += 1
            i0 = i1
        return acgt

    def run(self, binFiles, seqFile, outSeqFile, outStatsFile, minSeqLen):
        checkFileExists(seqFile)
        self.timing = {'read': 0.0, 'scan': 0.0, 'device': 0.0, 'write': 0.0, 'join_ms': 0.0, 'count_ms': 0.0, 'count_calls': 0}

        self.logger.info('Reading binned sequences.')
        t0 = time.perf_counter()
        files = list(binFiles) + [seqFile]
        raws = [self._read(f) for f in files]
        t1 = time.perf_counter()
        scans = [self._scan(f, raw) for f, raw in zip(files, raws)]
        del raws
        bins, (hdr, data, starts, lens) = scans[:-1], scans[-1]
        bin_nrec = np.array([len(b[3]) for b in bins], dtype=np.int64)
        text = b''.join(b[0] + b'\n' for b in scans if len(b[3]))
        eng = runtime.engine()
        t2 = time.perf_counter()
        try:
            id_start, id_len, flags, last, keep, nBinned, join_ms = eng.id_join(text, bin_nrec, len(lens))
        except _lib.CkmError as e:
            if e.record < 0:
                raise
            print(e)
            f = int(np.searchsorted(np.cumsum(bin_nrec), e.record, side='right'))
            self._fail("Failed to process sequence file: {}".format(files[f]))
        t3 = time.perf_counter()
        self.timing['join_ms'] = join_ms
        nb = int(bin_nrec.sum())
        bin_lens = np.concatenate([b[3] for b in bins]) if bins else np.zeros(0, dtype=np.int64)
        totalBinnedBases = int(bin_lens[keep].sum())
        self.logger.info('  Read %d (%.2f Mbp) binned sequences.' % (nBinned, float(totalBinnedBases) / 1e6))

        self.logger.info('Reading all sequences.')
        entries = np.flatnonzero(flags & 2)                  # the dict's keys, in dict order
        content = last[entries]                              # the record that supplies each key's sequence
        totalBases = int(lens[content].sum())
        self.logger.info('  Read %d (%.2f Mbp) sequences.' % (len(entries), float(totalBases) / 1e6))

        self.logger.info('Identifying unbinned sequences >= %d bp.' % minSeqLen)
        kept = (flags[entries] & 1) == 0
        kept &= lens[content] >= minSeqLen
        kept_ids, src = entries[kept] + nb, content[kept]
        unbinnedCount, unbinnedBases = len(src), int(lens[src].sum())
        t4c = time.perf_counter()
        acgt = self._count(data, starts[src], lens[src])
        t4 = time.perf_counter()
        empty = np.flatnonzero(acgt.sum(axis=1) == 0)
        if len(empty):
            r = kept_ids[empty[0]]
            seqId = text[id_start[r]:id_start[r] + id_len[r]].decode('utf-8')
            self._fail('Sequence %s in %s has no A, C, G, T or U bases, so its GC content is undefined.' % (seqId, seqFile))
        with open(outSeqFile, 'wb') as seqOut, open(outStatsFile, 'wb') as statsOut:
            statsOut.write(STATS_HEADER.encode())
            i0, ends = 0, np.cumsum(lens[src])
            while i0 < unbinnedCount:                        # output in pieces of about BATCH_BYTES of sequence
                i1 = max(i0 + 1, int(np.searchsorted(ends, (ends[i0 - 1] if i0 else 0) + BATCH_BYTES, side='right')))
                fasta, stats = format_records(text, id_start[kept_ids[i0:i1]], id_len[kept_ids[i0:i1]], data, starts[src[i0:i1]],
                                              lens[src[i0:i1]], acgt[i0:i1])
                seqOut.write(fasta)
                statsOut.write(stats)
                i0 = i1
        t5 = time.perf_counter()
        self.timing.update({'read': t1 - t0, 'scan': t2 - t1, 'device': (t3 - t2) + (t4 - t4c), 'write': t5 - t4,
                            'records': len(lens) + nb, 'bytes': sum(len(b[1]) for b in bins) + len(data)})

        self.logger.info('  Identified %d (%.2f Mbp) unbinned sequences.' % (unbinnedCount, float(unbinnedBases) / 1e6))

        if len(entries) == 0:
            self._fail('No sequences in %s.' % seqFile)
        self.logger.info('Percentage of unbinned sequences: %.2f%%' % (unbinnedCount * 100.0 / len(entries)))
        if totalBases == 0:
            self._fail('The sequences in %s hold no bases.' % seqFile)
        self.logger.info('Percentage of unbinned bases: %.2f%%' % (unbinnedBases * 100.0 / totalBases))
