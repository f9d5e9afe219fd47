"""Read depth per window for `checkm gc_bias_plot` behind the reference's CoverageWindows interface
(checkm/coverageWindows.py:30-255), without pysam.

The BAM is read through its BAI index and cut into batches exactly as for `checkm coverage` (checkm_b200/bam.py, at
most CKM_BAM_BATCH_MB compressed MiB each).  One device call per batch (`ckm_bam_windows`, csrc/bam.cu) inflates the
blocks, walks the records with coverageWindows' classification and adds, per reference, the nine counters (the ninth is
the number of covered bases, the sum of the per-base depth) and, per window, the sum of the depth over it.  Both are
exact integers; each value returned is one float64 division of one of them, as the reference's `sum(...) / windowSize`
and `float(sum(...)) / seqLen` are, so the values are the reference's bit for bit.

`run` returns {seqId: [coverage, windowCoverages]} for every reference in the BAM header, in header order; window k
covers [k W, (k + 1) W) and is taken only while (k + 1) W < seqLen, so a reference has (seqLen - 1) // W windows.
`binFiles` is not read (the reference does not read it either) and `threads` does not fork: the work is on the device.

Differences from the reference, on purpose: a read that reaches the edit-distance test without a numeric NM tag, the
alignment-length test without a CIGAR, or the depth update at a negative position stops the run with the read's name
(the reference's worker raises there, or indexes the array from its end); a window size below 1 is refused (the
reference loops forever)."""
import logging
import operator
import os
import sys
import time

import numpy as np

from ._lib import CkmError
from .coverage import CoverageStruct, bam_batches, print_summary  # noqa: F401 (CoverageStruct: the reference's name here)


def window_offsets(lengths, windowSize):
    """win_off (n_ref + 1 int64): reference r owns windows [win_off[r], win_off[r + 1]), (length - 1) // W of them."""
    lens = np.asarray(lengths, dtype=np.int64)
    off = np.zeros(len(lens) + 1, dtype=np.int64)
    np.cumsum(np.maximum(lens - 1, 0) // windowSize, out=off[1:])
    return off


class CoverageWindows():
    """Calculate coverage of all sequences."""

    def __init__(self, threads):
        self.logger = logging.getLogger('timestamp')
        self.totalThreads = threads
        self.timing = {}                  # seconds per phase of the last run, kernel ms and the number of batches
        self.counters = None              # (names, lengths, n_ref x 9 int64, window sums, win_off) of the last run

    def run(self, binFiles, bamFile, bAllReads, minAlignPer, maxEditDistPer, windowSize):
        """Calculate coverage of full sequences and windows."""
        if not os.path.exists(bamFile + '.bai'):
            self.logger.error('BAM file is not sorted: ' + bamFile + '\n')
            sys.exit(1)

        self.logger.info('Calculating coverage of windows.')
        try:
            W = operator.index(windowSize)
        except TypeError:
            W = 0
        if W < 1:
            self.logger.error('Window size must be a positive integer: %r\n' % (windowSize,))
            sys.exit(1)

        self.timing = {'read': 0.0, 'device_calls': 0.0, 'inflate_ms': 0.0, 'scan_ms': 0.0, 'format': 0.0, 'batches': 0,
                       'compressed_bytes': 0, 'inflated_bytes': 0, 'segments': 0, 'windows': 0}
        try:
            names, lengths, cnt, win, off = self._processBam(bamFile, bAllReads, minAlignPer, maxEditDistPer, W)
        except CkmError as e:
            self.logger.error('Failed to process BAM file %s: %s' % (bamFile, e))
            sys.exit(1)
        self.counters = (names, lengths, cnt, win, off)

        t0 = time.perf_counter()
        values = (win / W).tolist()                                    # one IEEE division per exact integer sum
        bases = cnt[:, 8].tolist()
        offs = off.tolist()
        coverageInfo = {}
        for r, (seqId, seqLen) in enumerate(zip(names, lengths)):
            coverageInfo[seqId] = [float(bases[r]) / seqLen, values[offs[r]:offs[r + 1]]]
        self.timing['format'] = time.perf_counter() - t0
        print_summary(self.logger, cnt, len(names))
        return coverageInfo

    def _processBam(self, bamFile, bAllReads, minAlignPer, maxEditDistPer, windowSize):
        """(names, lengths, n_ref x 9 int64 counters, int64 window sums, window offsets) of one BAM."""
        with bam_batches(bamFile, self.timing) as (header, run):
            names, lengths = header.names, header.lengths
            off = window_offsets(lengths, windowSize)
            cnt = np.zeros((len(names), 9), dtype=np.int64)
            win = np.zeros(int(off[-1]), dtype=np.int64)
            self.timing['windows'] = int(off[-1])
            run(lambda eng, comp, blocks, s, e, base: eng.bam_windows(
                comp, blocks, s, e, lengths, windowSize, off, cnt, win, comp_base=base, all_reads=bAllReads,
                min_align=minAlignPer, max_edit=maxEditDistPer))
            return names, lengths, cnt, win, off
