"""Read coverage (`checkm coverage`) behind the reference's Coverage interface (checkm/coverage.py:37-358), without pysam.

Each BAM is read through its BAI index (checkm_b200/bam.py) and cut into batches of at most CKM_BAM_BATCH_MB compressed
MiB (default 256, about 1.3 GB of device memory with the inflated stream: room next to a live search engine), always at
record anchors.  One device call per batch (`ckm_bam_coverage`, csrc/bam.cu) inflates the BGZF blocks, walks the records
and adds nine counters per reference; coverage = aligned bases / header length is formed here in float64.

The coverage file's rows, their order and their text are the reference's at threads=1: the bins' sequences in file order
(a later bin overrides an earlier one), then each BAM's references that are in no bin, in header order, with bin
`unbinned`; a BAM's header length replaces a sequence's length.  `threads` does not fork: the work is on the device.

Differences from the reference, on purpose: a read that reaches the edit-distance test without an integer NM tag stops
the run with the read's name (the reference's worker raises there and its contigs silently get 0), and the BAMs are
walked in file order rather than by forked workers per contig."""
import contextlib
import logging
import ntpath
import os
import sys
import time
from collections import defaultdict

import numpy as np

from . import bam, runtime, seqio
from ._lib import CkmError
from .common import binIdFromFilename

UNBINNED = 'unbinned'
DEFAULT_BATCH_MB = 256


class CoverageStruct():
    def __init__(self, seqLen, mappedReads, coverage):
        self.seqLen = seqLen
        self.mappedReads = mappedReads
        self.coverage = coverage


def batch_bytes():
    return int(float(os.environ.get('CKM_BAM_BATCH_MB', str(DEFAULT_BATCH_MB))) * (1 << 20))


@contextlib.contextmanager
def bam_batches(bamFile, timing):
    """Opens bamFile's index, block table and header (bam.Layout) and yields (header, run).  run(call) sends every batch
    through call(eng, comp, blocks, seg_start, seg_end, comp_base), one device call returning its inflate and scan ms.
    Adds to `timing`: 'read' (opening), 'device_calls' (the rest), the kernel ms, the batches and their sizes."""
    t0 = time.perf_counter()
    lay = bam.Layout(bamFile)
    t1 = time.perf_counter()

    def run(call):
        eng = runtime.engine()
        for b0, b1, s, e in lay.batches(batch_bytes()):
            comp, base = lay.comp(b0, b1)
            ms_inf, ms_scan = call(eng, comp, lay.blocks[b0:b1], s, e, base)
            timing['batches'] += 1
            timing['inflate_ms'] += ms_inf
            timing['scan_ms'] += ms_scan
            timing['compressed_bytes'] += comp.size
            timing['inflated_bytes'] += int(lay.U[b1] - lay.U[b0])
            timing['segments'] += len(s)
    try:
        yield lay.header, run
    finally:
        timing['read'] += t1 - t0
        timing['device_calls'] += time.perf_counter() - t1
        lay.close()


def print_summary(logger, cnt, numRefSeqs):
    """The summary the reference's writer prints per BAM (coverage.py:258-287, coverageWindows.py:243-255: the same text)
    from the n_ref x 9 counters, when the logger shows INFO."""
    if logger.getEffectiveLevel() > logging.INFO:
        return
    if numRefSeqs:
        sys.stderr.write('    Finished processing %d of %d (%.2f%%) reference sequences.\r' %
                         (numRefSeqs, numRefSeqs, 100.0))
    sys.stderr.write('\n')
    sys.stderr.flush()
    t = cnt.sum(axis=0).tolist() if len(cnt) else [0] * 9
    total = t[0]
    print('')
    print('    # total reads: %d' % total)
    if total == 0:                    # the reference divides by the total here and its writer process stops
        return
    for label, v in (('properly mapped reads', t[7]), ('duplicate reads', t[1]), ('secondary reads', t[2]),
                     ('reads failing QC', t[3]), ('reads failing alignment length', t[4]),
                     ('reads failing edit distance', t[5]), ('reads not properly paired', t[6])):
        print('      # %s: %d (%.1f%%)' % (label, v, float(v) * 100 / total))
    print('')


class Coverage():
    """Calculate coverage of all sequences."""

    def __init__(self, threads):
        self.logger = logging.getLogger('timestamp')
        self.totalThreads = threads
        self.timing = {}                  # seconds per phase of the last run, kernel ms and the number of batches
        self.counters = {}                # BAM path -> (names, lengths, n_ref x 9 int64) of the last run

    def run(self, binFiles, bamFiles, outFile, bAllReads, minAlignPer, maxEditDistPer, minQC):
        self.logger.info('Determining bin assignment of each sequence.')
        t0 = time.perf_counter()
        seqIdToBinId = {}
        seqIdToSeqLen = {}
        for binFile in binFiles:
            binId = binIdFromFilename(binFile)
            ids, _, _, lens = seqio.scan_nt_fasta(seqio.read_bytes(binFile))
            for seqId, n in zip(ids, lens.tolist()):
                seqIdToBinId[seqId] = binId
                seqIdToSeqLen[seqId] = n

        self.logger.info("Processing %d file(s) with %d threads.\n" % (len(bamFiles), self.totalThreads))
        for bamFile in bamFiles:
            if not os.path.exists(bamFile + '.bai'):
                self.logger.error('BAM file is either unsorted or not indexed: ' + bamFile + '\n')
                sys.exit(1)

        self.timing = {'bins': time.perf_counter() - t0, 'read': 0.0, 'device_calls': 0.0, 'inflate_ms': 0.0, 'scan_ms': 0.0,
                       'format_write': 0.0, 'batches': 0, 'compressed_bytes': 0, 'inflated_bytes': 0, 'segments': 0}
        coverageInfo = {}
        self.counters = {}
        for k, bamFile in enumerate(bamFiles):
            self.logger.info('Processing %s (%d of %d):' % (ntpath.basename(bamFile), k + 1, len(bamFiles)))
            try:
                names, lengths, cnt = self._processBam(bamFile, bAllReads, minAlignPer, maxEditDistPer, minQC)
            except CkmError as e:
                self.logger.error('Failed to process BAM file %s: %s' % (bamFile, e))
                sys.exit(1)
            self.counters[bamFile] = (names, lengths, cnt)
            info = {}
            for name, n, c in zip(names, lengths, cnt.tolist()):
                info[name] = CoverageStruct(seqLen=n, mappedReads=c[7], coverage=float(c[8]) / n)
            coverageInfo[bamFile] = info
            self._summary(cnt, len(names))

        self.logger.info('Writing coverage information to file.')
        t1 = time.perf_counter()
        for info in coverageInfo.values():
            for seqId, cs in info.items():
                seqIdToSeqLen[seqId] = cs.seqLen
        bamIds = [binIdFromFilename(b) for b in bamFiles]
        lines = ['Sequence Id\tBin Id\tSequence length (bp)' + '\tBam Id\tCoverage\tMapped reads' * len(bamFiles)]
        for seqId, seqLen in seqIdToSeqLen.items():
            row = seqId + '\t' + seqIdToBinId.get(seqId, UNBINNED) + '\t' + str(seqLen)
            for bamFile, bamId in zip(bamFiles, bamIds):
                cs = coverageInfo[bamFile].get(seqId)
                row += '\t%s\t%f\t%d' % ((bamId, cs.coverage, cs.mappedReads) if cs is not None else (bamId, 0, 0))
            lines.append(row)
        text = '\n'.join(lines) + '\n'
        if outFile == '':
            sys.stdout.write(text)
        else:
            try:
                with open(outFile, 'w') as f:
                    f.write(text)
            except IOError:
                self.logger.error("Error diverting stdout to file: " + outFile)
                sys.exit(1)
        self.timing['format_write'] = time.perf_counter() - t1

    def _processBam(self, bamFile, bAllReads, minAlignPer, maxEditDistPer, minQC):
        """(names, lengths, n_ref x 9 int64 counters) of one BAM: reads, duplicates, secondary, failed QC, failed alignment
        length, failed edit distance, failed proper pair, mapped, aligned bases."""
        with bam_batches(bamFile, self.timing) as (header, run):
            n_ref = len(header.names)
            cnt = np.zeros((n_ref, 9), dtype=np.int64)
            run(lambda eng, comp, blocks, s, e, base: eng.bam_coverage(
                comp, blocks, s, e, n_ref, cnt, comp_base=base, all_reads=bAllReads, min_qc=minQC, min_align=minAlignPer,
                max_edit=maxEditDistPer))
            return header.names, header.lengths, cnt

    def _summary(self, cnt, numRefSeqs):
        """The per-BAM summary of coverage.py:258-287 (stdout), when the logger shows INFO."""
        print_summary(self.logger, cnt, numRefSeqs)

    def parseCoverage(self, coverageFile):
        """{binId: {seqId: {bamId: coverage}}} of a coverage file."""
        coverageStats = {}
        with open(coverageFile) as f:
            next(f, None)
            for line in f:
                fields = line.split('\t')
                perSeq = coverageStats.setdefault(fields[1], {}).setdefault(fields[0], {})
                for i in range(3, len(fields), 3):
                    perSeq[fields[i]] = float(fields[i + 1])
        return coverageStats

    def binProfiles(self, coverageFile):
        """{binId: {bamId: [length-weighted mean coverage, standard deviation of the sequences' coverage]}}, with the
        reference's running weighted mean (coverage.py:315-358)."""
        coverages = defaultdict(lambda: defaultdict(list))
        stats = defaultdict(dict)
        with open(coverageFile) as f:
            next(f, None)
            for line in f:
                fields = line.split('\t')
                binId, seqLen = fields[1], int(fields[2])
                for i in range(3, len(fields), 3):
                    bamId, cov = fields[i], float(fields[i + 1])
                    coverages[binId][bamId].append(cov)
                    length, mean = stats[binId].get(bamId, [0, 0])
                    length += seqLen
                    w = float(seqLen) / length
                    stats[binId][bamId] = [length, cov * w + mean * (1 - w)]
        profiles = defaultdict(dict)
        for binId in stats:
            for bamId, (_, mean) in stats[binId].items():
                covs = coverages[binId][bamId]
                var = np.mean([(x - mean) ** 2 for x in covs]) if len(covs) > 1 else 0
                profiles[binId][bamId] = [mean, np.sqrt(var)]
        return profiles
