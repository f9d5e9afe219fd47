"""Exploring and modifying bins (`checkm outliers`, `checkm modify`, `checkm unique`) behind the reference's BinTools
interface (checkm/binTools.py:36-296).

`identifyOutliers` reads the tetranucleotide profile file once (`ckm_parse_kmer_profiles`; the reference re-reads it for
every bin) and keeps it on the device; the bins are read and their bases counted in batches (`ckm_scaffold_stats`, as
BinStatistics does), and every sequence of a batch is scored in one device call (`ckm_outlier_scores`, csrc/outliers.cu,
which states the arithmetic and the order of its sums).  Which table of the GC and CD distributions a bin is held to
depends on its mean GC and CD; those two means are ratios of integer totals, so they are formed here from the counts the
scan returned and the tables are resolved before the call.  Rows are written on the host, with Python's own `%` formats,
for the reported sequences only.  There is no CPU path for the scoring.

Where the reference ends in an uncaught exception -- a bin without sequences, a sequence without A/C/G/T (division by
zero), a sequence that is not in the profile file (KeyError) -- `identifyOutliers` logs an error naming the bin and the
sequence and exits with status 1; the dictionary-taking methods raise the reference's exception."""
import gzip
import logging
import os
import sys
import time

import numpy as np

from . import runtime, seqio
from .binStatistics import BATCH_BYTES, _from_dict, _GeneFeatures, _scan
from .common import binIdFromFilename, checkFileExists, findNearest, readDistribution
from .defaultValues import DefaultValues
from .genomicSignatures import parse_profiles

_COLS = 136
_NO_TABLE = (np.array([0, 1], dtype=np.int64), np.zeros(1), np.zeros(1), np.zeros(1))      # one key, bounds of 0


def readFasta(fastaFile):
    """util/seqUtils.py:180-211 through the library's scanner: {id: sequence}, ids in the reference's dictionary order."""
    try:
        ids, data, starts, lens = seqio.scan_nt_fasta(seqio.read_bytes(fastaFile))
    except Exception as e:
        print(e)
        logging.getLogger('timestamp').error("Failed to process sequence file: {}".format(fastaFile))
        sys.exit(1)
    raw = data.tobytes()
    return {i: raw[a:a + n].decode('latin-1') for i, a, n in zip(ids, starts.tolist(), lens.tolist())}


def writeFasta(seqs, outputFile):
    """util/seqUtils.py:266-276: `>id`, then the sequence on one line.  A name ending in .gz is written as gzip text (the
    reference opens it in binary mode and fails on the first write)."""
    fout = gzip.open(outputFile, 'wt') if outputFile.endswith('.gz') else open(outputFile, 'w')
    for seqId, seq in seqs.items():
        fout.write('>' + seqId + '\n')
        fout.write(seq + '\n')
    fout.close()


class _BoundTables(object):
    """The bound lists `ckm_outlier_scores` takes, resolved from the three distribution dictionaries: per distinct (mean
    key, percentile keys) one list of (length key, lower, upper), built the first time a bin needs it."""

    def __init__(self, gcBounds, cdBounds, tdBounds, distribution):
        self.gcBounds, self.cdBounds, self.distribution = gcBounds, cdBounds, distribution
        self.off, self.key, self.lo, self.hi, self.index = [0], [], [], [], {}
        tdKey = findNearest(list(tdBounds[list(tdBounds.keys())[0]].keys()), distribution)               # binTools.py:261
        self.td_table = self._add('td', [(n, 0.0, d[tdKey]) for n, d in tdBounds.items()])

    def _add(self, name, entries):
        if name not in self.index:
            self.index[name] = len(self.off) - 1
            for n, lo, hi in entries:
                self.key.append(float(n)); self.lo.append(float(lo)); self.hi.append(float(hi))
            self.off.append(len(self.key))
        return self.index[name]

    def gc_table(self, meanGC):
        """binTools.py:250-254: the table of the mean-GC key nearest to the bin's, the percentile keys taken from its first
        length entry."""
        closest = findNearest(np.array(list(self.gcBounds.keys())), meanGC)
        byLen = self.gcBounds[closest]
        d = byLen[list(byLen.keys())[0]]
        loKey = findNearest(list(d.keys()), (100 - self.distribution) / 2.0)
        hiKey = findNearest(list(d.keys()), (100 + self.distribution) / 2.0)
        return self._add(('gc', float(closest)), [(n, e[loKey], e[hiKey]) for n, e in byLen.items()])

    def cd_table(self, meanCD):
        """binTools.py:256-259."""
        closest = findNearest(np.array(list(self.cdBounds.keys())), meanCD)
        byLen = self.cdBounds[closest]
        d = byLen[list(byLen.keys())[0]]
        loKey = findNearest(list(d.keys()), (100 - self.distribution) / 2.0)
        return self._add(('cd', float(closest)), [(n, e[loKey], 0.0) for n, e in byLen.items()])

    def arrays(self):
        return np.array(self.off, dtype=np.int64), np.array(self.key), np.array(self.lo), np.array(self.hi)


class BinTools():
    """Functions for exploring and modifying bins (name, arguments and results of checkm.binTools.BinTools)."""

    def __init__(self, threads=1):
        self.logger = logging.getLogger('timestamp')
        self.totalThreads = threads
        self.timing = {}                  # seconds per phase of the last identifyOutliers

    def _fatal(self, message):
        self.logger.error(message)
        sys.exit(1)

    # ---- modifying bins (host only) ----
    def _removeSeqs(self, seqs, seqsToRemove):
        missingSeqIds = set(seqsToRemove).difference(set(seqs.keys()))
        if len(missingSeqIds) > 0:
            self._fatal('Missing sequence(s) specified for removal: ' + ', '.join(missingSeqIds) + '\n')
        for seqId in seqsToRemove:
            seqs.pop(seqId)

    def _addSeqs(self, seqs, refSeqs, seqsToAdd):
        missingSeqIds = set(seqsToAdd).difference(set(refSeqs.keys()))
        if len(missingSeqIds) > 0:
            self._fatal('Missing sequence(s) specified for addition: ' + ', '.join(missingSeqIds) + '\n')
        for seqId in seqsToAdd:
            seqs[seqId] = refSeqs[seqId]

    def modify(self, binFile, seqFile, seqsToAdd, seqsToRemove, outputFile):
        """Add and remove sequences from a file (binTools.py:61-75)."""
        binSeqs = readFasta(binFile)
        if seqsToAdd is not None:
            self._addSeqs(binSeqs, readFasta(seqFile), seqsToAdd)
        if seqsToRemove is not None:
            self._removeSeqs(binSeqs, seqsToRemove)
        writeFasta(binSeqs, outputFile)

    def removeOutliers(self, binFile, outlierFile, outputFile):
        """Remove the sequences the outlier file lists for this bin (binTools.py:77-104)."""
        binSeqs = readFasta(binFile)
        binIdToModify = binIdFromFilename(binFile)
        checkFileExists(outlierFile)
        seqsToRemove = []
        with open(outlierFile) as f:
            next(f, None)
            for line in f:
                lineSplit = line.split('\t')
                if lineSplit[0] == binIdToModify:
                    seqsToRemove.append(lineSplit[1])
        if len(seqsToRemove) > 0:
            self._removeSeqs(binSeqs, seqsToRemove)
        writeFasta(binSeqs, outputFile)

    def unique(self, binFiles):
        """Report sequences found twice in a bin or in two bins (binTools.py:106-146).  The reference compares the lines of
        a .gz bin as bytes with '>', so such a bin contributes no ids; that is kept."""
        binSeqs = {}
        for f in binFiles:
            binId = binIdFromFilename(f)
            seqIds = set()
            if not f.endswith('.gz'):
                for line in open(f):
                    if line[0] == '>':
                        seqId = line[1:].split(None, 1)[0]
                        if seqId in seqIds:
                            print('  [Warning] Sequence %s found multiple times in bin %s.' % (seqId, binId))
                        seqIds.add(seqId)
            binSeqs[binId] = seqIds

        bDuplicates = False
        binIds = list(binSeqs.keys())
        for i in range(0, len(binIds)):
            for j in range(i + 1, len(binIds)):
                seqInter = binSeqs[binIds[i]].intersection(binSeqs[binIds[j]])
                if len(seqInter) > 0:
                    bDuplicates = True
                    print('  Sequences shared between %s and %s: ' % (binIds[i], binIds[j]))
                    for seqId in seqInter:
                        print('    ' + seqId)
                    print('')
        if not bDuplicates:
            print('  No sequences assigned to multiple bins.')

    # ---- the reference's dictionary-taking methods ({sequence id: sequence string}), one-bin batches of the device call ----
    def _score_dict(self, seqs, coding=None, tetraSigs=None, binSig=None):
        sc = _scan([_from_dict(seqs)])[0]
        acgt = sc.stats[:, :4]
        n = len(sc.ids)
        if tetraSigs is None:
            matrix = np.zeros((1, _COLS))
            rows = np.zeros(n, dtype=np.int64)
        else:
            matrix = np.array([tetraSigs[seqId] for seqId in sc.ids], dtype=np.float64).reshape(n, _COLS)
            rows = np.arange(n, dtype=np.int64)
        if (acgt.sum(axis=1) == 0).any():                          # gcDist has refused these; the other methods do not ask for GC,
            acgt = acgt.copy()                                     # and the library refuses a sequence without a countable base
            acgt[acgt.sum(axis=1) == 0, 0] = 1
        eng = runtime.engine()
        sigs = eng.signatures(matrix)
        try:
            return eng.outlier_scores(sigs, [0, n], sc.lens, acgt, np.zeros(n, dtype=np.int64) if coding is None else coding, rows,
                                      [0], [0], 0, *_NO_TABLE, binsig_in=None if binSig is None else np.reshape(binSig, (1, _COLS)),
                                      want_binsig=True)
        finally:
            sigs.close()

    def gcDist(self, seqs):
        """GC statistics for bin (binTools.py:148-166): mean, each sequence's difference to it, each sequence's GC."""
        for seq in seqs.values():
            s = seq.upper()
            if not any(c in s for c in 'ACGTU'):
                raise ZeroDivisionError('float division by zero')
        means, _, values, _, _ = self._score_dict(seqs)
        return float(means[0, 0]), values[:, 1].copy(), values[:, 0].tolist()

    def codingDensityDist(self, seqs, prodigalParser):
        """Coding density statistics for bin (binTools.py:168-184)."""
        if any(len(seq) == 0 for seq in seqs.values()):
            raise ZeroDivisionError('float division by zero')
        coding = np.array([int(prodigalParser.codingBases(seqId)) for seqId in seqs], dtype=np.int64)
        means, _, values, _, _ = self._score_dict(seqs, coding=coding)
        return float(means[0, 1]), values[:, 3].copy(), values[:, 2].tolist()

    def binTetraSig(self, seqs, tetraSigs):
        """Tetranucleotide signature for bin (binTools.py:186-201)."""
        return self._score_dict(seqs, tetraSigs=tetraSigs)[1][0].copy()

    def tetraDiffDist(self, seqs, genomicSig, tetraSigs, binSig):
        """TD statistics for bin (binTools.py:203-209)."""
        means, _, values, _, _ = self._score_dict(seqs, tetraSigs=tetraSigs, binSig=binSig)
        return np.float64(means[0, 2]), values[:, 4].copy()

    # ---- checkm outliers ----
    def identifyOutliers(self, outDir, binFiles, tetraProfileFile, distribution, reportType, outputFile):
        """Identify sequences that are outliers (binTools.py:211-296)."""
        self.logger.info('Reading reference distributions.')
        tables = _BoundTables(readDistribution('gc_dist'), readDistribution('cd_dist'), readDistribution('td_dist'), distribution)

        fout = open(outputFile, 'w')
        fout.write('Bin Id\tSequence Id\tSequence length\tOutlying distributions')
        fout.write('\tSequence GC\tMean bin GC\tLower GC bound (%s%%)\tUpper GC bound (%s%%)' % (distribution, distribution))
        fout.write('\tSequence CD\tMean bin CD\tLower CD bound (%s%%)' % distribution)
        fout.write('\tSequence TD\tMean bin TD\tUpper TD bound (%s%%)\n' % distribution)

        t0 = time.perf_counter()
        with open(tetraProfileFile, 'rb') as f:
            profileIds, matrix = parse_profiles(f.read(), _COLS, self.totalThreads)
        rowOf = {seqId: r for r, seqId in enumerate(profileIds)}          # a repeated id keeps its last line, as the reference's dict
        self.timing = {'parse_profile': time.perf_counter() - t0, 'read_bins': 0.0, 'device_calls': 0.0,
                       'kernels_ms': [0.0, 0.0, 0.0], 'format_write': 0.0, 'rows': 0}
        eng = runtime.engine()
        sigs = eng.signatures(matrix if len(matrix) else np.zeros((1, _COLS)))
        try:
            pending, pending_bytes = [], 0
            for processedBins, binFile in enumerate(binFiles, 1):
                binId = binIdFromFilename(binFile)
                self.logger.info('Finding outliers in %s (%d of %d).' % (binId, processedBins, len(binFiles)))
                t1 = time.perf_counter()
                try:
                    parsed = seqio.scan_nt_fasta(seqio.read_bytes(binFile))
                except Exception as e:                        # util/seqUtils.py:205-209
                    print(e)
                    self._fatal("Failed to process sequence file: {}".format(binFile))
                gffFile = os.path.join(outDir, 'bins', binId, DefaultValues.PRODIGAL_GFF)
                if not os.path.exists(gffFile):
                    self._fatal('Missing gene feature file (%s). This plot if not compatible with the --genes option.\n'
                                % DefaultValues.PRODIGAL_GFF)
                if len(parsed[0]) == 0:
                    self._fatal('Bin %s has no sequences: its mean GC is undefined.' % binId)
                features = _GeneFeatures(gffFile)
                self.timing['read_bins'] += time.perf_counter() - t1
                pending.append((binId, parsed, features))
                pending_bytes += len(parsed[1])
                if pending_bytes >= BATCH_BYTES:
                    self._score_batch(pending, rowOf, tetraProfileFile, sigs, tables, reportType, fout)
                    pending, pending_bytes = [], 0
            if pending:
                self._score_batch(pending, rowOf, tetraProfileFile, sigs, tables, reportType, fout)
        finally:
            sigs.close()
        fout.close()

    def _score_batch(self, pending, rowOf, tetraProfileFile, sigs, tables, reportType, fout):
        """One device scan and one scoring call for the bins of `pending`, then their rows."""
        t0 = time.perf_counter()
        scanned = _scan([p[1] for p in pending])
        counts = [len(sc.ids) for sc in scanned]
        bin_off = np.concatenate([[0], np.cumsum(counts)]).astype(np.int64)
        lens = np.concatenate([sc.lens for sc in scanned]).astype(np.int64)
        acgt = np.ascontiguousarray(np.concatenate([sc.stats[:, :4] for sc in scanned]))
        coding = np.empty(len(lens), dtype=np.int64)
        rows = np.empty(len(lens), dtype=np.int64)
        bin_gc, bin_cd = [], []
        for b, ((binId, _, features), sc) in enumerate(zip(pending, scanned)):
            lo = int(bin_off[b])
            bases = acgt[lo:lo + len(sc.ids)].sum(axis=1)
            for i, seqId in enumerate(sc.ids):
                if bases[i] == 0:
                    self._fatal('Sequence %s of bin %s has no A, C, G or T: its GC is undefined.' % (seqId, binId))
                r = rowOf.get(seqId)
                if r is None:
                    self._fatal('Sequence %s of bin %s is not in the tetranucleotide profile file %s.' % (seqId, binId, tetraProfileFile))
                rows[lo + i] = r
                coding[lo + i] = int(features.codingBases(seqId))
            # the two means that choose the tables: integer totals divided once (binTools.py:163, 181)
            a = acgt[lo:lo + len(sc.ids)]
            meanGC = float(int(a[:, 1].sum() + a[:, 2].sum())) / int(a.sum())
            meanCD = float(int(coding[lo:lo + len(sc.ids)].sum())) / int(lens[lo:lo + len(sc.ids)].sum())
            bin_gc.append(tables.gc_table(meanGC))
            bin_cd.append(tables.cd_table(meanCD))
        t1 = time.perf_counter()
        means, _, values, mask, kernel_ms = runtime.engine().outlier_scores(sigs, bin_off, lens, acgt, coding, rows, bin_gc, bin_cd,
                                                                            tables.td_table, *tables.arrays())
        t2 = time.perf_counter()
        wanted = np.flatnonzero(mask == 7 if reportType == 'all' else mask != 0) if reportType in ('any', 'all') else []
        names = ('GC', 'CD', 'TD')
        b = 0
        for s in wanted:
            while s >= bin_off[b + 1]:
                b += 1
            binId, sc = pending[b][0], scanned[b]
            meanGC, meanCD, meanTD = means[b].tolist()
            GC, _, CD, _, TD, gcLower, gcUpper, cdLower, tdBound = values[s].tolist()
            outlying = [n for k, n in enumerate(names) if mask[s] >> k & 1]
            fout.write(binId + '\t' + sc.ids[s - int(bin_off[b])] + '\t%d' % lens[s] + '\t' + ','.join(outlying))
            fout.write('\t%.1f\t%.1f\t%.1f\t%.1f' % (GC * 100, meanGC * 100, (meanGC + gcLower) * 100, (meanGC + gcUpper) * 100))
            fout.write('\t%.1f\t%.1f\t%.1f' % (CD * 100, meanCD * 100, (meanCD + cdLower) * 100))
            fout.write('\t%.3f\t%.3f\t%.3f' % (TD, meanTD, tdBound) + '\n')
        t3 = time.perf_counter()
        self.timing['read_bins'] += t1 - t0
        self.timing['device_calls'] += t2 - t1
        self.timing['kernels_ms'] = [x + y for x, y in zip(self.timing['kernels_ms'], kernel_ms)]
        self.timing['format_write'] += t3 - t2
        self.timing['rows'] += len(wanted)
