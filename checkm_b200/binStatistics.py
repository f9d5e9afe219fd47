"""Bin statistics (GC, N50, contigs, coding density) behind the reference's BinStatistics interface
(checkm/binStatistics.py:37-290; SURVEY.md 8 row f4).  `analyze` writes these to storage/bin_stats.analyze.tsv, which
`ResultsParser.analyseResults` requires (resultsParser.py:63).

All the per-base work -- base counts, ambiguous bases, contig lengths of every scaffold of every bin of a batch -- is one
scan on the device (`ckm_scaffold_stats`); this module reads the files, forms the ratios from the integers with the same
float operations as the reference, and writes the same dictionary text.  There is no CPU path for the scan."""
import logging
import math
import os
import sys

import numpy as np

from . import runtime, seqio
from .common import binIdFromFilename, makeSurePathExists

# checkm/defaultValues.py:82-104
PRODIGAL_AA = 'genes.faa'
PRODIGAL_GFF = 'genes.gff'
MIN_SEQ_LEN_GC_STD = 1000

BATCH_BYTES = 1 << 29           # scaffold bytes of the bins scanned by one device call


def _n50(lengths):
    """util/seqUtils.py:289-301: the length at which the running sum of the lengths, longest first, reaches half the total."""
    ordered = np.sort(np.asarray(lengths, dtype=np.int64))[::-1]
    reached = np.cumsum(ordered)
    return int(ordered[int(np.searchsorted(reached, reached[-1] / 2.0, side='left'))])


class _Scaffolds(object):
    """Scaffolds of one bin after the device scan: ids in file order, their lengths, the 8 integers of each, its contigs."""
    __slots__ = ('ids', 'lens', 'stats', 'contig_scaffold', 'contig_len')

    def __init__(self, ids, lens, stats, contig_scaffold, contig_len):
        self.ids, self.lens, self.stats = ids, lens, stats
        self.contig_scaffold, self.contig_len = contig_scaffold, contig_len


def _scan(batches):
    """batches: list of (ids, data, starts, lens) as seqio.scan_nt_fasta returns them -> list of _Scaffolds, one device call."""
    sizes = [len(b[1]) for b in batches]
    data = np.concatenate([b[1] for b in batches]) if len(batches) > 1 else batches[0][1]
    shift = np.concatenate([[0], np.cumsum(sizes)[:-1]]).astype(np.int64)
    starts = np.concatenate([b[2] + s for b, s in zip(batches, shift)])
    lens = np.concatenate([b[3] for b in batches])
    stats, cscaf, clen, _ = runtime.engine().scaffold_stats(data, starts, lens)
    order = np.argsort(cscaf, kind='stable')
    cscaf, clen = cscaf[order], clen[order]
    out, first = [], 0
    for ids, _, _, blens in batches:
        k = len(ids)
        lo, hi = np.searchsorted(cscaf, [first, first + k])
        out.append(_Scaffolds(ids, blens, stats[first:first + k], cscaf[lo:hi] - first, clen[lo:hi]))
        first += k
    return out


def _from_dict(seqs):
    """{id: sequence string} -> the layout of seqio.scan_nt_fasta (for the reference's dictionary-taking methods)."""
    ids = list(seqs.keys())
    raw = [seqs[i].encode('latin-1', 'replace') for i in ids]
    lens = np.array([len(r) for r in raw], dtype=np.int64)
    padded = (lens + 63) // 64 * 64
    starts = np.concatenate([[0], np.cumsum(padded)[:-1]]).astype(np.int64) if ids else np.zeros(0, dtype=np.int64)
    data = np.zeros(int(padded.sum()), dtype=np.uint8)
    for r, s in zip(raw, starts):
        data[s:s + len(r)] = np.frombuffer(r, dtype=np.uint8)
    return ids, data, starts, lens


def _gc(sc, seqStats=None):
    """binStatistics.py:176-206 from the integer counts."""
    a, c, g, t = (sc.stats[:, k] for k in range(4))
    gc, at = g + c, a + t
    totalGC, totalAT = int(gc.sum()), int(at.sum())
    perSeq = []
    for i, seqId in enumerate(sc.ids):
        n = int(gc[i] + at[i])
        content = float(int(gc[i])) / n if n > 0 else 0.0
        if seqStats:
            seqStats[seqId]['GC'] = content
        if sc.lens[i] > MIN_SEQ_LEN_GC_STD:
            perSeq.append(content)
    GC = float(totalGC) / (totalGC + totalAT) if (totalGC + totalAT) > 0 else 0.0
    varGC = 0
    if len(perSeq) > 1:
        varGC = np.mean(list(map(lambda x: (x - GC) ** 2, perSeq)))
    return GC, math.sqrt(varGC)


def _seq_stats(sc, seqStats=None):
    """binStatistics.py:208-233 from the scaffold lengths and the contig list."""
    scaffoldLens = [int(v) for v in sc.lens]
    contigLens = [int(v) for v in sc.contig_len]
    if seqStats:
        for i, seqId in enumerate(sc.ids):
            seqStats[seqId]['Length'] = scaffoldLens[i]
            seqStats[seqId]['Total contig length'] = int(sc.stats[i, 7])
            seqStats[seqId]['# contigs'] = int(sc.stats[i, 6])
    ambiguous = int(sc.stats[:, 4].sum() + sc.stats[:, 5].sum())
    return (max(scaffoldLens), max(contigLens), sum(scaffoldLens), _n50(scaffoldLens), _n50(contigLens),
            np.mean(scaffoldLens), np.mean(contigLens), len(contigLens), ambiguous)


class _GeneFeatures(object):
    """What bin statistics and the plots take from Prodigal's GFF (prodigal.py:202-273): the translation table, per
    sequence the number of bases covered by at least one gene, and per sequence the coding-base mask as disjoint intervals
    (`intervals`, for `windowCodingBases`)."""

    def __init__(self, filename):
        self.translationTable = None
        genes, counter = {}, 0
        self.lastCodingBase = {}                  # the largest gene end of every line of the sequence (overwritten genes too)
        for line in open(filename):
            if line.startswith('# Model Data') and not self.translationTable:
                for token in line.split(';'):
                    if 'transl_table' in token:
                        self.translationTable = int(token[token.find('=') + 1:])
            if line[0] == '#' or line.strip() == '"' or not line.strip():
                continue
            fields = line.split('\t')
            seqId = fields[0]
            if seqId not in genes:
                counter = 0                       # the running gene number restarts with every sequence first seen
                genes[seqId] = {}
            genes[seqId][counter] = (int(fields[3]), int(fields[4]))
            self.lastCodingBase[seqId] = max(self.lastCodingBase.get(seqId, 0), int(fields[4]))
            counter += 1
        self._covered = {}
        for seqId, spans in genes.items():
            covered, reach = 0, 0                 # union of the 1-based closed intervals
            for start, end in sorted(spans.values()):
                start = max(start, 1)
                if end > reach:
                    covered += end - max(start - 1, reach)
                    reach = end
            self._covered[seqId] = covered
        self.intervals = {seqId: self._mask_intervals(spans.values(), self.lastCodingBase[seqId]) for seqId, spans in genes.items()}

    @staticmethod
    def _mask_intervals(spans, L):
        """prodigal.py:250-261: a mask of length L (the largest gene end) with mask[start-1:end] = 1 per gene, Python slice
        semantics (a start of 0 marks only the last base; a start past L marks nothing), as sorted disjoint [lo, hi) and the
        covered bases before each interval."""
        cut = [slice(s - 1, e).indices(L)[:2] for s, e in spans]
        merged = []
        for lo, hi in sorted(c for c in cut if c[1] > c[0]):
            if merged and lo <= merged[-1][1]:
                merged[-1][1] = max(merged[-1][1], hi)
            else:
                merged.append([lo, hi])
        lo = np.array([m[0] for m in merged], dtype=np.int64)
        hi = np.array([m[1] for m in merged], dtype=np.int64)
        before = np.concatenate([[0], np.cumsum(hi - lo)[:-1]]).astype(np.int64) if len(merged) else lo
        return lo, hi, before

    def codingBases(self, seqId):
        return float(self._covered.get(seqId, 0))

    def windowCodingBases(self, seqId, starts, ends):
        """Per window [start, end) of the sequence: the number of mask positions set in it, np.sum(mask[start:end]) of
        prodigal.py:263-273 (clipped to the mask; 0 for a sequence without a gene).  starts, ends: non-negative."""
        starts = np.asarray(starts, dtype=np.int64)
        ends = np.asarray(ends, dtype=np.int64)
        if seqId not in self.intervals:
            return np.zeros(len(starts), dtype=np.int64)
        lo, hi, before = self.intervals[seqId]

        def covered_below(pos):
            j = np.searchsorted(lo, pos, side='right') - 1
            jj = np.maximum(j, 0)
            return np.where(j >= 0, before[jj] + np.minimum(pos, hi[jj]) - lo[jj], 0) if len(lo) else np.zeros(len(pos), dtype=np.int64)
        return np.maximum(covered_below(ends) - covered_below(starts), 0)


class BinStatistics(object):
    """Statistics of putative genome bins (name, arguments and results of checkm.binStatistics.BinStatistics)."""

    def __init__(self, threads=1):
        self.logger = logging.getLogger('timestamp')
        self.totalThreads = threads

    def calculate(self, binFiles, outDir, binStatsFile):
        """Statistics of every bin -> <outDir>/storage/<binStatsFile>, one line `binId<TAB>dict` per bin, bins in the order
        given (the reference writes them in the order its worker processes finish)."""
        self.logger.info("Calculating genome statistics for %d bins with %d threads:" % (len(binFiles), self.totalThreads))
        storage = os.path.join(outDir, 'storage')
        makeSurePathExists(storage)
        show = self.logger.getEffectiveLevel() <= logging.INFO
        done = 0
        with open(os.path.join(storage, binStatsFile), 'w') as fout:
            pending, pending_bytes = [], 0

            def flush():
                nonlocal pending, pending_bytes, done
                live = [p for p in pending if len(p[1][0]) > 0]
                scanned = dict(zip([p[0] for p in live], _scan([p[1] for p in live]))) if live else {}
                for binFile, parsed in pending:
                    binId = binIdFromFilename(binFile)
                    binDir = os.path.join(outDir, 'bins', binId)
                    done += 1
                    if binFile not in scanned:
                        self.logger.error('No sequences in bin: ' + binFile)
                        continue
                    fout.write(binId + '\t' + str(self._bin_stats(binDir, scanned[binFile])) + '\n')
                    if show:
                        sys.stderr.write('    Finished processing %d of %d (%.2f%%) bins.\r' % (done, len(binFiles), float(done) * 100 / len(binFiles)))
                        sys.stderr.flush()
                pending, pending_bytes = [], 0

            for binFile in binFiles:
                makeSurePathExists(os.path.join(outDir, 'bins', binIdFromFilename(binFile)))
                parsed = self._read(binFile)
                pending.append((binFile, parsed))
                pending_bytes += len(parsed[1])
                if pending_bytes >= BATCH_BYTES:
                    flush()
            if pending:
                flush()
        if show:
            sys.stderr.write('\n')

    def _read(self, fastaFile):
        try:
            return seqio.scan_nt_fasta(seqio.read_bytes(fastaFile))
        except Exception as e:                        # util/seqUtils.py:205-209
            print(e)
            self.logger.error("Failed to process sequence file: {}".format(fastaFile))
            sys.exit(1)

    def _bin_stats(self, binDir, sc):
        """binStatistics.py:99-139: the dictionary of one bin, keys in the reference's order."""
        binStats = {}
        GC, stdGC = _gc(sc)
        binStats['GC'] = GC
        binStats['GC std'] = stdGC
        (maxScaffoldLen, maxContigLen, genomeSize, scaffold_N50, contig_N50, scaffoldAvgLen, contigAvgLen, numContigs,
         numAmbiguousBases) = _seq_stats(sc)
        binStats['Genome size'] = genomeSize
        binStats['# ambiguous bases'] = numAmbiguousBases
        binStats['# scaffolds'] = len(sc.ids)
        binStats['# contigs'] = numContigs
        binStats['Longest scaffold'] = maxScaffoldLen
        binStats['Longest contig'] = maxContigLen
        binStats['N50 (scaffolds)'] = scaffold_N50
        binStats['N50 (contigs)'] = contig_N50
        binStats['Mean scaffold length'] = float(scaffoldAvgLen)
        binStats['Mean contig length'] = float(contigAvgLen)
        codingDensity, translationTable, numORFs = self._coding_density(binDir, sc.ids, genomeSize)
        binStats['Coding density'] = codingDensity
        binStats['Translation table'] = translationTable
        binStats['# predicted genes'] = numORFs
        return binStats

    def _coding_density(self, binDir, scaffoldIds, genomeSize):
        """binStatistics.py:235-253."""
        gffFile = os.path.join(binDir, PRODIGAL_GFF)
        if not os.path.exists(gffFile):
            return -1, -1, -1                         # pre-called genes: nothing to measure the density against
        features = _GeneFeatures(gffFile)
        names = seqio.read_fasta(os.path.join(binDir, PRODIGAL_AA))[0]
        codingBasePairs = 0
        for scaffoldId in scaffoldIds:
            codingBasePairs += features.codingBases(scaffoldId)
        return float(codingBasePairs) / genomeSize, features.translationTable, len(set(names))

    # ---- the reference's dictionary-taking methods ({sequence id: sequence string}) ----
    def calculateGC(self, seqs, seqStats=None):
        """Fraction of A/C/G/T(U) that is G or C over all sequences, and its standard deviation over the sequences longer
        than 1000 (binStatistics.py:176-206)."""
        if not seqs:
            return 0.0, 0.0
        return _gc(_scan([_from_dict(seqs)])[0], seqStats)

    def calculateSeqStats(self, scaffolds, seqStats=None):
        """max scaffold, max contig, total length, scaffold N50, contig N50, mean scaffold, mean contig, contigs, ambiguous
        bases (binStatistics.py:208-233)."""
        return _seq_stats(_scan([_from_dict(scaffolds)])[0], seqStats)

    def calculateCodingDensity(self, outDir, scaffolds, genomeSize):
        return self._coding_density(outDir, list(scaffolds.keys()), genomeSize)

    def sequenceStats(self, outDir, binFile):
        """Per-sequence statistics of a bin (binStatistics.py:263-290)."""
        sc = _scan([self._read(binFile)])[0]
        seqStats = {seqId: {} for seqId in sc.ids}
        _gc(sc, seqStats)
        _seq_stats(sc, seqStats)
        aaFile = os.path.join(outDir, 'bins', binIdFromFilename(binFile), PRODIGAL_AA)
        if os.path.exists(aaFile):
            names, _, _, offsets = seqio.read_fasta(aaFile)
            for geneId, residues in zip(names, np.diff(offsets)):
                entry = seqStats[geneId[0:geneId.rfind('_')]]
                entry['# ORFs'] = entry.get('# ORFs', 0) + 1
                entry['Coding bases'] = entry.get('Coding bases', 0) + int(residues) * 3
        return seqStats
