"""HmmerAligner (mirror of checkm/hmmerAligner.py) with every alignment of a call made in one device pass.

The reference forks `threads` worker processes, fetches each marker's HMM into a temporary file and runs `hmmalign` once
per marker, or per (bin, multi-copy marker) pair for the strain-heterogeneity alignments (hmmerAligner.py:125-302).
Here the HMM file is loaded once (`runtime.models_for`), each marker is selected by accession, and one `ckm_align_groups`
call aligns every group: one group per marker for `makeAlignmentTopHit` / `makeAlignmentToPhyloMarkers`, one per (bin,
marker) for `makeAlignmentsOfMultipleHits`.  No process is started (a CUDA context cannot cross fork); `threads` is
accepted and ignored.  The masked FASTA the reference's `_maskAlignment` makes of the `hmmalign` Pfam output is built
straight from the per-residue states: column k holds the upper-case residue whose state is +k, else '-'.  Where a
reference worker would raise and leave a marker without its file, this logs an error naming bin, marker and sequence and
exits with status 1."""
import logging
import os
import sys
from collections import defaultdict

import numpy as np

from . import runtime
from ._lib import CkmError
from .binTools import readFasta
from .common import makeSurePathExists
from .defaultValues import DefaultValues
from .engine import digitize
from .hmmer import _LETTERS, format_alignment
from .resultsParser import ResultsParser

_SYMBOLS = np.frombuffer(_LETTERS.encode(), dtype=np.uint8)
_GAP = ord('-')


def masked_rows(residues, state, lens, M):
    """The masked alignment rows of sequences aligned to one model of M positions: an n x M uint8 array holding the residue
    symbol whose state is +k in column k - 1, '-' elsewhere (hmmerAligner.py:327-358 applied to hmmalign's Pfam output)."""
    lens = np.asarray(lens, dtype=np.int64)
    rows = np.full((len(lens), M), _GAP, dtype=np.uint8)
    seq_of = np.repeat(np.arange(len(lens)), lens)
    sel = state > 0
    rows[seq_of[sel], state[sel] - 1] = _SYMBOLS[residues[sel]]
    return rows


class _Group(object):
    """One `hmmalign` call of the reference: the sequences of one marker file, in the order the reference writes them."""
    __slots__ = ('markerId', 'outDir', 'names', 'descs', 'seqs', 'model')

    def __init__(self, markerId, outDir):
        self.markerId, self.outDir = markerId, outDir
        self.names, self.descs, self.seqs = [], [], []
        self.model = -1


class HmmerAligner(object):
    def __init__(self, threads):
        self.logger = logging.getLogger('timestamp')
        self.totalThreads = threads
        self.outputFormat = 'Pfam'

    def makeAlignmentTopHit(self, outDir, hmmModelFile, hmmTableFile, binIdToModels, bIgnoreThresholds, evalueThreshold,
                            lengthThreshold, bReportHitStats, alignOutputDir, bKeepUnmaskedAlign=False):
        """Align top hits in each bin. Assumes all bins are using the same marker genes."""
        self.logger.info("Extracting marker genes to align.")
        resultsParser = ResultsParser(binIdToModels)
        resultsParser.parseBinHits(outDir, hmmTableFile, False, bIgnoreThresholds, evalueThreshold, lengthThreshold)
        markerSeqs, markerStats = self._extractMarkerSeqsTopHits(outDir, resultsParser)
        self._alignMarkerGenes(markerSeqs, markerStats, bReportHitStats, hmmModelFile, binIdToModels, alignOutputDir,
                               bKeepUnmaskedAlign)
        return resultsParser

    def makeAlignmentToPhyloMarkers(self, outDir, hmmModelFile, hmmTableFile, binIdToModels, bIgnoreThresholds, evalueThreshold,
                                    lengthThreshold, bReportHitStats, alignOutputDir, bKeepUnmaskedAlign=False):
        """Align hits to a set of common marker genes."""
        self.logger.info("Extracting marker genes to align.")
        resultsParser = ResultsParser(binIdToModels)
        resultsParser.parseBinHits(outDir, hmmTableFile, False, bIgnoreThresholds, evalueThreshold, lengthThreshold)
        markerSeqs, markerStats = self._extractMarkerSeqsUnique(outDir, resultsParser)
        self._alignMarkerGenes(markerSeqs, markerStats, bReportHitStats, hmmModelFile, binIdToModels, alignOutputDir,
                               bKeepUnmaskedAlign)
        return resultsParser

    def makeAlignmentsOfMultipleHits(self, outDir, markerFile, hmmTableFile, binIdToModels, binIdToBinMarkerSets,
                                     bIgnoreThresholds, evalueThreshold, lengthThreshold, alignOutputDir):
        """Align markers with multiple hits within a bin: one group per (bin, marker), all in one device pass."""
        makeSurePathExists(alignOutputDir)
        resultsParser = ResultsParser(binIdToModels)
        resultsParser.parseBinHits(outDir, hmmTableFile, False, bIgnoreThresholds, evalueThreshold, lengthThreshold)
        self.logger.info('Aligning marker genes with multiple hits in a single bin:')
        groups = []
        for binId in binIdToModels:
            markers = self._extractMarkersWithMultipleHits(outDir, binId, resultsParser, binIdToBinMarkerSets[binId])
            if len(markers) == 0:
                continue
            binAlignOutputDir = os.path.join(alignOutputDir, binId)
            makeSurePathExists(binAlignOutputDir)
            for markerId, binSeqs in markers.items():
                groups.append(self._group(markerId, binSeqs, None, False, binAlignOutputDir))
        self._alignGroups(groups, markerFile, False)

    # ------------------------------------------------------------------ sequences, in the reference's order
    def _alignMarkerGenes(self, markerSeqs, markerStats, bReportHitStats, hmmModelFile, binIdToModels, alignOutputDir,
                          bKeepUnmaskedAlign):
        """One group per marker of the first bin's model set that has sequences (hmmerAligner.py:71-81, 229-302)."""
        markerIds = list(binIdToModels[list(binIdToModels.keys())[0]].keys())
        self.logger.info("Extracting %d HMMs with %d threads:" % (len(markerIds), self.totalThreads))
        makeSurePathExists(alignOutputDir)
        self.logger.info("Aligning %d marker genes with %d threads:" % (len(markerIds), self.totalThreads))
        groups = []
        for markerId in markerIds:
            g = self._group(markerId, markerSeqs.get(markerId, {}), markerStats.get(markerId, {}), bReportHitStats, alignOutputDir)
            if g.seqs:
                groups.append(g)
        self._alignGroups(groups, hmmModelFile, bKeepUnmaskedAlign)

    def _group(self, markerId, binSeqs, binStats, bReportHitStats, outDir):
        """The sequences and headers `_alignMarker` writes to the unaligned file (hmmerAligner.py:276-289)."""
        g = _Group(markerId, outDir)
        for binId, seqs in binSeqs.items():
            for seqId, seq in seqs.items():
                g.names.append(binId + DefaultValues.SEQ_CONCAT_CHAR + seqId)
                g.descs.append('[e-value=%.4g,score=%.1f]' % (binStats[binId][seqId][0], binStats[binId][seqId][1])
                               if bReportHitStats else '')
                g.seqs.append(seq)
        return g

    def _extractMarkerSeqsTopHits(self, outDir, resultsParser):
        """Per marker and bin, the hit left first by a descending in-place sort on the e-value: the LARGEST e-value, as in
        the reference (hmmerAligner.py:360-382)."""
        markerSeqs = defaultdict(dict)
        markerStats = defaultdict(dict)
        for binId in resultsParser.results:
            binORFs = readFasta(os.path.join(outDir, 'bins', binId, DefaultValues.PRODIGAL_AA))
            for markerId, hits in resultsParser.results[binId].markerHits.items():
                markerSeqs[markerId][binId] = {}
                markerStats[markerId][binId] = {}
                hits.sort(key=lambda x: x.full_e_value, reverse=True)
                topHit = hits[0]
                markerSeqs[markerId][binId][topHit.target_name] = self._extractSeq(topHit.target_name, binORFs, binId, markerId)
                markerStats[markerId][binId][topHit.target_name] = [topHit.full_e_value, topHit.full_score]
        return markerSeqs, markerStats

    def _extractMarkerSeqsUnique(self, outDir, resultsParser):
        """Per marker and bin, the hit of markers with exactly one hit (hmmerAligner.py:384-405)."""
        markerSeqs = defaultdict(dict)
        markerStats = defaultdict(dict)
        for binId in resultsParser.results:
            binORFs = readFasta(os.path.join(outDir, 'bins', binId, DefaultValues.PRODIGAL_AA))
            for markerId, hits in resultsParser.results[binId].markerHits.items():
                markerSeqs[markerId][binId] = {}
                markerStats[markerId][binId] = {}
                if len(hits) == 1:
                    hit = hits[0]
                    markerSeqs[markerId][binId][hit.target_name] = self._extractSeq(hit.target_name, binORFs, binId, markerId)
                    markerStats[markerId][binId][hit.target_name] = [hit.full_e_value, hit.full_score]
        return markerSeqs, markerStats

    def _extractMarkersWithMultipleHits(self, outDir, binId, resultsParser, binMarkerSet):
        """Markers of the bin's selected marker set with two or more hits; hits sorted by descending e-value in place, one
        sequence per target (hmmerAligner.py:430-452)."""
        markersWithMultipleHits = defaultdict(dict)
        binORFs = readFasta(os.path.join(outDir, 'bins', binId, DefaultValues.PRODIGAL_AA))
        markerGenes = binMarkerSet.selectedMarkerSet().getMarkerGenes()
        for markerId, hits in resultsParser.results[binId].markerHits.items():
            if markerId not in markerGenes or len(hits) < 2:
                continue
            hits.sort(key=lambda x: x.full_e_value, reverse=True)
            markersWithMultipleHits[markerId][binId] = {}
            for hit in hits:
                markersWithMultipleHits[markerId][binId][hit.target_name] = self._extractSeq(hit.target_name, binORFs, binId, markerId)
        return markersWithMultipleHits

    def _extractSeq(self, seqId, seqs, binId, markerId):
        """The ORF of a hit; an adjacent-ORF hit `A&&B` is the concatenation of its ORFs; a final '*' is dropped from each
        (hmmerAligner.py:407-428)."""
        seq = ''
        for part in seqId.split(DefaultValues.SEQ_CONCAT_CHAR):
            if part not in seqs:
                self.logger.error('Sequence %s of the hit of marker %s in bin %s is not in %s.'
                                  % (part, markerId, binId, DefaultValues.PRODIGAL_AA))
                sys.exit(1)
            s = seqs[part]
            seq += s[0:-1] if s[-1:] == '*' else s
        return seq

    # ------------------------------------------------------------------ one device pass, then the files
    def _alignGroups(self, groups, hmmModelFile, bKeepUnmaskedAlign):
        if not groups:
            return
        try:
            eng = runtime.engine()
            models = runtime.models_for(hmmModelFile)
            for g in groups:
                g.model = models.find(g.markerId)
                if g.model < 0:
                    self.logger.error('Marker %s is not in the HMM file %s.' % (g.markerId, hmmModelFile))
                    sys.exit(1)
            info = models.info()
            seqs = [s for g in groups for s in g.seqs]
            lens = np.array([len(s) for s in seqs], dtype=np.int64)
            offsets = np.zeros(len(seqs) + 1, dtype=np.int64)
            np.cumsum(lens, out=offsets[1:])
            residues = digitize(''.join(seqs))
            group_off = np.zeros(len(groups) + 1, dtype=np.int64)
            np.cumsum([len(g.seqs) for g in groups], out=group_off[1:])
            db = eng.seqdb(residues, offsets)
            try:
                state, _oasc = eng.align_groups(models, db, [g.model for g in groups], group_off)
            finally:
                db.close()
        except CkmError as err:
            self.logger.error('hmmalign engine exited with code: %d (%s)' % (err.code, err))
            sys.exit(err.code)
        for gi, g in enumerate(groups):
            s0, s1 = int(group_off[gi]), int(group_off[gi + 1])
            r0, r1 = int(offsets[s0]), int(offsets[s1])
            M = int(info[g.model].M)
            res, st = residues[r0:r1], state[r0:r1]
            rows = masked_rows(res, st, lens[s0:s1], M)
            with open(os.path.join(g.outDir, g.markerId + '.masked.faa'), 'w') as fout:
                for name, desc, row in zip(g.names, g.descs, rows):
                    fout.write(('>%s %s\n' % (name, desc)) if desc else ('>' + name + '\n'))
                    fout.write(row.tobytes().decode('ascii') + '\n')
            if bKeepUnmaskedAlign:
                text = format_alignment(g.names, g.descs, res, offsets[s0:s1 + 1] - r0, st, M, self.outputFormat, False)
                with open(os.path.join(g.outDir, g.markerId + '.aligned.faa'), 'w') as fout:
                    fout.write(text)
