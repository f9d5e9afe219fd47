"""AminoAcidIdentity (mirror of checkm/aminoAcidIdentity.py): AAI between the copies of every multi-copy marker of every
bin, and the strain heterogeneity the QA tables report.

The reference compares every pair of masked rows with a per-character Python loop (aminoAcidIdentity.py:64-93, 127-161).
Here `run` reads the `.masked.faa` files in the reference's order, packs every pair i < j of every file of every bin, and
one `ckm_aai_pairs` call returns each pair's mismatches and compared length; the AAI is then formed in float64 exactly as
the reference writes it.  `aai(seq1, seq2)` is a one-pair call of the same kernel."""
import logging
import os
import sys
from collections import defaultdict

import numpy as np

from . import runtime
from ._lib import CkmError
from .binTools import readFasta
from .common import getBinIdsFromOutDir
from .defaultValues import DefaultValues


def _identity(mismatches, seqLen):
    if seqLen == 0:
        return 0.0
    return 1.0 - (float(mismatches) / int(seqLen))


def _pair_counts(rows, pairs):
    """Mismatches and compared lengths of `pairs` (index pairs into the list of ASCII strings `rows`) in one device call."""
    data = ''.join(rows).encode('latin-1')
    row_off = np.zeros(len(rows) + 1, dtype=np.int64)
    np.cumsum([len(r) for r in rows], out=row_off[1:])
    return runtime.engine().aai_pairs(data, row_off, np.asarray(pairs, dtype=np.int32).reshape(-1, 2))


class AminoAcidIdentity(object):
    """Calculate AAI between sequences aligned to an HMM."""

    def __init__(self):
        self.logger = logging.getLogger('timestamp')
        self.aaiRawScores = defaultdict(dict)
        self.aaiHetero = defaultdict(dict)
        self.aaiMeanBinHetero = {}

    def run(self, aaiStrainThreshold, outDir, alignmentOutputFile):
        """Calculate AAI between input alignments."""
        self.logger.info('Calculating AAI between multi-copy marker genes.')
        if alignmentOutputFile:
            fout = open(alignmentOutputFile, 'w')

        rows, pairs, meta = [], [], []          # meta per pair: bin directory, marker, bin of the pair, row ids
        aaiOutputDir = os.path.join(outDir, 'storage', 'aai_qa')
        for binId in getBinIdsFromOutDir(outDir):
            binPath = os.path.join(aaiOutputDir, binId)
            if not os.path.exists(binPath):
                continue
            for f in os.listdir(binPath):
                if not f.endswith('.masked.faa'):
                    continue
                markerId = f[0:f.find('.')]
                seqs = readFasta(os.path.join(binPath, f))
                ids = list(seqs.keys())
                base = len(rows)
                rows.extend(seqs[seqId] for seqId in ids)
                for i in range(0, len(ids)):
                    seqIdI = ids[i]
                    binIdI = seqIdI[0:seqIdI.find(DefaultValues.SEQ_CONCAT_CHAR)]
                    for j in range(i + 1, len(ids)):
                        seqIdJ = ids[j]
                        binIdJ = seqIdJ[0:seqIdJ.find(DefaultValues.SEQ_CONCAT_CHAR)]
                        if binIdI != binIdJ:
                            # something is wrong as the bin Ids should always be the same
                            self.logger.error('Bin ids do not match.')
                            sys.exit(1)
                        if len(seqs[seqIdI]) != len(seqs[seqIdJ]):
                            self.logger.error('Aligned sequences %s and %s of %s differ in length (%d and %d).'
                                              % (seqIdI, seqIdJ, os.path.join(binPath, f), len(seqs[seqIdI]), len(seqs[seqIdJ])))
                            sys.exit(1)
                        pairs.append((base + i, base + j))
                        meta.append((binId, markerId, binIdI, seqIdI, seqIdJ))

        mismatches, lengths = np.zeros(0, dtype=np.int32), np.zeros(0, dtype=np.int32)
        if pairs:
            try:
                mismatches, lengths = _pair_counts(rows, pairs)
            except CkmError as err:
                self.logger.error('AAI engine exited with code: %d (%s)' % (err.code, err))
                sys.exit(1)

        for (i, j), (binId, markerId, binIdI, seqIdI, seqIdJ), m, n in zip(pairs, meta, mismatches.tolist(), lengths.tolist()):
            aai = _identity(m, n)
            if alignmentOutputFile:
                fout.write(binId + ',' + markerId + '\n')
                fout.write(seqIdI + '\t' + rows[i] + '\n')
                fout.write(seqIdJ + '\t' + rows[j] + '\n')
                fout.write('AAI: %.3f\n' % aai)
                fout.write('\n')
            if binIdI not in self.aaiRawScores:
                self.aaiRawScores[binIdI] = defaultdict(list)
            self.aaiRawScores[binIdI][markerId].append(aai)

        if alignmentOutputFile:
            fout.close()

        # calculate strain heterogeneity for each marker gene in each bin
        self.aaiHetero, self.aaiMeanBinHetero = self.strainHetero(self.aaiRawScores, aaiStrainThreshold)

    def strainHetero(self, aaiScores, aaiStrainThreshold):
        """Calculate strain heterogeneity."""
        aaiHetero = defaultdict(dict)
        aaiMeanBinHetero = {}
        for binId, markerIds in aaiScores.items():
            strainCount = 0
            multiCopyPairs = 0
            aaiHetero[binId] = {}
            for markerId, scores in markerIds.items():
                localStrainCount = 0
                for aaiScore in scores:
                    multiCopyPairs += 1
                    if aaiScore > aaiStrainThreshold:
                        strainCount += 1
                        localStrainCount += 1
                aaiHetero[binId][markerId] = float(localStrainCount) / len(scores)
            aaiMeanBinHetero[binId] = 100 * float(strainCount) / multiCopyPairs
        return aaiHetero, aaiMeanBinHetero

    def aai(self, seq1, seq2):
        """Calculate amino acid identity between sequences."""
        assert len(seq1) == len(seq2)
        mismatches, lengths = _pair_counts([seq1, seq2], [(0, 1)])
        return _identity(int(mismatches[0]), int(lengths[0]))
