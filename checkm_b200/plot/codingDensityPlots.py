"""`checkm coding_plot` (checkm/plot/codingDensityPlots.py): histogram of window coding density and delta-CD vs sequence
length.  Window base counts from the device (`BinWindows`); the coding bases of every window from the GFF's mask intervals
on the host (`_GeneFeatures.windowCodingBases`); CD = float(coding) / (a + c + g + t).  A window without A/C/G/T, where
the reference divides by zero, is refused with an error naming it."""
import logging
import os
import sys

import numpy as np

from ..binStatistics import _GeneFeatures
from ..binTools import BinTools
from ..common import binIdFromFilename, readDistribution
from ..defaultValues import DefaultValues
from .AbstractPlot import AbstractPlot, BinWindows
from .gcPlots import boundLines


class _MaskCodingBases(object):
    """codingBases(seqId) as the reference's parser counts it: the sum of the whole mask (prodigal.py:263-273)."""

    def __init__(self, features):
        self.features = features

    def codingBases(self, seqId):
        L = self.features.lastCodingBase.get(seqId, 0)
        return float(self.features.windowCodingBases(seqId, [0], [L])[0])


class CodingDensityPlots(AbstractPlot):
    def __init__(self, options):
        AbstractPlot.__init__(self, options)
        self.logger = logging.getLogger('timestamp')

    def plot(self, fastaFile, distributionsToPlot):
        self.fig.clear()
        self.fig.set_size_inches(self.options.width, self.options.height)
        axesHist = self.fig.add_subplot(121)
        axesDeltaCD = self.fig.add_subplot(122)
        self.plotOnAxes(fastaFile, distributionsToPlot, axesHist, axesDeltaCD)
        self.fig.tight_layout(pad=1, w_pad=1)
        self.draw()

    def plotOnAxes(self, fastaFile, distributionsToPlot, axesHist, axesDeltaCD, windows=None):
        gffFile = os.path.join(self.options.results_dir, 'bins', binIdFromFilename(fastaFile), DefaultValues.PRODIGAL_GFF)
        if not os.path.exists(gffFile):
            self.logger.error('Missing gene feature file (%s). This plot if not compatible with the --genes option.'
                              % DefaultValues.PRODIGAL_GFF)
            sys.exit(1)
        features = _GeneFeatures(gffFile)
        dist = readDistribution('cd_dist')
        bw = windows if windows is not None else BinWindows(fastaFile)
        W = self.options.cd_window_size
        off, acgt, _ = bw.windows(W)
        n, seqOf = bw.bases(W)
        bw.refuseEmpty(self, W, n, seqOf, 'coding density')
        coding = np.zeros(len(n), dtype=np.int64)
        for s, seqId in enumerate(bw.ids):
            k = np.arange(int(off[s + 1] - off[s]), dtype=np.int64)
            coding[off[s]:off[s + 1]] = features.windowCodingBases(seqId, k * W, (k + 1) * W)
        data = (coding.astype(np.float64) / n.astype(np.float64)).tolist()
        if len(data) == 0:
            axesHist.set_xlabel('[Error] No seqs >= %d, the specified window size' % W)
            return
        self._histogram(axesHist, data, self.options.cd_bin_width, '% coding density', W)

        meanCD, deltaCDs, _ = BinTools().codingDensityDist(bw.seqs, _MaskCodingBases(features))
        axesDeltaCD.scatter(deltaCDs, bw.lens.tolist(), c=abs(deltaCDs), s=10, lw=0.5, ec='black', cmap='gray_r')
        axesDeltaCD.set_xlabel(r'$\Delta$ CD (mean coding density = %.1f%%)' % (meanCD * 100))
        axesDeltaCD.set_ylabel('Sequence length (kbp)')
        _, yMaxSeqs = axesDeltaCD.get_ylim()
        xMinSeqs, xMaxSeqs = axesDeltaCD.get_xlim()
        for distToPlot in distributionsToPlot:
            xL, xU, y = boundLines(dist, meanCD, distToPlot)
            axesDeltaCD.plot(xL, y, 'r--', lw=0.5, zorder=0)
            axesDeltaCD.plot(xU, y, 'r--', lw=0.5, zorder=0)
        self._finishDelta(axesDeltaCD, yMaxSeqs, xMinSeqs, xMaxSeqs)
