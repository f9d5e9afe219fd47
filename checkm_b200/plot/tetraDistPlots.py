"""`checkm tetra_plot` (checkm/plot/tetraDistPlots.py): histogram of the windows' tetranucleotide distance to the bin
signature and delta-TD vs sequence length.  The bin signature is BinTools.binTetraSig (device); the distance of every
window comes from the same device call as its base counts (`BinWindows` at the TD window size)."""
import numpy as np

from ..binTools import BinTools
from ..common import findNearest, readDistribution
from ..genomicSignatures import GenomicSignatures
from .AbstractPlot import AbstractPlot, BinWindows


class TetraDistPlots(AbstractPlot):
    def __init__(self, options):
        AbstractPlot.__init__(self, options)

    def plot(self, fastaFile, tetraSigs, distributionsToPlot):
        self.fig.clear()
        self.fig.set_size_inches(self.options.width, self.options.height)
        axesHist = self.fig.add_subplot(121)
        axesDeltaTD = self.fig.add_subplot(122)
        self.plotOnAxes(fastaFile, tetraSigs, distributionsToPlot, axesHist, axesDeltaTD)
        self.fig.tight_layout(pad=1, w_pad=1)
        self.draw()

    def plotOnAxes(self, fastaFile, tetraSigs, distributionsToPlot, axesHist, axesDeltaTD, windows=None):
        dist = readDistribution('td_dist')
        W = self.options.td_window_size
        bw = windows if windows is not None else BinWindows(fastaFile, tetraSigs, W)
        binTools = BinTools()
        binSig = bw.binSig()
        genomicSig = GenomicSignatures(K=4, threads=1)
        for seqId in bw.ids:                          # the reference's per-sequence distances (unused; KeyError kept)
            genomicSig.distance(tetraSigs[seqId], binSig)
        data = bw.windows(W, signature=True)[2].tolist()
        if len(data) == 0:
            axesHist.set_xlabel('[Error] No seqs >= %d, the specified window size' % W)
            return
        self._histogram(axesHist, data, self.options.td_bin_width, r'$\Delta$ TD', W)

        meanTD, deltaTDs = binTools.tetraDiffDist(bw.seqs, genomicSig, tetraSigs, binSig)
        axesDeltaTD.scatter(deltaTDs, bw.lens.tolist(), c=abs(deltaTDs), s=10, lw=0.5, ec='black', cmap='gray_r')
        axesDeltaTD.set_xlabel(r'$\Delta$ TD (mean TD = %.2f)' % meanTD)
        axesDeltaTD.set_ylabel('Sequence length (kbp)')
        _, yMaxSeqs = axesDeltaTD.get_ylim()
        xMinSeqs, xMaxSeqs = axesDeltaTD.get_xlim()
        for distToPlot in distributionsToPlot:
            boundKey = findNearest(list(dist[list(dist.keys())[0]].keys()), distToPlot)
            y = list(dist)
            order = np.argsort(y)
            x = np.array([dist[n][boundKey] for n in y])[order]
            y = np.array(y)[order]
            # never rising with length: a value above an earlier one becomes the mean of its neighbours (the last one the
            # earlier value), and at most the earlier value
            for i in range(len(x) - 1):
                for j in range(i + 1, len(x)):
                    if x[j] > x[i]:
                        x[j] = x[i] if j == len(x) - 1 else (x[j - 1] + x[j + 1]) / 2
                        if x[j] > x[i]:
                            x[j] = x[i]
            axesDeltaTD.plot(x, y, 'r--', lw=0.5, zorder=0)
        self._finishDelta(axesDeltaTD, yMaxSeqs, xMinSeqs, xMaxSeqs)
