"""`checkm gc_plot` (checkm/plot/gcPlots.py): histogram of window GC and delta-GC vs sequence length.  The window base
counts come from the device (`BinWindows`); GC = float(g + c) / (a + c + g + t) per window on the host, a window without
A/C/G/T skipped as the reference's try/except skips it."""
import numpy as np

from ..binTools import BinTools
from ..common import findNearest, readDistribution
from .AbstractPlot import AbstractPlot, BinWindows


def windowGC(bw, windowSize, signature=False):
    """The window GC values of a bin in the reference's order, as Python floats, and the window base counts."""
    off, acgt, _ = bw.windows(windowSize, signature)
    n = acgt.sum(axis=1)
    return ((acgt[:, 1] + acgt[:, 2]).astype(np.float64) / n.astype(np.float64)), n


class GcPlots(AbstractPlot):
    def __init__(self, options):
        AbstractPlot.__init__(self, options)

    def plot(self, fastaFile, distributionsToPlot):
        self.fig.clear()
        self.fig.set_size_inches(self.options.width, self.options.height)
        axesHist = self.fig.add_subplot(121)
        axesDeltaGC = self.fig.add_subplot(122)
        self.plotOnAxes(fastaFile, distributionsToPlot, axesHist, axesDeltaGC)
        self.fig.tight_layout(pad=1, w_pad=1)
        self.draw()

    def plotOnAxes(self, fastaFile, distributionsToPlot, axesHist, axesDeltaGC, windows=None):
        dist = readDistribution('gc_dist')
        bw = windows if windows is not None else BinWindows(fastaFile)
        W = self.options.gc_window_size
        with np.errstate(divide='ignore', invalid='ignore'):
            gc, n = windowGC(bw, W)
        data = gc[n > 0].tolist()
        if len(data) == 0:
            axesHist.set_xlabel('[Error] No seqs >= %d, the specified window size' % W)
            return
        self._histogram(axesHist, data, self.options.gc_bin_width, '% GC', W)

        meanGC, deltaGCs, _ = BinTools().gcDist(bw.seqs)
        axesDeltaGC.scatter(deltaGCs, bw.lens.tolist(), c=abs(deltaGCs), s=10, lw=0.5, ec='black', cmap='gray_r')
        axesDeltaGC.set_xlabel(r'$\Delta$ GC (mean GC = %.1f%%)' % (meanGC * 100))
        axesDeltaGC.set_ylabel('Sequence length (kbp)')
        _, yMaxSeqs = axesDeltaGC.get_ylim()
        xMinSeqs, xMaxSeqs = axesDeltaGC.get_xlim()
        for distToPlot in distributionsToPlot:
            xL, xU, y = boundLines(dist, meanGC, distToPlot)
            axesDeltaGC.plot(xL, y, 'r--', lw=0.5, zorder=0)
            axesDeltaGC.plot(xU, y, 'r--', lw=0.5, zorder=0)
        self._finishDelta(axesDeltaGC, yMaxSeqs, xMinSeqs, xMaxSeqs)


def boundLines(dist, mean, distToPlot):
    """The lower and upper bound lines of a GC or CD distribution for one percentile range, sorted by length key."""
    closest = findNearest(np.array(list(dist.keys())), mean)
    byLen = dist[closest]
    d = byLen[list(byLen.keys())[0]]
    loKey = findNearest(list(d.keys()), (100 - distToPlot) / 2.0)
    hiKey = findNearest(list(d.keys()), (100 + distToPlot) / 2.0)
    xL = [byLen[n][loKey] for n in byLen]
    xU = [byLen[n][hiKey] for n in byLen]
    y = list(byLen)
    order = np.argsort(y)
    return np.array(xL)[order], np.array(xU)[order], np.array(y)[order]
