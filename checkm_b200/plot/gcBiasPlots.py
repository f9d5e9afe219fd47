"""`checkm gc_bias_plot` (checkm/plot/gcBiasPlots.py): GC against coverage per window and per sequence.  The window base
counts come from the device (`BinWindows`), the whole-sequence counts from the scaffold scan; the coverage profile is
CoverageWindows.run's.  A window or sequence without A/C/G/T, where the reference divides by zero, is refused with an
error naming it."""
import numpy as np
from numpy import array, log, mean, poly1d, polyfit

from ..binStatistics import _scan
from .AbstractPlot import AbstractPlot, BinWindows


class GcBiasPlot(AbstractPlot):
    def __init__(self, options):
        AbstractPlot.__init__(self, options)

    def plot(self, binFile, coverageProfile):
        self.fig.clear()
        self.fig.set_size_inches(self.options.width, self.options.height)
        windowAxes = self.fig.add_subplot(121)
        seqAxes = self.fig.add_subplot(122)
        self.plotOnAxes(binFile, coverageProfile, windowAxes, seqAxes)
        self.fig.tight_layout(pad=1)
        self.draw()

    def plotOnAxes(self, binFile, coverageProfile, windowAxes, seqAxes):
        bw = BinWindows(binFile)
        W = self.options.window_size
        off, acgt, _ = bw.windows(W)
        n, seqOf = bw.bases(W)
        bw.refuseEmpty(self, W, n, seqOf, 'GC')
        windowGC = ((acgt[:, 1] + acgt[:, 2]).astype(np.float64) / n.astype(np.float64)).tolist()
        whole = _scan([(bw.ids, bw.data, bw.starts, bw.lens)])[0].stats[:, :4] if bw.ids else np.zeros((0, 4), dtype=np.int64)
        seqN = whole.sum(axis=1)
        for s in np.flatnonzero(seqN == 0)[:1]:
            self._fatal('Sequence %s in bin %s has no A, C, G or T: its GC is undefined.' % (bw.ids[s], bw.binId))
        seqGC = ((whole[:, 1] + whole[:, 2]).astype(np.float64) / seqN.astype(np.float64)).tolist()

        offs = off.tolist()
        gc, coverage = [], []
        for s, seqId in enumerate(bw.ids):
            gc += windowGC[offs[s]:offs[s + 1]]
            coverage += coverageProfile[seqId][1]
        windowAxes.scatter(gc, coverage, c=abs(array(coverage)), s=10, lw=0.5, cmap='gray_r')
        windowAxes.set_xlabel('GC (mean = %.1f%%)' % (mean(gc) * 100))
        windowAxes.set_ylabel('Coverage (mean = %.1f)' % mean(coverage))
        if len(gc) > 1:
            slope, inter = polyfit(gc, coverage, 1)
            fit = poly1d([slope, inter])
            windowAxes.plot([min(gc), max(gc)], fit([min(gc), max(gc)]), '--r', lw=0.5)
            windowAxes.set_title('GC vs. Coverage\n(window size = %d bp, slope = %.2f)' % (W, slope))
        else:
            windowAxes.set_title('GC vs. Coverage\n(window size = %d bp, no best fit line)' % W)
        self._prettify(windowAxes)

        coverage = [coverageProfile[seqId][0] for seqId in bw.ids]
        seqLen = bw.lens.tolist()
        markerSize = log(array(seqLen))                               # log-scale, then onto 10 .. 210
        markerSize = (markerSize - min(markerSize)) / max(markerSize)
        markerSize = markerSize * 200 + 10
        seqAxes.scatter(seqGC, coverage, c=abs(array(coverage)), s=markerSize, lw=0.5, cmap='gray_r')
        seqAxes.set_xlabel('GC (mean = %.1f%%)' % (mean(seqGC) * 100))
        seqAxes.set_ylabel('Coverage (mean = %.1f)' % mean(coverage))
        seqAxes.set_title('GC vs. Coverage\nIndividual Sequences')
        self._prettify(seqAxes)
