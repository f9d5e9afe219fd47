"""`checkm dist_plot` (checkm/plot/distributionPlots.py): the GC, TD and CD plots of one bin on one figure.  The bin is
read once, and plots whose window sizes are equal share one device call."""
from .AbstractPlot import AbstractPlot, BinWindows
from .codingDensityPlots import CodingDensityPlots
from .gcPlots import GcPlots
from .tetraDistPlots import TetraDistPlots


class DistributionPlots(AbstractPlot):
    def __init__(self, options):
        AbstractPlot.__init__(self, options)
        self.options = options

    def plot(self, fastaFile, tetraSigs, distributionsToPlot):
        self.fig.clear()
        self.fig.set_size_inches(self.options.width, self.options.height)
        axesHistGC = self.fig.add_subplot(321)
        axesDeltaGC = self.fig.add_subplot(322)
        axesHistTD = self.fig.add_subplot(323)
        axesDeltaTD = self.fig.add_subplot(324)
        axesHistCD = self.fig.add_subplot(325)
        axesDeltaCD = self.fig.add_subplot(326)
        bw = BinWindows(fastaFile, tetraSigs, self.options.td_window_size)
        GcPlots(self.options).plotOnAxes(fastaFile, distributionsToPlot, axesHistGC, axesDeltaGC, windows=bw)
        TetraDistPlots(self.options).plotOnAxes(fastaFile, tetraSigs, distributionsToPlot, axesHistTD, axesDeltaTD, windows=bw)
        CodingDensityPlots(self.options).plotOnAxes(fastaFile, distributionsToPlot, axesHistCD, axesDeltaCD, windows=bw)
        self.fig.tight_layout(pad=1, w_pad=2, h_pad=2)
        self.draw()
