"""The part of the reference's plot base class (checkm/plot/AbstractPlot.py) that the window plots use: the rcParams, the
Figure on an Agg canvas, the axes colour and savePlot; plus the pieces the plots share -- one bin's window statistics from
the device (`BinWindows`), the histogram edges, the "prettify" block and the lower half of the delta-vs-length panels."""
import logging
import sys

import matplotlib as mpl
from matplotlib.backends.backend_agg import FigureCanvasAgg as FigureCanvas
from matplotlib.figure import Figure

import numpy as np

from .. import runtime, seqio
from .._lib import CkmError
from ..binTools import BinTools
from ..common import binIdFromFilename
from ..coverageWindows import window_offsets


class AbstractPlot(FigureCanvas):
    """Base class of the plots (name and constructor of checkm.plot.AbstractPlot.AbstractPlot)."""

    def __init__(self, options):
        self.options = options
        for key in ('font.size', 'axes.titlesize', 'axes.labelsize', 'xtick.labelsize', 'ytick.labelsize', 'legend.fontsize'):
            mpl.rcParams[key] = self.options.font_size
        mpl.rcParams['svg.fonttype'] = 'none'
        self.fig = Figure(facecolor='white', dpi=options.dpi)
        FigureCanvas.__init__(self, self.fig)
        self.cid = None
        self.type = '<none>'
        self.name = '<none>'
        self.axesColour = (0.5, 0.5, 0.5)

    def savePlot(self, filename, dpi=300):
        imgFormat = filename[filename.rfind('.') + 1:]
        if imgFormat in ('png', 'pdf', 'ps', 'eps', 'svg'):
            self.fig.savefig(filename, format=imgFormat, dpi=dpi, facecolor='white', edgecolor='white', bbox_inches='tight')

    # ---- shared by the plots ----
    def _fatal(self, message):
        logging.getLogger('timestamp').error(message)
        sys.exit(1)

    def _prettify(self, axes):
        """Ticks on the bottom and left only, tick lines and the two remaining spines in the axes colour."""
        for axis in (axes.yaxis, axes.xaxis):
            for tick in axis.majorTicks:
                tick.tick1On = True
                tick.tick2On = False
        for axis in (axes.yaxis, axes.xaxis):
            for line in axis.get_ticklines():
                line.set_color(self.axesColour)
        for loc, spine in axes.spines.items():
            spine.set_color('none' if loc in ('right', 'top') else self.axesColour)

    def _histogram(self, axes, data, binWidth, xLabel, windowSize):
        """The window histogram: edges 0, w, w + w, ... up to 1.0 by repeated float addition, density, grey bars."""
        edges = [0.0]
        edge = binWidth
        while edge <= 1.0:
            edges.append(edge)
            edge += binWidth
        axes.hist(data, bins=edges, density=True, color=(0.5, 0.5, 0.5))
        axes.set_xlabel(xLabel)
        axes.set_ylabel('% windows (' + str(windowSize) + ' bp)')
        self._prettify(axes)

    def _finishDelta(self, axes, yMaxSeqs, xMinSeqs, xMaxSeqs):
        """The delta-vs-length panel after its reference lines: the limits taken before them, a dashed line at 0 up to
        the last y tick, the y ticks relabelled in kbp."""
        axes.set_ylim([0, yMaxSeqs])
        axes.set_xlim([xMinSeqs, xMaxSeqs])
        yticks = axes.get_yticks()
        axes.vlines(0, 0, yticks[-1], linestyle='dashed', color=self.axesColour, zorder=0)
        labels = [('%.1f' % (float(v) / 1000)).replace('.0', '') for v in yticks]
        axes.set_yticks(yticks)
        axes.set_yticklabels(labels)
        self._prettify(axes)


class BinWindows(object):
    """One bin read once (seqio.scan_nt_fasta, the reference's readFasta) and its window statistics from the device, one
    `ckm_window_stats` call per window size.  At `sigWindowSize` the call also returns the tetranucleotide distances to the
    bin's signature (BinTools.binTetraSig over `tetraSigs`), so plots that share a window size share the call."""

    def __init__(self, fastaFile, tetraSigs=None, sigWindowSize=None):
        try:
            self.ids, self.data, self.starts, self.lens = seqio.scan_nt_fasta(seqio.read_bytes(fastaFile))
        except Exception as e:                        # util/seqUtils.py:205-209
            print(e)
            logging.getLogger('timestamp').error("Failed to process sequence file: {}".format(fastaFile))
            sys.exit(1)
        raw = self.data.tobytes()
        self.seqs = {i: raw[a:a + n].decode('latin-1') for i, a, n in zip(self.ids, self.starts.tolist(), self.lens.tolist())}
        self.binId = binIdFromFilename(fastaFile)
        self.tetraSigs, self.sigWindowSize = tetraSigs, sigWindowSize
        self._binSig = None
        self._calls = {}

    def binSig(self):
        if self._binSig is None:
            self._binSig = BinTools().binTetraSig(self.seqs, self.tetraSigs)
        return self._binSig

    def windows(self, windowSize, signature=False):
        """(win_off, nwin x 4 int64 A C G T counts, nwin distances or None) at this window size."""
        signature = signature or (self.tetraSigs is not None and windowSize == self.sigWindowSize)
        got = self._calls.get(windowSize)
        if got is None or (signature and got[2] is None):
            off = window_offsets(self.lens, windowSize)
            try:
                acgt, td, _ = runtime.engine().window_stats(self.data, self.starts, self.lens, windowSize, off,
                                                            self.binSig() if signature else None)
            except CkmError as e:
                logging.getLogger('timestamp').error('Window statistics of bin %s: %s' % (self.binId, e))
                sys.exit(1)
            got = self._calls[windowSize] = (off, acgt, td)
        return got

    def bases(self, windowSize, signature=False):
        """The A+C+G+T count of every window, and the sequence index of every window."""
        off, acgt, _ = self.windows(windowSize, signature)
        return acgt.sum(axis=1), np.repeat(np.arange(len(self.ids)), np.diff(off))

    def refuseEmpty(self, plot, windowSize, n, seqOf, what):
        """Logs an error naming the first window without A/C/G/T and exits (the reference divides by zero there)."""
        empty = np.flatnonzero(n == 0)
        if len(empty):
            w = int(empty[0])
            s = int(seqOf[w])
            off = self.windows(windowSize)[0]
            plot._fatal('Window %d (%d bp from position %d) of sequence %s in bin %s has no A, C, G or T: its %s is undefined.'
                        % (w - int(off[s]), windowSize, (w - int(off[s])) * windowSize, self.ids[s], self.binId, what))
