"""The part of the reference's plot base class (checkm/plot/AbstractPlot.py) that the plots use: the rcParams, the
Figure on an Agg canvas, the axes colour, savePlot and yLabelExtents; plus the pieces the plots share -- one bin's window
statistics from the device (`BinWindows`), the length profiles of many bins from one device call (`length_profiles`), the
histogram edges, the "prettify" block and the lower half of the delta-vs-length panels."""
import logging
import sys

import matplotlib as mpl
import matplotlib.transforms as mtransforms
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

    def yLabelExtents(self, labels, fontSize, rotation=0):
        """The bounds of the y tick labels in figure fractions, measured on a temporary axes that fills the figure."""
        self.fig.clear()
        tempAxes = self.fig.add_axes([0, 0, 1.0, 1.0])
        tempAxes.set_yticks(np.arange(len(labels)))
        yLabels = tempAxes.set_yticklabels(labels, size=fontSize, rotation=rotation)
        bboxes = [label.get_window_extent(self.get_renderer()).transformed(self.fig.transFigure.inverted()) for label in yLabels]
        yLabelBounds = mtransforms.Bbox.union(bboxes)
        self.fig.clear()
        return yLabelBounds

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
        self.ids, self.data, self.starts, self.lens = read_bin(fastaFile)
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


def read_bin(fastaFile):
    """A bin as the reference's readFasta sees it (seqio.scan_nt_fasta: ids in dict order, a repeated id keeping its last
    record); a file that cannot be read logs readFasta's error and exits with status 1."""
    try:
        return seqio.scan_nt_fasta(seqio.read_bytes(fastaFile))
    except Exception as e:                            # util/seqUtils.py:205-209
        print(e)
        logging.getLogger('timestamp').error("Failed to process sequence file: {}".format(fastaFile))
        sys.exit(1)


NX_OK, NX_INDEX, NX_SHORT = 0, 1, 2                   # ckm_length_profile's status of calculateNx


class LengthProfile(object):
    """One bin's share of a `ckm_length_profile` call: ids and lengths (readFasta's dict order), the total, the Nx list
    and its status (with `fail`: the rank of the record where calculateNx raises IndexError, or the number of thresholds
    reached), the 10 length-class counts of len_hist, and every record's rank in descending length order."""

    def __init__(self, binFile, ids, lens, total, nx, status, fail, classes, rank):
        self.binFile, self.binId = binFile, binIdFromFilename(binFile)
        self.ids, self.lens, self.total = ids, lens, total
        self.nx, self.status, self.fail, self.classes, self.rank = nx, status, fail, classes, rank

    def nxList(self):
        """calculateNx's return value when it returns (status NX_OK or NX_SHORT), as Python ints."""
        return self.nx[:len(self.nx) if self.status == NX_OK else self.fail].tolist()

    def sequenceAtRank(self, r):
        return self.ids[int(np.flatnonzero(self.rank == r)[0])]


def nx_fractions(step_size):
    """nx_plot's x: np.arange(0, 1 + step/2, step), as NxPlot.plot makes it."""
    return np.arange(0, 1.0 + 0.5 * step_size, step_size)


def length_profiles(binFiles, step_size=0.05, x=None):
    """The length profiles of many bins from one device call (ckm_length_profile): each bin read once as readFasta reads
    it, then the totals, the Nx lists at x (default: nx_fractions(step_size), sorted), the length classes and the ranks of
    every bin together.  Returns one LengthProfile per bin file, in order."""
    x = np.sort(nx_fractions(step_size) if x is None else np.asarray(x, dtype=np.float64))
    if len(x) == 0:
        raise ValueError('length_profiles: no Nx fractions')
    bins = [read_bin(f) for f in binFiles]
    counts = np.array([len(b[3]) for b in bins], dtype=np.int64)
    off = np.zeros(len(bins) + 1, dtype=np.int64)
    np.cumsum(counts, out=off[1:])
    lens = np.concatenate([b[3] for b in bins]) if bins else np.zeros(0, dtype=np.int64)
    try:
        total, nx, status, fail, classes, rank, _ = runtime.engine().length_profile(lens, off, x)
    except CkmError as e:
        logging.getLogger('timestamp').error('Length profile of bins %s: %s' % (', '.join(binIdFromFilename(f) for f in binFiles), e))
        sys.exit(1)
    return [LengthProfile(f, b[0], lens[off[i]:off[i + 1]], int(total[i]), nx[i], int(status[i]), int(fail[i]), classes[i],
                          rank[off[i]:off[i + 1]]) for i, (f, b) in enumerate(zip(binFiles, bins))]
