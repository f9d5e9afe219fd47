"""`checkm marker_plot` (checkm/plot/markerGenePosPlot.py): where each scaffold's marker genes lie, in 100 position bins
per row.  The scaffold lengths and their descending order come from the device (`length_profiles`, ckm_length_profile);
gene positions from the `genes.faa` header lines (`seqio.read_fasta`, ckm_fasta_parse), as ProdigalFastaParser reads
them.  Where the reference raises (a gene missing from genes.faa, a position past its row), the bin and the gene are
named in an error and the command exits with status 1."""
import logging
import math
import os

import matplotlib as mpl
import numpy as np
from matplotlib.patches import Rectangle

from .. import seqio
from ..common import binIdFromFilename
from ..defaultValues import DefaultValues
from .AbstractPlot import AbstractPlot, length_profiles

MAX_BINS = 100
COLOURS = [(1.0, 1.0, 1.0), (127 / 255.0, 201 / 255.0, 127 / 255.0), (255 / 255.0, 192 / 255.0, 134 / 255.0),
           (190 / 255.0, 174 / 255.0, 212 / 255.0), (0.0, 0.0, 0.0)]


def gene_positions(geneFile):
    """{gene id: [start, end]} from the header lines of a Prodigal protein file: fields 2 and 4 of the header's
    whitespace split (the text after the id is `# start # end # strand # ...`); a repeated id keeps its last header."""
    names, descs, _, _ = seqio.read_fasta(geneFile)
    gp = {}
    for name, desc in zip(names, descs):
        f = desc.split()
        gp[name] = [int(f[1]), int(f[3])]
    return gp


class MarkerGenePosPlot(AbstractPlot):
    def __init__(self, options):
        AbstractPlot.__init__(self, options)
        self.logger = logging.getLogger('timestamp')

    def getMarkerGenesPerSeq(self, markerGeneStats):
        """Per scaffold (the gene id up to its last '_'), one [geneId, markerId, start, end] per marker of each gene, the
        start and end of the marker's last hit; and the number of hits of each marker (the last gene's)."""
        markerGenePos, markerGeneNum = {}, {}
        start = end = None
        for geneId, markers in markerGeneStats.items():
            scaffoldId = geneId[0:geneId.rfind('_')]
            for markerId, hitList in markers.items():
                if hitList:
                    start, end = hitList[-1][0], hitList[-1][1]
                markerGenePos.setdefault(scaffoldId, []).append([geneId, markerId, start, end])
                markerGeneNum[markerId] = len(hitList)
        return markerGenePos, markerGeneNum

    def roundUpToNearest100(self, x):
        return int(math.ceil(x / 100.0)) * 100

    def plot(self, binFile, markerGeneStats, binStats):
        binId = binIdFromFilename(binFile)
        markerGenesPerSeq, _ = self.getMarkerGenesPerSeq(markerGeneStats)
        if len(markerGenesPerSeq) == 0:
            return False

        prof = length_profiles([binFile])[0]
        lens = prof.lens.tolist()
        onMarkers = [i for i, seqId in enumerate(prof.ids) if seqId in markerGenesPerSeq]
        seqLens = {prof.ids[i]: lens[i] for i in onMarkers}
        longestSeq = max([0] + list(seqLens.values()))
        binSize = prof.total
        sortedSeqLens = [(prof.ids[i], lens[i]) for i in sorted(onMarkers, key=lambda i: prof.rank[i])]

        markerBases = sum(seqLens.values())
        if binSize == 0:
            self._fatal('Marker gene position plot of bin %s: its sequences have no bases.' % binId)
        result_str = 'Markers reside on {:,} of {:,} sequences which span {:.2f} of {:.2f} ({:.1f}%) Mb'.format(
            len(seqLens), len(prof.ids), markerBases / 1e6, binSize / 1e6, markerBases * 100.0 / binSize)
        self.logger.info(result_str)

        plotBinSize = self.roundUpToNearest100(float(longestSeq) / MAX_BINS)
        if plotBinSize == 0:
            self._fatal('Marker gene position plot of bin %s: the sequences with marker genes have no bases.' % binId)
        yLabels = [seqId for seqId, _ in sortedSeqLens]

        geneFile = os.path.join(self.options.results_dir, 'bins', binId, DefaultValues.PRODIGAL_AA)
        if not os.path.exists(geneFile):
            self._fatal('Input file does not exists: ' + geneFile)
        try:
            genePos = gene_positions(geneFile)
        except (IndexError, ValueError):
            self._fatal('Marker gene position plot of bin %s: a header of %s has no start and end positions.' % (binId, geneFile))

        # every row's marker counts first: where the reference fails part-way through, nothing below is drawn
        rows = []
        for seqId, seqLen in sortedSeqLens:
            markerCount = [0] * int(math.ceil(float(seqLen) / plotBinSize))
            for geneId, _markerId, geneStartPos, _geneEndPos in markerGenesPerSeq[seqId]:
                if geneId not in genePos:
                    self._fatal('Marker gene position plot of bin %s: gene %s is not in %s.' % (binId, geneId, geneFile))
                binPos = int(float(genePos[geneId][0] + geneStartPos) / plotBinSize)
                if not -len(markerCount) <= binPos < len(markerCount):
                    self._fatal('Marker gene position plot of bin %s: gene %s lies at position bin %d of sequence %s, '
                                'which has %d.' % (binId, geneId, binPos, seqId, len(markerCount)))
                markerCount[binPos] += 1
            rows.append(markerCount)

        self.fig.clear()
        self.fig.set_size_inches(self.options.width, self.options.height)
        yLabelBounds = self.yLabelExtents(yLabels, self.options.font_size)

        pad, width = self.options.fig_padding, self.options.width
        heightBottomLabels = 0.4 + pad
        widthSideLabel = yLabelBounds.width * width + pad
        widthPerBin = (width - widthSideLabel - pad) / MAX_BINS
        titleHeight = 0.2
        HEIGHT_PER_ROW = 0.2
        height = HEIGHT_PER_ROW * len(sortedSeqLens) + heightBottomLabels + pad + titleHeight
        rowBinHeight = widthPerBin / HEIGHT_PER_ROW

        self.fig.set_size_inches(width, height)
        axes = self.fig.add_axes([widthSideLabel / width, heightBottomLabels / height,
                                  1.0 - (widthSideLabel + pad) / width,
                                  1.0 - (heightBottomLabels + pad + titleHeight) / height])
        axes.set_xlim([0, MAX_BINS + 0.1])
        axes.set_xlabel('Position ({:,} bp/bin)'.format(plotBinSize))
        axes.set_ylim([0, len(sortedSeqLens)])
        axes.set_yticks(np.arange(0.5, len(sortedSeqLens) + 0.5, 1.0))
        axes.set_yticklabels(yLabels)

        discreteColourMap = mpl.colors.ListedColormap(COLOURS)
        axisColourMap = self.fig.add_axes([pad / width, pad / height, 0.15, 0.03 * (width / height)])
        colourBar = mpl.colorbar.ColorbarBase(axisColourMap, cmap=discreteColourMap, norm=mpl.colors.Normalize(vmin=0, vmax=1),
                                              orientation='horizontal', drawedges=True)
        colourBar.set_ticks([0.1, 0.3, 0.5, 0.7, 0.9])
        colourBar.set_ticklabels(['0', '1', '2', '3', '4+'])
        colourBar.outline.set_linewidth(0.5)
        colourBar.dividers.set_linewidth(0.5)
        for a in axisColourMap.xaxis.majorTicks:
            a.tick1On = False
            a.tick2On = False

        binPosX = 0.5
        for markerCount in rows:
            for i, n in enumerate(markerCount):
                axes.add_patch(Rectangle((i + 0.1, binPosX - 0.4 * rowBinHeight), 0.8, 0.8 * rowBinHeight,
                                         facecolor=COLOURS[n] if n < len(COLOURS) else COLOURS[-1], lw=0.2))
            binPosX += 1.0

        titleStr = binId + '\n'
        titleStr += '({:.1f}% complete, {:.1f}% contamination)'.format(binStats['Completeness'], binStats['Contamination'])
        titleStr += '\n({})'.format(result_str)
        axes.set_title(titleStr)

        for a in axes.yaxis.majorTicks:
            a.tick1On = False
            a.tick2On = False
        for a in axes.xaxis.majorTicks:
            a.tick1On = True
            a.tick2On = False
        for line in axes.yaxis.get_ticklines():
            line.set_color(self.axesColour)
        for line in axes.xaxis.get_ticklines():
            line.set_color(self.axesColour)
            line.set_ms(2)
        for loc, spine in axes.spines.items():
            spine.set_color('none' if loc in ('left', 'right', 'top') else self.axesColour)

        self.draw()
        return True
