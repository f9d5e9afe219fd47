"""Plain-Python restatement of the three length plots' computations (checkm/plot/nxPlot.py, lengthHistogram.py,
markerGenePosPlot.py), for the tests: the Nx loop with its exceptions, the length classes by np.histogram's edge rule, and
the marker rows of marker_plot.  Lengths are Python ints, thresholds Python floats, so every comparison is exact."""
import math

EDGES = [0, 1, 2, 5, 10, 20, 50, 100, 200, 500, 1e12]


def nx(x, lens):
    """(nx list, exception name or None) of calculateNx at the ascending fractions x: threshold j is x[j] * total; the loop
    appends the current length while the running sum reaches the threshold, stops appending thresholds after the last but
    goes on with the sequences, so a sequence after the one reaching the last threshold raises IndexError."""
    lens = sorted(lens, reverse=True)
    total = sum(lens)
    thresholds = [float(v) * total for v in x]
    out, j, run = [], 0, 0
    for L in lens:
        run += L
        while run >= thresholds[j]:
            out.append(L)
            if len(out) == len(thresholds):
                break
            j += 1
            if j >= len(thresholds):
                return out, 'IndexError'
    return out, None


def plot_nx(x, lens):
    """What NxPlot.plot makes of it: the list, or the exception (a list shorter than x fails in axes.plot)."""
    if len(x) == 0:
        return None, 'IndexError'
    out, exc = nx(x, lens)
    if exc is None and len(out) != len(x):
        exc = 'ValueError'
    return out, exc


def length_classes(lens):
    """np.histogram(float(len) / 1e3, EDGES): class c holds EDGES[c] <= v < EDGES[c + 1], the last class also v == 1e12."""
    counts = [0] * (len(EDGES) - 1)
    for L in lens:
        v = float(L) / 1e3
        for c in range(len(counts)):
            last = c == len(counts) - 1
            if EDGES[c] <= v and (v < EDGES[c + 1] or (last and v == EDGES[c + 1])):
                counts[c] += 1
                break
    return counts


def marker_rows(markerGeneStats, seqLens, genePos):
    """marker_plot's rows: (the scaffolds with markers longest first, ties in dict order, with their lengths), the
    position bin size and the marker count of every cell of every row; or the exception the reference raises.
    seqLens: {scaffold: length} in the bin's dict order; genePos: {gene: [start, end]} from genes.faa."""
    perSeq, start = {}, None
    for geneId, markers in markerGeneStats.items():
        scaffold = geneId[:geneId.rfind('_')]
        for markerId, hits in markers.items():
            for hit in hits:
                start = hit[0]
            perSeq.setdefault(scaffold, []).append((geneId, start))
    if not perSeq:
        return None, None, None, None
    onMarkers = [(s, n) for s, n in seqLens.items() if s in perSeq]
    longest = max([0] + [n for _, n in onMarkers])
    order = sorted(onMarkers, key=lambda sn: -sn[1])
    binSize = int(math.ceil(float(longest) / 100 / 100.0)) * 100
    if binSize == 0:
        return order, binSize, None, 'ZeroDivisionError'
    rows = []
    for s, n in order:
        row = [0] * int(math.ceil(float(n) / binSize))
        for geneId, hitStart in perSeq[s]:
            if geneId not in genePos:
                return order, binSize, None, 'KeyError'
            k = int(float(genePos[geneId][0] + hitStart) / binSize)
            if not -len(row) <= k < len(row):
                return order, binSize, None, 'IndexError'
            row[k] += 1
        rows.append(row)
    return order, binSize, rows, None
