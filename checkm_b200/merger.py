"""Bin mergers (`checkm merge`) behind the reference's Merger interface (checkm/merger.py:30-110).

The reference scores every pair of bins with three ResultsManager.geneCounts calls, one of them on a merged copy of the
two hit dicts.  Here each bin's hits become one row of copy numbers over the shared marker union, once per bin, and every
pair is scored in one device call (`ckm_merge_pairs`, csrc/merge.cu, which states the arithmetic); the rows of
merger.tsv are written from the passing pairs by the library's host formatter (`ckm_format_merger_rows`, the reference's
'%.2f' values).  The hits come from this package's ResultsParser, so the reduction runs on the device too."""
import ctypes as C
import logging
import os
import sys
import time

import numpy as np

from . import _lib, runtime
from .common import checkDirExists
from .resultsParser import ResultsParser

HEADER = ('Bin Id 1\tBin Id 2'
          '\tBin 1 completeness\tBin 1 contamination'
          '\tBin 2 completeness\tBin 2 contamination'
          '\tDelta completeness\tDelta contamination\tMerger delta'
          '\tMerged completeness\tMerged contamination\n')


def copy_number_matrix(binIds, binMarkerHits, markers):
    """nbins x len(markers) int32: the number of hits of each bin to each marker (0 when the marker has no entry)."""
    col = {m: c for c, m in enumerate(markers)}
    counts = np.zeros((len(binIds), len(markers)), dtype=np.int32)
    for b, binId in enumerate(binIds):
        for marker, hits in binMarkerHits[binId].items():
            c = col.get(marker)
            if c is not None:
                counts[b, c] = len(hits)
    return counts


def format_rows(binIds, p, s, n_markers, pairs):
    """The merger.tsv rows (without the header) of the pairs `Engine.merge_pairs` returned, as bytes."""
    enc = [b.encode() for b in binIds]
    offsets = np.zeros(len(enc) + 1, dtype=np.int64)
    offsets[1:] = np.cumsum([len(b) for b in enc])
    blob = b''.join(enc)
    p = np.ascontiguousarray(p, dtype=np.int32)
    s = np.ascontiguousarray(s, dtype=np.int32)
    n_markers = np.ascontiguousarray(n_markers, dtype=np.int32)
    pairs = np.ascontiguousarray(pairs)
    cap = len(pairs) * 160 + 2 * int(offsets[-1]) + 1
    while True:
        out = C.create_string_buffer(cap)
        used = C.c_int64()
        rc = _lib.lib().ckm_format_merger_rows(blob, offsets.ctypes.data, len(enc), p.ctypes.data, s.ctypes.data,
                                               n_markers.ctypes.data, pairs.ctypes.data if len(pairs) else None, len(pairs),
                                               out, cap, C.byref(used))
        if rc == 8 and used.value > cap:               # CKM_ECAPACITY: the size needed came back
            cap = used.value
            continue
        _lib.check(rc)
        return out.raw[:used.value]


class Merger():
    def __init__(self):
        self.logger = logging.getLogger('timestamp')
        self.timing = {}                  # seconds per phase of the last run

    def run(self, binFiles, outDir, hmmTableFile,
            binIdToModels, binIdToBinMarkerSets,
            minDeltaComp, maxDeltaCont,
            minMergedComp, maxMergedCont):
        checkDirExists(outDir)

        self.logger.info('Comparing marker sets between all pairs of bins.')

        # ensure all bins are using the same marker set
        markerGenesI = binIdToBinMarkerSets[list(binIdToBinMarkerSets.keys())[0]].mostSpecificMarkerSet().getMarkerGenes()
        for binIdJ in binIdToBinMarkerSets:
            if markerGenesI != binIdToBinMarkerSets[binIdJ].mostSpecificMarkerSet().getMarkerGenes():
                self.logger.error('All bins must use the same marker set to assess potential mergers.')
                sys.exit(1)

        t0 = time.perf_counter()
        resultsParser = ResultsParser(binIdToModels)
        resultsParser.parseBinHits(outDir, hmmTableFile)
        t1 = time.perf_counter()

        binMarkerHits = {binId: rm.markerHits for binId, rm in resultsParser.results.items()}
        binIds = sorted(binMarkerHits.keys())
        counts = copy_number_matrix(binIds, binMarkerHits, sorted(markerGenesI))
        n_markers = np.array([binIdToBinMarkerSets[b].mostSpecificMarkerSet().numMarkers() for b in binIds], dtype=np.int32)
        t2 = time.perf_counter()

        pairs, kernel_ms = runtime.engine().merge_pairs(counts, n_markers, minDeltaComp, maxDeltaCont, minMergedComp,
                                                        maxMergedCont)
        t3 = time.perf_counter()

        rows = format_rows(binIds, (counts > 0).sum(axis=1), counts.sum(axis=1, dtype=np.int64), n_markers, pairs)
        outputFile = os.path.join(outDir, "merger.tsv")
        with open(outputFile, 'wb') as fout:
            fout.write(HEADER.encode())
            fout.write(rows)
        t4 = time.perf_counter()
        self.timing = {'parse_reduce': t1 - t0, 'counts': t2 - t1, 'device_call': t3 - t2, 'kernel_ms': kernel_ms,
                       'format_write': t4 - t3, 'pairs': len(pairs)}

        return outputFile
