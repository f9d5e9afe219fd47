"""CPU restatement of CheckM's bin-merger search (checkm/merger.py:34-110 with ResultsManager.geneCounts and
MarkerSet.genomeCheck in individual mode, markerSets.py:206-217) -- TEST INFRASTRUCTURE ONLY.

Only tests/ and bench legs that time a CPU baseline may import this; the product (checkm_b200/merger.py) scores the pairs
on the device.  Pinned: tests/test_merge_cpu.py holds it to the merger.tsv files the reference's own Merger wrote
(tests/golden/merge/, made by tests/golden/make_merge_goldens.py).

One merged dict and two completeness/contamination evaluations per pair, as in the reference."""


def genome_check(markers, n_markers, hits):
    """(completeness, contamination) of a {marker: copy number} dict over the marker union, individual mode."""
    present = 0
    multi = 0
    for m in markers:
        if m in hits:
            present += 1
            multi += hits[m] - 1
    return 100 * float(present) / n_markers, 100 * float(multi) / n_markers


def merge_pairs(binIds, copy_numbers, n_markers, markers, minDeltaComp, maxDeltaCont, minMergedComp, maxMergedCont):
    """copy_numbers[binId]: {marker: number of hits >= 1}; n_markers[binId]: numMarkers() of its marker set; markers: the
    shared marker union.  Returns the merger.tsv data lines, in the reference's order, and the (i, j) index pairs."""
    ids = sorted(binIds)
    lines, pairs = [], []
    for i in range(len(ids)):
        bi = ids[i]
        compI, contI = genome_check(markers, n_markers[bi], copy_numbers[bi])
        for j in range(i + 1, len(ids)):
            bj = ids[j]
            compJ, contJ = genome_check(markers, n_markers[bj], copy_numbers[bj])
            merged = dict(copy_numbers[bi])
            for m, c in copy_numbers[bj].items():
                merged[m] = merged.get(m, 0) + c
            compM, contM = genome_check(markers, n_markers[bj], merged)
            if not (compM >= minMergedComp and contM < maxMergedCont):
                continue
            deltaComp = compM - max(compI, compJ)
            deltaCont = contM - max(contI, contJ)
            if deltaComp >= minDeltaComp and deltaCont < maxDeltaCont:
                lines.append('%s\t%s\t%.2f\t%.2f\t%.2f\t%.2f\t%.2f\t%.2f\t%.2f\t%.2f\t%.2f\n' %
                             (bi, bj, compI, contI, compJ, contJ, deltaComp, deltaCont, deltaComp - deltaCont, compM, contM))
                pairs.append((i, j))
    return lines, pairs
