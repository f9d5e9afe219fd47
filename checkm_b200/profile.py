"""Community profile (`checkm profile`) behind the reference's Profile interface (checkm/profile.py:30-149): per bin, the
reads mapped to it in each BAM file of a `checkm coverage` file, as a share of all mapped reads, of the binned
populations (normalised by bin size) and of the community.  Host only: the work is one pass over the coverage file.

Where the reference stops with an uncaught exception, an error naming the file is logged and the run exits with status
1: a coverage file without rows (IndexError), and a BAM file without mapped reads or a bin of total length 0
(ZeroDivisionError)."""
import logging
import sys

from .common import checkFileExists, reassignStdOut, restoreStdOut
from .coverage import UNBINNED
from .resultsParser import _FrameTable


class Profile():
    def __init__(self):
        self.logger = logging.getLogger('timestamp')

    def _fail(self, message):
        self.logger.error(message)
        sys.exit(1)

    def _read(self, coverageFile):
        """{bin: {bam: mapped reads}} and {bin: summed sequence length}, both in order of first appearance, and
        {bam: mapped reads over all bins}."""
        reads, size, total = {}, {}, {}
        with open(coverageFile) as f:
            next(f, None)                                   # the header line
            for line in f:
                fields = line.split('\t')
                binId = fields[1]
                size[binId] = size.get(binId, 0) + int(fields[2])
                perBam = reads.setdefault(binId, {})
                for bamId, mapped in zip(fields[3::3], fields[5::3]):
                    mapped = int(mapped)
                    perBam[bamId] = perBam.get(bamId, 0) + mapped
                    total[bamId] = total.get(bamId, 0) + mapped
        return reads, size, total

    def run(self, coverageFile, outFile, bTabTable):
        checkFileExists(coverageFile)

        self.logger.info('Determining number of reads mapped to each bin.')
        reads, size, total = self._read(coverageFile)
        if not reads:
            self._fail('No sequences in coverage file %s.' % coverageFile)
        for bamId, n in total.items():
            if n == 0:
                self._fail('No reads of BAM file %s are mapped in coverage file %s.' % (bamId, coverageFile))

        # share of each BAM's mapped reads per bin; for the binned populations, the same per base of the bin, then as a
        # share of its sum over the bins (summed in order of first appearance, as the reference does)
        share, norm, normSum = {}, {}, {}
        for binId, perBam in reads.items():
            share[binId] = {bamId: float(n) / total[bamId] for bamId, n in perBam.items()}
            if binId == UNBINNED:
                continue
            if size[binId] == 0:
                self._fail('Bin %s has no bases in coverage file %s.' % (binId, coverageFile))
            norm[binId] = {bamId: s / size[binId] for bamId, s in share[binId].items()}
            for bamId, v in norm[binId].items():
                normSum[bamId] = normSum.get(bamId, 0) + v
        for perBam in norm.values():
            for bamId in perBam:
                perBam[bamId] = perBam[bamId] / normSum[bamId] if normSum[bamId] != 0 else 0

        oldStdOut = reassignStdOut(outFile)

        binIds = sorted(reads)
        bamIds = sorted(reads[binIds[0]])
        header = ['Bin Id', 'Bin size (Mbp)']
        for bamId in bamIds:
            header += [bamId + ': mapped reads', bamId + ': % mapped reads', bamId + ': % binned populations',
                       bamId + ': % community']
        table = None
        if bTabTable:
            print('\t'.join(header))
        else:
            table = _FrameTable(header)

        for binId in binIds:
            row = [binId, float(size[binId]) / 1e6]
            for bamId in bamIds:
                unbinned = share[UNBINNED][bamId] if UNBINNED in share else 0
                row += [reads[binId][bamId], share[binId][bamId] * 100.0]
                if binId == UNBINNED:
                    row += ['NA', unbinned * 100.0]
                else:
                    row += [norm[binId][bamId] * 100.0, norm[binId][bamId] * 100.0 * (1.0 - unbinned)]
            if table is None:
                print('\t'.join(map(str, row)))
            else:
                table.add_row(row)
        if table is not None:
            print(table.get_string())

        restoreStdOut(outFile, oldStdOut)
