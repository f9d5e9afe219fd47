"""`checkm nx_plot` (checkm/plot/nxPlot.py): the Nx curve of a bin.  The sort, the prefix sums and the Nx loop run on the
device (`length_profiles`, ckm_length_profile); where the reference's loop or its plot call raises, the bin and the
sequence are named in an error and the command exits with status 1."""
import numpy as np

from .AbstractPlot import AbstractPlot, NX_INDEX, NX_OK, length_profiles, nx_fractions
from .. import runtime


class NxPlot(AbstractPlot):
    def __init__(self, options):
        AbstractPlot.__init__(self, options)

    def calculateNx(self, x, seqs):
        """The reference's Nx list of the sequences `seqs` (a dict) at the fractions x, which is sorted in place; raises
        IndexError where the reference's loop does."""
        x.sort()
        if len(x) == 0:
            raise IndexError('index 0 is out of bounds for axis 0 with size 0')
        lens = np.array([len(s) for s in seqs.values()], dtype=np.int64)
        _, nx, status, fail, _, _, _ = runtime.engine().length_profile(lens, np.array([0, len(lens)], dtype=np.int64), x)
        if status[0] == NX_INDEX:
            raise IndexError('index %d is out of bounds for axis 0 with size %d' % (len(x), len(x)))
        return nx[0][:len(x) if status[0] == NX_OK else int(fail[0])].tolist()

    def plot(self, fastaFile):
        self.fig.clear()
        self.fig.set_size_inches(self.options.width, self.options.height)
        axes = self.fig.add_subplot(111)

        x = nx_fractions(self.options.step_size)
        if len(x) == 0:
            self._fatal('Nx-plot of %s: the step size %r gives no Nx fractions.' % (fastaFile, self.options.step_size))
        prof = length_profiles([fastaFile], x=x)[0]
        if prof.status == NX_INDEX:
            self._fatal('Nx-plot of bin %s: the reference\'s Nx loop reaches its last threshold before sequence %s and '
                        'fails there (IndexError).' % (prof.binId, prof.sequenceAtRank(prof.fail)))
        if prof.status != NX_OK:
            self._fatal('Nx-plot of bin %s: %s, so the plot has %d Nx values for %d fractions.'
                        % (prof.binId, 'the bin has no sequences' if not len(prof.ids) else
                           'the bin\'s total length never reaches its threshold at Nx = %r' % float(x[prof.fail]),
                           prof.fail, len(x)))
        axes.plot(x, prof.nxList(), 'ko-', ms=4)
        axes.set_xlabel('Nx')
        axes.set_ylabel('Sequence length (kbp)')

        yticks = axes.get_yticks()
        axes.set_yticklabels([('%.1f' % (float(v) / 1000)).replace('.0', '') for v in yticks])
        self._prettify(axes)
        self.fig.tight_layout(pad=1)
        self.draw()
