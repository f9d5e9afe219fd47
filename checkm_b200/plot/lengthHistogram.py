"""`checkm len_hist` (checkm/plot/lengthHistogram.py): the bin's sequences counted in ten length classes.  The classes
are counted on the device (`length_profiles`, ckm_length_profile) with np.histogram's edge rule."""
import numpy as np
from matplotlib.ticker import MaxNLocator

from .AbstractPlot import AbstractPlot, length_profiles

CLASS_LABELS = ['<1', '1-2', '2-5', '5-10', '10-20', '20-50', '50-100', '100-200', '200-500', '>500']


class LengthHistogram(AbstractPlot):
    def __init__(self, options):
        AbstractPlot.__init__(self, options)

    def plot(self, fastaFile):
        self.fig.clear()
        self.fig.set_size_inches(self.options.width, self.options.height)
        axes = self.fig.add_subplot(111)

        prof = length_profiles([fastaFile])[0]
        counts = prof.classes
        axes.bar(x=np.arange(0.1, len(counts)), height=counts, width=0.8, color=(0.5, 0.5, 0.5))
        axes.set_xlabel('Sequence length (kbp)')
        axes.set_ylabel('Number sequences (out of %d)' % len(prof.ids))

        _, end = axes.get_ylim()
        axes.set_ylim([0, end])
        axes.get_yaxis().set_major_locator(MaxNLocator(integer=True))

        axes.set_xlim([0, len(counts)])
        axes.set_xticks(np.arange(0.5, len(counts)))
        axes.set_xticklabels(CLASS_LABELS)
        self._prettify(axes)
        self.fig.tight_layout(pad=1)
        self.draw()
