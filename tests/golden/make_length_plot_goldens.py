"""Generates the length-plot goldens by running the REFERENCE's own NxPlot, LengthHistogram and MarkerGenePosPlot
(checkm/plot/nxPlot.py, lengthHistogram.py, markerGenePosPlot.py, imported read-only from the reference checkout,
CHECKM_REFERENCE or /root/reference) over tools/axes_recorder.py, the stand-in matplotlib.  Run in the build container
only:

    python tests/golden/make_length_plot_goldens.py

Bins: the nine outlier bins (tests/golden/outliers/bins), plots/bins/p1_edges.fna, and the edge bins written here to
length_plots/bins/: duplicate ids, a single record, equal lengths, lengths around the class edges (999, 1000, 1001, 1999,
2000, 2001 bp), an empty record (also trailing the longest ones), an empty file, two bins whose Nx loop raises IndexError
at steps 0.3 and 0.07 ([5, 4, 3, 2, 1] and [100, 1, 1, 1] bp), and a gzipped bin with records of exactly 999, 1000, 2000,
500000 and 500001 bp.  Per bin and Nx step in STEPS: the reference's calculateNx(x, seqs) (its list, or the exception's
name) and the call log of NxPlot.plot; per bin the call log of LengthHistogram.plot.

marker_plot: the three protein bins of tests/golden/aai/ with their oracle domtblouts as `bins/<id>/genes.faa` and
`hmmer.analyze.txt`; the reference's ResultsParser.analyseResults and cacheResults write `storage/marker_gene_stats.tsv` and
`bin_stats_ext.tsv` (kept in length_plots/markers/storage/); nucleotide bins length_plots/markers/<id>.fna hold one
scaffold per gene-id prefix (two of strainA's of equal length, one scaffold without genes).  Recorded: each bin's
MarkerGenePosPlot.plot on the parsed files, and on hand-made marker dicts -- a marker with several hits, two markers on
one gene, no markers, a gene missing from genes.faa (KeyError) and a hit past its row (IndexError) -- with the INFO lines
and the return value.

A log whose compact JSON is larger than FULL_LOG_MAX bytes is kept as its SHA-256 (make_plot_goldens.log_digest)."""
import gzip
import json
import logging
import os
import shutil
import sys
import tempfile
import types

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
OUT = os.path.join(HERE, 'length_plots')
AAI = os.path.join(HERE, 'aai')
CPR = os.path.join(HERE, 'cpr_43_markers.hmm')
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)
sys.path.insert(0, os.environ.get('CHECKM_REFERENCE', '/root/reference'))

import numpy as np  # noqa: E402

STEPS = [0.01, 0.05, 0.07, 0.1, 0.25, 0.3, 0.5, 1.0]
FULL_LOG_MAX = 60000
MARKER_BINS = ['strainA', 'strainB', 'strainC']


def options(results_dir='', step=0.05):
    return types.SimpleNamespace(font_size=8, dpi=600, width=6.5, height=6.5, fig_padding=0.2, step_size=step,
                                 results_dir=results_dir, image_type='png')


def seq_of(rng, n):
    return ''.join(np.array(list('ACGT'))[rng.integers(0, 4, size=n)])


def edge_bins(rng):
    """{file name: records} of the new edge bins."""
    return {
        'l1_dups.fna': [('d1', seq_of(rng, 3000)), ('d2', seq_of(rng, 700)), ('d1', seq_of(rng, 1200)),
                        ('d3', seq_of(rng, 2500)), ('d2', seq_of(rng, 5200))],
        'l2_single.fna': [('only', seq_of(rng, 4321))],
        'l3_equal.fna': [('e%d' % i, seq_of(rng, 1000)) for i in range(6)] + [('f1', seq_of(rng, 2000)), ('f2', seq_of(rng, 2000))],
        'l4_edges.fna': [('s%d' % n, seq_of(rng, n)) for n in (999, 1000, 1001, 1999, 2000, 2001, 1, 50)],
        'l5_empty_record.fna': [('a', seq_of(rng, 800)), ('nothing', ''), ('b', seq_of(rng, 1500)), ('c', seq_of(rng, 1500))],
        'l6_trailing_empty.fna': [('a', seq_of(rng, 800)), ('z1', ''), ('z2', '')],
        'l7_empty.fna': [],
        'l8_raise_step03.fna': [('r%d' % n, seq_of(rng, n)) for n in (5, 4, 3, 2, 1)],
        'l9_raise_step007.fna': [('q%d' % i, seq_of(rng, n)) for i, n in enumerate((100, 1, 1, 1))],
        'l10_big.fna.gz': [('g%d' % n, ('ACGTTGCA' * (n // 8 + 1))[:n]) for n in (999, 1000, 2000, 500000, 500001, 20000)],
    }


def bin_files():
    og = os.path.join(HERE, 'outliers', 'bins')
    out = [os.path.join(og, f) for f in sorted(os.listdir(og))]
    out.append(os.path.join(HERE, 'plots', 'bins', 'p1_edges.fna'))
    lb = os.path.join(OUT, 'bins')
    return out + [os.path.join(lb, f) for f in sorted(os.listdir(lb))]


def scaffold_bin(rng, binId):
    """One scaffold per gene-id prefix of the bin's genes.faa, long enough for its genes (two of strainA's of equal
    length), and one scaffold without genes."""
    ends = {}
    for line in open(os.path.join(AAI, 'bins', binId + '.faa')):
        if line.startswith('>'):
            f = line[1:].split()
            scaffold = f[0][:f[0].rfind('_')]
            ends[scaffold] = max(ends.get(scaffold, 0), int(f[4]))
    lens = {s: e + int(rng.integers(50, 4000)) for s, e in ends.items()}
    names = list(lens)
    if binId == 'strainA' and len(names) >= 3:
        lens[names[2]] = lens[names[1]] = max(lens[names[1]], lens[names[2]])
    records = [(s, seq_of(rng, n)) for s, n in lens.items()]
    records.insert(1, ('%s_nogenes' % binId, seq_of(rng, 1234)))
    return records


def main():
    from make_outlier_goldens import write_bin
    from make_plot_goldens import log_digest
    from tools import axes_recorder as rec
    os.environ['CHECKM_DATA_PATH'] = os.path.join(HERE, 'reduction', 'data')     # make_plot_goldens points it elsewhere
    rng = np.random.default_rng(20261019)
    shutil.rmtree(OUT, ignore_errors=True)
    os.makedirs(os.path.join(OUT, 'bins'))
    for name, records in edge_bins(rng).items():
        write_bin(os.path.join(OUT, 'bins', name), records)
    os.makedirs(os.path.join(OUT, 'markers', 'storage'))
    for binId in MARKER_BINS:
        write_bin(os.path.join(OUT, 'markers', binId + '.fna'), scaffold_bin(rng, binId))

    # storage/ from the reference's own ResultsParser over the oracle's hit tables
    from checkm.hmmerModelParser import HmmModelParser
    from checkm.markerSets import MarkerSetParser
    from checkm.resultsParser import ResultsParser
    work = tempfile.mkdtemp(prefix='lenplot_gold_')
    out = os.path.join(work, 'out')
    os.makedirs(os.path.join(out, 'storage'))
    for binId in MARKER_BINS:
        bdir = os.path.join(out, 'bins', binId)
        os.makedirs(bdir)
        shutil.copyfile(os.path.join(AAI, 'bins', binId + '.faa'), os.path.join(bdir, 'genes.faa'))
        shutil.copyfile(os.path.join(AAI, 'bins', binId + '.hmmer.analyze.txt'), os.path.join(bdir, 'hmmer.analyze.txt'))
    with open(os.path.join(AAI, 'expected.json')) as f:
        stats_lines = json.load(f)['bin_stats']
    with open(os.path.join(out, 'storage', 'bin_stats.analyze.tsv'), 'w') as f:
        f.write(''.join(l + '\n' for l in stats_lines))
    models = HmmModelParser(CPR).models()
    RP = ResultsParser({b: models for b in MARKER_BINS})
    RP.analyseResults(out, 'bin_stats.analyze.tsv', 'hmmer.analyze.txt')
    RP.cacheResults(out, MarkerSetParser().getMarkerSets(out, MARKER_BINS, CPR), False)
    for name in ('marker_gene_stats.tsv', 'bin_stats_ext.tsv'):
        shutil.copyfile(os.path.join(out, 'storage', name), os.path.join(OUT, 'markers', 'storage', name))
    RP = ResultsParser(None)
    markerGeneStats = RP.parseMarkerGeneStats(out)
    binStats = RP.parseBinStatsExt(out)

    infos = []

    class Capture(logging.Handler):
        def emit(self, record):
            infos.append(record.getMessage())
    logger = logging.getLogger('timestamp')
    logger.addHandler(Capture())
    logger.setLevel(logging.INFO)

    rec.install()
    from checkm.plot.lengthHistogram import LengthHistogram
    from checkm.plot.markerGenePosPlot import MarkerGenePosPlot
    from checkm.plot.nxPlot import NxPlot
    from checkm.util.seqUtils import readFasta

    runs, values = {}, {}

    def run(key, fn):
        rec.reset()
        del infos[:]
        try:
            ret = fn()
            text = json.dumps(rec.LOG, sort_keys=True, separators=(',', ':'))
            runs[key] = {'log': list(rec.LOG)} if len(text) <= FULL_LOG_MAX else {'sha256': log_digest(rec.LOG)}
            runs[key]['returns'] = ret
        except (IndexError, KeyError, ValueError, ZeroDivisionError, SystemExit) as e:
            runs[key] = {'raises': type(e).__name__}
        runs[key]['info'] = list(infos)
        print(key, runs[key].get('raises', '%d calls' % len(rec.LOG)))

    for binFile in bin_files():
        binId = os.path.basename(binFile).split('.')[0]
        seqs = readFasta(binFile)
        values[binId] = {}
        for step in STEPS:
            x = np.arange(0, 1.0 + 0.5 * step, step)
            try:
                values[binId][str(step)] = {'nx': NxPlot(options(step=step)).calculateNx(x, seqs)}
            except IndexError as e:
                values[binId][str(step)] = {'raises': type(e).__name__}
            run('nx|%s|%r' % (binId, step), lambda: NxPlot(options(step=step)).plot(binFile))
        run('len|%s' % binId, lambda: LengthHistogram(options()).plot(binFile))

    mdir = os.path.join(OUT, 'markers')
    cases = {}
    for binId in MARKER_BINS:
        cases['files|' + binId] = markerGeneStats[binId]
    a = dict(markerGeneStats['strainA'])
    genes = list(a)
    first = genes[0]
    marker = list(a[first])[0]
    multi = dict(a)
    multi[first] = {marker: [[3, 40], [55, 90], [120, 160]]}                       # several hits: the last one counts
    multi[genes[1]] = dict(list(a[genes[1]].items()) + [('PF99999.1', [[10, 20]])])  # two markers on one gene
    cases['multihit|strainA'] = multi
    cases['nomarkers|strainA'] = {}
    cases['missinggene|strainA'] = dict(list(a.items()) + [(genes[0].rsplit('_', 1)[0] + '_999', {marker: [[1, 5]]})])
    cases['pastend|strainA'] = dict(list(a.items()) + [(first, {marker: [[10 ** 6, 10 ** 6 + 50]]})])
    for key, mgs in cases.items():
        binId = key.split('|')[1]
        run('marker|' + key, lambda: MarkerGenePosPlot(options(out)).plot(os.path.join(mdir, binId + '.fna'), mgs, binStats[binId]))
    rec.uninstall()

    with gzip.open(os.path.join(OUT, 'expected.json.gz'), 'wt') as f:
        json.dump({'runs': runs, 'values': values, 'steps': STEPS, 'marker_cases': {k: [[g, list(m.items())] for g, m in c.items()] for k, c in cases.items()},
                   'bin_stats': {b: binStats[b] for b in MARKER_BINS}}, f, sort_keys=True)
    shutil.rmtree(work)


if __name__ == '__main__':
    main()
