"""Generates the plot goldens by running the REFERENCE's own GcPlots, CodingDensityPlots, TetraDistPlots,
DistributionPlots and GcBiasPlot (checkm/plot/*.py, imported read-only from the reference checkout, CHECKM_REFERENCE or
/root/reference) over tools/axes_recorder.py, the stand-in matplotlib.  Run in the build container only:

    python tests/golden/make_plot_goldens.py

Inputs: the nine bins of tests/golden/outliers/ with their GFFs and synthetic distribution files, and one more bin,
plots/bins/p1_edges.fna (sequences of length exactly 2 x 2048 and 2 x 2048 + 1, 300 and 301, shorter than most window
sizes, a run of 250 N, lower case, U and IUPAC codes) with plots/out/bins/p1_edges/genes.gff (overlapping genes, a gene
starting at 0, a gene past its sequence's end, a sequence without genes).  The tetranucleotide profile is
oracle.outliers_oracle.profile_text over outliers/extra.fna, the outlier bins and p1_edges; the coverage profile of
gc_bias_plot is oracle.plot_windows_oracle.synthetic_coverage, with the right number of windows per sequence.

It writes plots/expected.json.gz: per run (plot, bin, window sizes) the recorded call log of `plot(...)` -- for window
sizes below 100, which log one value per window, the SHA-256 of its compact JSON instead -- or the name of the exception
the reference raised; and per bin and window size the reference's own window values (baseCount,
ProdigalGeneFeatureParser.codingBases(seqId, start, end), and genomicSig.distance(seqSignature(window), binSig)) as
float.hex, for the oracle and the device to be held to."""
import gzip
import hashlib
import json
import os
import shutil
import sys
import types

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
OG = os.path.join(HERE, 'outliers')
OUT = os.path.join(HERE, 'plots')
sys.path.insert(0, ROOT)
sys.path.insert(0, os.environ.get('CHECKM_REFERENCE', '/root/reference'))
os.environ['CHECKM_DATA_PATH'] = os.path.join(OG, 'data')

import numpy as np   # noqa: E402

WINDOWS = [1, 7, 100, 2048, 5000, 10000]
DIST_SIZES = [(w, w, w) for w in WINDOWS] + [(5000, 5000, 10000), (7, 100, 7)]   # (gc, td, cd); the last two mixed
DISTRIBUTIONS = [95, 85]
FULL_LOG_FROM = 100                    # smaller window sizes log one value per window: their logs are kept as digests


def options(results_dir, gc=5000, td=5000, cd=10000, window=5000):
    return types.SimpleNamespace(font_size=8, dpi=600, width=6.5, height=8, gc_window_size=gc, td_window_size=td,
                                 cd_window_size=cd, window_size=window, gc_bin_width=0.01, cd_bin_width=0.01,
                                 td_bin_width=0.01, results_dir=results_dir)


def seq_of(rng, n, gc):
    p = np.array([(1 - gc) / 2, gc / 2, gc / 2, (1 - gc) / 2])
    return ''.join(np.array(list('ACGT'))[rng.choice(4, size=n, p=p)])


def edge_bin(rng):
    mixed = seq_of(rng, 1200, 0.5)
    mixed = mixed[:100].lower() + 'N' * 250 + mixed[100:500] + 'RYKMSWnnbdhv' + mixed[500:].replace('T', 'U', 60)
    return [('k2048', seq_of(rng, 4096, 0.45)), ('k2048p1', seq_of(rng, 4097, 0.6)), ('k300', seq_of(rng, 300, 0.5)),
            ('k301', seq_of(rng, 301, 0.5)), ('short', seq_of(rng, 50, 0.5)), ('mixed', mixed),
            ('nogenes', seq_of(rng, 900, 0.3))]


def write_edge_bin(records):
    sys.path.insert(0, HERE)
    from make_outlier_goldens import write_bin
    os.makedirs(os.path.join(OUT, 'bins'))
    write_bin(os.path.join(OUT, 'bins', 'p1_edges.fna'), records)
    gdir = os.path.join(OUT, 'out', 'bins', 'p1_edges')
    os.makedirs(gdir)
    genes = {'k2048': [(10, 900), (500, 1500), (1400, 1402), (3000, 4096)],      # overlaps
             'k2048p1': [(0, 700), (1000, 2000), (0, 4097)],                    # starts at 0
             'k300': [(5, 200), (250, 420)],                                     # past the end
             'k301': [(1, 301)],
             'short': [(3, 40)],
             'mixed': [(1, 300), (290, 800), (1000, 1700)]}
    with open(os.path.join(gdir, 'genes.gff'), 'w') as f:
        f.write('##gff-version  3\n')
        for name, spans in genes.items():
            f.write('# Model Data: version=Prodigal.v2.6.3;run_type=Single;transl_table=11;uses_sd=1\n')
            for k, (s, e) in enumerate(spans):
                f.write('%s\tProdigal_v2.6.3\tCDS\t%d\t%d\t50.0\t+\t0\tID=1_%d;partial=00;\n' % (name, s, e, k + 1))


def log_digest(log):
    """What a call log of a window size below FULL_LOG_FROM is kept as: the SHA-256 of its compact JSON."""
    return hashlib.sha256(json.dumps(log, sort_keys=True, separators=(',', ':')).encode()).hexdigest()


def main():
    from oracle import outliers_oracle as oo, plot_windows_oracle as pw
    from tools import axes_recorder as rec
    rng = np.random.default_rng(20240811)
    shutil.rmtree(OUT, ignore_errors=True)
    write_edge_bin(edge_bin(rng))
    bins = [(os.path.join(OG, 'bins', f), os.path.join(OG, 'out')) for f in sorted(os.listdir(os.path.join(OG, 'bins')))]
    bins.append((os.path.join(OUT, 'bins', 'p1_edges.fna'), os.path.join(OUT, 'out')))
    profile = os.path.join(OUT, 'tetra.tsv')
    with open(profile, 'w') as f:
        f.write(oo.profile_text([os.path.join(OG, 'extra.fna')] + [b for b, _ in bins]))

    rec.install()
    from checkm.binTools import BinTools
    from checkm.genomicSignatures import GenomicSignatures
    from checkm.plot.codingDensityPlots import CodingDensityPlots
    from checkm.plot.distributionPlots import DistributionPlots
    from checkm.plot.gcBiasPlots import GcBiasPlot
    from checkm.plot.gcPlots import GcPlots
    from checkm.plot.tetraDistPlots import TetraDistPlots
    from checkm.prodigal import ProdigalGeneFeatureParser
    from checkm.util.seqUtils import baseCount, readFasta
    gs = GenomicSignatures(K=4, threads=1)
    tetraSigs = gs.read(profile)
    os.remove(profile)

    def run(key, fn, W):
        rec.reset()
        try:
            fn()
            runs[key] = {'log': list(rec.LOG)} if W >= FULL_LOG_FROM else {'sha256': log_digest(rec.LOG)}
        except (ZeroDivisionError, SystemExit) as e:
            runs[key] = {'raises': type(e).__name__}
        print(key, runs[key].get('raises', '%d calls' % len(rec.LOG)))

    runs, values = {}, {}
    for binFile, resultsDir in bins:
        binId = oo.bin_id(binFile)
        seqs = readFasta(binFile)
        parser = ProdigalGeneFeatureParser(os.path.join(resultsDir, 'bins', binId, 'genes.gff'))
        binSig = BinTools().binTetraSig(seqs, tetraSigs)
        values[binId] = {}
        for W in WINDOWS:
            v = {'acgt': [], 'coding': [], 'td': []}
            for seqId, seq in seqs.items():
                for start in range(0, max(len(seq) - 1, 0) // W * W, W):
                    v['acgt'].append(list(baseCount(seq[start:start + W])))
                    v['coding'].append(float.hex(float(parser.codingBases(seqId, start, start + W))))
                    v['td'].append(float.hex(float(gs.distance(gs.seqSignature(seq[start:start + W]), binSig))))
            values[binId][str(W)] = v
            for dist in ([DISTRIBUTIONS] if W != 1 else [[95]]):
                o = options(resultsDir, gc=W, td=W, cd=W, window=W)
                d = '_'.join(str(x) for x in dist)
                run('gc|%s|%d|%s' % (binId, W, d), lambda: GcPlots(o).plot(binFile, dist), W)
                run('cd|%s|%d|%s' % (binId, W, d), lambda: CodingDensityPlots(o).plot(binFile, dist), W)
                run('td|%s|%d|%s' % (binId, W, d), lambda: TetraDistPlots(o).plot(binFile, tetraSigs, dist), W)
            cov = pw.synthetic_coverage({i: len(s) for i, s in seqs.items()}, W)
            run('bias|%s|%d' % (binId, W), lambda: GcBiasPlot(options(resultsDir, window=W)).plot(binFile, cov), W)
        for gc, td, cd in DIST_SIZES:
            o = options(resultsDir, gc=gc, td=td, cd=cd)
            run('dist|%s|%d_%d_%d' % (binId, gc, td, cd), lambda: DistributionPlots(o).plot(binFile, tetraSigs, DISTRIBUTIONS),
                min(gc, td, cd))
    rec.uninstall()
    with gzip.open(os.path.join(OUT, 'expected.json.gz'), 'wt') as f:
        json.dump({'runs': runs, 'values': values, 'windows': WINDOWS, 'dist_sizes': DIST_SIZES,
                   'distributions': DISTRIBUTIONS}, f, sort_keys=True)


if __name__ == '__main__':
    main()
