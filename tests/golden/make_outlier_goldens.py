"""Generates the `checkm outliers` goldens by running the REFERENCE's own BinTools (checkm/binTools.py, imported read-only
from the reference checkout, CHECKM_REFERENCE or /root/reference) on synthetic bins.  Run in the build container only:

    python tests/golden/make_outlier_goldens.py

CheckM's data bundle is not available, so the three distribution files (data/distributions/{gc,cd,td}_dist.txt) are
SYNTHETIC: their shape is taken from how binTools.py:250-276 indexes them (gc, cd: mean key -> length key -> percentile ->
bound; td: length key -> percentile -> bound), their numbers are made up.  They are deliberately not rectangular: one mean-GC
key has an extra length key, and the percentile keys of later length entries are in another order than the first entry's.

It writes under tests/golden/outliers/: bins/ (nine bins), out/bins/<bin>/genes.gff, extra.fna (an unbinned sequence and a
decoy under the id z1), the distribution files, and expected.json: the outlier file per (report type, distribution), what
gcDist / codingDensityDist / binTetraSig / tetraDiffDist return for four of the bins, the SHA-256 and the ids of what
removeOutliers and modify write, and what unique prints.  The profile file is not kept: it is
oracle.outliers_oracle.profile_text([extra.fna] + bins), which the tests write again -- every binned sequence, the unbinned
one, and z1 twice with different values, the last line counting.  Bins:

  b1_plain     six sequences: one of another GC and composition without a gene (outlying in all three), one without a gene
  b2_one       one sequence
  b3_repeat    an id that occurs twice (first place, last record)
  b4_mixed     lower case, N, IUPAC codes and U
  b5_gz        gzip
  b6_nan       a sequence of three bases: its signature is nan, and so are the bin's signature and every TD of the bin
  b7_tie       mean GC exactly 5/16, halfway between the keys 0.25 and 0.375; lengths 600 and 1200, halfway between length keys
  b8_edge      three sequences whose delta GC, delta CD and TD are exactly bounds of the tables (`<` and `>` are strict)
  b9_shared    shares one sequence with b1_plain (for `unique`)
"""
import contextlib
import gzip
import hashlib
import io
import json
import os
import re
import shutil
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
OUT = os.path.join(HERE, 'outliers')
sys.path.insert(0, ROOT)
sys.path.insert(0, os.environ.get('CHECKM_REFERENCE', '/root/reference'))
os.environ['CHECKM_DATA_PATH'] = os.path.join(OUT, 'data')

import numpy as np   # noqa: E402

LEN_KEYS = [200, 400, 800, 1600, 3200]
GC_KEYS = [0.125, 0.25, 0.375, 0.5, 0.625, 0.75]
CD_KEYS = [0.25, 0.5, 0.75, 0.9]
GC_PCT = [0.5, 2.5, 5.0, 10.0, 50, 90.0, 95.0, 97.5, 99.5]
TD_PCT = [50, 80.5, 90, 95, 99, 100]
DISTRIBUTIONS = [90, 95, 99, 85]          # 85 is not a key: 7.5 and 92.5 lie halfway between percentile keys
REPORTS = ['any', 'all']


def seq_of(rng, n, gc, skew=None):
    p = np.array([(1 - gc) / 2, gc / 2, gc / 2, (1 - gc) / 2])
    if skew is not None:
        p = p * skew
        p /= p.sum()
    return ''.join(np.array(list('ACGT'))[rng.choice(4, size=n, p=p)])


def exact(rng, n, gc_count):
    """n bases of A/C/G/T with exactly gc_count of G or C."""
    s = list('G' * (gc_count // 2) + 'C' * (gc_count - gc_count // 2) + 'A' * ((n - gc_count) // 2) +
             'T' * (n - gc_count - (n - gc_count) // 2))
    rng.shuffle(s)
    return ''.join(s)


def bins(rng):
    b = {}
    b['b1_plain.fna'] = [('p%d' % i, seq_of(rng, n, 0.5)) for i, n in enumerate((1100, 300, 650, 2900, 900))]
    b['b1_plain.fna'].insert(3, ('p_odd', seq_of(rng, 1000, 0.8, skew=[4, 1, 3, 0.5])))
    b['b2_one.fna'] = [('solo', seq_of(rng, 700, 0.4))]
    b['b3_repeat.fna'] = [('r0', seq_of(rng, 450, 0.45)), ('r1', seq_of(rng, 500, 0.45)), ('r2', seq_of(rng, 900, 0.45)),
                          ('r1', seq_of(rng, 350, 0.7))]
    mixed = seq_of(rng, 900, 0.55)
    mixed = mixed[:150].lower() + 'NNNNNNNNNNNN' + mixed[150:400] + 'RYKMSWnnbdhv' + mixed[400:].replace('T', 'U', 40)
    b['b4_mixed.fna'] = [('m0', mixed), ('m1', seq_of(rng, 500, 0.55).lower()), ('m3', 'ACGU' * 60 + 'acgu' * 40)]
    b['b5_gz.fna.gz'] = [('z%d' % i, seq_of(rng, n, 0.62)) for i, n in enumerate((1500, 420, 800))]
    b['b6_nan.fna'] = [('n0', seq_of(rng, 600, 0.5)), ('n_short', 'ACG'), ('n2', seq_of(rng, 1000, 0.5))]
    b['b7_tie.fna'] = [('t600', exact(rng, 600, 200)), ('t1200', exact(rng, 1200, 350)), ('t760', exact(rng, 760, 250))]
    b['b8_edge.fna'] = [('e_gc', seq_of(rng, 420, 0.56)), ('e_cd', seq_of(rng, 850, 0.5)), ('e_td', seq_of(rng, 1500, 0.5)),
                        ('e_rest', seq_of(rng, 3000, 0.5))]
    b['b9_shared.fna'] = [('s0', seq_of(rng, 400, 0.5)), b['b1_plain.fna'][1]]
    return b


def write_bin(path, records, width=70):
    lines = []
    for name, seq in records:
        lines.append('>%s some description\n' % name)
        lines.extend(seq[i:i + width] + '\n' for i in range(0, len(seq), width))
    opener = gzip.open if path.endswith('.gz') else open
    with opener(path, 'wt') as f:
        f.write(''.join(lines))


def write_gff(path, records, rng, no_gene):
    """Prodigal-style: genes of 150..600 bases with gaps and the odd overlap, none on the sequences of `no_gene`."""
    with open(path, 'w') as f:
        f.write('##gff-version  3\n')
        for name, seq in dict(records).items():
            f.write('# Sequence Data: seqnum=1;seqlen=%d;seqhdr="%s"\n' % (len(seq), name))
            f.write('# Model Data: version=Prodigal.v2.6.3;run_type=Single;model="Ab initio";gc_cont=50.00;transl_table=11;uses_sd=1\n')
            if name in no_gene or len(seq) < 200:
                continue
            at, k = int(rng.integers(1, 40)), 1
            while at + 150 < len(seq):
                end = min(len(seq), at + int(rng.integers(150, 600)))
                f.write('%s\tProdigal_v2.6.3\tCDS\t%d\t%d\t50.0\t+\t0\tID=1_%d;partial=00;\n' % (name, at, end, k))
                at, k = end + int(rng.integers(-30, 120)), k + 1


def tables(rng):
    def pct(keys, lo, hi, order):
        vals = dict(zip(keys, np.linspace(lo, hi, len(keys)).tolist()))
        return {k: vals[k] for k in order}
    gc, cd, td = {}, {}, {}
    for g in GC_KEYS:
        gc[g] = {}
        for i, n in enumerate(LEN_KEYS + ([6400] if g == 0.5 else [])):
            w = 0.22 / (1 + i) + 0.02 * g
            gc[g][n] = pct(GC_PCT, -w, w, GC_PCT if i == 0 else GC_PCT[::-1])
    for c in CD_KEYS:
        cd[c] = {}
        for i, n in enumerate(LEN_KEYS):
            w = 0.5 / (1 + i) + 0.05 * c
            cd[c][n] = pct(GC_PCT, -w, w, GC_PCT if i == 0 else GC_PCT[3:] + GC_PCT[:3])
    for i, n in enumerate(LEN_KEYS):
        td[n] = pct(TD_PCT, 0.05 + 0.3 / (1 + i), 0.2 + 0.5 / (1 + i), TD_PCT if i == 0 else TD_PCT[::-1])
    return gc, cd, td


def digest(path):
    """What a written FASTA file is held to: the SHA-256 of its bytes, and its ids for a readable failure."""
    text = open(path).read()
    return {'sha256': hashlib.sha256(text.encode()).hexdigest(), 'ids': [l[1:].split()[0] for l in text.split('\n') if l.startswith('>')]}


def write_tables(gc, cd, td):
    d = os.path.join(OUT, 'data', 'distributions')
    os.makedirs(d, exist_ok=True)
    for name, t in (('gc_dist', gc), ('cd_dist', cd), ('td_dist', td)):
        with open(os.path.join(d, name + '.txt'), 'w') as f:
            f.write(repr(t) + '\n')


def main():
    from oracle import outliers_oracle as oo
    from oracle.binstats_oracle import coding_bases, read_fasta
    rng = np.random.default_rng(20240607)
    shutil.rmtree(OUT, ignore_errors=True)
    os.makedirs(os.path.join(OUT, 'bins'))
    all_bins = bins(rng)
    for fname, records in all_bins.items():
        write_bin(os.path.join(OUT, 'bins', fname), records)
        gdir = os.path.join(OUT, 'out', 'bins', oo.bin_id(fname))
        os.makedirs(gdir)
        write_gff(os.path.join(gdir, 'genes.gff'), records, rng, no_gene={'p_odd', 'p4', 'e_rest'})
    write_bin(os.path.join(OUT, 'extra.fna'), [('unbinned0', seq_of(rng, 500, 0.35)), ('z1', seq_of(rng, 450, 0.2))])
    tmp = tempfile.mkdtemp(prefix='outlier_gold_')
    profileFile = os.path.join(tmp, 'tetra.tsv')
    with open(profileFile, 'w') as f:
        f.write(oo.profile_text([os.path.join(OUT, 'extra.fna')] + [os.path.join(OUT, 'bins', f) for f in all_bins]))

    # the tables, then three bounds moved onto values b8_edge reaches
    gc, cd, td = tables(rng)
    edge = os.path.join(OUT, 'bins', 'b8_edge.fna')
    seqs = read_fasta(edge)
    sigs = oo.read_profile(profileFile)
    _, covered = coding_bases(os.path.join(OUT, 'out', 'bins', 'b8_edge', 'genes.gff'))
    s = oo.bin_scores(seqs, sigs, covered)
    ids = list(seqs)
    kgc, kcd = oo.find_nearest(GC_KEYS, s['meanGC']), oo.find_nearest(CD_KEYS, s['meanCD'])
    i = ids.index('e_gc')
    assert s['deltaGC'][i] > 0
    gc[kgc][oo.find_nearest(LEN_KEYS, len(seqs['e_gc']))][97.5] = s['deltaGC'][i]
    i = ids.index('e_cd')
    cd[kcd][oo.find_nearest(LEN_KEYS, len(seqs['e_cd']))][2.5] = s['deltaCD'][i]
    i = ids.index('e_td')
    td[oo.find_nearest(LEN_KEYS, len(seqs['e_td']))][95] = s['TD'][i]
    write_tables(gc, cd, td)

    from checkm.binTools import BinTools
    from checkm.genomicSignatures import GenomicSignatures
    from checkm.prodigal import ProdigalGeneFeatureParser
    bt = BinTools()
    binFiles = [os.path.join(OUT, 'bins', f) for f in all_bins]
    outDir = os.path.join(OUT, 'out')
    expected = {'bins': list(all_bins), 'outliers': {}, 'helpers': {}}
    for report in REPORTS:
        for dist in DISTRIBUTIONS:
            path = os.path.join(tmp, 'outliers.tsv')
            bt.identifyOutliers(outDir, binFiles, profileFile, dist, report, path)
            expected['outliers']['%s_%d' % (report, dist)] = open(path).read()
            print(report, dist, expected['outliers']['%s_%d' % (report, dist)].count('\n') - 1, 'rows')

    from checkm.util.seqUtils import readFasta
    gs = GenomicSignatures(K=4, threads=1)
    tetraSigs = gs.read(profileFile)
    for f in [binFiles[k] for k in (0, 1, 5, 6)]:
        seqs = readFasta(f)
        binId = oo.bin_id(f)
        meanGC, deltaGCs, GCs = bt.gcDist(seqs)
        meanCD, deltaCDs, CDs = bt.codingDensityDist(seqs, ProdigalGeneFeatureParser(os.path.join(outDir, 'bins', binId, 'genes.gff')))
        binSig = bt.binTetraSig(seqs, tetraSigs)
        binSigCopy = np.array(binSig)
        meanTD, deltaTDs = bt.tetraDiffDist(seqs, gs, tetraSigs, binSigCopy)
        expected['helpers'][binId] = {'meanGC': float(meanGC), 'deltaGCs': deltaGCs.tolist(), 'GCs': [float(x) for x in GCs],
                                      'meanCD': float(meanCD), 'deltaCDs': deltaCDs.tolist(), 'CDs': [float(x) for x in CDs],
                                      'binSig': binSigCopy.tolist(), 'meanTD': float(meanTD), 'deltaTDs': deltaTDs.tolist()}

    # removeOutliers / modify / unique
    with open(os.path.join(tmp, 'o.tsv'), 'w') as f:
        f.write(expected['outliers']['any_95'])
    cleaned = {}
    for fname in ('b1_plain.fna', 'b5_gz.fna.gz', 'b2_one.fna'):
        path = os.path.join(tmp, 'cleaned.fna')
        bt.removeOutliers(os.path.join(OUT, 'bins', fname), os.path.join(tmp, 'o.tsv'), path)
        cleaned[fname] = digest(path)
    expected['removeOutliers'] = cleaned
    path = os.path.join(tmp, 'modified.fna')
    bt.modify(os.path.join(OUT, 'bins', 'b1_plain.fna'), os.path.join(OUT, 'bins', 'b5_gz.fna.gz'), ['z1', 'z2'], ['p0', 'p_odd'], path)
    expected['modify'] = dict(digest(path), add=['z1', 'z2'], remove=['p0', 'p_odd'])
    buf = io.StringIO()
    with contextlib.redirect_stdout(buf):
        bt.unique(binFiles)
    expected['unique_all'] = buf.getvalue()
    buf = io.StringIO()
    with contextlib.redirect_stdout(buf):
        bt.unique(binFiles[1:4])
    expected['unique_none'] = buf.getvalue()
    shutil.rmtree(tmp)
    text = json.dumps(expected, indent=1, sort_keys=True)
    text = re.sub(r'\[\n\s*([^\[\]{}]*?)\n\s*\]', lambda mt: '[' + ' '.join(mt.group(1).split()) + ']', text)   # flat lists on one line
    with open(os.path.join(OUT, 'expected.json'), 'w') as f:
        f.write(text + '\n')


if __name__ == '__main__':
    main()
