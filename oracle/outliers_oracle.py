"""CPU restatement of `checkm outliers` (checkm/binTools.py:148-296) -- TEST INFRASTRUCTURE ONLY.

Only tests/ and tools/bench_outliers.py's CPU leg may import this; the product (checkm_b200/binTools.py) scores the
sequences on the device and never comes here.  Pinned: tests/test_outliers_cpu.py holds it to the outlier files the
reference's own BinTools wrote (tests/golden/outliers/, made by tests/golden/make_outlier_goldens.py) and holds
`pairwise_sum` to the installed numpy's np.sum bit for bit.

Plain Python floats (IEEE doubles) throughout; numpy is not used for any arithmetic, so the order of every sum is written
out here."""
import ast
import os

from oracle.binstats_oracle import base_counts, coding_bases, read_fasta

PRODIGAL_GFF = 'genes.gff'
HEADER = ('Bin Id\tSequence Id\tSequence length\tOutlying distributions'
          '\tSequence GC\tMean bin GC\tLower GC bound (%s%%)\tUpper GC bound (%s%%)'
          '\tSequence CD\tMean bin CD\tLower CD bound (%s%%)'
          '\tSequence TD\tMean bin TD\tUpper TD bound (%s%%)\n')


def pairwise_sum(a, lo=0, n=None):
    """np.sum of a contiguous float64 vector: below 8 elements a loop from 0.0; up to 128 elements eight running sums
    combined as ((r0+r1)+(r2+r3))+((r4+r5)+(r6+r7)) and the tail added one by one; above 128 the vector is halved, the
    first half rounded down to a multiple of 8."""
    if n is None:
        n = len(a)
    if n < 8:
        res = 0.0
        for i in range(lo, lo + n):
            res += a[i]
        return res
    if n <= 128:
        r = [a[lo + j] for j in range(8)]
        i = 8
        while i < n - n % 8:
            for j in range(8):
                r[j] += a[lo + i + j]
            i += 8
        res = ((r[0] + r[1]) + (r[2] + r[3])) + ((r[4] + r[5]) + (r[6] + r[7]))
        while i < n:
            res += a[lo + i]
            i += 1
        return res
    n2 = n // 2
    n2 -= n2 % 8
    return pairwise_sum(a, lo, n2) + pairwise_sum(a, lo + n2, n - n2)


def find_nearest(keys, value):
    """common.py:58-62: the key at the first minimum of |key - value| (a nan distance never wins, as in argmin unless it
    comes first)."""
    best = 0
    d0 = abs(keys[0] - value)
    if d0 != d0:
        return keys[0]                   # np.argmin returns the first nan
    for i in range(1, len(keys)):
        d = abs(keys[i] - value)
        if d != d:
            return keys[i]
        if d < d0:
            best, d0 = i, d
    return keys[best]


def read_distribution(data_root, prefix):
    with open(os.path.join(data_root, 'distributions', prefix + '.txt')) as f:
        return ast.literal_eval(f.read())


def read_profile(path):
    """genomicSignatures.py:189-200: id -> list of floats, a repeated id keeping its last line."""
    sig = {}
    with open(path) as f:
        next(f)
        for line in f:
            parts = line.split('\t')
            sig[parts[0]] = [float(x) for x in parts[1:]]
    return sig


def profile_text(fasta_files):
    """A profile file over the sequences of `fasta_files`, one line per sequence and file in the files' order, so an id
    that two files hold gets two lines (tests/golden/outliers/ keeps the FASTA files and not the 2.6 kB per line of the
    profile).  The lines are oracle/tetra_oracle.py's, which tests/test_tetra_cpu.py holds to the reference."""
    from oracle import tetra_oracle
    text = [tetra_oracle.profile_text({}, 4)]
    for path in fasta_files:
        text.append(tetra_oracle.profile_text(read_fasta(path), 4).split('\n', 1)[1])
    return ''.join(text)


def gc_dist(seqs):
    GCs, gc_total, bases_total = [], 0, 0
    for seq in seqs.values():
        a, c, g, t = base_counts(seq)
        GCs.append(float(g + c) / (a + c + g + t))
        gc_total += g + c
        bases_total += a + c + g + t
    mean = float(gc_total) / bases_total
    return mean, [x - mean for x in GCs], GCs


def cd_dist(seqs, covered):
    CDs, coding_total, bases_total = [], 0.0, 0
    for seq_id, seq in seqs.items():
        coding = float(covered.get(seq_id, 0))
        CDs.append(coding / len(seq))
        coding_total += coding
        bases_total += len(seq)
    mean = float(coding_total) / bases_total
    return mean, [x - mean for x in CDs], CDs


def bin_tetra_sig(seqs, sigs):
    """binTools.py:186-201: the first sequence's weighted signature, then the others added to it in dictionary order."""
    bin_size = sum(len(s) for s in seqs.values())
    bin_sig = None
    for seq_id, seq in seqs.items():
        w = float(len(seq)) / bin_size
        weighted = [v * w for v in sigs[seq_id]]
        bin_sig = weighted if bin_sig is None else [x + y for x, y in zip(bin_sig, weighted)]
    return bin_sig


def td_dist(seqs, sigs, bin_sig):
    TDs = [pairwise_sum([abs(x - y) for x, y in zip(sigs[seq_id], bin_sig)]) for seq_id in seqs]
    return pairwise_sum(TDs) / len(TDs), TDs


def bin_scores(seqs, sigs, covered):
    """Everything binTools.py:234-247 computes for one bin."""
    meanGC, deltaGCs, GCs = gc_dist(seqs)
    bin_sig = bin_tetra_sig(seqs, sigs)
    meanTD, TDs = td_dist(seqs, sigs, bin_sig)
    meanCD, deltaCDs, CDs = cd_dist(seqs, covered)
    return {'meanGC': meanGC, 'deltaGC': deltaGCs, 'GC': GCs, 'meanCD': meanCD, 'deltaCD': deltaCDs, 'CD': CDs,
            'binSig': bin_sig, 'meanTD': meanTD, 'TD': TDs}


def bounds(dists, meanGC, meanCD, distribution, seq_lens):
    """binTools.py:250-276: per sequence (gcLower, gcUpper, cdLower, tdUpper)."""
    gcB, cdB, tdB = dists
    closestGC = find_nearest(list(gcB.keys()), meanGC)
    d = gcB[closestGC][list(gcB[closestGC].keys())[0]]
    gcLo = find_nearest(list(d.keys()), (100 - distribution) / 2.0)
    gcHi = find_nearest(list(d.keys()), (100 + distribution) / 2.0)
    closestCD = find_nearest(list(cdB.keys()), meanCD)
    d = cdB[closestCD][list(cdB[closestCD].keys())[0]]
    cdLo = find_nearest(list(d.keys()), (100 - distribution) / 2.0)
    tdKey = find_nearest(list(tdB[list(tdB.keys())[0]].keys()), distribution)
    out = []
    for n in seq_lens:
        g = gcB[closestGC][find_nearest(list(gcB[closestGC].keys()), n)]
        c = cdB[closestCD][find_nearest(list(cdB[closestCD].keys()), n)]
        t = tdB[find_nearest(list(tdB.keys()), n)]
        out.append((g[gcLo], g[gcHi], c[cdLo], t[tdKey]))
    return out


def bin_id(path):
    base = os.path.basename(path)
    base = base[:-3] if base.endswith('.gz') else base
    return os.path.splitext(base)[0]


def identify_outliers(out_dir, bin_files, profile_file, distribution, report_type, data_root):
    """The text of the outlier file (binTools.py:211-296)."""
    dists = [read_distribution(data_root, p) for p in ('gc_dist', 'cd_dist', 'td_dist')]
    sigs = read_profile(profile_file)
    text = [HEADER % ((distribution,) * 4)]
    for path in bin_files:
        seqs = read_fasta(path)
        _, covered = coding_bases(os.path.join(out_dir, 'bins', bin_id(path), PRODIGAL_GFF))
        s = bin_scores(seqs, sigs, covered)
        bnd = bounds(dists, s['meanGC'], s['meanCD'], distribution, [len(q) for q in seqs.values()])
        for i, (seq_id, seq) in enumerate(seqs.items()):
            gcLo, gcHi, cdLo, tdHi = bnd[i]
            out = []
            if s['deltaGC'][i] < gcLo or s['deltaGC'][i] > gcHi:
                out.append('GC')
            if s['deltaCD'][i] < cdLo:
                out.append('CD')
            if s['TD'][i] > tdHi:
                out.append('TD')
            if (report_type == 'any' and len(out) >= 1) or (report_type == 'all' and len(out) == 3):
                text.append(bin_id(path) + '\t' + seq_id + '\t%d' % len(seq) + '\t' + ','.join(out))
                text.append('\t%.1f\t%.1f\t%.1f\t%.1f' % (s['GC'][i] * 100, s['meanGC'] * 100, (s['meanGC'] + gcLo) * 100,
                                                          (s['meanGC'] + gcHi) * 100))
                text.append('\t%.1f\t%.1f\t%.1f' % (s['CD'][i] * 100, s['meanCD'] * 100, (s['meanCD'] + cdLo) * 100))
                text.append('\t%.3f\t%.3f\t%.3f' % (s['TD'][i], s['meanTD'], tdHi) + '\n')
    return ''.join(text)
