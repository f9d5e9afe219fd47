"""Strain heterogeneity on the device: (a) one `ckm_align_groups` call against one `ckm_align` call per (bin, marker) on
the same sequences, (b) `ckm_aai_pairs` against the reference's per-character Python loop on the CPU, and (c)
`HmmerAligner.makeAlignmentsOfMultipleHits` + `AminoAcidIdentity.run` end to end on bins searched by `MarkerGeneFinder`.

    python tools/bench_strain.py [--bins 1000] [--multi 6] [--reps 3]

Workload: `--bins` synthetic protein bins over the 43 CPR markers: each bin carries `--multi` multi-copy markers (2-3
copies of one emitted homolog at 60-99 % identity, with background flanks), 12 single-copy markers and 20 background ORFs.
One JSON line per measurement, each with the card's name and power limit read in the same run; times are host clocks
around calls that end in a device synchronise, best of --reps after one warm-up call."""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
CPR = os.path.join(ROOT, 'tests', 'golden', 'cpr_43_markers.hmm')


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else 'unknown'


def workload(nbins, nmulti, seed=5):
    """Per bin: a list of ORFs (code arrays) and the groups [(model, [orf indices])] of its multi-copy markers."""
    from tools import synth
    rng = np.random.default_rng(seed)
    hm = synth.read_hmms(CPR)
    pool = [[synth.emit_homolog(h, rng, sharpen=0.5) for _ in range(4)] for h in hm]
    bg = lambda n: rng.choice(20, size=n, p=synth.BG).astype(np.uint8)      # noqa: E731
    bins = []
    for _ in range(nbins):
        ms = rng.permutation(len(hm))
        orfs, groups = [bg(int(rng.integers(80, 400))) for _ in range(20)], []
        for m in ms[:nmulti]:
            base = pool[m][int(rng.integers(0, 4))]
            idx = []
            for f in rng.choice([0.01, 0.07, 0.12, 0.4], size=int(rng.integers(2, 4))):
                t = base.copy()
                mut = rng.random(len(t)) < f
                t[mut] = (t[mut] + rng.integers(1, 20, size=int(mut.sum()))) % 20
                idx.append(len(orfs))
                orfs.append(np.concatenate([bg(int(rng.integers(3, 40))), t, bg(int(rng.integers(3, 40)))]))
            groups.append((int(m), idx))
        for m in ms[nmulti:nmulti + 12]:
            orfs.append(np.concatenate([bg(10), pool[m][int(rng.integers(0, 4))], bg(10)]))
        bins.append((orfs, groups))
    return bins


def best_of(fn, reps):
    fn()
    t = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        t.append(time.perf_counter() - t0)
    return min(t)


def python_aai(a, b):
    """checkm/aminoAcidIdentity.py:127-161, the loop the reference runs per pair."""
    startIndex = 0
    for i in range(0, len(a)):
        if a[i] == '-' or b[i] == '-':
            startIndex = i + 1
        else:
            break
    endIndex = len(a)
    for i in range(len(a) - 1, 0, -1):
        if a[i] == '-' or b[i] == '-':
            endIndex = i
        else:
            break
    mismatches = 0
    seqLen = 0
    for i in range(startIndex, endIndex):
        if a[i] != b[i]:
            mismatches += 1
            seqLen += 1
        elif a[i] == '-' and b[i] == '-':
            pass
        else:
            seqLen += 1
    return 0.0 if seqLen == 0 else 1.0 - (float(mismatches) / seqLen)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--bins', type=int, default=1000)
    ap.add_argument('--multi', type=int, default=6)
    ap.add_argument('--reps', type=int, default=3)
    args = ap.parse_args()
    from checkm_b200 import runtime
    from checkm_b200.hmmerAligner import masked_rows
    gpu = card()
    eng = runtime.engine()
    models = runtime.models_for(CPR)
    info = models.info()
    bins = workload(args.bins, args.multi)
    base = {'card': gpu, 'bins': args.bins, 'multi_copy_markers_per_bin': args.multi}

    def emit(**kv):
        print(json.dumps(dict(base, **kv)), flush=True)

    # ---- (a) groups: one call against one call per group ----
    seqs, gmodel, goff = [], [], [0]
    for orfs, groups in bins:
        for m, idx in groups:
            seqs += [orfs[i] for i in idx]
            gmodel.append(m)
            goff.append(len(seqs))
    off = np.zeros(len(seqs) + 1, np.int64)
    off[1:] = np.cumsum([len(s) for s in seqs])
    res = np.concatenate(seqs)
    db = eng.seqdb(res, off)
    state = [None]

    def one_call():
        state[0] = eng.align_groups(models, db, gmodel, goff)[0]
    t_groups = best_of(one_call, args.reps)
    sub = []
    for g in range(len(gmodel)):
        o = off[goff[g]:goff[g + 1] + 1] - off[goff[g]]
        sub.append(eng.seqdb(res[off[goff[g]]:off[goff[g + 1]]], o))

    def per_group():
        for g, d in enumerate(sub):
            eng.align(models, d, gmodel[g])
    t_per = best_of(per_group, 1)
    for d in sub:
        d.close()
    db.close()
    emit(step='align', groups=len(gmodel), sequences=len(seqs), residues=int(off[-1]), align_groups_s=round(t_groups, 4),
         align_per_group_s=round(t_per, 4), speedup=round(t_per / t_groups, 2))

    # ---- (b) AAI: one device call against the Python loop ----
    rows, pairs = [], []
    for g, m in enumerate(gmodel):
        r0, r1 = off[goff[g]], off[goff[g + 1]]
        mr = masked_rows(res[r0:r1], state[0][r0:r1], np.diff(off[goff[g]:goff[g + 1] + 1]), int(info[m].M))
        b = len(rows)
        rows += [r.tobytes().decode() for r in mr]
        pairs += [(b + i, b + j) for i in range(len(mr)) for j in range(i + 1, len(mr))]
    roff = np.zeros(len(rows) + 1, np.int64)
    roff[1:] = np.cumsum([len(r) for r in rows])
    data = ''.join(rows).encode()
    parr = np.array(pairs, np.int32)
    out = [None]

    def dev():
        out[0] = eng.aai_pairs(data, roff, parr)
    t_dev = best_of(dev, args.reps)
    t0 = time.perf_counter()
    ref = [python_aai(rows[i], rows[j]) for i, j in pairs]
    t_py = time.perf_counter() - t0
    got = [0.0 if n == 0 else 1.0 - (float(m) / n) for m, n in zip(out[0][0].tolist(), out[0][1].tolist())]
    emit(step='aai', pairs=len(pairs), columns=int(roff[-1]), aai_pairs_s=round(t_dev, 5), python_loop_s=round(t_py, 3),
         speedup=round(t_py / t_dev, 1), identical=got == ref)

    # ---- (c) end to end on searched bins ----
    from checkm_b200.aminoAcidIdentity import AminoAcidIdentity
    from checkm_b200.defaultValues import DefaultValues
    from checkm_b200.hmmerAligner import HmmerAligner
    from checkm_b200.markerGeneFinder import MarkerGeneFinder
    from checkm_b200.markerSets import MarkerSetParser
    from tools import synth
    work = tempfile.mkdtemp(prefix='bench_strain_')
    try:
        DefaultValues.set_data_root(os.path.join(ROOT, 'tests', 'golden', 'reduction', 'data'))
        files = []
        for b, (orfs, _) in enumerate(bins):
            p = os.path.join(work, 'bin%04d.faa' % b)
            with open(p, 'w') as f:
                for i, s in enumerate(orfs):
                    f.write('>c1_%d # 1 # 3 # 1 # ID=1_%d;partial=00\n%s*\n' % (i + 1, i + 1, ''.join(synth.ALPHABET[c] for c in s)))
            files.append(p)
        out_dir = os.path.join(work, 'out')
        os.makedirs(os.path.join(out_dir, 'storage', 'aai_qa'))
        t0 = time.perf_counter()
        b2m = MarkerGeneFinder(1).find(files, out_dir, 'hmmer.analyze.txt', 'hmmer.analyze.ali.txt', CPR, False, False, True)
        t_find = time.perf_counter() - t0
        bms = MarkerSetParser(1).getMarkerSets(out_dir, list(b2m.keys()), CPR)
        t0 = time.perf_counter()
        HmmerAligner(1).makeAlignmentsOfMultipleHits(out_dir, CPR, 'hmmer.analyze.txt', b2m, bms, False, DefaultValues.E_VAL,
                                                     DefaultValues.LENGTH, os.path.join(out_dir, 'storage', 'aai_qa'))
        t_align = time.perf_counter() - t0
        aai = AminoAcidIdentity()
        t0 = time.perf_counter()
        aai.run(0.9, out_dir, None)
        t_aai = time.perf_counter() - t0
        npairs = sum(len(v) for ms in aai.aaiRawScores.values() for v in ms.values())
        emit(step='end_to_end', find_s=round(t_find, 2), multiple_hits_s=round(t_align, 3), aai_run_s=round(t_aai, 3),
             bins_with_pairs=len(aai.aaiMeanBinHetero), aai_pairs=npairs)
    finally:
        shutil.rmtree(work, ignore_errors=True)


if __name__ == '__main__':
    main()
