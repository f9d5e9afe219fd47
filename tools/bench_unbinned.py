"""Measures `checkm unbinned` on a seeded synthetic metagenome: about 2 Gbp in 1.5 M records (log-normal lengths, 200 bp
to 500 kb, one sequence line per record), 35 % of the records spread over 150 bins, a few ids repeated in the assembly.
Prints one JSON line: the join kernels' and the count kernel's milliseconds by CUDA events, the wall time of
Unbinned.run split into read / scan / device / write with records per second and GB/s, the pure-Python oracle's time on
a 1 % slice scaled to the whole, and the card's name and power limit read in the same run.  The files go to a temporary
directory that is removed at the end.

    python tools/bench_unbinned.py [--records 1500000] [--runs 2] [--out bench_unbinned.json]"""
import argparse
import json
import logging
import os
import shutil
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
HDR = 20                                   # '>ctg000000123 len=1\n' is 20 bytes


def card():
    try:
        return subprocess.check_output(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], text=True).strip()
    except Exception as e:
        return 'unknown (%s)' % e


def fasta(lens, names, rng):
    """One FASTA file as bytes: record i is '>ctg<names[i]:09d> len=1\\n' and lens[i] random bases and '\\n'."""
    n = len(lens)
    rec = HDR + lens + 1
    start = np.concatenate([[0], np.cumsum(rec)[:-1]]).astype(np.int64)
    out = np.frombuffer(b'ACGT', dtype=np.uint8)[rng.integers(0, 4, size=int(rec.sum()), dtype=np.uint8)]
    head = np.empty((n, HDR), dtype=np.uint8)
    head[:] = np.frombuffer(b'>ctg000000000 len=1\n', dtype=np.uint8)
    v = np.asarray(names, dtype=np.int64)
    for k in range(9):
        head[:, 12 - k] = 48 + v % 10
        v = v // 10
    out[(start[:, None] + np.arange(HDR)).ravel()] = head.ravel()
    out[start + rec - 1] = 10
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--records', type=int, default=1_500_000)
    ap.add_argument('--bins', type=int, default=150)
    ap.add_argument('--runs', type=int, default=2)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    from checkm_b200.unbinned import Unbinned
    from oracle import unbinned_oracle
    logging.getLogger('timestamp').setLevel(logging.WARNING)
    rng = np.random.default_rng(2027)
    n = args.records
    lens = np.clip(rng.lognormal(np.log(700), 1.1, size=n), 200, 500_000).astype(np.int64)
    names = np.arange(n, dtype=np.int64)
    names[rng.choice(np.arange(1000, n), size=200, replace=False)] = rng.integers(0, 1000, size=200)   # repeated ids
    binned = rng.random(n) < 0.35
    bin_of = rng.integers(0, args.bins, size=n)
    tmp = tempfile.mkdtemp(prefix='bench_unbinned_')
    try:
        asm = os.path.join(tmp, 'assembly.fna')
        fasta(lens, names, rng).tofile(asm)
        binFiles = []
        for b in range(args.bins):
            sel = np.flatnonzero(binned & (bin_of == b))
            path = os.path.join(tmp, 'bin%03d.fna' % b)
            fasta(lens[sel], names[sel], rng).tofile(path)
            binFiles.append(path)
        in_bytes = os.path.getsize(asm) + sum(os.path.getsize(p) for p in binFiles)

        # warm-up on a small slice (module load, first allocations), then the timed runs
        small = os.path.join(tmp, 'small.fna')
        fasta(lens[:2000], names[:2000], rng).tofile(small)
        Unbinned().run(binFiles[:2], small, os.path.join(tmp, 'w.fna'), os.path.join(tmp, 'w.tsv'), 0)
        runs = []
        for _ in range(args.runs):
            u = Unbinned()
            t0 = time.perf_counter()
            u.run(binFiles, asm, os.path.join(tmp, 'out.fna'), os.path.join(tmp, 'out.tsv'), 0)
            wall = time.perf_counter() - t0
            t = dict(u.timing)
            t['wall'] = wall
            t['records_per_s'] = t['records'] / wall
            t['GBps'] = in_bytes / wall / 1e9
            runs.append(t)

        # the oracle on the first 1 % of the records, with the bins restricted to them, scaled by 100
        k = n // 100
        sub_asm = fasta(lens[:k], names[:k], rng).tobytes()
        sub_bins = [fasta(lens[:k][m], names[:k][m], rng).tobytes() for m in ((binned[:k] & (bin_of[:k] == b)) for b in range(args.bins))]
        t0 = time.perf_counter()
        unbinned_oracle.run(sub_bins, sub_asm, 0)
        oracle_s = (time.perf_counter() - t0) * n / k
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    out = {'card': card(), 'records': int(n), 'assembly_bp': int(lens.sum()), 'input_bytes': int(in_bytes),
           'binned_share': float(binned.mean()), 'bins': args.bins, 'runs': runs, 'oracle_s_scaled_from_1pct': oracle_s}
    line = json.dumps(out)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(args.out) or '.', exist_ok=True)
        with open(args.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
