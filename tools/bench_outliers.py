"""`checkm outliers` on the device (checkm_b200/binTools.py over csrc/outliers.cu), end to end on a synthetic assembly:
log-normal contigs in bins (one of them, "unbinned", holding a fifth of the contigs), the profile file written by this
package's GenomicSignatures, synthetic distribution files and one-gene-per-contig GFFs.

    python tools/bench_outliers.py [--contigs 200000] [--bins 500] [--reps 5] [--threads 8]

Prints one JSON line per measurement, each with the card's name, power limit and maximum SM clock read in the same run:
after a warm-up run, `identifyOutliers` by phase (profile parse, bin read + base scan, device calls ended by a stream
synchronise, row format + write, total); the three kernels by CUDA events, median of --reps replays of every batch's
scoring call; and the oracle (oracle/outliers_oracle.py, one core) on every 50th bin -- its time is for that sample and is
not extrapolated.  Needs a GPU; no device or host setting is changed."""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

LEN_KEYS = [500, 1000, 2000, 5000, 10000, 50000]
PCT = [0.5, 2.5, 5.0, 50.0, 95.0, 97.5, 99.5]


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else 'unknown'


def write_distributions(root):
    d = os.path.join(root, 'distributions')
    os.makedirs(d)
    spread = {n: 0.3 / (1 + i) for i, n in enumerate(LEN_KEYS)}
    tables = {'gc_dist': {round(float(g), 2): {n: dict(zip(PCT, np.linspace(-w, w, len(PCT)).tolist())) for n, w in spread.items()}
                          for g in np.arange(0.2, 0.81, 0.05)},
              'cd_dist': {round(float(c), 2): {n: dict(zip(PCT, np.linspace(-2 * w, 2 * w, len(PCT)).tolist())) for n, w in spread.items()}
                          for c in np.arange(0.5, 1.0, 0.1)},
              'td_dist': {n: {p: 0.05 + w * p / 100 for p in (50, 90, 95, 99)} for n, w in spread.items()}}
    for name, t in tables.items():
        with open(os.path.join(d, name + '.txt'), 'w') as f:
            f.write(repr(t))


def write_assembly(root, ncontigs, nbins, seed=1):
    """Bins as FASTA files with a genes.gff each, and all contigs as one assembly file.  Returns the bin files."""
    rng = np.random.default_rng(seed)
    lens = np.clip(rng.lognormal(7.5, 1.0, ncontigs), 300, 300000).astype(np.int64)
    share = rng.dirichlet(np.full(nbins - 1, 1.0)) * 0.8
    owner = rng.choice(nbins, size=ncontigs, p=np.concatenate([share, [0.2]]))
    letters = np.frombuffer(b'ACGT', dtype=np.uint8)
    binFiles = []
    with open(os.path.join(root, 'assembly.fna'), 'wb') as asm:
        for b in range(nbins):
            binId = 'bin%04d' % b if b < nbins - 1 else 'unbinned'
            gc = rng.uniform(0.3, 0.7)
            os.makedirs(os.path.join(root, 'bins', binId))
            parts, gff = [], []
            for c in np.flatnonzero(owner == b):
                p = gc if rng.random() > 0.02 else 1 - gc              # the odd foreign contig
                n = int(lens[c])
                seq = letters[rng.choice(4, size=n, p=[(1 - p) / 2, p / 2, p / 2, (1 - p) / 2])].tobytes()
                parts.append(b'>c%d\n' % c + seq + b'\n')
                gff.append('c%d\tbench\tCDS\t%d\t%d\t1.0\t+\t0\tID=1_1;\n' % (c, 1 + n // 20, n - n // 10))
            path = os.path.join(root, binId + '.fna')
            with open(path, 'wb') as f:
                f.write(b''.join(parts))
            asm.write(b''.join(parts))
            with open(os.path.join(root, 'bins', binId, 'genes.gff'), 'w') as f:
                f.write(''.join(gff))
            if parts:
                binFiles.append(path)
    return binFiles, int(lens.sum())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--contigs', type=int, default=200000)
    ap.add_argument('--bins', type=int, default=500)
    ap.add_argument('--reps', type=int, default=5)
    ap.add_argument('--threads', type=int, default=8)
    args = ap.parse_args()
    from checkm_b200 import runtime
    from checkm_b200.binTools import BinTools
    from checkm_b200.defaultValues import DefaultValues
    from checkm_b200.genomicSignatures import GenomicSignatures
    from oracle import outliers_oracle
    dev = card()
    eng = runtime.engine()                                          # fails here without a GPU

    def emit(rec):
        rec['card'] = dev
        print(json.dumps(rec), flush=True)

    with tempfile.TemporaryDirectory(prefix='bench_outliers_') as root:
        write_distributions(root)
        DefaultValues.set_data_root(root)
        t0 = time.perf_counter()
        binFiles, bases = write_assembly(root, args.contigs, args.bins)
        profile = os.path.join(root, 'tetra.tsv')
        t1 = time.perf_counter()
        GenomicSignatures(4, args.threads).calculate(os.path.join(root, 'assembly.fna'), profile)
        emit({'contigs': args.contigs, 'bins': len(binFiles), 'bases': bases, 'synthesis_s': round(t1 - t0, 2),
              'tetra_s': round(time.perf_counter() - t1, 2), 'profile_bytes': os.path.getsize(profile)})

        calls = []
        scores = eng.outlier_scores

        def recording(*a, **k):
            calls.append((a, k))
            return scores(*a, **k)
        out = os.path.join(root, 'outliers.tsv')
        bt = BinTools(threads=args.threads)
        bt.identifyOutliers(root, binFiles, profile, 95, 'any', out)          # warm-up: module load, workspaces
        eng.outlier_scores = recording
        t2 = time.perf_counter()
        bt.identifyOutliers(root, binFiles, profile, 95, 'any', out)
        total = time.perf_counter() - t2
        eng.outlier_scores = scores
        rec = {'identifyOutliers_total_s': round(total, 3), 'device_call_batches': len(calls)}
        rec.update({k: ([round(x, 3) for x in v] if isinstance(v, list) else round(v, 4) if isinstance(v, float) else v)
                    for k, v in bt.timing.items()})
        emit(rec)

        # the kernels alone: every batch's scoring call replayed against a resident copy of the profile matrix
        from checkm_b200.genomicSignatures import parse_profiles
        with open(profile, 'rb') as f:
            _, matrix = parse_profiles(f.read(), 136, args.threads)
        sigs = eng.signatures(matrix)
        per_rep = []
        for _ in range(max(5, args.reps)):
            ms = np.zeros(3)
            for a, k in calls:
                ms += scores(sigs, *a[1:], **k)[4]
            per_rep.append(ms)
        sigs.close()
        med = np.median(np.array(per_rep), axis=0)
        emit({'kernel_ms_median': {'outlier_bin_kernel': round(float(med[0]), 3), 'outlier_seq_kernel': round(float(med[1]), 3),
                                   'outlier_mean_kernel': round(float(med[2]), 3)}, 'reps': len(per_rep),
              'signature_bytes_read_by_seq_kernel': int(sum(len(a[2]) for a, _ in calls)) * 136 * 8})

        sample = binFiles[::50]
        t3 = time.perf_counter()
        want = outliers_oracle.identify_outliers(root, sample, profile, 95, 'any', root)
        oracle_s = time.perf_counter() - t3
        bt.identifyOutliers(root, sample, profile, 95, 'any', out)
        emit({'oracle_bins': len(sample), 'oracle_s_for_that_sample': round(oracle_s, 2), 'equal_to_oracle': open(out).read() == want})
    runtime.shutdown()


if __name__ == '__main__':
    main()
