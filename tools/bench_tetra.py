"""Throughput of the genomic-signature scan (`checkm tetra`; checkm_b200/csrc/kmers.cu) against HBM bandwidth and against
the bin-statistics scan (ntstats_kernel) on the same layout, the low-complexity worst case, `GenomicSignatures.calculate`
end to end, and the reference's algorithm (oracle/tetra_oracle.py, one core) on a bounded sample.

    python tools/bench_tetra.py [--gbases 1.0] [--median 3000] [--steps 5] [--e2e-mb 256] [--cpu-seconds 10]

One JSON line: `value` = sequence bytes / kernel time (CUDA events, K = 4), with the card's name and power limit read in the
same run."""
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

HBM_GBS = 3350.0                # H100 SXM data sheet


def contigs(total, median, seed=7, alphabet=b'ACGT', repeat=None):
    """Log-normal lengths (median `median`, sigma 1) up to `total` bases; bases drawn once (64 MB) and reused at random
    offsets, or `repeat` tiled (the low-complexity case)."""
    rng = np.random.default_rng(seed)
    lens = np.maximum(rng.lognormal(np.log(median), 1.0, size=int(total / median * 1.2) + 16).astype(np.int64), 50)
    lens = lens[:int(np.searchsorted(np.cumsum(lens), total)) + 1]
    src = np.frombuffer((repeat * ((64 << 20) // len(repeat) + 1))[:64 << 20], dtype=np.uint8) if repeat else \
        rng.choice(np.frombuffer(alphabet, dtype=np.uint8), size=64 << 20)
    pool = np.concatenate([src, src[:int(lens.max())]])
    padded = (lens + 63) // 64 * 64
    starts = np.concatenate([[0], np.cumsum(padded)[:-1]]).astype(np.int64)
    data = np.zeros(int(padded.sum()) + 64, dtype=np.uint8)
    offs = rng.integers(0, 64 << 20, size=len(lens)) // 4 * 4
    for s, n, at in zip(starts, lens, offs):
        data[s:s + n] = pool[at:at + n]
    return data, starts, lens


def timed(fn, steps):
    fn()                                                      # warm-up: workspace allocation
    return float(np.median([fn() for _ in range(steps)]))


def card():
    try:
        out = subprocess.run(['nvidia-smi', '-i', os.environ.get('CKM_DEVICE', '0'), '--query-gpu=name,power.limit',
                              '--format=csv,noheader,nounits'], capture_output=True, text=True, timeout=10).stdout.strip()
        name, watts = [v.strip() for v in out.split(',')]
        return {"name": name, "power_limit_w": float(watts)}
    except Exception as e:                                    # the measurement stands without it, marked as such
        return {"name": None, "power_limit_w": None, "error": str(e)}


def end_to_end(data, starts, lens, mb, threads):
    """FASTA file on disk (60-column lines) -> GenomicSignatures.calculate -> profile file, split into its stages."""
    from checkm_b200.genomicSignatures import GenomicSignatures
    root = tempfile.mkdtemp(prefix='ckm_tetra_')
    try:
        path = os.path.join(root, 'seqs.fna')
        n, nbytes = 0, 0
        with open(path, 'wb') as f:
            while n < len(lens) and nbytes < mb * 1e6:
                seq = data[starts[n]:starts[n] + lens[n]].tobytes()
                f.write(b'>contig_%d\n' % n + b'\n'.join(seq[k:k + 60] for k in range(0, len(seq), 60)) + b'\n')
                nbytes += len(seq)
                n += 1
        gs = GenomicSignatures(4, threads)
        gs.calculate(path, os.path.join(root, 'warm.tsv'))
        t0 = time.perf_counter()
        gs.calculate(path, os.path.join(root, 'tetra.tsv'))
        wall = time.perf_counter() - t0
        t = dict(gs.timings)
        return {"sequences": n, "MB": nbytes / 1e6, "threads": threads, "seconds": wall, "MB_per_s": nbytes / 1e6 / wall,
                "read_and_layout_s": t['read_and_layout'], "h2d_and_other_device_call_s": t['device_calls'] - t['kernels'],
                "kernel_s": t['kernels'], "format_and_write_s": t['format_and_write'],
                "output_MB": os.path.getsize(os.path.join(root, 'tetra.tsv')) / 1e6}
    finally:
        shutil.rmtree(root, ignore_errors=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--gbases', type=float, default=1.0)
    ap.add_argument('--median', type=int, default=3000)
    ap.add_argument('--steps', type=int, default=5)
    ap.add_argument('--worst-gbases', type=float, default=0.25)
    ap.add_argument('--e2e-mb', type=float, default=256)
    ap.add_argument('--threads', type=int, default=8)
    ap.add_argument('--cpu-seconds', type=float, default=10.0)
    a = ap.parse_args()
    from checkm_b200 import runtime
    eng = runtime.engine()
    data, starts, lens = contigs(a.gbases * 1e9, a.median)
    total = int(lens.sum())
    k4 = timed(lambda: eng.kmer_counts(data, starts, lens, 4)[1], a.steps)
    k1 = timed(lambda: eng.kmer_counts(data, starts, lens, 1)[1], a.steps)
    nt = timed(lambda: eng.scaffold_stats(data, starts, lens)[3], a.steps)
    t0 = time.perf_counter()
    counts, _ = eng.kmer_counts(data, starts, lens, 4)
    call_s = time.perf_counter() - t0
    worst = {}
    for name, rep in (('homopolymer A', b'A'), ('dinucleotide AC', b'AC'), ('tetranucleotide GATC', b'GATC')):
        wd, ws, wl = contigs(a.worst_gbases * 1e9, a.median, seed=9, repeat=rep)
        ms = timed(lambda: eng.kmer_counts(wd, ws, wl, 4)[1], a.steps)
        worst[name] = {"GB_per_s": int(wl.sum()) / ms / 1e6, "kernel_ms": ms, "GB": int(wl.sum()) / 1e9}
    e2e = end_to_end(data, starts, lens, a.e2e_mb, a.threads) if a.e2e_mb > 0 else None
    from oracle import tetra_oracle as to
    index = to.kmer_index(4)
    t0, done, i = time.perf_counter(), 0, 0
    while time.perf_counter() - t0 < a.cpu_seconds and i < len(lens):
        s = data[starts[i]:starts[i] + lens[i]].tobytes().decode('latin-1')
        '\t'.join(map(str, to.seq_signature(s, 4, index)))
        done += int(lens[i])
        i += 1
    cpu = time.perf_counter() - t0
    print(json.dumps({
        "metric": "sequence bytes scanned per second, K = 4", "value": total / k4 / 1e6, "unit": "GB/s", "kernel_ms": k4, "steps": a.steps,
        "card": card(),
        "config": {"workload": "%d contigs, log-normal lengths (median %d, sigma 1), %.2f Gbases resident; input larger than L2" % (len(lens), a.median, total / 1e9)},
        "roofline": {"bound": "hbm", "achieved": total / k4 / 1e6, "peak": HBM_GBS, "unit": "GB/s", "frac": total / k4 / 1e6 / HBM_GBS,
                     "peak_source": "H100 SXM data sheet, 3350", "algorithmic_bytes": "1 byte read per base; 544 B written per sequence"},
        "k1": {"GB_per_s": total / k1 / 1e6, "kernel_ms": k1},
        "ntstats_same_layout": {"GB_per_s": total / nt / 1e6, "kernel_ms": nt, "tetra_over_ntstats": nt / k4},
        "engine_call_s": call_s, "counts_checksum": int(counts.sum(dtype=np.int64)),
        "low_complexity": worst,
        "e2e": e2e,
        "cpu_baseline": {"value": done / cpu / 1e6, "unit": "MB/s", "cores": 1, "kind": "port",
                         "sample": "%d contigs (%.1f MB) through oracle/tetra_oracle.py seq_signature + str() of the 136 values" % (i, done / 1e6)},
    }))


if __name__ == '__main__':
    main()
