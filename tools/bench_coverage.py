"""`checkm coverage` on the device (checkm_b200/csrc/bam.cu): the inflate kernel in GB/s of compressed input and of
inflated output, the record scan in records/s, `Coverage.run` end to end split into reading (index, block table, header),
device calls (host-to-device copies and kernels) and formatting; and two CPU baselines measured in the same run: the same
blocks inflated by the stdlib zlib on all cores (zlib releases the GIL: the floor any CPU path pays), and the oracle's
record loop (oracle/coverage_oracle.py) on one core.

    python tools/bench_coverage.py [--gb 1.0] [--oracle-mb 64] [--json out.json]

Two seeded workloads of about --gb compressed GB each, written to a temporary directory at level 6:
  short  a metagenome assembly: one contig of 1-20 kb per 150 reads (~48,000 contigs at 1 GB), ~2x
  long   six contigs of 5 Mb at ~36x (1 GB): the fewest anchors per record (one per 16 kb window)
The oracle runs on a smaller sample of the same shape (--oracle-mb of records) and its rate is reported for that sample.
One JSON line per workload, with the card's name and power limit read in the same run."""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time
import zlib
from concurrent.futures import ThreadPoolExecutor

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

RECORD_BYTES = 292                    # one bulk record (150 bp, 3 CIGAR ops, NM:C)
COMPRESSED_RATIO = 0.48               # compressed / inflated for these records at level 6 (sizes the workloads)


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else 'unknown'


def workload(kind, nrec, seed):
    rng = np.random.default_rng(seed)
    if kind == 'short':
        n = max(10, nrec // 150)
        lens = rng.integers(1000, 20000, size=n)
        reads = np.maximum(1, (lens * nrec / lens.sum()).astype(np.int64))
    else:
        lens = np.full(6, 5_000_000)
        reads = np.full(6, nrec // 6)
    return rng, lens, reads


def write(path, kind, nrec, seed):
    from tools import bamsynth as bs
    rng, lens, reads = workload(kind, nrec, seed)
    body, ref, pos, end = bs.bulk_records(rng, lens, reads)
    tail = b''.join(bs.record(rng, -1, -1, 't%d' % i, flag=0x4, cigar=(), l_seq=150, nm=None)[0] for i in range(1000))
    refs = [('%s%d' % (kind, i), int(n)) for i, n in enumerate(lens)]
    bs.write_bam(path, refs, body, ref, pos, end, np.zeros(len(ref), bool), n_unplaced=1000, unplaced=tail, levels=(6,),
                 threads=os.cpu_count() or 1)
    return len(ref)


def host_zlib(path, threads):
    from checkm_b200 import bam
    with open(path, 'rb') as f:
        raw = f.read()
    blocks, _ = bam.bgzf_blocks(raw)
    spans = [(c + 18, c + n - 8) for c, n, _ in blocks.tolist()]
    chunks = [spans[i::threads] for i in range(threads)]

    def work(part):
        return sum(len(zlib.decompress(raw[a:b], -15)) for a, b in part)
    t0 = time.perf_counter()
    with ThreadPoolExecutor(threads) as ex:
        out = sum(ex.map(work, chunks))
    return time.perf_counter() - t0, len(raw), out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--gb', type=float, default=1.0)
    ap.add_argument('--oracle-mb', type=float, default=64)
    ap.add_argument('--json', default=None)
    a = ap.parse_args()
    from checkm_b200 import runtime
    from checkm_b200.coverage import Coverage
    from oracle import coverage_oracle as co
    name = card()
    runtime.engine()
    tmp = tempfile.mkdtemp(prefix='bench_coverage_')
    results = []
    try:
        for i, kind in enumerate(('short', 'long')):
            path = os.path.join(tmp, kind + '.bam')
            nrec = int(a.gb * 1e9 / COMPRESSED_RATIO / RECORD_BYTES)
            t0 = time.perf_counter()
            nrec = write(path, kind, nrec, 100 + i)
            t_gen = time.perf_counter() - t0
            size = os.path.getsize(path)
            cov = Coverage(1)
            out = os.path.join(tmp, kind + '.tsv')
            cov.run([], [path], out, False, 0.98, 0.02, 15)              # warm-up: module load, pool growth, page cache
            runs = []
            for _ in range(2):
                t0 = time.perf_counter()
                cov.run([], [path], out, False, 0.98, 0.02, 15)
                runs.append((time.perf_counter() - t0, dict(cov.timing)))
            wall, tm = min(runs, key=lambda r: r[0])
            kern_s = (tm['inflate_ms'] + tm['scan_ms']) / 1e3
            threads = os.cpu_count() or 1
            zt, zc, zu = host_zlib(path, threads)
            opath = os.path.join(tmp, kind + '_oracle.bam')
            onrec = write(opath, kind, int(a.oracle_mb * 1e6 / RECORD_BYTES), 200 + i)
            t0 = time.perf_counter()
            co.counters(opath)
            ot = time.perf_counter() - t0
            r = {'workload': kind, 'card': name, 'file_bytes': size, 'records': nrec, 'segments': tm['segments'],
                 'batches': tm['batches'], 'compressed_bytes': tm['compressed_bytes'], 'inflated_bytes': tm['inflated_bytes'],
                 'inflate_ms': round(tm['inflate_ms'], 2), 'scan_ms': round(tm['scan_ms'], 2),
                 'inflate_GBps_compressed': round(tm['compressed_bytes'] / tm['inflate_ms'] / 1e6, 2),
                 'inflate_GBps_inflated': round(tm['inflated_bytes'] / tm['inflate_ms'] / 1e6, 2),
                 'scan_Mrecords_per_s': round(nrec / tm['scan_ms'] / 1e3, 1),
                 'run_s': round(wall, 3), 'read_s': round(tm['read'], 3), 'device_calls_s': round(tm['device_calls'], 3),
                 'kernels_s': round(kern_s, 3), 'copies_and_host_in_calls_s': round(tm['device_calls'] - kern_s, 3),
                 'format_write_s': round(tm['format_write'], 3),
                 'host_zlib_threads': threads, 'host_zlib_s': round(zt, 3),
                 'host_zlib_GBps_inflated': round(zu / zt / 1e9, 2),
                 'oracle_records': onrec, 'oracle_s': round(ot, 2), 'oracle_Mrecords_per_s_one_core': round(onrec / ot / 1e6, 3),
                 'generate_s': round(t_gen, 1)}
            print(json.dumps(r), flush=True)
            results.append(r)
            os.remove(path)
            os.remove(opath)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    if a.json:
        with open(a.json, 'w') as f:
            json.dump(results, f, indent=1)


if __name__ == '__main__':
    main()
