"""Read depth per window (`checkm gc_bias_plot`'s coverage profile) on the device (bam_window_kernel, csrc/bam.cu): the
inflate and window-scan kernels at W = 5000, 100 and 1, `CoverageWindows.run` split into reading (index, block table,
header), device calls and formatting, `Coverage.run` on the same file (the record scan without windows), and parity of
the window sums with the oracle (oracle/coverage_windows_oracle.py) on a smaller sample of the same shape.

    python tools/bench_coverage_windows.py [--gb 1.0] [--oracle-mb 16] [--json out.json]

The two seeded workloads of tools/bench_coverage.py (about --gb compressed GB each, level 6):
  short  one contig of 1-20 kb per 150 reads (~48,000 contigs at 1 GB), ~2x
  long   six contigs of 5 Mb at ~36x
At W = 1 the reference's return value is one Python float per base (about 500 M of them for `short`), so W = 1 times the
device calls of `_processBam` only and leaves the formatting out.  One JSON line per workload, with the card's name and
power limit read in the same run."""
import argparse
import json
import os
import shutil
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tools.bench_coverage import COMPRESSED_RATIO, RECORD_BYTES, card, write  # noqa: E402

WINDOWS = (5000, 100, 1)


def best_of(fn, n=2):
    runs = []
    for _ in range(n):
        t0 = time.perf_counter()
        timing = fn()
        runs.append((time.perf_counter() - t0, timing))
    return min(runs, key=lambda r: r[0])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--gb', type=float, default=1.0)
    ap.add_argument('--oracle-mb', type=float, default=16)
    ap.add_argument('--json', default=None)
    a = ap.parse_args()
    from checkm_b200 import runtime
    from checkm_b200.coverage import Coverage
    from checkm_b200.coverageWindows import CoverageWindows
    from oracle import coverage_windows_oracle as cwo
    name = card()
    runtime.engine()
    tmp = tempfile.mkdtemp(prefix='bench_coverage_windows_')
    results = []
    try:
        for i, kind in enumerate(('short', 'long')):
            path = os.path.join(tmp, kind + '.bam')
            nrec = write(path, kind, int(a.gb * 1e9 / COMPRESSED_RATIO / RECORD_BYTES), 100 + i)
            r = {'workload': kind, 'card': name, 'file_bytes': os.path.getsize(path), 'records': nrec}

            cov = Coverage(1)
            out = os.path.join(tmp, kind + '.tsv')
            cov.run([], [path], out, False, 0.98, 0.02, 15)              # warm-up: module load, pool growth, page cache

            def coverage_run():
                cov.run([], [path], out, False, 0.98, 0.02, 15)
                return dict(cov.timing)
            wall, tm = best_of(coverage_run)
            r['coverage'] = {'run_s': round(wall, 3), 'inflate_ms': round(tm['inflate_ms'], 2),
                             'scan_ms': round(tm['scan_ms'], 2), 'batches': tm['batches']}

            cw = CoverageWindows(1)
            cw.run([], path, False, 0.98, 0.02, 5000)                      # warm-up
            for W in WINDOWS:
                def windows_run():
                    cw.timing = {'read': 0.0, 'device_calls': 0.0, 'inflate_ms': 0.0, 'scan_ms': 0.0, 'format': 0.0,
                                 'batches': 0, 'compressed_bytes': 0, 'inflated_bytes': 0, 'segments': 0, 'windows': 0}
                    if W == 1:
                        cw._processBam(path, False, 0.98, 0.02, W)
                    else:
                        cw.run([], path, False, 0.98, 0.02, W)
                    return dict(cw.timing)
                wall, tm = best_of(windows_run)
                kern_s = (tm['inflate_ms'] + tm['scan_ms']) / 1e3
                r['W%d' % W] = {'windows': tm['windows'], 'run_s': round(wall, 3), 'read_s': round(tm['read'], 3),
                                'device_calls_s': round(tm['device_calls'], 3), 'kernels_s': round(kern_s, 3),
                                'format_s': round(tm['format'], 3) if W != 1 else 'not measured',
                                'inflate_ms': round(tm['inflate_ms'], 2), 'window_scan_ms': round(tm['scan_ms'], 2),
                                'window_scan_over_inflate': round(tm['scan_ms'] / tm['inflate_ms'], 3),
                                'batches': tm['batches']}
            os.remove(path)

            opath = os.path.join(tmp, kind + '_oracle.bam')
            onrec = write(opath, kind, int(a.oracle_mb * 1e6 / RECORD_BYTES), 200 + i)
            t0 = time.perf_counter()
            names, lens, want_cnt, deps = cwo.depths(opath)
            ot = time.perf_counter() - t0
            parity = True
            for W in (100, 1):
                cw.timing = {'read': 0.0, 'device_calls': 0.0, 'inflate_ms': 0.0, 'scan_ms': 0.0, 'batches': 0,
                             'compressed_bytes': 0, 'inflated_bytes': 0, 'segments': 0, 'windows': 0}
                _, _, cnt, win, _ = cw._processBam(opath, False, 0.98, 0.02, W)
                want = np.concatenate([cwo.window_sums(d, W) for d in deps])
                parity &= bool(np.array_equal(cnt, want_cnt) and np.array_equal(win, want))
            r.update({'oracle_records': onrec, 'oracle_s': round(ot, 2), 'parity_W100_W1': parity})
            os.remove(opath)
            print(json.dumps(r), flush=True)
            results.append(r)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    if a.json:
        with open(a.json, 'w') as f:
            json.dump(results, f, indent=1)


if __name__ == '__main__':
    main()
