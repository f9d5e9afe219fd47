"""Length profiles on the device (ckm_length_profile): 1,000 seeded bins of 10^2-10^5 records each (log-uniform counts,
log-normal lengths), Nx at step 0.05.  Prints the GPU's name and power limit, the kernel time of one call for all bins
(median of --reps after a warm-up), the call with its copies, and the pure-Python oracle (oracle/length_plots_oracle.py)
on the same bins for comparison.  With --plots N, also NxPlot / LengthHistogram .plot() on recording axes
(tools/axes_recorder.py) for the first N bins of up to 20 Mb written as FASTA files to a temporary directory.

    python tools/bench_length_plots.py [--bins 1000] [--reps 20] [--plots 20]"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time
import types

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def make_bins(nbins, seed=1):
    rng = np.random.default_rng(seed)
    counts = np.exp(rng.uniform(np.log(100), np.log(100000), nbins)).astype(np.int64)
    return [np.maximum(1, rng.lognormal(8.0, 1.2, n)).astype(np.int64) for n in counts]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--bins', type=int, default=1000)
    ap.add_argument('--reps', type=int, default=20)
    ap.add_argument('--plots', type=int, default=20)
    ap.add_argument('--oracle-bins', type=int, default=50)
    a = ap.parse_args()
    from checkm_b200 import runtime
    from oracle import length_plots_oracle as lo
    gpu = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True,
                         text=True).stdout.strip()
    bins = make_bins(a.bins)
    lens = np.concatenate(bins)
    off = np.zeros(len(bins) + 1, np.int64)
    off[1:] = np.cumsum([len(b) for b in bins])
    x = np.arange(0, 1.025, 0.05)
    eng = runtime.engine()
    eng.length_profile(lens, off, x)
    ms, wall = [], []
    for _ in range(a.reps):
        t0 = time.perf_counter()
        ms.append(eng.length_profile(lens, off, x)[-1])
        wall.append(time.perf_counter() - t0)
    t0 = time.perf_counter()
    for L in bins[:a.oracle_bins]:
        ll = L.tolist()
        lo.nx(x.tolist(), ll)
        lo.length_classes(ll)
    oracle_s = (time.perf_counter() - t0) / a.oracle_bins
    out = {'gpu': gpu, 'bins': a.bins, 'records': int(len(lens)), 'kernel_ms': float(np.median(ms)),
           'call_s': float(np.median(wall)), 'kernel_us_per_bin': 1e3 * float(np.median(ms)) / a.bins,
           'oracle_s_per_bin': oracle_s}
    if a.plots:
        from tools import axes_recorder as rec
        rec.install()
        from checkm_b200.plot.lengthHistogram import LengthHistogram
        from checkm_b200.plot.nxPlot import NxPlot
        o = types.SimpleNamespace(font_size=8, dpi=600, width=6.5, height=6.5, step_size=0.05)
        with tempfile.TemporaryDirectory() as tmp:
            files = []
            for i, L in enumerate([L for L in bins if L.sum() < 2e7][:a.plots]):      # bins of up to 20 Mb on disk
                path = os.path.join(tmp, 'b%d.fna' % i)
                with open(path, 'w') as f:
                    f.write(''.join('>s%d\n%s\n' % (k, 'A' * int(n)) for k, n in enumerate(L)))
                files.append(path)
            for name, cls in (('nx_plot', NxPlot), ('len_hist', LengthHistogram)):
                cls(o).plot(files[0])
                t0 = time.perf_counter()
                for f in files:
                    rec.reset()
                    cls(o).plot(f)
                out[name + '_s_per_bin'] = (time.perf_counter() - t0) / len(files)
        rec.uninstall()
    print(json.dumps(out))


if __name__ == '__main__':
    main()
