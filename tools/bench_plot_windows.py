"""Measures the plot windows on the device: 1,000 seeded bins of 2-6 Mb, one ckm_window_stats call per bin at W = 5,000
with a bin signature (what tetra_plot and dist_plot make per bin).  Prints one JSON line: the kernels' time by CUDA
events, the bytes scanned over it against 3.35 TB/s (the H100 SXM data sheet's HBM3 bandwidth), the wall time per bin
of TetraDistPlots.plotOnAxes on recording axes (tools/axes_recorder.py), the CPU oracle's time per bin (on a 1 Mb slice,
scaled), and the card's name and power limit read in the same run.

    python tools/bench_plot_windows.py [--bins 1000] [--out bench_plot_windows.json]"""
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


def card():
    try:
        return subprocess.check_output(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], text=True).strip()
    except Exception as e:
        return 'unknown (%s)' % e


def make_bin(rng):
    size = int(rng.integers(2_000_000, 6_000_000))
    lens = []
    while sum(lens) < size:
        lens.append(int(rng.integers(1000, 400_000)))
    g = rng.uniform(0.3, 0.7)
    seq = rng.choice(np.frombuffer(b'ACGT', dtype=np.uint8), size=sum(lens), p=[(1 - g) / 2, g / 2, g / 2, (1 - g) / 2])
    lens = np.array(lens, dtype=np.int64)
    starts = np.concatenate([[0], np.cumsum((lens + 63) // 64 * 64)[:-1]]).astype(np.int64)
    data = np.zeros(int(starts[-1] + (lens[-1] + 63) // 64 * 64), dtype=np.uint8)
    at = 0
    for a, n in zip(starts, lens):
        data[a:a + n] = seq[at:at + n]
        at += n
    return data, starts, lens


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--bins', type=int, default=1000)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    from checkm_b200 import runtime
    from checkm_b200.coverageWindows import window_offsets
    from oracle import plot_windows_oracle as pw
    eng = runtime.engine()
    rng = np.random.default_rng(5000)
    W = 5000
    sig = rng.dirichlet(np.ones(136))
    kernel_ms, scanned, calls = 0.0, 0, 0.0
    first = None
    for b in range(args.bins):
        data, starts, lens = make_bin(rng)
        first = first or (data, starts, lens)
        off = window_offsets(lens, W)
        t0 = time.perf_counter()
        _, _, ms = eng.window_stats(data, starts, lens, W, off, sig)
        calls += time.perf_counter() - t0
        if b:                                         # the first call loads the module
            kernel_ms += ms
            scanned += int(lens.sum())
    n = max(args.bins - 1, 1)

    # plotOnAxes on recording axes, per bin, over bins written as FASTA
    from tools import axes_recorder as rec
    rec.install()
    from checkm_b200.plot.tetraDistPlots import TetraDistPlots
    from checkm_b200.defaultValues import DefaultValues
    tmp = tempfile.mkdtemp()
    os.makedirs(os.path.join(tmp, 'distributions'))
    with open(os.path.join(tmp, 'distributions', 'td_dist.txt'), 'w') as f:
        f.write(repr({1000: {95: 0.2}, 5000: {95: 0.1}}))
    DefaultValues.set_data_root(tmp)
    data, starts, lens = first
    path = os.path.join(tmp, 'bin.fna')
    with open(path, 'wb') as f:
        for i, (a, m) in enumerate(zip(starts, lens)):
            f.write(b'>s%d\n' % i + data[a:a + m].tobytes() + b'\n')
    tetraSigs = {'s%d' % i: sig for i in range(len(lens))}
    opts = types.SimpleNamespace(font_size=8, dpi=600, width=6.5, height=8, td_window_size=W, td_bin_width=0.01)
    plot_s = []
    for _ in range(4):
        rec.reset()
        p = TetraDistPlots(opts)
        t0 = time.perf_counter()
        p.plotOnAxes(path, tetraSigs, [95], rec.Axes('h'), rec.Axes('d'))
        plot_s.append(time.perf_counter() - t0)
    rec.uninstall()

    # the CPU oracle on 1 Mb of the first bin, scaled to the bin
    seq = data[starts[0]:starts[0] + lens[0]].tobytes().decode('latin-1')[:1_000_000]
    t0 = time.perf_counter()
    pw.window_stats(seq, W, sig.tolist())
    oracle_s = (time.perf_counter() - t0) * lens.sum() / max(len(seq), 1)
    out = {'bins': args.bins, 'window': W, 'card': card(), 'kernel_ms_per_bin': kernel_ms / n,
           'bytes_per_bin': scanned / n, 'scan_TBps': scanned / (kernel_ms / 1e3) / 1e12 if kernel_ms else None,
           'share_of_3.35TBps': (scanned / (kernel_ms / 1e3) / 3.35e12) if kernel_ms else None,
           'call_s_per_bin': calls / args.bins, 'plotOnAxes_s_per_bin': sorted(plot_s)[1],
           'oracle_s_per_bin': oracle_s}
    line = json.dumps(out)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(args.out) or '.', exist_ok=True)
        with open(args.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
