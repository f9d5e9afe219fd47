"""Per-class measurement of the packed ViterbiFilter (vitp_kernel<W>, checkm_b200/csrc/kernels_vitp.cu) on the batch of
bench.py --config 3 (16 bins x 2,900 ORFs x 5,000 models, built with bench.py's own generators).

    python tools/bench_viterbi.py [--bins 16] [--reps 5] [--out FILE.json] [--dry-run]

Reports, per class W: the pairs that reach the packed kernel (bias survivors, from the dense pass bits of
ckm_filter_scores), their padded cells (64 W per row), the kernel time (torch.profiler, in a run of its own after the timed
ones), cells/s, and the bound of the DPX instructions alone (7 VIADDMNMX per word and row; 2 warp-instructions/clk/SM at
the card's maximum SM clock) as a floor on the time.  The stage time (ms_vit, CUDA events in the engine) is the median of
--reps searches.  --dry-run builds the workload and the class table on the host and stops before the device.
"""
import argparse
import json
import os
import re
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402

WS = (1, 2, 3, 4, 6, 8, 10, 12, 14, 16)


def vq_of(M):
    for lim, q in ((64, 2), (128, 4), (192, 6), (256, 8), (384, 12), (512, 16), (640, 20), (768, 24), (896, 28), (1024, 32)):
        if M <= lim:
            return q
    return 0


def card():
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader,nounits'],
                             capture_output=True, text=True, timeout=30).stdout.strip().split('\n')[0]
        name, pl, mhz = [x.strip() for x in out.split(',')]
        return {"name": name, "power_limit_w": float(pl), "sm_max_mhz": float(mhz)}
    except Exception as ex:                                  # noqa: BLE001
        return {"error": str(ex)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--bins', type=int, default=bench.BINS_PER_STEP)
    ap.add_argument('--reps', type=int, default=5)
    ap.add_argument('--out', help='also write the report to this JSON file')
    ap.add_argument('--dry-run', action='store_true')
    args = ap.parse_args()

    t0 = time.perf_counter()
    db_path = bench.model_db(bench.N_MODELS)
    from tools import synth
    Ms = np.asarray([h.M for h in synth.read_hmms(db_path)])
    bt = bench.Batch(bench.make_bins(args.bins, 10000, bench.CFG[3]['orfs']))
    W_of = np.asarray([vq_of(int(M)) // 2 for M in Ms])
    rep = {"workload": "%d bins x %d ORFs (%d residues) x %d models" % (args.bins, len(bt.off) - 1, len(bt.res), len(Ms)),
           "models_per_class": {str(w): int((W_of == w).sum()) for w in WS}, "models_without_class": int((W_of == 0).sum()),
           "host_setup_s": time.perf_counter() - t0}
    if args.dry_run:
        print(json.dumps(rep, indent=1))
        return

    import torch
    from checkm_b200 import engine as E
    eng = E.Engine()
    models = eng.load_models(db_path)
    db = eng.seqdb(bt.res, bt.off, bt.binof, args.bins)
    rep["card"] = card()
    for _ in range(2):
        eng.search(models, db)
    vit_ms = []
    for _ in range(args.reps):
        eng.search(models, db)
        st = eng.stats()
        vit_ms.append(st.ms_vit)
    rep["ms_vit"] = {"median": float(np.median(vit_ms)), "min": float(min(vit_ms)), "max": float(max(vit_ms)), "runs": vit_ms}
    rep["vit_int32_redo"] = int(st.n_vit_redo)

    # pairs and padded cells of every class: bias survivors from the dense pass bits
    _, _, _, ps = eng.filter_scores(models, db)
    L = np.diff(bt.off)
    surv = (ps & 2) != 0
    pairs = surv.sum(axis=1)
    rows = surv.astype(np.int64) @ L
    del ps, surv

    # kernel times: torch.profiler in a run of its own
    from torch.profiler import profile, ProfilerActivity
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        eng.search(models, db)
        torch.cuda.synchronize()
    kt = {}
    for ev in prof.key_averages():
        m = re.search(r'vitp_kernel<(\d+)', ev.key)
        if m:
            kt[int(m.group(1))] = kt.get(int(m.group(1)), 0.0) + ev.device_time_total / 1e3   # ms
    mhz = rep["card"].get("sm_max_mhz")
    nsm = torch.cuda.get_device_properties(0).multi_processor_count
    cls = {}
    for w in WS:
        sel = W_of == w
        cells = float(rows[sel].sum()) * 64 * w
        ms = kt.get(w)
        # DPX floor: 7 VIADDMNMX per word and row, 2 warp-instructions/clk/SM
        floor_ms = float(rows[sel].sum()) * 7 * w / (2.0 * nsm * mhz * 1e6) * 1e3 if mhz else None
        cls[str(w)] = {"pairs": int(pairs[sel].sum()), "padded_cells": cells, "kernel_ms": ms,
                       "gcells_per_s": cells / ms / 1e6 if ms else None, "dpx_floor_ms": floor_ms}
    rep["classes"] = cls
    rep["kernel_ms_total"] = sum(kt.values())
    if args.out:
        with open(args.out, 'w') as f:
            json.dump(rep, f, indent=1)
    print(json.dumps(rep, indent=1))
    db.close()
    models.close()
    eng.close()


if __name__ == '__main__':
    main()
