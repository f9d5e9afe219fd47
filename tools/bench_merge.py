"""`checkm merge` on the device (checkm_b200/csrc/merge.cu): the all-pairs scoring kernel at B bins x |G| markers, its
share of the POPC issue bound, `Merger.run` end to end, and two baselines in pairs/s -- the drop-in loop of
checkm/merger.py:66-106 with three `geneCounts` device calls per pair, and the oracle loop (oracle/merge_oracle.py) on
one core.

    python tools/bench_merge.py [--bins 1000,10000,30000] [--markers 104,1500,5000] [--reps 3] [--popc-rate R]

--popc-rate: POPC warp-instructions per clock per SM as `tools/ubench` (mode 14) measured it on this card; the share of
the issue bound is reported only when it is given.  One JSON line per measurement, each with the card's name, power limit and
maximum SM clock read in the same run."""
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

DEFAULT = (5.0, 10.0, 50.0, 20.0)
PERMISSIVE = (-1e9, 1e9, -1e9, 1e9)


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else 'unknown'


def synthetic(nb, ng, seed=1):
    """Bins as a binning run leaves them: most nearly complete with little contamination, some fragments; a few pairs per
    bin pass the CLI defaults."""
    rng = np.random.default_rng(seed)
    level = np.where(rng.random(nb) < 0.8, rng.uniform(0.85, 1.0, nb), rng.uniform(0.05, 0.5, nb))[:, None]
    counts = (rng.random((nb, ng)) < level).astype(np.int32)
    counts += (rng.random((nb, ng)) < 0.01).astype(np.int32)
    return counts, np.full(nb, ng, dtype=np.int32)


def sm_clock_mhz():
    q = subprocess.run(['nvidia-smi', '--query-gpu=clocks.max.sm', '--format=csv,noheader,nounits'],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return float(q[0]) if q else float('nan')


def device_sizes(eng, args, emit):
    nsm = eng_sm_count()
    mhz = sm_clock_mhz()
    for nb in args.bins:
        for ng in args.markers:
            counts, nm = synthetic(nb, ng)
            pairs_total = nb * (nb - 1) // 2
            w = ((ng + 31) // 32 + 7) // 8 * 8
            for label, thr in (('default', DEFAULT), ('all_pairs', PERMISSIVE)):
                try:
                    eng.merge_pairs(counts, nm, *thr)            # warm-up (module load, allocations)
                    ks, walls = [], []
                    for _ in range(args.reps):
                        t0 = time.perf_counter()
                        pairs, ms = eng.merge_pairs(counts, nm, *thr)
                        walls.append(time.perf_counter() - t0)
                        ks.append(ms)
                except (MemoryError, RuntimeError) as err:
                    emit({'bins': nb, 'markers': ng, 'thresholds': label, 'error': str(err)[:200]})
                    continue
                k = float(np.median(ks))
                rec = {'bins': nb, 'markers': ng, 'thresholds': label, 'pairs_kept': int(len(pairs)), 'kernel_ms': round(k, 3),
                       'call_s': round(float(np.median(walls)), 4), 'pairs_per_s': pairs_total / (k / 1e3)}
                if args.popc_rate:
                    bound_ms = pairs_total * w / 32.0 / (args.popc_rate * nsm * mhz * 1e3)   # warp-POPCs / (rate x SMs x clk)
                    rec['popc_bound_ms'] = round(bound_ms, 3)
                    rec['share_of_popc_bound'] = round(bound_ms / k, 3)
                emit(rec)
                del pairs


def eng_sm_count():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def write_bins(root, nb, seed=3):
    """nb bins as domtblout files over the 43 CPR models: one hit per present marker, each on its own ORF."""
    from checkm_b200.hmmerModelParser import HmmModelParser
    models = HmmModelParser(os.path.join(ROOT, 'tests', 'golden', 'cpr_43_markers.hmm')).models()
    accs = sorted(models)
    counts, _ = synthetic(nb, len(accs), seed)
    ids = ['bin%05d' % b for b in range(nb)]
    for b, binId in enumerate(ids):
        d = os.path.join(root, 'bins', binId)
        os.makedirs(d)
        lines = ['# target name accession ...']
        for g, acc in enumerate(accs):
            m = models[acc]
            thr = (m.nc if ('TIGR' in acc and m.nc) else (m.ga or m.tc or m.nc))[0]
            for c in range(counts[b, g]):
                lines.append('k%d_%d - %d %s %s %d 1e-40 %.1f 0.1 1 1 1e-43 1e-40 %.1f 0.1 1 %d 11 %d 9 %d 0.95 # 1 # 2 # 1 # ID=x'
                             % (c, 10 * g + 1, m.leng + 60, m.name, acc, m.leng, thr + 80.0, thr + 79.0, m.leng, m.leng + 10, m.leng + 12))
        with open(os.path.join(d, 'merger.table.txt'), 'w') as f:
            f.write('\n'.join(lines) + '\n#\n# [ok]\n')
    os.makedirs(os.path.join(root, 'storage'))
    return ids, {b: models for b in ids}


def end_to_end(nb, dropin_bins, emit):
    from checkm_b200.defaultValues import DefaultValues
    from checkm_b200.markerSets import MarkerSetParser
    from checkm_b200.merger import Merger
    from oracle.merge_oracle import merge_pairs as oracle_pairs
    DefaultValues.set_data_root(os.path.join(ROOT, 'tests', 'golden', 'e2e', 'data'))
    root = tempfile.mkdtemp(prefix='bench_merge_')
    try:
        ids, b2m = write_bins(root, nb)
        hmm = os.path.join(ROOT, 'tests', 'golden', 'cpr_43_markers.hmm')
        ms = MarkerSetParser().getMarkerSets(root, ids, hmm)
        for label, thr in (('default', DEFAULT), ('all_pairs', PERMISSIVE)):
            m = Merger()
            t0 = time.perf_counter()
            path = m.run([], root, 'merger.table.txt', b2m, ms, *thr)
            total = time.perf_counter() - t0
            rec = {'e2e_bins': nb, 'thresholds': label, 'total_s': round(total, 4)}
            rec.update({k: (round(v, 4) if isinstance(v, float) else v) for k, v in m.timing.items()})
            # the same pairs by the oracle loop, from the copy numbers the device path used
            from checkm_b200.resultsParser import ResultsParser
            rp = ResultsParser(b2m)
            rp.parseBinHits(root, 'merger.table.txt')
            markers = sorted(ms[ids[0]].mostSpecificMarkerSet().getMarkerGenes())
            cn = {b: {k: len(v) for k, v in rp.results[b].markerHits.items() if k in markers} for b in ids}
            nm = {b: ms[b].mostSpecificMarkerSet().numMarkers() for b in ids}
            t1 = time.perf_counter()
            lines, _ = oracle_pairs(ids, cn, nm, markers, *thr)
            rec['oracle_s'] = round(time.perf_counter() - t1, 3)
            rec['oracle_pairs_per_s'] = nb * (nb - 1) / 2 / rec['oracle_s']
            rec['equal_to_oracle'] = open(path).read().splitlines(keepends=True)[1:] == lines
            emit(rec)
            os.remove(path)
        # today's drop-in loop: merger.py:66-106 with three ResultsManager.geneCounts device calls per pair, on a prefix
        sub = ids[:dropin_bins]
        t2 = time.perf_counter()
        npairs = dropin_loop(sub, rp, ms, *DEFAULT)
        dt = time.perf_counter() - t2
        emit({'dropin_bins': len(sub), 'pairs': npairs, 'dropin_s': round(dt, 3), 'dropin_pairs_per_s': npairs / dt})
    finally:
        shutil.rmtree(root, ignore_errors=True)


def dropin_loop(binIds, rp, ms, minDeltaComp, maxDeltaCont, minMergedComp, maxMergedCont):
    res = rp.results
    n = 0
    for i in range(len(binIds)):
        bi = binIds[i]
        compI, contI = res[bi].geneCounts(ms[bi].mostSpecificMarkerSet(), res[bi].markerHits, True)[6:8]
        for j in range(i + 1, len(binIds)):
            bj = binIds[j]
            compJ, contJ = res[bj].geneCounts(ms[bj].mostSpecificMarkerSet(), res[bj].markerHits, True)[6:8]
            merged = {k: list(v) for k, v in res[bi].markerHits.items()}
            for k, v in res[bj].markerHits.items():
                if k in merged:
                    merged[k].extend(v)
                else:
                    merged[k] = v
            compM, contM = res[bi].geneCounts(ms[bj].mostSpecificMarkerSet(), merged, True)[6:8]
            n += 1
            if not (compM >= minMergedComp and contM < maxMergedCont):
                continue
            _ = (compM - max(compI, compJ), contM - max(contI, contJ))
    return n



def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--bins', default='1000,10000,30000')
    ap.add_argument('--markers', default='104,1500,5000')
    ap.add_argument('--reps', type=int, default=3)
    ap.add_argument('--e2e-bins', type=int, default=1000)
    ap.add_argument('--dropin-bins', type=int, default=150)
    ap.add_argument('--popc-rate', type=float, default=0.0)
    args = ap.parse_args()
    args.bins = [int(x) for x in args.bins.split(',')]
    args.markers = [int(x) for x in args.markers.split(',')]
    from checkm_b200 import runtime
    dev = card()

    def emit(rec):
        rec['card'] = dev
        print(json.dumps(rec), flush=True)
    device_sizes(runtime.engine(), args, emit)
    end_to_end(args.e2e_bins, args.dropin_bins, emit)


if __name__ == '__main__':
    main()
