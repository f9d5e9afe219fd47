"""Generates the `checkm merge` goldens by running the REFERENCE's own Merger (checkm/merger.py, with its ResultsParser,
MarkerSetParser and PFAM code, imported read-only from /root/reference) on domtblout inputs.  Run in the build container
only:

    python tests/golden/make_merge_goldens.py

It writes tests/golden/merge/merge_goldens.json and twosets.ms; tests/test_merge_gpu.py replays them through
checkm_b200.merger.Merger and tests/test_merge_cpu.py through oracle/merge_oracle.py.  The Pfam clan file is the e2e one
(tests/golden/e2e/data).  Cases:

  synth   22 bins over the 43 CPR models, each bin's domtblout kept in the json (`inputs`): complementary halves,
          overlapping ranges, full multi-copy bins, sparse bins, two empty bins and two ids that differ only in case
          (`binQ`, `BinQ`).  Per marker a bin holds one hit, and sometimes a second copy on another contig, a hit split
          over two adjacent ORFs (merged by the reduction), a row below the model's threshold (dropped), or, for a Pfam
          marker with clan mates, a weaker overlapping hit of a clan mate on the same ORF (dropped by the clan filter).
          Marker files: the CPR HMM file, the e2e taxon file and twosets.ms, a taxon file with one marker in two sets.
  e2e_hmm, e2e_taxon   the oracle's domtblout of the three e2e bins, read from tests/golden/e2e/expected.json.
Per case and marker file the json holds the bins in sorted() order, the marker union, numMarkers() per bin, the copy
numbers after the reference's reduction (one row per bin over the union) and merger.tsv per threshold setting
(minDeltaComp, maxDeltaCont, minMergedComp, maxMergedCont): the CLI defaults; a permissive one that writes every pair;
`edge`, whose four values are values the data reaches (so `>=` and `<` are both pinned); and `negative`, which writes
pairs with negative deltas.
"""
import json
import os
import re
import shutil
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
OUT = os.path.join(HERE, 'merge')
sys.path.insert(0, ROOT)
sys.path.insert(0, '/root/reference')
os.environ['CHECKM_DATA_PATH'] = os.path.join(HERE, 'e2e', 'data')

import numpy as np   # noqa: E402

CPR = os.path.join(HERE, 'cpr_43_markers.hmm')
TABLE = 'merger.table.txt'
DEFAULT = (5.0, 10.0, 50.0, 20.0)
PERMISSIVE = (-1e9, 1e9, -1e9, 1e9)
NEGATIVE = (-60.0, 15.0, 0.0, 100.0)
CLAN_MATES = {'PF00276.21': 'PF00281.20', 'PF00281.20': 'PF00276.21', 'PF00380.20': 'PF00411.20',
              'PF00411.20': 'PF00380.20', 'PF01409.21': 'PF13393.7', 'PF01411.20': 'PF01409.21'}


def row(orf, m, acc, score, evalue, hmm, ali):
    return ('%s - %d %s %s %d %.2g %.1f 0.1 1 1 %.2g %.2g %.1f 0.1 %d %d %d %d %d %d 0.95 # 1 # 2 # 1 # ID=x'
            % (orf, m.leng + 60, m.name, acc, m.leng, evalue, score, evalue / 10, evalue, score - 1.0, hmm[0], hmm[1], ali[0], ali[1],
               max(1, ali[0] - 2), ali[1] + 2))


def planted_table(models, markers, seed, copies=0.1):
    """One bin's domtblout over `markers`, rows grouped by query as hmmsearch writes them."""
    rng = np.random.default_rng(seed)
    per_acc = {}
    for n, acc in enumerate(markers):
        m = models[acc]
        thr = (m.nc if ('TIGR' in acc and m.nc) else (m.ga or m.tc or m.nc))[0]
        orf = 1 + 10 * n
        full = (1, m.leng)
        r = rng.random()
        if r < 0.15:                                         # split over two adjacent ORFs: the reduction merges them
            h = m.leng // 2
            per_acc.setdefault(acc, []).append(row('c1_%d' % orf, m, acc, thr + 40, 1e-30, (1, h), (5, h + 4)))
            per_acc[acc].append(row('c1_%d' % (orf + 1), m, acc, thr + 30, 1e-25, (h + 1, m.leng), (3, m.leng - h + 2)))
        else:
            per_acc.setdefault(acc, []).append(row('c1_%d' % orf, m, acc, thr + 60, 1e-40, full, (11, m.leng + 10)))
        if rng.random() < copies:                            # a second copy on another contig
            per_acc[acc].append(row('c2_%d' % orf, m, acc, thr + 50, 1e-35, full, (11, m.leng + 10)))
        if rng.random() < 0.1:                               # below the model's threshold: dropped
            per_acc[acc].append(row('c3_%d' % orf, m, acc, thr - 5, 1e-5, full, (11, m.leng + 10)))
        mate = CLAN_MATES.get(acc)
        if mate and r >= 0.15 and rng.random() < 0.5:        # a weaker clan mate on the same ORF: the clan filter drops it
            mm = models[mate]
            mthr = (mm.ga or mm.tc or mm.nc)[0]
            per_acc.setdefault(mate, []).append(row('c1_%d' % orf, mm, mate, mthr + 30, 1e-20, (1, mm.leng), (12, m.leng)))
    lines = [l for acc in sorted(per_acc) for l in per_acc[acc]]
    return '# target name accession tlen query name accession qlen ...\n' + ''.join(l + '\n' for l in lines) + '#\n# [ok]\n'


def synth_inputs(models):
    accs = sorted(models)
    rng = np.random.default_rng(2024)
    spans = {'half0': (0, 22), 'half1': (22, 43), 'mid': (10, 35), 'head': (0, 12), 'lo30': (0, 30), 'hi30': (13, 43),
             'core': (5, 38), 'binQ': (0, 20), 'BinQ': (20, 43)}
    tables = {b: planted_table(models, accs[lo:hi], 100 + k) for k, (b, (lo, hi)) in enumerate(spans.items())}
    for k in range(4):
        tables['full%d' % k] = planted_table(models, accs, 200 + k, copies=(0.05, 0.2, 0.5, 0.8)[k])
    for k in range(5):
        picks = sorted(rng.choice(43, size=int(rng.integers(4, 30)), replace=False).tolist())
        tables['sparse%d' % k] = planted_table(models, [accs[p] for p in picks], 300 + k, copies=0.3)
    for k in range(2):
        tables['empty%d' % k] = planted_table(models, [], 400 + k)
    return tables


def layout(tables):
    root = tempfile.mkdtemp(prefix='merge_gold_')
    for binId, text in tables.items():
        os.makedirs(os.path.join(root, 'bins', binId))
        with open(os.path.join(root, 'bins', binId, TABLE), 'w') as f:
            f.write(text)
    os.makedirs(os.path.join(root, 'storage'))
    return root


def edge_thresholds(copy_numbers, n_markers, markers):
    """Four thresholds taken from values the pairs reach: the 40th percentile of delta completeness and of merged
    completeness, the 60th of delta contamination and of merged contamination."""
    from oracle.merge_oracle import genome_check
    ids = sorted(copy_numbers)
    mc, mk, dc, dk = [], [], [], []
    for i in range(len(ids)):
        ci, ki = genome_check(markers, n_markers[ids[i]], copy_numbers[ids[i]])
        for j in range(i + 1, len(ids)):
            cj, kj = genome_check(markers, n_markers[ids[j]], copy_numbers[ids[j]])
            merged = dict(copy_numbers[ids[i]])
            for m, c in copy_numbers[ids[j]].items():
                merged[m] = merged.get(m, 0) + c
            c, k = genome_check(markers, n_markers[ids[j]], merged)
            mc.append(c); mk.append(k); dc.append(c - max(ci, cj)); dk.append(k - max(ki, kj))
    pick = lambda v, q: sorted(v)[int(q * (len(v) - 1))]   # noqa: E731
    return [pick(dc, 0.4), pick(dk, 0.6), pick(mc, 0.4), pick(mk, 0.6)]


def main():
    from checkm.hmmerModelParser import HmmModelParser
    from checkm.markerSets import MarkerSetParser
    from checkm.merger import Merger
    from checkm.resultsParser import ResultsParser

    models = HmmModelParser(CPR).models()
    accs = sorted(models)
    os.makedirs(OUT, exist_ok=True)
    sets = [set(accs[0:6]), set(accs[5:14]), set(accs[14:30]), set(accs[30:43])]     # accs[5] is in two sets
    with open(os.path.join(OUT, 'twosets.ms'), 'w') as f:
        f.write('# [Taxon Marker File]\nBacteria\t1\t43\tk__Bacteria\t5449\t%s\n' % str(sets))
    taxon = os.path.join(HERE, 'e2e', 'markers', 'taxon.ms')
    with open(os.path.join(HERE, 'e2e', 'expected.json')) as f:
        e2e = json.load(f)

    synth = synth_inputs(models)
    cases = {'synth': (synth, {b: models for b in synth}, {'hmm': CPR, 'taxon': taxon, 'twosets': os.path.join(OUT, 'twosets.ms')})}
    for mode, mfile in (('hmm', CPR), ('taxon', taxon)):
        tables = {b: ''.join(l + '\n' for l in lines) for b, lines in e2e[mode]['domtblout'].items()}
        cases['e2e_' + mode] = (tables, {b: {a: models[a] for a in e2e[mode]['subset'][b]} for b in tables}, {mode: mfile})

    golden = {'inputs': synth, 'cases': {}}
    for case, (tables, binIdToModels, mfiles) in cases.items():
        cdir = layout(tables)
        binIds = sorted(tables)
        g = {}
        for which, mfile in mfiles.items():
            ms = MarkerSetParser().getMarkerSets(cdir, binIds, mfile)
            rp = ResultsParser(binIdToModels)
            rp.parseBinHits(cdir, TABLE)
            markers = sorted(ms[binIds[0]].mostSpecificMarkerSet().getMarkerGenes())
            cn = {b: {m: len(h) for m, h in rp.results[b].markerHits.items() if m in markers} for b in binIds}
            nm = {b: ms[b].mostSpecificMarkerSet().numMarkers() for b in binIds}
            settings = {'default': list(DEFAULT), 'permissive': list(PERMISSIVE)}
            if case == 'synth':
                settings['edge'] = edge_thresholds(cn, nm, markers)
                settings['negative'] = list(NEGATIVE)
            entry = {'bins': binIds, 'markers': markers, 'n_markers': [nm[b] for b in binIds],
                     'copy_numbers': [[cn[b].get(m, 0) for m in markers] for b in binIds], 'thresholds': settings, 'tsv': {}}
            for label, thr in settings.items():
                path = Merger().run([], cdir, TABLE, binIdToModels, ms, *thr)
                entry['tsv'][label] = open(path).read()
            g[which] = entry
            print(case, which, len(markers), 'markers', {k: v.count('\n') - 1 for k, v in entry['tsv'].items()})
        shutil.rmtree(cdir)
        golden['cases'][case] = g
    text = json.dumps(golden, indent=1, sort_keys=True)
    text = re.sub(r'\[\n\s*([^\[\]{}]*?)\n\s*\]', lambda mt: '[' + ' '.join(mt.group(1).split()) + ']', text)   # flat lists on one line
    with open(os.path.join(OUT, 'merge_goldens.json'), 'w') as f:
        f.write(text + '\n')


if __name__ == '__main__':
    main()
