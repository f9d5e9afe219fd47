"""Goldens for strain heterogeneity (HmmerAligner + AminoAcidIdentity): run in the build container only (imports the
reference read-only).

    python tests/golden/make_aai_goldens.py

Fixture (tests/golden/aai/): three protein bins with Prodigal-style headers.  Copies of chosen CPR markers are planted
at controlled identity to a first copy (about 99 %, 93 %, 88 % and 60 %), one marker of `strainA` has a copy split over
two adjacent ORFs (an `A&&B` hit after the adjacent-ORF merge), one copy of `strainB` is cut at both ends (its alignment
starts and ends in gaps), and `strainC` has no multi-copy marker.  Each bin is searched against cpr_43_markers.hmm by the
oracle (bins/<id>.hmmer.analyze.txt).

expected.json holds what the REFERENCE's own code makes of them, with `checkm.hmmer.HMMERRunner` replaced inside
checkm.hmmerAligner by an oracle-backed hmmfetch / hmmalign (oracle.pyoracle.align, formatted as hmmalign's Pfam output,
as make_align_goldens.py does):
  * the files HmmerAligner.makeAlignmentsOfMultipleHits, makeAlignmentTopHit (with bKeepUnmaskedAlign) and
    makeAlignmentToPhyloMarkers leave behind;
  * the marker sequences each extraction step collects, and the hit order the top-hit sort leaves;
  * AminoAcidIdentity.run at --aai_strain 0.9 and 0.95: the -a file, aaiRawScores / aaiHetero / aaiMeanBinHetero as float
    reprs, and QA tables 1-3 (plain and tab) from ResultsParser.printSummary with that aai;
  * aai() on the string vectors of checkm/test/test_aminoAcidIdentity.py and on edge rows, and strainHetero on that
    file's cases.
Directory listings are taken in sorted order while the reference runs (the tests do the same), so the order of bins and
files does not depend on the file system."""
import io
import json
import os
import shutil
import sys
import tempfile
from collections import defaultdict
from contextlib import redirect_stdout

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
OUT = os.path.join(HERE, 'aai')
CPR = os.path.join(HERE, 'cpr_43_markers.hmm')
sys.path.insert(0, ROOT)
sys.path.insert(0, '/root/reference')
os.environ.setdefault('CHECKM_DATA_PATH', os.path.join(HERE, 'reduction', 'data'))

import numpy as np  # noqa: E402

L = "ACDEFGHIKLMNPQRSTVWY-BJZOUX*~"
BIN_IDS = ['strainA', 'strainB', 'strainC']
BIN_STATS = ("{'GC': %r, 'GC std': 0.0213, 'Genome size': %d, '# ambiguous bases': 0, '# scaffolds': 4, '# contigs': 4, "
             "'Longest scaffold': 90000, 'Longest contig': 90000, 'N50 (scaffolds)': 60000, 'N50 (contigs)': 60000, "
             "'Mean scaffold length': 45000.5, 'Mean contig length': 45000.5, 'Coding density': 0.8812, 'Translation table': 11, "
             "'# predicted genes': %d}")
THRESHOLDS = ('0.9', '0.95')

AAI_VECTORS = [('ACGT', 'ACGT'), ('ACGT', 'TGCA'), ('ACGT----', '----TGCA'), ('ACGT--', '--GTAC'), ('AAAACGTTTT', '---ACGG---'),
               ('ACGT', 'ACGG'), ('A-C-G-T', 'A-C-G-T'), ('A-C-G-T', 'AACCGGT'),
               ('-----', '-----'), ('-ACGT', 'AACGT'), ('-ACGT', '-ACGA'), ('A', 'A'), ('A', 'C'), ('-', 'A'), ('', ''),
               ('AC--GT', 'AC--GA'), ('A--C-T', 'A--C-T'), ('AXXC', 'AXXC'), ('XAX', 'XCX'), ('A-', 'A-'), ('A-', 'AC'),
               ('-A', 'CA'), ('A' * 700 + '-' * 30, 'A' * 600 + 'C' * 100 + '-' * 30), ('-' * 513 + 'AC', 'C' * 514 + 'C')]
STRAIN_CASES = [({'b1': {'g1': [0.1], 'g2': [0.1], 'g3': [0.1]}}, 0.9),
                ({'b1': {'g1': [0.95], 'g2': [0.95], 'g3': [0.95]}}, 0.9),
                ({'b1': {'g1': [0.95], 'g2': [0.1], 'g3': [0.1]}}, 0.9),
                ({'b1': {'g1': [0.95, 0.95, 0.95], 'g2': [0.1, 0.1, 0.1], 'g3': [0.95, 0.1, 0.1]}}, 0.9),
                ({'b1': {'g1': [0.9, 0.95]}, 'b2': {'g2': [0.5]}}, 0.9)]


def build_bins(hm, accs):
    """Marker ORFs planted among background ORFs; returns {binId: (names, descs, seqs)}, seqs as code arrays ending in '*'."""
    from tools import synth
    rng = np.random.default_rng(4242)
    bg = lambda n: rng.choice(20, size=n, p=synth.BG).astype(np.uint8)          # noqa: E731

    def mutate(s, f):
        t = s.copy()
        m = rng.random(len(t)) < f
        t[m] = (t[m] + rng.integers(1, 20, size=int(m.sum()))) % 20
        return t

    def homolog(mi):
        return synth.emit_homolog(hm[mi], rng, sharpen=0.6)

    plan = {}
    a1, a3, a10, a5 = homolog(1), homolog(3), homolog(10), homolog(5)
    cut = len(a5) // 2
    plan['strainA'] = [('full', a1), ('full', mutate(a1, 0.01)), ('full', a3), ('full', mutate(a3, 0.07)),
                       ('full', a10), ('full', mutate(a10, 0.12)), ('full', mutate(a10, 0.40)), ('full', homolog(27)),
                       ('split', (a5[:cut], a5[cut:])), ('full', mutate(a5, 0.05))]
    b1, b3 = homolog(1), homolog(3)
    k = len(b1) // 10
    plan['strainB'] = [('full', b1), ('bare', mutate(b1[k:len(b1) - k], 0.03)), ('full', b3), ('full', mutate(b3, 0.05)),
                       ('full', homolog(12))]
    plan['strainC'] = [('full', homolog(1)), ('full', homolog(3)), ('full', homolog(20))]
    bins = {}
    for binId, items in plan.items():
        orfs = [bg(int(rng.integers(80, 400))) for _ in range(24)]
        slot = 1
        for kind, s in items:
            if kind == 'split':
                orfs.insert(slot, np.concatenate([bg(12), s[0], bg(6)]))
                orfs.insert(slot + 1, np.concatenate([bg(5), s[1], bg(15)]))
                slot += 4
            elif kind == 'bare':
                orfs.insert(slot, s)
                slot += 3
            else:
                orfs.insert(slot, np.concatenate([bg(int(rng.integers(3, 40))), s, bg(int(rng.integers(3, 40)))]))
                slot += 3
        names, descs, seqs = [], [], []
        pos = 1
        for i, s in enumerate(orfs):
            contig, n = i // 12 + 1, i % 12 + 1
            if n == 1:
                pos = 1
            nt = 3 * (len(s) + 1)
            names.append('%s_c%d_%d' % (binId[-1], contig, n))
            descs.append('# %d # %d # %d # ID=%d_%d;partial=00;start_type=ATG;rbs_motif=None;rbs_spacer=None;gc_cont=0.480'
                         % (pos, pos + nt - 1, 1 if i % 3 else -1, contig, n))
            pos += nt + 37
            seqs.append(np.concatenate([s, [27]]).astype(np.uint8))
        bins[binId] = (names, descs, seqs)
    return bins


class _SortedListdir(object):
    def __enter__(self):
        self.saved = os.listdir
        os.listdir = lambda p='.': sorted(self.saved(p))

    def __exit__(self, *a):
        os.listdir = self.saved


def tree(root):
    out = {}
    for d, _, files in os.walk(root):
        for f in files:
            p = os.path.join(d, f)
            out[os.path.relpath(p, root)] = open(p).read()
    return out


def main():
    from oracle import pyoracle as po
    from tools import synth
    from checkm_b200.hmmer import format_alignment
    import checkm.hmmerAligner as ref_ha
    from checkm.aminoAcidIdentity import AminoAcidIdentity
    from checkm.hmmerModelParser import HmmModelParser
    from checkm.markerSets import MarkerSetParser
    from checkm.resultsParser import ResultsParser
    from checkm.defaultValues import DefaultValues

    hf = po.HmmFile(CPR)
    accs = hf.accs()
    hm = synth.read_hmms(CPR)

    class OracleRunner(object):
        """hmmfetch writes the key; hmmalign aligns every sequence with the oracle and writes hmmalign's Pfam format."""
        def __init__(self, mode='dom'):
            self.mode = mode

        def fetch(self, db, key, fetchFileName, bKeyFile=False):
            with open(fetchFileName, 'w') as f:
                f.write(key)

        def align(self, db, query, outputFile, writeMode='>', outputFormat='Pfam', trim=False):
            m = accs.index(open(db).read())
            names, descs, seqs = [], [], []
            for line in open(query):
                line = line.rstrip('\n')
                if line.startswith('>'):
                    parts = line[1:].split(None, 1)
                    names.append(parts[0])
                    descs.append(parts[1] if len(parts) > 1 else '')
                    seqs.append('')
                else:
                    seqs[-1] += line
            codes = [np.array([L.index(c) if c in L else 26 for c in s.upper()], dtype=np.uint8) for s in seqs]
            off = np.zeros(len(codes) + 1, dtype=np.int64)
            off[1:] = np.cumsum([len(c) for c in codes])
            state = np.concatenate([po.align(hf, m, c)[0] if len(c) else np.zeros(0, np.int32) for c in codes])
            with open(outputFile, 'w') as f:
                f.write(format_alignment(names, descs, np.concatenate(codes), off, state, hm[m].M, outputFormat, trim))

    ref_ha.HMMERRunner = OracleRunner

    shutil.rmtree(OUT, ignore_errors=True)
    os.makedirs(os.path.join(OUT, 'bins'))
    bins = build_bins(hm, accs)
    work = tempfile.mkdtemp(prefix='aai_gold_')
    out = os.path.join(work, 'out')
    os.makedirs(os.path.join(out, 'storage', 'aai_qa'))
    for binId in BIN_IDS:
        names, descs, seqs = bins[binId]
        text = ''.join('>%s %s\n%s\n' % (n, d, ''.join(L[c] for c in s)) for n, d, s in zip(names, descs, seqs))
        with open(os.path.join(OUT, 'bins', binId + '.faa'), 'w') as f:
            f.write(text)
        bdir = os.path.join(out, 'bins', binId)
        os.makedirs(bdir)
        shutil.copyfile(os.path.join(OUT, 'bins', binId + '.faa'), os.path.join(bdir, 'genes.faa'))
        res = np.concatenate(seqs)
        offs = np.zeros(len(seqs) + 1, dtype=np.int64)
        offs[1:] = np.cumsum([len(s) for s in seqs])
        rp = po.search(hf, res, offs, nthreads=8)
        table = os.path.join(bdir, 'hmmer.analyze.txt')
        po.write_domtblout(rp, hf, names, descs, table)
        po.free_results(rp)
        shutil.copyfile(table, os.path.join(OUT, 'bins', binId + '.hmmer.analyze.txt'))
    stats_lines = [binId + '\t' + BIN_STATS % (0.45 + 0.03 * i, 150000 + 999 * i, len(bins[binId][2])) for i, binId in enumerate(BIN_IDS)]
    with open(os.path.join(out, 'storage', 'bin_stats.analyze.tsv'), 'w') as f:
        f.write(''.join(l + '\n' for l in stats_lines))

    exp = {'bin_stats': stats_lines}
    models = HmmModelParser(CPR).models()
    binIdToModels = {b: models for b in BIN_IDS}
    bms = MarkerSetParser().getMarkerSets(out, BIN_IDS, CPR)
    HA = ref_ha.HmmerAligner(2)

    # ---- the extraction steps on the reference's reduced hits ----
    RP = ResultsParser(binIdToModels)
    RP.parseBinHits(out, 'hmmer.analyze.txt', False, False, DefaultValues.E_VAL, DefaultValues.LENGTH)
    hits_in = {b: [[m, [[h.target_name, h.full_e_value, h.full_score] for h in hits]] for m, hits in RP.results[b].markerHits.items()]
               for b in BIN_IDS}

    def dump(markerSeqs):
        return [[m, [[b, [[sid, seq] for sid, seq in seqs.items()]] for b, seqs in bs.items()]] for m, bs in markerSeqs.items()]
    multi = {b: dump(HA._extractMarkersWithMultipleHits(out, b, RP, bms[b])) for b in BIN_IDS}
    RP = ResultsParser(binIdToModels)
    RP.parseBinHits(out, 'hmmer.analyze.txt', False, False, DefaultValues.E_VAL, DefaultValues.LENGTH)
    unique_seqs, unique_stats = HA._extractMarkerSeqsUnique(out, RP)
    top_seqs, top_stats = HA._extractMarkerSeqsTopHits(out, RP)
    exp['extract'] = {'hits': hits_in, 'multi': multi, 'unique': dump(unique_seqs), 'tophit': dump(top_seqs),
                      'tophit_stats': [[m, [[b, [[sid, repr(v[0]), repr(v[1])] for sid, v in s.items()]] for b, s in bs.items()]] for m, bs in top_stats.items()],
                      'tophit_sorted': {b: [[m, [h.target_name for h in hits]] for m, hits in RP.results[b].markerHits.items()] for b in BIN_IDS}}

    # ---- the three methods ----
    with _SortedListdir():
        HA.makeAlignmentsOfMultipleHits(out, CPR, 'hmmer.analyze.txt', binIdToModels, bms, False, DefaultValues.E_VAL,
                                        DefaultValues.LENGTH, os.path.join(out, 'storage', 'aai_qa'))
        exp['multi_files'] = tree(os.path.join(out, 'storage', 'aai_qa'))
        top = os.path.join(work, 'tophit')
        HA.makeAlignmentTopHit(out, CPR, 'hmmer.analyze.txt', binIdToModels, False, DefaultValues.E_VAL, DefaultValues.LENGTH,
                               True, top, True)
        exp['tophit_files'] = tree(top)
        phy = os.path.join(work, 'phylo')
        HA.makeAlignmentToPhyloMarkers(out, CPR, 'hmmer.analyze.txt', binIdToModels, False, DefaultValues.E_VAL,
                                       DefaultValues.LENGTH, True, phy)
        exp['phylo_files'] = tree(phy)

        # ---- AAI and the QA tables ----
        exp['aai'] = {}
        RP = ResultsParser(binIdToModels)
        RP.analyseResults(out, 'bin_stats.analyze.tsv', 'hmmer.analyze.txt')
        for thr in THRESHOLDS:
            aai = AminoAcidIdentity()
            afile = os.path.join(work, 'aai_%s.txt' % thr)
            aai.run(float(thr), out, afile)
            e = {'alignment_file': open(afile).read(),
                 'raw': {b: {m: [repr(v) for v in vs] for m, vs in ms.items()} for b, ms in aai.aaiRawScores.items()},
                 'hetero': {b: {m: repr(v) for m, v in ms.items()} for b, ms in aai.aaiHetero.items()},
                 'mean': {b: repr(v) for b, v in aai.aaiMeanBinHetero.items()}, 'tables': {}}
            for fmt in (1, 2, 3):
                for tab in (True, False):
                    buf = io.StringIO()
                    with redirect_stdout(buf):
                        RP.printSummary(fmt, aai, bms, False, None, tab, '', out)
                    e['tables']['%d%s' % (fmt, 't' if tab else 'p')] = buf.getvalue()
            exp['aai'][thr] = e

    one = AminoAcidIdentity()
    exp['aai_vectors'] = [[a, b, repr(one.aai(a, b))] for a, b in AAI_VECTORS]
    cases = []
    for scores, thr in STRAIN_CASES:
        d = defaultdict(dict)
        d.update(scores)
        het, mean = one.strainHetero(d, thr)
        cases.append([scores, thr, {b: {m: repr(v) for m, v in ms.items()} for b, ms in het.items()}, {b: repr(v) for b, v in mean.items()}])
    exp['strain_cases'] = cases
    with open(os.path.join(OUT, 'expected.json'), 'w') as f:
        json.dump(exp, f, indent=0, sort_keys=True)
    shutil.rmtree(work)
    print({thr: exp['aai'][thr]['mean'] for thr in THRESHOLDS})
    print({thr: exp['aai'][thr]['raw'] for thr in THRESHOLDS[:1]})
    print(sorted(exp['multi_files']), len(exp['tophit_files']), len(exp['phylo_files']))


if __name__ == '__main__':
    main()
