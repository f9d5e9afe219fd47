"""Strain heterogeneity, host side (checkm/hmmerAligner.py, checkm/aminoAcidIdentity.py).

Expected values come from tests/golden/make_aai_goldens.py (the reference's own extraction steps and strainHetero) and
tests/golden/make_align_goldens.py (the masked FASTA the reference makes of an alignment)."""
import json
import os
import shutil
from collections import defaultdict

import numpy as np
import pytest

from conftest import CPR_HMM, GOLDEN

AAI = os.path.join(GOLDEN, 'aai')
ALI = os.path.join(GOLDEN, 'align')
BIN_IDS = ['strainA', 'strainB', 'strainC']


@pytest.fixture(scope='module')
def expected():
    with open(os.path.join(AAI, 'expected.json')) as f:
        return json.load(f)


class _Hit(object):
    def __init__(self, target_name, full_e_value, full_score):
        self.target_name, self.full_e_value, self.full_score = target_name, full_e_value, full_score


class _Results(object):
    """The part of ResultsParser the extraction steps read: results[binId].markerHits, from the recorded hits."""
    def __init__(self, hits):
        self.results = {}
        for binId, markers in hits.items():
            rm = type('RM', (), {})()
            rm.markerHits = {m: [_Hit(*h) for h in hs] for m, hs in markers}
            self.results[binId] = rm


class _MarkerSets(object):
    def __init__(self, genes):
        self.genes = genes

    def selectedMarkerSet(self):
        return self

    def getMarkerGenes(self):
        return self.genes


def _accs():
    return [l.split()[1] for l in open(CPR_HMM) if l.startswith('ACC ')]


def _dump(markerSeqs):
    return [[m, [[b, [[sid, seq] for sid, seq in seqs.items()]] for b, seqs in bs.items()]] for m, bs in markerSeqs.items()]


@pytest.fixture()
def outdir(tmp_path):
    for b in BIN_IDS:
        os.makedirs(str(tmp_path / 'bins' / b))
        shutil.copyfile(os.path.join(AAI, 'bins', b + '.faa'), str(tmp_path / 'bins' / b / 'genes.faa'))
    return str(tmp_path)


def test_extraction_order(expected, outdir):
    """Sequences per marker in the reference's order: `A&&B` targets concatenated, the final '*' stripped, one sequence
    per target, the multi-copy markers of the selected set, and the top hit = the largest e-value after the sort."""
    from checkm_b200.hmmerAligner import HmmerAligner
    ex = expected['extract']
    HA = HmmerAligner(1)
    genes = set(_accs())
    rp = _Results(ex['hits'])
    for b in BIN_IDS:
        assert _dump(HA._extractMarkersWithMultipleHits(outdir, b, rp, _MarkerSets(genes))) == ex['multi'][b], b
    assert '&&' in json.dumps(ex['multi']['strainA'])
    rp = _Results(ex['hits'])
    seqs, _stats = HA._extractMarkerSeqsUnique(outdir, rp)
    assert _dump(seqs) == ex['unique']
    seqs, stats = HA._extractMarkerSeqsTopHits(outdir, rp)
    assert _dump(seqs) == ex['tophit']
    assert [[m, [[b, [[sid, repr(v[0]), repr(v[1])] for sid, v in s.items()]] for b, s in bs.items()]] for m, bs in stats.items()] \
        == ex['tophit_stats']
    assert {b: [[m, [h.target_name for h in hits]] for m, hits in rp.results[b].markerHits.items()] for b in BIN_IDS} \
        == ex['tophit_sorted']
    assert all(not s.endswith('*') for m, bs in ex['tophit'] for b, ss in bs for _, s in ss)


def test_missing_target_exits(expected, outdir):
    from checkm_b200.hmmerAligner import HmmerAligner
    hits = {b: ex for b, ex in expected['extract']['hits'].items()}
    hits['strainA'] = [[m, [['nosuchorf', 1e-30, 80.0]] + hs] for m, hs in hits['strainA']]
    with pytest.raises(SystemExit) as e:
        HmmerAligner(1)._extractMarkersWithMultipleHits(outdir, 'strainA', _Results(hits), _MarkerSets(set(_accs())))
    assert e.value.code == 1


@pytest.mark.parametrize('acc', ['PF00281.20', 'PF00380.20', 'PF01411.20', 'TIGR01024'])
def test_states_to_masked_rows(acc):
    """States -> masked rows equals the masked FASTA the reference made of the same alignment."""
    from checkm_b200.engine import digitize
    from checkm_b200.hmmerAligner import masked_rows
    names, descs, seqs = [], [], []
    for line in open(os.path.join(ALI, acc + '.unaligned.faa')):
        line = line.rstrip('\n')
        if line.startswith('>'):
            p = line[1:].split(None, 1)
            names.append(p[0])
            descs.append(p[1] if len(p) > 1 else '')
            seqs.append('')
        else:
            seqs[-1] += line
    state = np.load(os.path.join(ALI, acc + '.state.npy'))
    M, cur = None, None
    for line in open(CPR_HMM):
        if line.startswith('ACC '):
            cur = line.split()[1]
        if line.startswith('LENG ') and cur == acc:
            M = int(line.split()[1])
            break
    rows = masked_rows(digitize(''.join(seqs)), state, [len(s) for s in seqs], M)
    text = ''.join(('>%s %s\n' % (n, d) if d else '>%s\n' % n) + r.tobytes().decode() + '\n' for n, d, r in zip(names, descs, rows))
    assert text == open(os.path.join(ALI, acc + '.masked.faa')).read()


def test_strain_hetero_cases(expected):
    from checkm_b200.aminoAcidIdentity import AminoAcidIdentity
    for scores, thr, het, mean in expected['strain_cases']:
        d = defaultdict(dict)
        d.update(scores)
        got_het, got_mean = AminoAcidIdentity().strainHetero(d, thr)
        assert {b: {m: repr(v) for m, v in ms.items()} for b, ms in got_het.items()} == het
        assert {b: repr(v) for b, v in got_mean.items()} == mean


def _write_masked(root, binId, name, text):
    d = os.path.join(root, 'storage', 'aai_qa', binId)
    os.makedirs(d, exist_ok=True)
    with open(os.path.join(d, name), 'w') as f:
        f.write(text)


def test_aai_run_refusals(outdir):
    """Rows of another bin in a bin's file, and rows of unequal width: an error and exit status 1, before any device work."""
    from checkm_b200.aminoAcidIdentity import AminoAcidIdentity
    _write_masked(outdir, 'strainA', 'PF00281.20.masked.faa', '>strainA&&x1\nAC-D\n>strainB&&x2\nACGD\n')
    with pytest.raises(SystemExit) as e:
        AminoAcidIdentity().run(0.9, outdir, None)
    assert e.value.code == 1
    _write_masked(outdir, 'strainA', 'PF00281.20.masked.faa', '>strainA&&x1\nAC-D\n>strainA&&x2\nACGDE\n')
    with pytest.raises(SystemExit) as e:
        AminoAcidIdentity().run(0.9, outdir, None)
    assert e.value.code == 1


def test_aai_run_without_pairs(outdir, tmp_path):
    """Files with one row, and bins without a directory, give no scores and an empty -a file."""
    from checkm_b200.aminoAcidIdentity import AminoAcidIdentity
    _write_masked(outdir, 'strainB', 'PF00281.20.masked.faa', '>strainB&&x1\nAC-D\n')
    aai = AminoAcidIdentity()
    out = str(tmp_path / 'a.txt')
    aai.run(0.9, outdir, out)
    assert dict(aai.aaiRawScores) == {} and aai.aaiMeanBinHetero == {} and open(out).read() == ''
