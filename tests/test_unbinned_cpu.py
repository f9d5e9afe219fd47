"""`checkm unbinned` and `checkm profile`, CPU side: the oracle port and Profile against the files the reference's own
Unbinned.run and Profile.run wrote (tests/golden/unbinned/, made by tests/golden/make_unbinned_goldens.py), the library's
host formatter against Python's '%.2f', and Profile's refusals."""
import glob
import gzip
import json
import logging
import os

import numpy as np
import pytest

from conftest import GOLDEN

UB = os.path.join(GOLDEN, 'unbinned')
INPUTS = os.path.join(UB, 'inputs')
EXPECTED = os.path.join(UB, 'expected')


def _raw(path):
    with (gzip.open if path.endswith('.gz') else open)(path, 'rb') as f:
        return f.read()


def _expected(name):
    with open(os.path.join(EXPECTED, name), 'rb') as f:
        return f.read()


def _cases():
    with open(os.path.join(UB, 'cases.json')) as f:
        return json.load(f)


def _profile_inputs():
    paths = sorted(glob.glob(os.path.join(INPUTS, 'cov_*.tsv')))
    paths += [os.path.join(GOLDEN, 'coverage', 'coverage_%s.tsv' % o) for o in ('all_reads', 'defaults', 'loose', 'strict')]
    return paths


@pytest.mark.parametrize('case', sorted(_cases()))
def test_oracle_matches_reference(case):
    from oracle import unbinned_oracle
    c = _cases()[case]
    fasta, stats, info = unbinned_oracle.run([_raw(os.path.join(INPUTS, b)) for b in c['bins']],
                                             _raw(os.path.join(INPUTS, c['seqFile'])), c['minSeqLen'])
    assert fasta == _expected('unbinned_%s.fna' % case)
    assert stats == _expected('unbinned_%s.tsv' % case)
    assert info == c['info']


@pytest.mark.parametrize('style', ['tab', 'table'])
@pytest.mark.parametrize('path', _profile_inputs(), ids=lambda p: os.path.basename(p)[:-4])
def test_profile_matches_reference(path, style, tmp_path):
    from checkm_b200.profile import Profile
    out = str(tmp_path / 'profile.txt')
    Profile().run(path, out, style == 'tab')
    with open(out, 'rb') as f:
        assert f.read() == _expected('profile_%s_%s.txt' % (os.path.basename(path)[:-4], style))


def test_profile_to_stdout(capsys):
    from checkm_b200.profile import Profile
    path = os.path.join(INPUTS, 'cov_three_bams.tsv')
    Profile().run(path, '', True)
    assert capsys.readouterr().out.encode() == _expected('profile_cov_three_bams_tab.txt')


@pytest.mark.parametrize('text,needle', [
    ('', 'No sequences'),
    ('Sequence Id\tBin Id\tSequence length (bp)\tBam Id\tCoverage\tMapped reads\n', 'No sequences'),
    ('h\na\tbin1\t100\ts1\t0.0\t0\nb\tunbinned\t10\ts1\t0.0\t0\n', 's1'),
    ('h\na\tbin1\t0\ts1\t0.0\t4\n', 'bin1'),
])
def test_profile_refusals(text, needle, tmp_path, caplog):
    from checkm_b200.profile import Profile
    path = str(tmp_path / 'coverage.tsv')
    with open(path, 'w') as f:
        f.write(text)
    with caplog.at_level(logging.ERROR, logger='timestamp'), pytest.raises(SystemExit) as e:
        Profile().run(path, str(tmp_path / 'out.txt'), True)
    assert e.value.code == 1
    assert needle in caplog.text and path in caplog.text


def _format_gc(gc, total):
    """The stats rows the library writes for (g + c, a + c + g + t) pairs, one empty id each."""
    from checkm_b200.unbinned import format_records
    n = len(gc)
    acgt = np.zeros((n, 4), dtype=np.int64)
    acgt[:, 1] = gc
    acgt[:, 0] = total - gc
    zeros = np.zeros(n, dtype=np.int64)
    _, stats = format_records(b'', zeros, zeros, np.zeros(0, dtype=np.uint8), zeros, zeros, acgt)
    return stats.decode().splitlines()


def test_formatter_prints_as_python_for_every_small_ratio():
    """Every (g + c, total) with 0 <= g + c <= total <= 2000."""
    total = np.concatenate([np.full(t + 1, t, dtype=np.int64) for t in range(1, 2001)])
    gc = np.concatenate([np.arange(t + 1, dtype=np.int64) for t in range(1, 2001)])
    got = _format_gc(gc, total)
    want = ['\t0\t%.2f' % (float(g) * 100 / t) for g, t in zip(gc.tolist(), total.tolist())]
    assert got == want


def test_formatter_prints_as_python_on_random_ratios():
    rng = np.random.default_rng(11)
    total = rng.integers(1, 1 << 40, size=1_000_000, dtype=np.int64)
    gc = (rng.random(1_000_000) * (total + 1)).astype(np.int64).clip(0, total)
    got = _format_gc(gc, total)
    want = ['\t0\t%.2f' % (float(g) * 100 / t) for g, t in zip(gc.tolist(), total.tolist())]
    assert got == want


def test_formatter_writes_ids_sequences_and_lengths():
    from checkm_b200.unbinned import format_records
    text = b'x c\xc3\xa9 y\n'
    data = np.frombuffer(b'ACGTN' + b'\0' * 59 + b'ac gu' + b'\0' * 59, dtype=np.uint8)
    fasta, stats = format_records(text, [2, 0], [3, 1], data, [0, 64], [5, 5], [[1, 1, 1, 1], [1, 1, 1, 1]])
    assert fasta == b'>c\xc3\xa9\nACGTN\n>x\nac gu\n'
    assert stats == b'c\xc3\xa9\t5\t50.00\nx\t5\t50.00\n'


def test_formatter_refuses_a_sequence_without_bases():
    from checkm_b200 import _lib
    from checkm_b200.unbinned import format_records
    with pytest.raises(_lib.CkmError):
        format_records(b'x', [0], [1], np.zeros(64, dtype=np.uint8), [0], [3], [[0, 0, 0, 0]])
