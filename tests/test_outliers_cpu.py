"""`checkm outliers` without a device: the places where byte identity with the reference is easy to lose, each pinned on
the host.  The order of numpy's sums (which the device reduction follows), ties in findNearest, the profile parser against
float(), the resolution of the distribution tables, the oracle against the outlier files the reference's own BinTools wrote
(tests/golden/outliers/, made by tests/golden/make_outlier_goldens.py), and the host-only methods of BinTools."""
import gzip
import hashlib
import json
import os

import numpy as np
import pytest

from conftest import GOLDEN

OG = os.path.join(GOLDEN, 'outliers')
TETRA = os.path.join(GOLDEN, 'tetra')
OUTDIR = os.path.join(OG, 'out')
PROFILE = None


@pytest.fixture(scope='module', autouse=True)
def profile_file(tmp_path_factory, expected):
    """The fixture's profile file, written from its FASTA files as the golden generator wrote it."""
    from oracle.outliers_oracle import profile_text
    global PROFILE
    PROFILE = str(tmp_path_factory.mktemp('outliers') / 'tetra.tsv')
    with open(PROFILE, 'w') as f:
        f.write(profile_text([os.path.join(OG, 'extra.fna')] + _bin_files(expected)))


@pytest.fixture(scope='module')
def expected():
    with open(os.path.join(OG, 'expected.json')) as f:
        return json.load(f)


def _bits(x):
    return np.float64(x).view(np.uint64)


def _digest(text):
    return {'sha256': hashlib.sha256(text.encode()).hexdigest(), 'ids': [l[1:].split()[0] for l in text.split('\n') if l.startswith('>')]}


def _bin_files(expected):
    return [os.path.join(OG, 'bins', f) for f in expected['bins']]


def test_reduction_order_is_numpys():
    """np.sum / np.mean of a contiguous float64 vector, restated in oracle.outliers_oracle.pairwise_sum, bit for bit on the
    installed numpy: every length 1..2000 and a few of 1e5..1e6, random magnitudes and cancelling values."""
    from oracle.outliers_oracle import pairwise_sum
    rng = np.random.default_rng(11)
    for n in list(range(1, 2001)) + [100000, 100003, 262144, 1000000]:
        x = rng.standard_normal(n) * 10.0 ** rng.integers(-8, 8, n)
        y = rng.standard_normal(n)
        cancelling = np.concatenate([x[:n // 2], -x[:n // 2][::-1], x[2 * (n // 2):]]) if n < 3000 else x
        for v in (x, cancelling):
            lst = v.tolist()
            assert _bits(pairwise_sum(lst)) == _bits(np.sum(v)), n
            assert _bits(pairwise_sum(lst) / n) == _bits(np.mean(v)), n
        d = np.abs(x - y)
        assert _bits(pairwise_sum([abs(a - b) for a, b in zip(x.tolist(), y.tolist())])) == _bits(np.sum(d)), n


def test_distance_of_136_terms_is_two_blocks():
    """The shape the sequence kernel hard-codes: 136 terms are summed as 64 + 72, each block as eight running sums."""
    from oracle.outliers_oracle import pairwise_sum
    rng = np.random.default_rng(5)
    for _ in range(200):
        a = (rng.random(136) * 10.0 ** rng.integers(-6, 0, 136)).tolist()
        halves = []
        for lo, n in ((0, 64), (64, 72)):
            r = [sum_ for sum_ in a[lo:lo + 8]]
            for i in range(8, n, 8):
                for j in range(8):
                    r[j] += a[lo + i + j]
            halves.append(((r[0] + r[1]) + (r[2] + r[3])) + ((r[4] + r[5]) + (r[6] + r[7])))
        assert _bits(halves[0] + halves[1]) == _bits(pairwise_sum(a)) == _bits(np.sum(np.array(a)))


def test_find_nearest_takes_the_first_of_two_equally_near_keys():
    from checkm_b200.common import findNearest
    from oracle.outliers_oracle import find_nearest
    for f in (findNearest, find_nearest):
        assert f([500, 1000, 2000], 750) == 500
        assert f([1000, 500, 2000], 750) == 1000
        assert f([0.25, 0.375, 0.5], 0.3125) == 0.25
        assert f([5.0, 10.0, 2.5], 7.5) == 5.0
        assert f([0.5, 2.5, 5.0, 97.5], (100 - 95) / 2.0) == 2.5          # an int from the command line
        assert f([50, 90, 95, 99], 95) == 95
        assert f([500], 10 ** 9) == 500


def _profile_text(ids, matrix):
    return ('Sequence Id\tcols\n' + ''.join(i + '\t' + '\t'.join(map(str, row)) + '\n' for i, row in zip(ids, matrix))).encode()


def test_profile_parser_gives_what_float_gives():
    from checkm_b200.genomicSignatures import parse_profiles
    rng = np.random.default_rng(7)
    n = 7353                                                                 # x 136: a million values
    m = rng.random((n, 136)) * 10.0 ** rng.integers(-12, 1, (n, 136))
    m[0, :6] = [np.nan, 0.0, 1.0, 1e-05, 0.0001, 2.2250738585072014e-308]
    m[1] = np.nan
    ids = ['contig_%d' % i for i in range(n)]
    ids[5] = 'id with blanks |and| pipes'
    text = _profile_text(ids, m)
    for threads in (1, 4):
        got_ids, got = parse_profiles(text, 136, threads)
        assert got_ids == ids
        want = np.array([[float(x) for x in line.split('\t')[1:]] for line in text.decode().split('\n')[1:-1]])
        assert np.array_equal(got.view(np.uint64), want.view(np.uint64))
    # the last line without a newline, CRLF, inf
    got_ids, got = parse_profiles(b'h\na\t1.5\tinf\r\nb\t-0.0\tnan', 2)
    assert got_ids == ['a', 'b'] and got[0].tolist() == [1.5, np.inf] and np.signbit(got[1, 0]) and np.isnan(got[1, 1])
    assert parse_profiles(b'only a header\n', 136)[1].shape == (0, 136)


@pytest.mark.parametrize('name', ['fixture.fna.tetra.tsv', 'bin1.fna.tetra.tsv', 'bin2.fna.tetra.tsv', 'bin3.fna.tetra.tsv'])
def test_profile_parser_equals_genomic_signatures_read(name):
    from checkm_b200.genomicSignatures import GenomicSignatures, parse_profiles
    path = os.path.join(TETRA, name)
    want = GenomicSignatures(4, 1).read(path)
    with open(path, 'rb') as f:
        ids, got = parse_profiles(f.read())
    assert ids == list(want.keys())
    for i, row in zip(ids, got):
        assert np.array_equal(row.view(np.uint64), want[i].view(np.uint64)), i


@pytest.mark.parametrize('text,line', [(b'', 1), (b'h\na\t1\t2\t3\n', 2), (b'h\na\t1\t2\nb\t1\n', 3), (b'h\na\t1\t2\n\nb\t1\t2\n', 3),
                                       (b'h\na\t1\tx\n', 2), (b'h\na\t1\t0x10\n', 2), (b'h\na\t1\t\n', 2), (b'h\na\t1\t2 3\n', 2),
                                       (b'h\nnotabs\n', 2)])
def test_profile_parser_refuses_malformed_files(text, line):
    from checkm_b200._lib import CkmError
    from checkm_b200.genomicSignatures import parse_profiles
    with pytest.raises(CkmError) as err:
        parse_profiles(text, 2)
    assert err.value.code == 3 and 'line %d' % line in str(err.value)


@pytest.mark.parametrize('report', ['any', 'all'])
@pytest.mark.parametrize('distribution', [90, 95, 99, 85])
def test_oracle_reproduces_the_reference(expected, report, distribution):
    from oracle import outliers_oracle as oo
    got = oo.identify_outliers(OUTDIR, _bin_files(expected), PROFILE, distribution, report, os.path.join(OG, 'data'))
    assert got == expected['outliers']['%s_%d' % (report, distribution)]


def test_goldens_cover_the_edges(expected):
    """The fixture still holds what it was built for: a nan bin, a value on each kind of bound, all-three outliers."""
    rows = {l.split('\t')[1]: l.split('\t') for l in expected['outliers']['any_95'].split('\n')[1:-1]}
    assert rows['n_short'][11] == 'nan' and rows['n_short'][3] == 'CD'
    assert rows['e_gc'][3] == 'TD' and rows['e_gc'][4] == rows['e_gc'][7]          # GC sits on its upper bound: not outlying
    assert rows['e_cd'][3] == 'TD' and rows['e_cd'][8] == rows['e_cd'][10]         # CD sits on its lower bound
    assert 'e_td' not in rows
    assert rows['p_odd'][3] == 'GC,CD,TD'
    assert expected['helpers']['b7_tie']['meanGC'] == 0.3125


@pytest.mark.parametrize('distribution', [90, 95, 99, 85])
def test_bound_tables_resolve_as_the_reference_indexes_them(expected, monkeypatch, distribution):
    """The lists the device call takes -- per bin the (length key, lower, upper) entries of the table its means select --
    give every sequence the bounds binTools.py:250-276 look up."""
    from checkm_b200.binTools import _BoundTables
    from checkm_b200.common import readDistribution
    from checkm_b200.defaultValues import DefaultValues
    from oracle import outliers_oracle as oo
    monkeypatch.setattr(DefaultValues, 'DISTRIBUTION_DIR', os.path.join(OG, 'data', 'distributions'))
    dists = [readDistribution(p) for p in ('gc_dist', 'cd_dist', 'td_dist')]
    tables = _BoundTables(*dists, distribution)
    from oracle.binstats_oracle import coding_bases
    for path in _bin_files(expected):
        seqs = oo.read_fasta(path)
        h = {'meanGC': oo.gc_dist(seqs)[0],
             'meanCD': oo.cd_dist(seqs, coding_bases(os.path.join(OUTDIR, 'bins', oo.bin_id(path), 'genes.gff'))[1])[0]}
        lens = [len(s) for s in seqs.values()]
        want = oo.bounds(dists, h['meanGC'], h['meanCD'], distribution, lens)
        g, c = tables.gc_table(h['meanGC']), tables.cd_table(h['meanCD'])
        off, key, lo, hi = tables.arrays()

        def nearest(t, n):
            return int(off[t]) + int(np.argmin(np.abs(key[off[t]:off[t + 1]] - n)))
        got = [(lo[nearest(g, n)], hi[nearest(g, n)], lo[nearest(c, n)], hi[nearest(tables.td_table, n)]) for n in lens]
        assert got == [tuple(float(v) for v in w) for w in want]


def test_remove_outliers_modify_and_unique(expected, tmp_path, capsys):
    from checkm_b200.binTools import BinTools
    bt = BinTools()
    outliers = str(tmp_path / 'outliers.tsv')
    with open(outliers, 'w') as f:
        f.write(expected['outliers']['any_95'])
    for name, want in expected['removeOutliers'].items():
        out = str(tmp_path / 'cleaned.fna')
        bt.removeOutliers(os.path.join(OG, 'bins', name), outliers, out)
        assert _digest(open(out).read()) == want, name
    m = expected['modify']
    out = str(tmp_path / 'modified.fna.gz')
    bt.modify(os.path.join(OG, 'bins', 'b1_plain.fna'), os.path.join(OG, 'bins', 'b5_gz.fna.gz'), m['add'], m['remove'], out)
    assert _digest(gzip.open(out, 'rt').read()) == {'ids': m['ids'], 'sha256': m['sha256']}
    capsys.readouterr()
    bt.unique(_bin_files(expected))
    assert capsys.readouterr().out == expected['unique_all']
    bt.unique(_bin_files(expected)[1:4])
    assert capsys.readouterr().out == expected['unique_none']


def test_removing_a_sequence_the_bin_does_not_hold_exits(tmp_path):
    from checkm_b200.binTools import BinTools
    with pytest.raises(SystemExit) as err:
        BinTools().modify(os.path.join(OG, 'bins', 'b2_one.fna'), None, None, ['absent'], str(tmp_path / 'x.fna'))
    assert err.value.code == 1
