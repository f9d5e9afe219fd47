"""`checkm unbinned` on the device (checkm_b200.unbinned.Unbinned over ckm_id_join, csrc/idjoin.cu, and the scaffold scan):
both output files byte for byte and the INFO lines against the reference's own Unbinned.run (tests/golden/unbinned/,
made by tests/golden/make_unbinned_goldens.py), also with the base counts split into many device calls; every refusal;
the join against a Python dict/set restatement on about 10^6 records and on ids built to collide; and the community
profile workflow unbinned -> coverage -> profile against the oracles."""
import gzip
import json
import logging
import os

import numpy as np
import pytest

from conftest import GOLDEN

pytestmark = pytest.mark.gpu
UB = os.path.join(GOLDEN, 'unbinned')
INPUTS = os.path.join(UB, 'inputs')
EXPECTED = os.path.join(UB, 'expected')

# every str.isspace() character, and non-space characters whose UTF-8 shares lead bytes with them
WHITESPACE = [chr(c) for c in (0x9, 0xa, 0xb, 0xc, 0xd, 0x1c, 0x1d, 0x1e, 0x1f, 0x20, 0x85, 0xa0, 0x1680, 0x2000, 0x2001,
                               0x2002, 0x2003, 0x2004, 0x2005, 0x2006, 0x2007, 0x2008, 0x2009, 0x200a, 0x2028, 0x2029,
                               0x202f, 0x205f, 0x3000)]
HEADER_SPACE = [w for w in WHITESPACE if w not in '\n\r']          # a header line cannot hold a line end
NEAR_MISSES = ['\x84', '\xa1', '\x86', 'ᚁ', 'ᙿ', '​', '‧', '‪', '‮', '‰', '⁞',
               '⁠', '、', '⿿', '\xe9', '€', '\xdf', '\U0001f600']
ID_CHARS = list('ACGTacgtxyz_.|:0123456789') + NEAR_MISSES


def _cases():
    with open(os.path.join(UB, 'cases.json')) as f:
        return json.load(f)


def _read(path):
    with open(path, 'rb') as f:
        return f.read()


def _raw(path):
    with (gzip.open if path.endswith('.gz') else open)(path, 'rb') as f:
        return f.read()


def _run(tmp_path, bins, seq, min_len, caplog=None):
    from checkm_b200.unbinned import Unbinned
    fna, tsv = str(tmp_path / 'unbinned.fna'), str(tmp_path / 'unbinned.tsv')
    u = Unbinned()
    if caplog is None:
        u.run(bins, seq, fna, tsv, min_len)
    else:
        with caplog.at_level(logging.INFO, logger='timestamp'):
            u.run(bins, seq, fna, tsv, min_len)
    return _read(fna), _read(tsv), u


@pytest.mark.parametrize('case', sorted(_cases()))
def test_files_and_log_equal_the_reference(case, tmp_path, caplog):
    c = _cases()[case]
    fasta, stats, _ = _run(tmp_path, [os.path.join(INPUTS, b) for b in c['bins']], os.path.join(INPUTS, c['seqFile']),
                           c['minSeqLen'], caplog)
    assert fasta == _read(os.path.join(EXPECTED, 'unbinned_%s.fna' % case))
    assert stats == _read(os.path.join(EXPECTED, 'unbinned_%s.tsv' % case))
    assert [r.getMessage() for r in caplog.records if r.name == 'timestamp'] == c['info']


@pytest.mark.parametrize('case', ['base', 'gzip'])
def test_small_device_batches(case, tmp_path, monkeypatch):
    from checkm_b200 import unbinned
    monkeypatch.setattr(unbinned, 'BATCH_BYTES', 100)
    c = _cases()[case]
    fasta, stats, u = _run(tmp_path, [os.path.join(INPUTS, b) for b in c['bins']], os.path.join(INPUTS, c['seqFile']),
                           c['minSeqLen'])
    assert fasta == _read(os.path.join(EXPECTED, 'unbinned_%s.fna' % case))
    assert stats == _read(os.path.join(EXPECTED, 'unbinned_%s.tsv' % case))
    assert u.timing['count_calls'] >= 3


BIN_OK = b'>b1\nACGT\n'
REFUSALS = [
    # (assembly bytes, bin bytes, minSeqLen, which file or sequence the message names)
    (b'>a\nACGT\n>n\nNNNN\n', BIN_OK, 0, 'n'),                     # a kept sequence without A/C/G/T/U
    (b'>a\nACGT\n>e\n>b1\nAC\n', BIN_OK, 0, 'e'),                  # an empty kept sequence at the default minSeqLen
    (b'', BIN_OK, 0, 'asm'),                                       # no records
    (b'\n\n  \n', BIN_OK, 0, 'asm'),                               # blank lines only: no records
    (b'>b1\n\n', BIN_OK, 0, 'asm'),                                # no bases
    (b'>a\nAC\xff\xfeGT\n', BIN_OK, 0, 'asm'),                      # not UTF-8
    (b'ACGT\n>a\nACGT\n', BIN_OK, 0, 'asm'),                       # sequence before the first header
    (b'>a\nACGT\n> \t\nACGT\n', BIN_OK, 0, 'asm'),                 # a header without an id
    (b'>a\nACGT\n>\xe3\x80\x80\nACGT\n', BIN_OK, 0, 'asm'),         # ... whose only character is U+3000
    (b'>a\nACGT\n', b'>b1\nAC\n>\nGT\n', 0, 'bin'),                # a bin's header without an id
    (b'>a\nACGT\n', b'\xc3\x28', 0, 'bin'),                        # a bin that is not UTF-8
    (b'>a\nAC\xc3\xa9GT\n', BIN_OK, 0, 'asm'),                      # non-ASCII in a sequence line
]


@pytest.mark.parametrize('asm,bin_,min_len,named', REFUSALS)
def test_refusals(asm, bin_, min_len, named, tmp_path, caplog):
    paths = {'asm': str(tmp_path / 'asm.fna'), 'bin': str(tmp_path / 'bin.fna')}
    with open(paths['asm'], 'wb') as f:
        f.write(asm)
    with open(paths['bin'], 'wb') as f:
        f.write(bin_)
    with caplog.at_level(logging.INFO, logger='timestamp'), pytest.raises(SystemExit) as e:
        _run(tmp_path, [paths['bin']], paths['asm'], min_len)
    assert e.value.code == 1
    errors = ' '.join(r.getMessage() for r in caplog.records if r.levelno >= logging.ERROR)
    assert (paths[named] if named in paths else 'Sequence %s ' % named) in errors


def _python_join(bin_headers, asm_headers):
    """The reference's dicts restated: per assembly record (binned, first of its id, last record of its id), per bin record
    whether it is the last of its id in its file, and the number of binned ids."""
    binned, keep = set(), []
    for headers in bin_headers:
        ids = [h.split(None, 1)[0] for h in headers]
        last = {i: r for r, i in enumerate(ids)}
        keep += [last[i] == r for r, i in enumerate(ids)]
        binned.update(ids)
    ids = [h.split(None, 1)[0] for h in asm_headers]
    first, last = {}, {}
    for r, i in enumerate(ids):
        first.setdefault(i, r)
        last[i] = r
    flags = [(1 if i in binned else 0) | (2 if first[i] == r else 0) for r, i in enumerate(ids)]
    return np.array(flags, dtype=np.uint8), np.array([last[i] for i in ids], dtype=np.int64), np.array(keep, bool), len(binned)


def _check_join(engine, bin_headers, asm_headers):
    text = b''.join(h.encode() + b'\n' for hs in bin_headers for h in hs) + b''.join(h.encode() + b'\n' for h in asm_headers)
    id_start, id_len, flags, last, keep, nbinned, ms = engine.id_join(text, [len(h) for h in bin_headers], len(asm_headers))
    want_flags, want_last, want_keep, want_n = _python_join(bin_headers, asm_headers)
    assert np.array_equal(flags, want_flags)
    assert np.array_equal(last, want_last)
    assert np.array_equal(keep, want_keep)
    assert nbinned == want_n
    every = [h for hs in bin_headers for h in hs] + list(asm_headers)
    got_ids = [text[s:s + n] for s, n in zip(id_start.tolist(), id_len.tolist())]
    assert got_ids == [h.split(None, 1)[0].encode() for h in every]
    return ms


def test_join_equals_python_on_a_million_records(engine):
    rng = np.random.default_rng(7)
    chars = np.array(ID_CHARS, dtype=object)
    pool = [''.join(chars[rng.integers(0, len(chars), size=int(k))]) for k in rng.integers(1, 24, size=400_000)]
    space = np.array(HEADER_SPACE, dtype=object)

    def header(i):
        lead = ''.join(space[rng.integers(0, len(space), size=int(rng.integers(0, 3)))]) if rng.random() < 0.1 else ''
        tail = space[rng.integers(0, len(space))] + 'd' + chars[rng.integers(0, len(chars))] if rng.random() < 0.5 else ''
        return lead + pool[i] + tail

    bins = [[header(i) for i in rng.integers(0, len(pool), size=int(k))] for k in rng.integers(100, 4000, size=150)]
    asm = [header(i) for i in rng.integers(0, len(pool), size=700_000)]
    assert sum(len(b) for b in bins) + len(asm) > 900_000
    _check_join(engine, bins, asm)


def test_join_on_colliding_ids(engine):
    rng = np.random.default_rng(8)
    prefix = 'x' * 1500
    long_ids = [prefix + chr(c) for c in range(33, 127)] + [prefix + 'é', prefix + '、']     # > 1 KB, last byte differs
    common = ['contig_' + 'A' * 200 + '%07d' % i for i in range(20_000)]                         # long common prefix
    asm = list(long_ids) + list(common)
    for d in range(1, 300):                                                                      # repeats at every distance
        asm.insert(int(rng.integers(0, len(asm))), asm[-d])
    asm += [i + ' tail' for i in long_ids[::-1]]
    bins = [long_ids[::3] + common[::7], [prefix] + common[5::11] + common[::7][:50], []]
    _check_join(engine, bins, asm)


def test_long_ids_and_empty_sequences_equal_the_oracle(tmp_path):
    from oracle import unbinned_oracle
    rng = np.random.default_rng(9)
    ids = ['q' * 1100 + '%04d' % i for i in range(300)] + ['p%d' % i for i in range(300)]
    recs = []
    for r in range(1500):
        i = ids[int(rng.integers(0, len(ids)))]
        n = int(rng.choice([0, 0, 1, 5, 70, 300]))
        seq = ''.join(rng.choice(list('ACGTNacgtuRY'), size=n))
        seq = 'g' + seq[1:] if n else seq                      # every non-empty sequence has a base to count
        lines = [seq[k:k + 60] for k in range(0, n, 60)]
        recs.append('>' + i + ' r%d\n' % r + ''.join(line + '\n' for line in lines))
    asm = ''.join(recs).encode()
    bin_ = ''.join('>%s\nACGT\n' % i for i in ids[::5]).encode()
    with open(str(tmp_path / 'asm.fna'), 'wb') as f:
        f.write(asm)
    with open(str(tmp_path / 'bin.fna'), 'wb') as f:
        f.write(bin_)
    fasta, stats, _ = _run(tmp_path, [str(tmp_path / 'bin.fna')], str(tmp_path / 'asm.fna'), 1)
    want_fasta, want_stats, _ = unbinned_oracle.run([bin_], asm, 1)
    assert fasta == want_fasta and stats == want_stats


def test_community_profile_workflow(tmp_path):
    """unbinned -> coverage (the BAM's references include the unbinned contigs) -> profile, against the oracles."""
    from checkm_b200.coverage import Coverage
    from checkm_b200.profile import Profile
    from oracle import coverage_oracle, unbinned_oracle
    from tools import bamsynth as bs
    rng = np.random.default_rng(10)
    lens = rng.integers(500, 6000, size=60)
    names = ['ctg%d' % i for i in range(len(lens))]
    seqs = [''.join(rng.choice(list('ACGT'), size=int(n))) for n in lens]
    rec = lambda idx: ''.join('>%s\n%s\n' % (names[i], seqs[i]) for i in idx)     # noqa: E731
    asm = str(tmp_path / 'assembly.fna')
    binFiles = [str(tmp_path / ('bin%d.fna' % b)) for b in range(3)]
    with open(asm, 'w') as f:
        f.write(rec(range(len(lens))) + '\n')
    for b, path in enumerate(binFiles):
        with open(path, 'w') as f:
            f.write(rec(range(b * 12, b * 12 + 12)))
    fna = str(tmp_path / 'unbinned.fna')
    from checkm_b200.unbinned import Unbinned
    Unbinned().run(binFiles, asm, fna, str(tmp_path / 'unbinned.tsv'), 0)
    want_fasta, _, _ = unbinned_oracle.run([_raw(p) for p in binFiles], _raw(asm), 0)
    assert _read(fna) == want_fasta
    bams = []
    for s in range(2):
        body, ref, pos, end = bs.bulk_records(rng, lens, lens // (100 + 100 * s))
        path = str(tmp_path / ('sample%d.bam' % s))
        bs.write_bam(path, list(zip(names, lens.tolist())), body, ref, pos, end, np.zeros(len(ref), bool))
        bams.append(path)
    cov = str(tmp_path / 'coverage.tsv')
    Coverage(1).run(binFiles, bams, cov, False, 0.98, 0.02, 15)
    want_cov = coverage_oracle.coverage_tsv(binFiles, bams)
    assert _read(cov).decode() == want_cov
    unbinned_rows = {line.split('\t')[0] for line in want_cov.splitlines()[1:] if line.split('\t')[1] == 'unbinned'}
    assert unbinned_rows == {line[1:] for line in want_fasta.decode().splitlines() if line.startswith('>')}
    ref_cov = str(tmp_path / 'coverage_oracle.tsv')
    with open(ref_cov, 'w') as f:
        f.write(want_cov)
    for tab in (True, False):
        Profile().run(cov, str(tmp_path / 'profile.txt'), tab)
        Profile().run(ref_cov, str(tmp_path / 'profile_oracle.txt'), tab)
        assert _read(str(tmp_path / 'profile.txt')) == _read(str(tmp_path / 'profile_oracle.txt'))
        assert b'unbinned' in _read(str(tmp_path / 'profile.txt'))
