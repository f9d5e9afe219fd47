"""Fixtures for read coverage (`checkm coverage`) and what the REFERENCE's own Coverage computes for them.

Run in the build container (needs /root/reference):  python tests/golden/make_coverage_goldens.py

The reference's `checkm.coverage` reads BAM files through `pysam`, which is not installed here (and its `Coverage.run`
cannot run in CheckM 1.2.4 even with pysam: `import pysam` sits inside `__init__`, so the module-global name the worker
processes use is unbound).  This script installs a STAND-IN `pysam` -- a small BAM reader written here with the stdlib
gzip and struct, independent of checkm_b200/bam.py and oracle/coverage_oracle.py -- both in sys.modules and as the module
global `checkm.coverage.pysam`, and then runs the reference's own `Coverage.run` (threads=1) and `binProfiles`.  The
classification and the file layout that are frozen are the reference's; only the BAM reader underneath is a stand-in.
Its read attributes follow the SAM specification and pysam's documented definitions: query_length is l_seq;
query_alignment_length is the query end minus the query start (leading soft clips, hard clips skipped, give the start;
l_seq minus the trailing soft clips gives the end); without SEQ the M, I, =, X ops of the CIGAR give it (unpinned against
real pysam); `fetch(ref, beg, end)` yields the reference's records that overlap [beg, end) under htslib's rule (end
position = pos + reference span of the CIGAR, or pos + 1 for an unmapped read or an empty span).

Writes tests/golden/coverage/:
  bin1.fna, bin2.fna          two bins; c2 is in both (the later bin wins), c9 is in no BAM
  sample1.bam(.bai)           refs c1 c2 c3 c5 c6: every filter branch with values on the min_align, max_edit and min_qc
                              boundaries, soft and hard clips, a read without SEQ, NM of types c C s S i I, a placed
                              unmapped read, an unplaced unmapped tail, a contig without reads (c6), c5 in no bin, records
                              across small blocks and one 75 kB record spanning three blocks; stored, fixed-Huffman and
                              dynamic blocks; a sparse contig (c3) whose linear index has empty windows (htslib-filled)
  sample2.bam(.bai)           refs c3 c1 c7 (another set and order), linear index left with zeros in empty windows
  coverage_<opt>.tsv          Coverage(1).run([bin1, bin2], [sample1, sample2], ...) for every option set
  expected.json               the option sets; binProfiles as [repr(mean), repr(std)]; parseCoverage of the defaults;
                              the INFO summary text of the defaults; the writer's block tables, record starts, header ends
                              and linear-index anchors"""
import gzip
import json
import logging
import os
import shutil
import struct
import sys
import tempfile
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
OUT = os.path.join(HERE, 'coverage')
sys.path.insert(0, ROOT)
sys.path.insert(0, '/root/reference')

from tools import bamsynth as bs  # noqa: E402

OPTIONS = {
    'defaults': dict(bAllReads=False, minAlignPer=0.98, maxEditDistPer=0.02, minQC=15),
    'all_reads': dict(bAllReads=True, minAlignPer=0.98, maxEditDistPer=0.02, minQC=15),
    'loose': dict(bAllReads=False, minAlignPer=0.5, maxEditDistPer=0.1, minQC=0),
    'strict': dict(bAllReads=True, minAlignPer=0.99, maxEditDistPer=0.0, minQC=30),
}


# ------------------------------------------------------------------ stand-in pysam (test infrastructure) ----
class _Read(object):
    def __init__(self, flag, mapq, cigar, l_seq, tags):
        self.flag, self.mapping_quality, self._cigar, self.query_length, self._tags = flag, mapq, cigar, l_seq, tags

    is_unmapped = property(lambda self: bool(self.flag & 0x4))
    is_duplicate = property(lambda self: bool(self.flag & 0x400))
    is_secondary = property(lambda self: bool(self.flag & 0x100))
    is_supplementary = property(lambda self: bool(self.flag & 0x800))
    is_qcfail = property(lambda self: bool(self.flag & 0x200))
    is_proper_pair = property(lambda self: bool(self.flag & 0x2))

    @property
    def query_alignment_length(self):
        ops = self._cigar
        if self.query_length == 0:
            return sum(n for op, n in ops if op in 'MI=X')
        start = 0
        for op, n in ops:
            if op == 'S':
                start += n
            elif op != 'H':
                break
        end = self.query_length
        for op, n in reversed(ops[1:]):
            if op == 'S':
                end -= n
            elif op != 'H':
                break
        return end - start

    def get_tag(self, tag):
        if tag not in self._tags:
            raise KeyError(tag)
        return self._tags[tag]


class _Samfile(object):
    def __init__(self, path, mode='rb'):
        data = gzip.decompress(open(path, 'rb').read())
        l_text, = struct.unpack_from('<i', data, 4)
        p = 8 + l_text
        n_ref, = struct.unpack_from('<i', data, p)
        p += 4
        self.references, self.lengths = [], []
        for _ in range(n_ref):
            ln, = struct.unpack_from('<i', data, p)
            self.references.append(data[p + 4:p + 3 + ln].decode())
            self.lengths.append(struct.unpack_from('<i', data, p + 4 + ln)[0])
            p += 8 + ln
        self.references, self.lengths = tuple(self.references), tuple(self.lengths)
        self._recs = []
        while p < len(data):
            bs_, = struct.unpack_from('<i', data, p)
            self._recs.append(data[p + 4:p + 4 + bs_])
            p += 4 + bs_

    def fetch(self, ref, beg, end):
        tid = self.references.index(ref)
        for r in self._recs:
            rid, pos, l_name, mapq, _, n_cig, flag, l_seq = struct.unpack_from('<iiBBHHHi', r, 0)
            if rid != tid:
                continue
            cig = [('MIDNSHP=X'[v & 15], v >> 4) for v in struct.unpack_from('<%dI' % n_cig, r, 32 + l_name)]
            span = 0 if flag & 0x4 else sum(n for op, n in cig if op in 'MDN=X')
            rend = pos + (span or 1)
            if not (pos < end and rend > beg):
                continue
            a = 32 + l_name + 4 * n_cig + (l_seq + 1) // 2 + l_seq
            tags = {}
            while a < len(r):
                tag, ty = r[a:a + 2].decode(), chr(r[a + 2])
                a += 3
                if ty in 'cCsSiI':
                    fmt = '<' + {'c': 'b', 'C': 'B', 's': 'h', 'S': 'H', 'i': 'i', 'I': 'I'}[ty]
                    tags[tag], = struct.unpack_from(fmt, r, a)
                    a += struct.calcsize(fmt)
                elif ty == 'A':
                    tags[tag] = chr(r[a])
                    a += 1
                elif ty == 'f':
                    tags[tag], = struct.unpack_from('<f', r, a)
                    a += 4
                elif ty in 'ZH':
                    z = r.index(b'\x00', a)
                    tags[tag] = r[a:z].decode()
                    a = z + 1
                else:                                        # B: subtype, count, values
                    sub, cnt = chr(r[a]), struct.unpack_from('<I', r, a + 1)[0]
                    size = {'c': 1, 'C': 1, 's': 2, 'S': 2, 'i': 4, 'I': 4, 'f': 4}[sub]
                    tags[tag] = list(r[a + 5:a + 5 + cnt * size])
                    a += 5 + cnt * size
            yield _Read(flag, mapq, cig, l_seq, tags)

    def close(self):
        pass


def stand_in_pysam():
    m = types.ModuleType('pysam')
    m.Samfile = _Samfile
    m.AlignmentFile = _Samfile
    return m


# ------------------------------------------------------------------ fixtures ----
def sample1(rng):
    refs = [('c1', 50000), ('c2', 3000), ('c3', 120000), ('c5', 8000), ('c6', 1000)]
    recs = []

    def add(ref, pos, name, **kw):
        b, e = bs.record(rng, ref, pos, name, **kw)
        recs.append((ref, pos, e, b, bool(kw.get('flag', 0x3) & 0x4)))

    # c1: every branch, boundary values at l_seq = 100 (0.98 * 100, 0.02 * 100, MAPQ 15) and at l_seq = 150
    p = 100
    for name, kw in [
        ('mapped', {}),
        ('unmapped_placed', dict(flag=0x1 | 0x4 | 0x20, cigar=(), l_seq=100, nm=None)),
        ('dup', dict(flag=0x403)),
        ('secondary', dict(flag=0x103)),
        ('supplementary', dict(flag=0x803)),
        ('qcfail', dict(flag=0x203)),
        ('mapq14', dict(mapq=14)), ('mapq15', dict(mapq=15)), ('mapq0', dict(mapq=0)), ('mapq30', dict(mapq=30)),
        ('mapq255', dict(mapq=255)),
        ('aln98', dict(cigar=((1, 'S'), (98, 'M'), (1, 'S')))), ('aln97', dict(cigar=((2, 'S'), (97, 'M'), (1, 'S')))),
        ('aln147of150', dict(cigar=((3, 'S'), (147, 'M')))), ('aln146of150', dict(cigar=((4, 'S'), (146, 'M')))),
        ('aln99_hard', dict(cigar=((5, 'H'), (1, 'S'), (99, 'M'), (7, 'H')))),
        ('aln_hard_soft', dict(cigar=((3, 'H'), (2, 'S'), (96, 'M'), (2, 'S'), (4, 'H')))),
        ('aln_indel', dict(cigar=((40, 'M'), (2, 'I'), (30, 'M'), (5, 'D'), (28, 'M')))),
        ('aln_eqx', dict(cigar=((50, '='), (1, 'X'), (49, '=')))),
        ('aln_n', dict(cigar=((50, 'M'), (300, 'N'), (50, 'M')))),
        ('nm2', dict(nm=(2, 'C'))), ('nm3', dict(nm=(3, 'C'))), ('nm3_of150', dict(cigar=((150, 'M'),), nm=(3, 'c'))),
        ('nm4_of150', dict(cigar=((150, 'M'),), nm=(4, 's'))), ('nm_S', dict(nm=(1, 'S'))), ('nm_i', dict(nm=(2, 'i'))),
        ('nm_I', dict(nm=(5, 'I'))), ('nm_c_neg', dict(nm=(-1, 'c'))),
        ('nm_after_tags', dict(nm=None, aux=b'XAZabc\x00RGZgrp1\x00XBB' + struct.pack('<BI', ord('C'), 3) + b'abc'
                               + bs.aux_int('NM', 1, 's'))),
        ('unpaired', dict(flag=0x1)), ('unpaired_single', dict(flag=0x0)),
        ('noseq', dict(l_seq=0, cigar=((100, 'M'),), nm=(0, 'C'))),
        ('noseq_clipped', dict(l_seq=0, cigar=((10, 'S'), (80, 'M'), (10, 'S')), nm=(0, 'C'))),
        ('noseq_nm1', dict(l_seq=0, cigar=((100, 'M'),), nm=(1, 'C'))),
        ('allsoft', dict(cigar=((100, 'S'),), l_seq=100)),
    ]:
        add(0, p, name, **kw)
        p += int(rng.integers(20, 400))
    # bulk on c1 and c2 with small blocks (records cross block boundaries)
    for ref, L, n in ((0, 50000, 300), (1, 3000, 60)):
        lo = p if ref == 0 else 0
        for pos in sorted(rng.integers(lo, L - 160, size=n).tolist()):
            a, b = int(rng.integers(0, 4)), int(rng.integers(0, 4))
            cig = tuple(x for x in ((a, 'S'), (150 - a - b, 'M'), (b, 'S')) if x[0])
            add(ref, pos, 'r%d_%d' % (ref, pos), flag=int(rng.choice([0x3, 0x3, 0x3, 0x1, 0x403, 0x103])),
                mapq=int(rng.choice([60, 60, 10])), cigar=cig, nm=(int(rng.integers(0, 5)), str(rng.choice(list('cCsi')))))
    # c3: sparse windows, and one 75 kB read
    for pos in (10, 500, 16390, 90000, 90010, 119000):
        add(2, pos, 'sparse%d' % pos)
    big_at = len(recs)
    add(2, 119500, 'huge', cigar=((50000, 'S'),), l_seq=50000)
    recs.sort(key=lambda t: (t[0], t[1]))
    # c5 (in no bin): a few reads; c6: none
    for pos in sorted(rng.integers(0, 7800, size=40).tolist()):
        add(3, pos, 'u5_%d' % pos, cigar=((150, 'M'),), nm=(0, 'C'))
    return refs, recs, big_at


def sample2(rng):
    refs = [('c3', 120000), ('c1', 50000), ('c7', 20000)]
    recs = []
    for ref, L, n in ((0, 120000, 80), (1, 50000, 200), (2, 20000, 50)):
        for pos in sorted(rng.integers(0, L - 200, size=n).tolist()):
            if ref == 0 and 30000 < pos < 80000:
                continue                                     # empty windows: zeros in the linear index
            b, e = bs.record(rng, ref, pos, 's%d_%d' % (ref, pos), flag=int(rng.choice([0x3, 0x3, 0x1, 0x5])),
                             cigar=((1, 'S'), (99, 'M')), nm=(int(rng.integers(0, 3)), 'C'))
            recs.append((ref, pos, e, b, False))
    return refs, recs


def write(path, refs, recs, rng, unplaced=0, **kw):
    tail = [bs.record(rng, -1, -1, 'unplaced%d' % i, flag=0x4, cigar=(), l_seq=80, nm=None)[0] for i in range(unplaced)]
    table, starts = bs.write_bam(path, refs, [r[3] for r in recs], [r[0] for r in recs], [r[1] for r in recs],
                                 [r[2] for r in recs], np.array([r[4] for r in recs]), n_unplaced=unplaced,
                                 unplaced=b''.join(tail), **kw)
    return table, starts


def write_fasta(path, recs):
    with open(path, 'w') as f:
        for name, n in recs:
            f.write('>%s desc\n' % name)
            s = 'ACGT' * (n // 4) + 'ACGT'[:n % 4]
            for i in range(0, len(s), 70):
                f.write(s[i:i + 70] + '\n')


def main():
    rng = np.random.default_rng(20261016)
    shutil.rmtree(OUT, ignore_errors=True)
    os.makedirs(OUT)
    write_fasta(os.path.join(OUT, 'bin1.fna'), [('c1', 49000), ('c2', 3000), ('c9', 700)])
    write_fasta(os.path.join(OUT, 'bin2.fna'), [('c3', 1000), ('c2', 2500)])
    refs1, recs1, _ = sample1(rng)
    recs1.sort(key=lambda t: (t[0], t[1]))
    huge = [i for i, r in enumerate(recs1) if len(r[3]) > 65536][0]
    hstart = sum(len(r[3]) for r in recs1[:huge])
    head = len(bs.header_bytes(refs1))
    hend = hstart + len(recs1[huge][3])
    total = sum(len(r[3]) for r in recs1)
    cuts = [head + x for x in range(0, total, 2500) if not hstart <= x < hend + 2500] + [head + hstart + 300, head + hstart + 40000]
    known = {}
    t1, s1 = write(os.path.join(OUT, 'sample1.bam'), refs1, recs1, rng, unplaced=5, levels=(0, 1, 6, 9, 4),
                   strategies=('default', 'fixed', 'huffman', 'rle', 'filtered', 'default'), cuts=cuts, payload=60000)
    refs2, recs2 = sample2(rng)
    t2, s2 = write(os.path.join(OUT, 'sample2.bam'), refs2, recs2, rng, unplaced=3, levels=(6,), payload=4000,
                   fill_linear=False)
    for name, t, s, refs in (('sample1', t1, s1, refs1), ('sample2', t2, s2, refs2)):
        known[name] = {'blocks': t.tolist(), 'record_starts': s.tolist(), 'header_end': len(bs.header_bytes(refs)),
                       'names': [r[0] for r in refs], 'lengths': [r[1] for r in refs]}

    os.environ['CHECKM_DATA_PATH'] = tempfile.mkdtemp()
    pysam = stand_in_pysam()
    sys.modules['pysam'] = pysam
    import checkm.coverage as cc
    cc.pysam = pysam
    bins = [os.path.join(OUT, 'bin1.fna'), os.path.join(OUT, 'bin2.fna')]
    bams = [os.path.join(OUT, 'sample1.bam'), os.path.join(OUT, 'sample2.bam')]
    logger = logging.getLogger('timestamp')
    expected = {'options': OPTIONS, 'known': known, 'profiles': {}}
    for label, opt in OPTIONS.items():
        out = os.path.join(OUT, 'coverage_%s.tsv' % label)
        logger.setLevel(logging.INFO if label == 'defaults' else logging.WARNING)
        cap = tempfile.TemporaryFile(mode='w+')
        sys.stdout.flush()
        saved = os.dup(1)
        os.dup2(cap.fileno(), 1)
        try:
            cc.Coverage(1).run(bins, bams, out, opt['bAllReads'], opt['minAlignPer'], opt['maxEditDistPer'], opt['minQC'])
            sys.stdout.flush()
        finally:
            os.dup2(saved, 1)
            os.close(saved)
        cap.seek(0)
        if label == 'defaults':
            expected['summary'] = cap.read()
            expected['parseCoverage'] = cc.Coverage(1).parseCoverage(out)
        prof = cc.Coverage(1).binProfiles(out)
        expected['profiles'][label] = {b: {k: [repr(float(v[0])), repr(float(v[1]))] for k, v in d.items()} for b, d in prof.items()}
    # the profiles' dict order is part of what printSummary writes
    expected['profile_order'] = {label: [[b, list(d.keys())] for b, d in p.items()] for label, p in expected['profiles'].items()}
    with open(os.path.join(OUT, 'expected.json'), 'w') as f:
        json.dump(expected, f, indent=0, sort_keys=False)
    print(sum(os.path.getsize(os.path.join(OUT, f)) for f in os.listdir(OUT)), 'bytes in', OUT)


if __name__ == '__main__':
    main()
