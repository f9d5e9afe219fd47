"""Fixtures for read depth per window (`checkm gc_bias_plot`'s coverage profile) and what the REFERENCE's own
CoverageWindows computes for them.

Run in the build container (needs /root/reference):  python tests/golden/make_coverage_windows_goldens.py

The reference's `checkm.coverageWindows` reads the BAM through `pysam`, which is not installed here (and its
`_processBam` cannot run in CheckM 1.2.4 even with pysam: `import pysam` sits inside `ReadLoader.__init__`, so the module
global it uses is unbound).  This script installs a STAND-IN `pysam` -- the BAM reader of make_coverage_goldens.py,
extended with what coverageWindows asks of a read (`pos`, `alen`, `rlen`, `opt`) and `fetch(..., callback=)` -- both in
sys.modules and as the module global `checkm.coverageWindows.pysam`, and then runs the reference's own
`CoverageWindows(1).run`.  Only the BAM reader underneath is a stand-in.  Its attributes follow pysam's documented
definitions: `pos` is reference_start; `alen` is reference_length, the CIGAR's M, D, N, =, X lengths, None without a
CIGAR; `rlen` is query_length, l_seq; `opt` is get_tag: an int for the integer types, a float for `f`, KeyError when the
tag is absent; `fetch(ref, beg, end)` yields the records overlapping [beg, end) under htslib's rule and calls `callback`
with each; `is_secondary` is flag 0x100.

Writes tests/golden/coverage_windows/:
  windows.bam(.bai)   seeded: refs of length k W, k W + 1, <= W and 1, a reference without reads, reads across window
                      boundaries, reads longer than W, reads running past the reference end and lying wholly past it,
                      D, N, I and S operations, an I/S-only CIGAR (alen 0), supplementary and MAPQ-0 reads (mapped here),
                      NM of type f on and off the threshold, l_seq == 0, and the other filter branches
  expected.json.gz    per BAM (this one and tests/golden/coverage/sample1.bam, sample2.bam), per option set and per W
                      in (1, 7, 100, 5000): {seqId: [repr(coverage), run-length-encoded windows [[repr(value), run]...]]};
                      the INFO summary text of windows.bam at the defaults, W = 5000"""
import gzip
import json
import logging
import os
import shutil
import struct
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
OUT = os.path.join(HERE, 'coverage_windows')
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)
sys.path.insert(0, '/root/reference')

from tools import bamsynth as bs  # noqa: E402
import make_coverage_goldens as mcg  # noqa: E402

OPTIONS = {
    'defaults': dict(bAllReads=False, minAlignPer=0.98, maxEditDistPer=0.02),
    'all_reads': dict(bAllReads=True, minAlignPer=0.98, maxEditDistPer=0.02),
    'loose': dict(bAllReads=False, minAlignPer=0.5, maxEditDistPer=0.1),
    'strict': dict(bAllReads=True, minAlignPer=0.99, maxEditDistPer=0.0),
}
WINDOWS = (1, 7, 100, 5000)
BAMS = {'windows': os.path.join(OUT, 'windows.bam'), 'sample1': os.path.join(HERE, 'coverage', 'sample1.bam'),
        'sample2': os.path.join(HERE, 'coverage', 'sample2.bam')}


# ------------------------------------------------------------------ stand-in pysam (test infrastructure) ----
class _Read(mcg._Read):
    def __init__(self, pos, flag, mapq, cigar, l_seq, tags):
        mcg._Read.__init__(self, flag, mapq, cigar, l_seq, tags)
        self.pos = self.reference_start = pos

    @property
    def reference_length(self):
        if not self._cigar:
            return None
        return sum(n for op, n in self._cigar if op in 'MDN=X')

    alen = reference_length
    rlen = property(lambda self: self.query_length)

    def opt(self, tag):
        return self.get_tag(tag)


class _Samfile(mcg._Samfile):
    def fetch(self, ref, beg, end, callback=None):
        """The reads overlapping [beg, end): passed to `callback` one by one (and their number returned), or an iterator."""
        tid = self.references.index(ref)
        reads = []
        for r in self._recs:
            rid, pos, l_name, mapq, _, n_cig, flag, l_seq = struct.unpack_from('<iiBBHHHi', r, 0)
            if rid != tid:
                continue
            cig = [('MIDNSHP=X'[v & 15], v >> 4) for v in struct.unpack_from('<%dI' % n_cig, r, 32 + l_name)]
            span = 0 if flag & 0x4 else sum(k for op, k in cig if op in 'MDN=X')
            if not (pos < end and pos + (span or 1) > beg):
                continue
            tags = self._tags_of(r, 32 + l_name + 4 * n_cig + (l_seq + 1) // 2 + l_seq)
            reads.append(_Read(pos, flag, mapq, cig, l_seq, tags))
        if callback is None:
            return iter(reads)
        for read in reads:
            callback(read)
        return len(reads)

    @staticmethod
    def _tags_of(r, a):
        tags = {}
        while a < len(r):
            tag, ty = r[a:a + 2].decode(), chr(r[a + 2])
            a += 3
            if ty in 'cCsSiIf':
                fmt = '<' + {'c': 'b', 'C': 'B', 's': 'h', 'S': 'H', 'i': 'i', 'I': 'I', 'f': 'f'}[ty]
                tags[tag], = struct.unpack_from(fmt, r, a)
                a += struct.calcsize(fmt)
            elif ty == 'A':
                tags[tag] = chr(r[a])
                a += 1
            elif ty in 'ZH':
                z = r.index(b'\x00', a)
                tags[tag] = r[a:z].decode()
                a = z + 1
            else:
                sub, cnt = chr(r[a]), struct.unpack_from('<I', r, a + 1)[0]
                size = {'c': 1, 'C': 1, 's': 2, 'S': 2, 'i': 4, 'I': 4, 'f': 4}[sub]
                tags[tag] = list(r[a + 5:a + 5 + cnt * size])
                a += 5 + cnt * size
        return tags


def stand_in_pysam():
    m = mcg.stand_in_pysam()
    m.Samfile = m.AlignmentFile = _Samfile
    return m


# ------------------------------------------------------------------ the fixture ----
def f_nm(v):
    return b'NMf' + struct.pack('<f', v)


def windows_bam(rng, path):
    refs = [('w1', 15000), ('w2', 10001), ('w3', 4000), ('w4', 2000), ('w5', 30000), ('w6', 700), ('w7', 701), ('w8', 1)]
    recs = []

    def add(ref, pos, name, **kw):
        b, e = bs.record(rng, ref, pos, name, **kw)
        recs.append((ref, pos, e, b, bool(kw.get('flag', 0x3) & 0x4)))

    # w1 (3 x 5000): hand-made cases
    for pos, name, kw in [
        (0, 'first', {}),
        (100, 'longer_than_w', dict(cigar=((6000, 'M'),), l_seq=6000, nm=(50, 'S'))),
        (4950, 'across_5000', {}),
        (4990, 'dni_s', dict(cigar=((10, 'S'), (40, 'M'), (5, 'D'), (30, 'M'), (2, 'I'), (20, 'M'), (100, 'N'), (30, 'M')),
                             nm=(2, 'C'))),
        (5000, 'is_only', dict(cigar=((50, 'S'), (50, 'I')), l_seq=100)),
        (5001, 'is_only_noseq', dict(cigar=((10, 'I'),), l_seq=0, nm=(0, 'C'))),
        (5100, 'supplementary', dict(flag=0x803)),
        (5200, 'mapq0', dict(mapq=0)),
        (5300, 'secondary', dict(flag=0x103)),
        (5350, 'qcfail', dict(flag=0x203)),
        (5400, 'duplicate', dict(flag=0x403)),
        (5450, 'unmapped_placed', dict(flag=0x1 | 0x4 | 0x20, cigar=(), l_seq=100, nm=None)),
        (5500, 'not_paired', dict(flag=0x1)),
        (5600, 'nm_f_on', dict(nm=None, aux=f_nm(2.0))),
        (5700, 'nm_f_off', dict(nm=None, aux=f_nm(2.5))),
        (5750, 'nm_f_mid', dict(nm=None, aux=b'XAZx\x00' + f_nm(1.0))),
        (5800, 'nm_f_loose', dict(nm=None, aux=f_nm(9.5))),
        (5900, 'noseq', dict(l_seq=0, cigar=((100, 'M'),), nm=(0, 'C'))),
        (5950, 'noseq_nm1', dict(l_seq=0, cigar=((100, 'M'),), nm=(1, 'C'))),
        (6000, 'aln98', dict(cigar=((2, 'S'), (98, 'M')))), (6050, 'aln97', dict(cigar=((3, 'S'), (97, 'M')))),
        (6100, 'aln_with_d', dict(cigar=((5, 'S'), (50, 'M'), (3, 'D'), (45, 'M')))),
        (6200, 'nm_i', dict(nm=(2, 'i'))), (6250, 'nm_c_neg', dict(nm=(-1, 'c'))), (6300, 'nm3', dict(nm=(3, 'C'))),
        (9999, 'across_10000', dict(cigar=((150, 'M'),), nm=(1, 'C'))),
        (14950, 'past_end', {}),
        (14999, 'last_base', dict(cigar=((1, 'S'), (99, 'M')), nm=(0, 's'))),
    ]:
        add(0, pos, name, **kw)
    # w2 (2 x 5000 + 1): reads over the last base and past the end
    for pos in (0, 4999, 5000, 9900, 9950, 9999, 10000):
        add(1, pos, 'w2_%d' % pos)
    # w3 (<= 5000): a read longer than the reference, reads lying wholly past the end (fetch does not yield them)
    add(2, 0, 'w3_long', cigar=((5000, 'M'),), l_seq=5000, nm=(10, 'I'))
    add(2, 3950, 'w3_edge')
    add(2, 4000, 'w3_past', flag=0x3)
    add(2, 4500, 'w3_far_past', flag=0x403)
    # w4: no reads.  w5: a random population over 30 kbp
    for pos in sorted(rng.integers(0, 29950, size=400).tolist()):
        a, b = int(rng.integers(0, 4)), int(rng.integers(0, 4))
        d = int(rng.integers(0, 3))
        mid = 150 - a - b
        cig = [(a, 'S'), (mid // 2, 'M'), (d, 'D'), (mid - mid // 2, 'M'), (b, 'S')]
        if rng.random() < 0.1:
            cig = [(a, 'S'), (mid // 2, 'M'), (int(rng.integers(10, 400)), 'N'), (mid - mid // 2, 'M'), (b, 'S')]
        cig = tuple(x for x in cig if x[0])
        if rng.random() < 0.15:
            kw = dict(nm=None, aux=f_nm(float(rng.integers(0, 8)) / 2))
        else:
            kw = dict(nm=(int(rng.integers(0, 5)), str(rng.choice(list('cCsSiI')))))
        add(4, pos, 'r5_%d' % pos, flag=int(rng.choice([0x3, 0x3, 0x3, 0x1, 0x403, 0x103, 0x803, 0x203])),
            mapq=int(rng.choice([60, 60, 0])), cigar=cig, **kw)
    # w6 (7 x 100), w7 (7 x 100 + 1), w8 (length 1)
    for ref, L in ((5, 700), (6, 701)):
        for pos in (0, 93, 600, L - 50, L - 1):
            add(ref, pos, 'w%d_%d' % (ref + 1, pos))
    add(7, 0, 'w8_0')
    recs.sort(key=lambda t: (t[0], t[1]))
    tail = [bs.record(rng, -1, -1, 'unplaced%d' % i, flag=0x4, cigar=(), l_seq=80, nm=None)[0] for i in range(3)]
    bs.write_bam(path, refs, [r[3] for r in recs], [r[0] for r in recs], [r[1] for r in recs], [r[2] for r in recs],
                 np.array([r[4] for r in recs]), n_unplaced=3, unplaced=b''.join(tail), levels=(6, 1), payload=3000)


def rle(values):
    out = []
    for v in values:
        r = repr(float(v))
        if out and out[-1][0] == r:
            out[-1][1] += 1
        else:
            out.append([r, 1])
    return out


def main():
    rng = np.random.default_rng(20261017)
    shutil.rmtree(OUT, ignore_errors=True)
    os.makedirs(OUT)
    windows_bam(rng, BAMS['windows'])

    os.environ['CHECKM_DATA_PATH'] = tempfile.mkdtemp()
    pysam = stand_in_pysam()
    sys.modules['pysam'] = pysam
    import checkm.coverageWindows as cw
    cw.pysam = pysam
    logger = logging.getLogger('timestamp')
    expected = {'options': OPTIONS, 'windows': list(WINDOWS), 'values': {}}
    for bam_label, path in BAMS.items():
        per = expected['values'][bam_label] = {}
        for label, opt in OPTIONS.items():
            per[label] = {}
            for W in WINDOWS:
                want_summary = bam_label == 'windows' and label == 'defaults' and W == 5000
                logger.setLevel(logging.INFO if want_summary else logging.WARNING)
                cap = tempfile.TemporaryFile(mode='w+')
                sys.stdout.flush()
                saved = os.dup(1)
                os.dup2(cap.fileno(), 1)
                try:
                    info = dict(cw.CoverageWindows(1).run([], path, opt['bAllReads'], opt['minAlignPer'],
                                                          opt['maxEditDistPer'], W))
                    sys.stdout.flush()
                finally:
                    os.dup2(saved, 1)
                    os.close(saved)
                cap.seek(0)
                if want_summary:
                    expected['summary'] = cap.read()
                per[label][str(W)] = {k: [repr(float(v[0])), rle(v[1])] for k, v in info.items()}
    # compact and gzip-compressed (mtime 0, so the bytes depend only on the values): a few hundred thousand window
    # values, most of them in runs, would otherwise be tens of thousands of text lines
    with open(os.path.join(OUT, 'expected.json.gz'), 'wb') as f:
        f.write(gzip.compress(json.dumps(expected, separators=(',', ':')).encode(), 9, mtime=0))
    print(sum(os.path.getsize(os.path.join(OUT, f)) for f in os.listdir(OUT)), 'bytes in', OUT)


if __name__ == '__main__':
    main()
