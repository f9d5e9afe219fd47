"""CPU restatement of `checkm gc_bias_plot`'s read depth (checkm/coverageWindows.py:30-205) for the tests and the
benchmark's parity check: the BAM inflated and its header read with coverage_oracle's helpers, each record kept when
`fetch(ref, 0, len)` would yield it, classified as ReadLoader.__call__ does, the mapped reads' clipped spans put into a
difference array per reference, then `cumsum` for the depth and window sums of it.  The product never imports this
module."""
import struct

import numpy as np

from oracle import coverage_oracle as co

_FLOAT_NM = ord('f')


def nm_number(stream, a, e):
    """NM as pysam's get_tag returns it to a numeric comparison: an integer type or the float of type f; None otherwise."""
    v = co.nm_tag(stream, a, e)
    if v is not None:
        return v
    while a < e:                                       # an integer NM was not found: look for one of type f
        tag, ty = stream[a:a + 2], stream[a + 2]
        a += 3
        if ty in (ord('Z'), ord('H')):
            a = stream.index(b'\x00', a, e) + 1
        elif ty == ord('B'):
            cnt, = struct.unpack_from('<i', stream, a + 1)
            a += 5 + cnt * co._SIZE[stream[a]]
        else:
            if tag == b'NM':
                return struct.unpack_from('<f', stream, a)[0] if ty == _FLOAT_NM else None
            a += co._SIZE[ty]
    return None


def depths(path, all_reads=False, min_align=0.98, max_edit=0.02):
    """(names, lengths, n_ref x 9 int64 counters, [per-reference int64 depth arrays]).  The ninth counter is the bases
    covered, the sum of the depth.  Raises ValueError where the reference raises or indexes from the array's end."""
    stream = co.inflate(path)
    names, lens, p = co.parse_header(stream)
    cnt = np.zeros((len(names), 9), dtype=np.int64)
    diff = [np.zeros(n + 1, dtype=np.int64) for n in lens]
    n = len(stream)
    while p + 4 <= n:
        bs, ref, pos, l_name, mapq, _, n_cigar, flag, l_seq = struct.unpack_from('<iiiBBHHHi', stream, p)
        if ref == -1:
            break
        rec = p + 4
        p = rec + bs
        cig = rec + 32 + l_name
        cigar = [(v >> 4, v & 15) for v in struct.unpack_from('<%dI' % n_cigar, stream, cig)]
        alen = sum(k for k, op in cigar if op in (0, 2, 3, 7, 8))
        L = lens[ref]
        fend = pos + (1 if flag & 0x4 or alen == 0 else alen)
        if not (pos < L and fend > 0):
            continue                                   # fetch(ref, 0, L) does not yield it
        c = cnt[ref]
        c[0] += 1
        if flag & 0x4:
            continue
        if flag & 0x400:
            c[1] += 1
        elif flag & 0x100:
            c[2] += 1
        elif flag & 0x200:
            c[3] += 1
        elif n_cigar == 0:
            raise ValueError('read %s has no CIGAR' % stream[cig - l_name:cig - 1].decode())
        elif alen < min_align * l_seq:
            c[4] += 1
        else:
            nm = nm_number(stream, cig + 4 * n_cigar + (l_seq + 1) // 2 + l_seq, rec + bs)
            if nm is None:
                raise ValueError('read %s has no numeric NM tag' % stream[cig - l_name:cig - 1].decode())
            if nm > max_edit * l_seq:
                c[5] += 1
            elif not all_reads and not flag & 0x2:
                c[6] += 1
            elif pos < 0:
                raise ValueError('read %s is mapped at position %d' % (stream[cig - l_name:cig - 1].decode(), pos))
            else:
                c[7] += 1
                b = min(pos + alen, L)
                if b > pos:
                    c[8] += b - pos
                    diff[ref][pos] += 1
                    diff[ref][b] -= 1
    return names, lens, cnt, [np.cumsum(d[:-1]) for d in diff]


def window_sums(depth, W):
    """The depth summed over windows [k W, (k + 1) W) while (k + 1) W < len(depth)."""
    nwin = (len(depth) - 1) // W
    return depth[:nwin * W].reshape(nwin, W).sum(axis=1) if nwin else np.zeros(0, dtype=np.int64)


def coverage_windows(path, W, all_reads=False, min_align=0.98, max_edit=0.02):
    """{seqId: [coverage, windowCoverages]} as CoverageWindows.run returns it, and the counters."""
    names, lens, cnt, deps = depths(path, all_reads, min_align, max_edit)
    out = {}
    for name, L, c, d in zip(names, lens, cnt, deps):
        out[name] = [float(int(c[8])) / L, [float(int(v)) / W for v in window_sums(d, W)]]
    return out, cnt
