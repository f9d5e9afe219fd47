"""Host-side BAM readers for `checkm coverage`: the BGZF block table (`ckm_bgzf_blocks`), the BAM header, the BAI index,
the record anchors it yields, and the cut of a file into device batches.

Record starts cannot be found in parallel from the bytes alone: records chain through `block_size` across block
boundaries.  The index gives them.  Every non-zero linear-index offset is the start of a record (the first one
overlapping a 16 kbp window), and so is the end of the header; these anchors, sorted and made unique, cut the placed
reads into segments that the device walks independently (csrc/bam.cu).  The reference requires `<bam>.bai` as well
(coverage.py:78-81).  CSI indexes and CRAM are not read."""
import ctypes as C
import mmap
import os
import struct
import zlib

import numpy as np

from . import _lib

BLOCK_DTYPE = np.dtype([('coffset', '<i8'), ('clen', '<i4'), ('isize', '<i4')])
PSEUDO_BIN = 37450
MAX_BLOCK = 65536
CKM_EFORMAT = 3


def format_error(msg):
    return _lib.CkmError(CKM_EFORMAT, msg)


def bgzf_blocks(data, base=0, cap=None):
    """The BGZF blocks wholly inside `data` (a bytes-like object or uint8 array holding the file from offset `base`):
    a BLOCK_DTYPE array and the number of bytes they cover."""
    buf = np.frombuffer(data, dtype=np.uint8) if not isinstance(data, np.ndarray) else data
    n = buf.size
    cap = n // 28 + 1 if cap is None else int(cap)
    out = np.empty(max(cap, 1), dtype=BLOCK_DTYPE)
    nb, used = C.c_int64(), C.c_int64()
    _lib.check(_lib.lib().ckm_bgzf_blocks(buf.ctypes.data if n else None, n, int(base), out.ctypes.data, cap, C.byref(nb),
                                          C.byref(used)))
    return out[:nb.value].copy(), used.value


class Header(object):
    """names, lengths and `end`: the position of the first record in the decompressed stream."""

    def __init__(self, names, lengths, end, text):
        self.names, self.lengths, self.end, self.text = names, lengths, end, text


def read_header(buf, blocks):
    """The BAM header, inflated with the stdlib zlib from the first blocks (it is small)."""
    stream = bytearray()
    need = 12
    parsed = None
    for k in range(len(blocks)):
        c, n = int(blocks['coffset'][k]), int(blocks['clen'][k])
        blk = bytes(buf[c:c + n])
        xlen, = struct.unpack_from('<H', blk, 10)
        try:
            stream += zlib.decompress(blk[12 + xlen:n - 8], -15)
        except zlib.error as e:
            raise format_error('BAM header: BGZF block at file offset %d does not inflate (%s)' % (c, e))
        if len(stream) < need:
            continue
        if stream[:4] != b'BAM\x01':
            raise format_error('not a BAM file (magic %r)' % bytes(stream[:4]))
        parsed = _parse_header(stream)
        if parsed is not None:
            break
        need = len(stream) + 1
    if parsed is None:
        raise format_error('BAM header is truncated')
    return parsed


def _parse_header(s):
    if len(s) < 12:
        return None
    l_text, = struct.unpack_from('<i', s, 4)
    if l_text < 0:
        raise format_error('BAM header: negative l_text')
    p = 8 + l_text
    if len(s) < p + 4:
        return None
    n_ref, = struct.unpack_from('<i', s, p)
    if n_ref < 0:
        raise format_error('BAM header: negative n_ref')
    p += 4
    names, lens = [], []
    for _ in range(n_ref):
        if len(s) < p + 4:
            return None
        l_name, = struct.unpack_from('<i', s, p)
        if l_name < 1:
            raise format_error('BAM header: reference name length %d' % l_name)
        if len(s) < p + 8 + l_name:
            return None
        names.append(bytes(s[p + 4:p + 3 + l_name]).decode())
        ln, = struct.unpack_from('<i', s, p + 4 + l_name)
        if ln < 1:
            raise format_error('BAM header: reference %s has length %d' % (names[-1], ln))
        lens.append(ln)
        p += 8 + l_name
    return Header(names, lens, p, bytes(s[8:8 + l_text]).decode(errors='replace'))


class Index(object):
    """linear: the non-zero linear-index virtual offsets of every reference (uint64); placed_end: the largest end offset of
    the pseudo-bins (the end of the placed reads), or None when the index has none."""

    def __init__(self, n_ref, linear, placed_end, n_no_coor):
        self.n_ref, self.linear, self.placed_end, self.n_no_coor = n_ref, linear, placed_end, n_no_coor


def read_bai(path):
    with open(path, 'rb') as f:
        b = f.read()
    if b[:4] != b'BAI\x01':
        raise format_error('%s is not a BAI index' % path)
    try:
        n_ref, = struct.unpack_from('<i', b, 4)
        p = 8
        linear, placed_end = [], None
        for _ in range(n_ref):
            n_bin, = struct.unpack_from('<i', b, p)
            p += 4
            for _ in range(n_bin):
                bn, n_chunk = struct.unpack_from('<Ii', b, p)
                p += 8
                if bn == PSEUDO_BIN and n_chunk >= 1:          # metadata: (first, end) offsets of the reference's reads
                    _, end = struct.unpack_from('<QQ', b, p)
                    placed_end = end if placed_end is None else max(placed_end, end)
                p += 16 * n_chunk
            n_intv, = struct.unpack_from('<i', b, p)
            p += 4
            if n_intv:
                lin = np.frombuffer(b, dtype='<u8', count=n_intv, offset=p)
                linear.append(lin[lin != 0])
            p += 8 * n_intv
        if p > len(b):
            raise struct.error('index runs past its end')
        n_no_coor = struct.unpack_from('<Q', b, p)[0] if len(b) >= p + 8 else None
    except (struct.error, ValueError) as e:
        raise format_error('%s is truncated or malformed (%s)' % (path, e))
    lin = np.unique(np.concatenate(linear)) if linear else np.zeros(0, dtype=np.uint64)
    return Index(n_ref, lin.astype(np.uint64), placed_end, n_no_coor)


def voff_to_u(voffs, blocks, U, what):
    """Virtual offsets -> positions in the decompressed stream, U[block(coffset)] + uoffset.  A coffset that is not a block
    start, or a uoffset past its block, means the index does not belong to this file."""
    v = np.asarray(voffs, dtype=np.uint64)
    coff = (v >> np.uint64(16)).astype(np.int64)
    uoff = (v & np.uint64(0xffff)).astype(np.int64)
    k = np.searchsorted(blocks['coffset'], coff)
    ok = (k < len(blocks))
    ok[ok] &= blocks['coffset'][k[ok]] == coff[ok]
    ok[ok] &= uoff[ok] <= blocks['isize'][k[ok]]
    if not ok.all():
        bad = int(v[~ok][0])
        raise format_error('%s: virtual offset %d (file offset %d + %d) is not in a BGZF block of this file; the index '
                           'does not belong to it' % (what, bad, bad >> 16, bad & 0xffff))
    return U[k] + uoff


class Layout(object):
    """What the device needs for one BAM: its block table, the segments to walk (stream positions) and the header."""

    def __init__(self, path):
        self.path = path
        self.index = read_bai(path + '.bai')
        size = os.path.getsize(path)
        self._f = open(path, 'rb')
        self.buf = np.frombuffer(mmap.mmap(self._f.fileno(), 0, access=mmap.ACCESS_READ), dtype=np.uint8) if size \
            else np.zeros(0, dtype=np.uint8)
        # the blocks up to the end of the placed reads; the unplaced tail is neither walked nor inflated
        limit = size
        if self.index.placed_end is not None:
            limit = min(size, (int(self.index.placed_end) >> 16) + MAX_BLOCK)
        self.blocks, used = bgzf_blocks(self.buf[:limit])
        if limit == size and used != size:
            raise format_error('%s: truncated BGZF block at file offset %d' % (path, used))
        self.U = np.zeros(len(self.blocks) + 1, dtype=np.int64)
        self.U[1:] = np.cumsum(self.blocks['isize'])
        self.header = read_header(self.buf, self.blocks)
        if self.index.n_ref != len(self.header.names):
            raise format_error('%s.bai: %d references, the BAM header has %d; the index does not belong to this file'
                               % (path, self.index.n_ref, len(self.header.names)))
        total = int(self.U[-1])
        anchors = voff_to_u(self.index.linear, self.blocks, self.U, path + '.bai')
        self.anchors = np.unique(np.concatenate([[self.header.end], anchors])).astype(np.int64)
        if self.index.placed_end is not None:
            end = int(voff_to_u([self.index.placed_end], self.blocks, self.U, path + '.bai')[0])
        else:
            end = total
        if self.anchors[0] < self.header.end or self.anchors[-1] > end:
            raise format_error('%s.bai: a linear-index offset lies outside the placed reads; the index does not belong to '
                               'this file' % path)
        self.seg_start = self.anchors
        self.seg_end = np.append(self.anchors[1:], end).astype(np.int64)
        keep = self.seg_end > self.seg_start
        self.seg_start, self.seg_end = self.seg_start[keep], self.seg_end[keep]

    def batches(self, budget):
        """Cuts the segments into batches of at most `budget` compressed bytes, always at anchors (a single segment larger
        than the budget is one batch).  Yields (b0, b1, seg_start, seg_end): blocks [b0, b1) and the segments relative to
        U[b0]."""
        if len(self.seg_start) == 0:
            return
        iend = self.U[1:]                                              # end of each block in the stream
        first = np.searchsorted(iend, self.seg_start, side='right')   # block holding the segment's first byte
        last = np.searchsorted(iend, self.seg_end - 1, side='right')  # block holding its last byte
        cend = self.blocks['coffset'][last] + self.blocks['clen'][last]
        j0 = 0
        n = len(first)
        while j0 < n:
            cstart = int(self.blocks['coffset'][first[j0]])
            j1 = int(np.searchsorted(cend, cstart + budget, side='right'))
            j1 = max(j1, j0 + 1)
            b0, b1 = int(first[j0]), int(last[j1 - 1]) + 1
            base = int(self.U[b0])
            yield b0, b1, self.seg_start[j0:j1] - base, self.seg_end[j0:j1] - base
            j0 = j1

    def comp(self, b0, b1):
        """The compressed bytes of blocks [b0, b1) and the file offset of the first."""
        c0 = int(self.blocks['coffset'][b0])
        c1 = int(self.blocks['coffset'][b1 - 1] + self.blocks['clen'][b1 - 1])
        return self.buf[c0:c1], c0

    def close(self):
        self.buf = None
        self._f.close()
