"""Seeded synthetic BAM + BAI files (test and benchmark infrastructure; the product never imports this module).

Records are built with numpy: one at a time for hand-made fixtures (`record`), or as one fixed-layout structured array for
large samples (`bulk_records`).  `write_bam` splits the stream into BGZF blocks compressed with the stdlib zlib as raw
deflate, at a level and strategy chosen per block (level 0 gives stored blocks, Z_FIXED fixed-Huffman ones, the rest
mostly dynamic ones), appends the 28-byte EOF block and writes the BAI the SAM specification describes: bins by
`reg2bin`, chunks, the 16 kbp linear index and the pseudo-bin 37450 with each reference's offset range and read counts."""
import struct
import zlib
from concurrent.futures import ThreadPoolExecutor

import numpy as np

EOF_BLOCK = bytes.fromhex('1f8b08040000000000ff0600424302001b0003000000000000000000')
BLOCK_PAYLOAD = 0xff00                     # htslib's BGZF_BLOCK_SIZE
PSEUDO_BIN = 37450
CIGAR_OPS = 'MIDNSHP=X'
STRATEGIES = {'default': zlib.Z_DEFAULT_STRATEGY, 'filtered': zlib.Z_FILTERED, 'huffman': zlib.Z_HUFFMAN_ONLY,
              'rle': zlib.Z_RLE, 'fixed': zlib.Z_FIXED}


def reg2bin(beg, end):
    """SAM spec 5.3: the bin of the 0-based half-open interval [beg, end) (numpy arrays or ints)."""
    beg = np.asarray(beg, dtype=np.int64)
    end = np.asarray(end, dtype=np.int64) - 1
    out = np.zeros(np.broadcast(beg, end).shape, dtype=np.int64)
    done = np.zeros(out.shape, dtype=bool)
    for shift, off in ((14, 4681), (17, 585), (20, 73), (23, 9), (26, 1)):
        m = ~done & ((beg >> shift) == (end >> shift))
        out = np.where(m, off + (beg >> shift), out)
        done |= m
    return out


def ref_span(cigar):
    """Reference bases a CIGAR consumes (M, D, N, =, X)."""
    return sum(n for n, op in cigar if op in 'MDN=X')


def bgzf_block(payload, level=6, strategy='default'):
    c = zlib.compressobj(level, zlib.DEFLATED, -15, 9, STRATEGIES[strategy])
    cdata = c.compress(payload) + c.flush()
    bsize = 18 + len(cdata) + 8 - 1
    if bsize > 65535:
        raise ValueError('payload does not fit one BGZF block')
    head = b'\x1f\x8b\x08\x04\x00\x00\x00\x00\x00\xff\x06\x00BC\x02\x00' + struct.pack('<H', bsize)
    return head + cdata + struct.pack('<II', zlib.crc32(payload) & 0xffffffff, len(payload))


def header_bytes(refs, text=''):
    t = text.encode()
    out = [b'BAM\x01', struct.pack('<i', len(t)), t, struct.pack('<i', len(refs))]
    for name, ln in refs:
        n = name.encode() + b'\x00'
        out += [struct.pack('<i', len(n)), n, struct.pack('<i', ln)]
    return b''.join(out)


def aux_int(tag, value, typ):
    fmt = {'c': '<b', 'C': '<B', 's': '<h', 'S': '<H', 'i': '<i', 'I': '<I'}[typ]
    return tag.encode() + typ.encode() + struct.pack(fmt, value)


def record(rng, ref, pos, name, flag=0x3, mapq=60, cigar=((100, 'M'),), l_seq=None, nm=(0, 'C'), aux=b'',
           next_ref=-1, next_pos=-1, tlen=0):
    """One BAM record (with its block_size) and its reference end.  l_seq defaults to the query length of the CIGAR;
    nm=None leaves out the NM tag."""
    if l_seq is None:
        l_seq = sum(n for n, op in cigar if op in 'MIS=X')
    span = ref_span(cigar)
    end = pos + (span if span > 0 and not flag & 0x4 else 1)
    b = int(reg2bin(max(pos, 0), max(end, pos + 1))) if pos >= 0 else 4680
    nb = name.encode() + b'\x00'
    cig = b''.join(struct.pack('<I', n << 4 | CIGAR_OPS.index(op)) for n, op in cigar)
    seq = rng.integers(0, 256, size=(l_seq + 1) // 2, dtype=np.uint8).tobytes()
    qual = rng.integers(20, 41, size=l_seq, dtype=np.uint8).tobytes()
    tags = (aux_int('NM', nm[0], nm[1]) if nm is not None else b'') + aux
    body = struct.pack('<iiBBHHHiiii', ref, pos, len(nb), mapq, b, len(cigar), flag, l_seq, next_ref, next_pos, tlen)
    body += nb + cig + seq + qual + tags
    return struct.pack('<i', len(body)) + body, end


def bulk_records(rng, ref_lens, reads_per_ref, read_len=150, name_len=15):
    """Fixed-layout records sorted by (ref, pos): CIGAR `aS mM bS` (a, b in 1..4, so every read has soft clips), flags and
    MAPQ drawn so that every filter branch fires, an NM:C tag.  Returns (stream bytes, ref, pos, end)."""
    ref_lens = np.asarray(ref_lens, dtype=np.int64)
    counts = np.asarray(reads_per_ref, dtype=np.int64)
    n = int(counts.sum())
    ref = np.repeat(np.arange(len(ref_lens), dtype=np.int32), counts)
    a = rng.integers(1, 5, size=n)
    b = rng.integers(1, 5, size=n)
    m = read_len - a - b
    pos = (rng.random(n) * np.maximum(ref_lens[ref] - m, 1)).astype(np.int64)
    order = np.lexsort((pos, ref))
    pos, a, b, m = pos[order], a[order], b[order], m[order]
    end = pos + m
    l_seq_b = (read_len + 1) // 2
    dt = np.dtype([('bs', '<i4'), ('ref', '<i4'), ('pos', '<i4'), ('l_name', 'u1'), ('mapq', 'u1'), ('bin', '<u2'),
                   ('n_cigar', '<u2'), ('flag', '<u2'), ('l_seq', '<i4'), ('nref', '<i4'), ('npos', '<i4'), ('tlen', '<i4'),
                   ('name', 'S%d' % name_len), ('cigar', '<u4', (3,)), ('seq', 'u1', (l_seq_b,)), ('qual', 'u1', (read_len,)),
                   ('nm_tag', 'S3'), ('nm', 'u1')])
    r = np.zeros(n, dtype=dt)
    r['bs'] = dt.itemsize - 4
    r['ref'] = ref
    r['pos'] = pos
    r['l_name'] = name_len
    u = rng.random(n)
    r['mapq'] = np.where(u < 0.05, rng.integers(0, 15, size=n), 60)
    r['bin'] = reg2bin(pos, end)
    r['n_cigar'] = 3
    f = rng.random(n)
    flag = np.full(n, 0x3, dtype=np.int64)
    flag = np.where(f < 0.02, 0x1 | 0x4, flag)                       # placed unmapped
    flag = np.where((f >= 0.02) & (f < 0.05), 0x403, flag)           # duplicate
    flag = np.where((f >= 0.05) & (f < 0.07), 0x103, flag)           # secondary
    flag = np.where((f >= 0.07) & (f < 0.08), 0x803, flag)           # supplementary
    flag = np.where((f >= 0.08) & (f < 0.09), 0x203, flag)           # QC fail
    flag = np.where((f >= 0.09) & (f < 0.14), 0x1, flag)             # not properly paired
    r['flag'] = flag
    r['l_seq'] = read_len
    r['nref'] = ref
    r['npos'] = pos
    names = np.char.add(b'r', np.char.zfill(np.arange(n).astype('S%d' % (name_len - 2)), name_len - 2))
    r['name'] = names
    r['cigar'][:, 0] = (a << 4) | 4
    r['cigar'][:, 1] = (m << 4) | 0
    r['cigar'][:, 2] = (b << 4) | 4
    r['seq'] = rng.choice(np.array([0x11, 0x12, 0x14, 0x18, 0x21, 0x22, 0x24, 0x28, 0x41, 0x42, 0x44, 0x48, 0x81, 0x82, 0x84, 0x88],
                                   dtype=np.uint8), size=(n, l_seq_b))
    r['qual'] = rng.integers(30, 38, size=(n, read_len), dtype=np.uint8)
    r['nm_tag'] = b'NMC'
    r['nm'] = np.minimum(rng.geometric(0.5, size=n) - 1, 255)
    end = np.where(flag & 0x4, pos + 1, end)
    r['bin'] = reg2bin(pos, end)
    return r.tobytes(), ref.astype(np.int64), pos, end


def _compress_all(payloads, levels, strategies, threads):
    jobs = [(p, levels[i % len(levels)], strategies[i % len(strategies)]) for i, p in enumerate(payloads)]
    if threads <= 1 or len(jobs) < 64:
        return [bgzf_block(*j) for j in jobs]
    with ThreadPoolExecutor(threads) as ex:                      # zlib releases the GIL
        return list(ex.map(lambda j: bgzf_block(*j), jobs, chunksize=64))


def write_bam(path, refs, records, rec_ref, rec_pos, rec_end, rec_unmapped=None, n_unplaced=0, unplaced=b'', text='',
              levels=(6,), strategies=('default',), cuts=None, payload=BLOCK_PAYLOAD, fill_linear=True, pseudo_bin=True,
              threads=1, index=True):
    """Writes `path` and `path.bai`.  records: the placed records' bytes, sorted by (ref, pos), with per-record ref, pos
    and reference end (exclusive); unplaced: the bytes of the n_unplaced records with refID -1 that follow them.  Blocks:
    the header in blocks of its own, then `payload` bytes each, also cut at the stream positions in `cuts` (records then
    span blocks).
    Returns the block table (coffset, clen, isize) and the stream positions of the records."""
    head = header_bytes(refs, text)
    rec_ref = np.asarray(rec_ref, dtype=np.int64)
    rec_pos = np.asarray(rec_pos, dtype=np.int64)
    rec_end = np.asarray(rec_end, dtype=np.int64)
    nrec = len(rec_ref)
    body = records if isinstance(records, (bytes, bytearray)) else b''.join(records)
    if isinstance(records, (bytes, bytearray)):
        sizes = None
    else:
        sizes = np.array([len(r) for r in records], dtype=np.int64)
    stream = head + body + unplaced
    total = len(stream)
    if sizes is None:
        rsize = len(body) // nrec if nrec else 0
        starts = len(head) + np.arange(nrec, dtype=np.int64) * rsize
        ends = starts + rsize
    else:
        starts = len(head) + np.concatenate([[0], np.cumsum(sizes)[:-1]]).astype(np.int64) if nrec else np.zeros(0, np.int64)
        ends = starts + sizes
    bounds = {0, len(head), total}
    bounds.update(range(0, len(head), payload))
    bounds.update(range(len(head), total, payload))
    for c in (cuts or ()):
        bounds.add(int(c))
    bounds = sorted(b for b in bounds if 0 <= b <= total)
    payloads = [stream[a:b] for a, b in zip(bounds[:-1], bounds[1:]) if b > a]
    blocks = _compress_all(payloads, list(levels), list(strategies), threads)
    coff = np.zeros(len(blocks) + 1, dtype=np.int64)
    coff[1:] = np.cumsum([len(b) for b in blocks])
    ustart = np.zeros(len(blocks) + 1, dtype=np.int64)
    ustart[1:] = np.cumsum([len(p) for p in payloads])
    with open(path, 'wb') as f:
        for b in blocks:
            f.write(b)
        f.write(EOF_BLOCK)
    eof_coff = int(coff[-1])
    table = np.array([(int(coff[i]), len(blocks[i]), len(payloads[i])) for i in range(len(blocks))] + [(eof_coff, 28, 0)],
                     dtype=[('coffset', '<i8'), ('clen', '<i4'), ('isize', '<i4')])

    def voff(u):
        u = np.asarray(u, dtype=np.int64)
        k = np.searchsorted(ustart[:-1], u, side='right') - 1
        at_end = u >= total
        c = np.where(at_end, eof_coff, coff[np.clip(k, 0, len(blocks) - 1)])
        off = np.where(at_end, 0, u - ustart[np.clip(k, 0, len(blocks) - 1)])
        return (c.astype(np.uint64) << np.uint64(16)) | off.astype(np.uint64)

    if index:
        write_bai(path + '.bai', len(refs), rec_ref, rec_pos, rec_end, voff(starts), voff(ends),
                  rec_unmapped if rec_unmapped is not None else np.zeros(nrec, dtype=bool), n_unplaced, fill_linear, pseudo_bin)
    return table, starts


def write_bai(path, n_ref, ref, pos, end, vbeg, vend, unmapped, n_unplaced, fill_linear=True, pseudo_bin=True):
    n = len(ref)
    binv = reg2bin(pos, np.maximum(end, pos + 1)) if n else np.zeros(0, np.int64)
    new_chunk = np.ones(n, dtype=bool)
    if n > 1:
        new_chunk[1:] = (ref[1:] != ref[:-1]) | (binv[1:] != binv[:-1])
    cstart = np.flatnonzero(new_chunk)
    cend = np.concatenate([cstart[1:], [n]]) - 1
    w0 = pos >> 14
    w1 = (np.maximum(end, pos + 1) - 1) >> 14
    out = [b'BAI\x01', struct.pack('<i', n_ref)]
    ref_first = np.searchsorted(ref, np.arange(n_ref + 1)) if n else np.zeros(n_ref + 1, dtype=np.int64)
    chunk_ref = ref[cstart] if n else np.zeros(0, np.int64)
    chunk_lo = np.searchsorted(chunk_ref, np.arange(n_ref + 1))
    for r in range(n_ref):
        a, b = int(ref_first[r]), int(ref_first[r + 1])
        bins = {}
        for c in range(int(chunk_lo[r]), int(chunk_lo[r + 1])):
            i, j = int(cstart[c]), int(cend[c])
            bins.setdefault(int(binv[i]), []).append((int(vbeg[i]), int(vend[j])))
        if b > a and pseudo_bin:
            um = int(np.count_nonzero(unmapped[a:b]))
            bins[PSEUDO_BIN] = [(int(vbeg[a]), int(vend[b - 1])), (b - a - um, um)]
        out.append(struct.pack('<i', len(bins)))
        for bn, chunks in bins.items():
            out.append(struct.pack('<Ii', bn, len(chunks)))
            out.append(np.array(chunks, dtype='<u8').tobytes())
        if b > a:
            nint = int(w1[a:b].max()) + 1
            lin = np.full(nint, np.iinfo(np.uint64).max, dtype=np.uint64)
            np.minimum.at(lin, w0[a:b], vbeg[a:b])
            span = w1[a:b] - w0[a:b]
            for k in np.flatnonzero(span > 0):
                for w in range(int(w0[a + k]) + 1, int(w1[a + k]) + 1):
                    lin[w] = min(lin[w], vbeg[a + k])
            empty = lin == np.iinfo(np.uint64).max
            lin[empty] = 0
            if fill_linear:                                      # htslib: an empty window takes its predecessor's offset
                for w in range(1, nint):
                    if lin[w] == 0:
                        lin[w] = lin[w - 1]
        else:
            lin = np.zeros(0, dtype=np.uint64)
        out.append(struct.pack('<i', len(lin)))
        out.append(lin.astype('<u8').tobytes())
    out.append(struct.pack('<Q', n_unplaced))
    with open(path, 'wb') as f:
        f.write(b''.join(out))
