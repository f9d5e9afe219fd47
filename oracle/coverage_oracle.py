"""CPU restatement of `checkm coverage` (checkm/coverage.py:57-287) for the tests and the benchmark's CPU arm: each BGZF
block inflated by the stdlib zlib, the records walked with struct, classified as coverage.py:206-230 does, nine counters
per reference.  The product never imports this module."""
import os
import struct
import zlib

import numpy as np

FIELDS = ('reads', 'duplicates', 'secondary', 'failed_qc', 'failed_align', 'failed_edit', 'failed_pair', 'mapped',
          'aligned_bases')


def bgzf_blocks(raw):
    """[(coffset, clen, isize)] of every BGZF block of the file bytes."""
    out, p = [], 0
    while p < len(raw):
        if raw[p:p + 4] != b'\x1f\x8b\x08\x04':
            raise ValueError('not a BGZF block at file offset %d' % p)
        xlen, = struct.unpack_from('<H', raw, p + 10)
        q, bsize = p + 12, None
        while q < p + 12 + xlen:
            si, slen = raw[q:q + 2], struct.unpack_from('<H', raw, q + 2)[0]
            if si == b'BC':
                bsize, = struct.unpack_from('<H', raw, q + 4)
            q += 4 + slen
        clen = bsize + 1
        isize, = struct.unpack_from('<I', raw, p + clen - 4)
        out.append((p, clen, isize))
        p += clen
    return out


def inflate_block(raw, coffset, clen):
    xlen, = struct.unpack_from('<H', raw, coffset + 10)
    data = zlib.decompress(raw[coffset + 12 + xlen:coffset + clen - 8], -15)
    crc, isize = struct.unpack_from('<II', raw, coffset + clen - 8)
    if zlib.crc32(data) & 0xffffffff != crc or len(data) != isize:
        raise ValueError('BGZF block at file offset %d fails its CRC or ISIZE' % coffset)
    return data


def inflate(path):
    with open(path, 'rb') as f:
        raw = f.read()
    return b''.join(inflate_block(raw, c, n) for c, n, _ in bgzf_blocks(raw))


def parse_header(stream):
    """(names, lengths, position of the first record)."""
    if stream[:4] != b'BAM\x01':
        raise ValueError('not a BAM file')
    l_text, = struct.unpack_from('<i', stream, 4)
    p = 8 + l_text
    n_ref, = struct.unpack_from('<i', stream, p)
    p += 4
    names, lens = [], []
    for _ in range(n_ref):
        l_name, = struct.unpack_from('<i', stream, p)
        names.append(stream[p + 4:p + 4 + l_name - 1].decode())
        lens.append(struct.unpack_from('<i', stream, p + 4 + l_name)[0])
        p += 8 + l_name
    return names, lens, p


def query_alignment_length(cigar, l_seq):
    """pysam's query_alignment_end - query_alignment_start; without SEQ the length the CIGAR's M, I, =, X ops give."""
    if l_seq == 0:
        return sum(n for n, op in cigar if op in (0, 1, 7, 8))
    start, end = 0, l_seq
    for n, op in cigar:
        if op == 4:
            start += n
        elif op != 5:
            break
    for n, op in reversed(cigar[1:]):
        if op == 4:
            end -= n
        elif op != 5:
            break
    return end - start


_INT = {ord('c'): '<b', ord('C'): '<B', ord('s'): '<h', ord('S'): '<H', ord('i'): '<i', ord('I'): '<I'}
_SIZE = {ord('A'): 1, ord('c'): 1, ord('C'): 1, ord('s'): 2, ord('S'): 2, ord('i'): 4, ord('I'): 4, ord('f'): 4}


def nm_tag(stream, a, e):
    while a < e:
        tag, ty = stream[a:a + 2], stream[a + 2]
        a += 3
        if ty in (ord('Z'), ord('H')):
            z = stream.index(b'\x00', a, e)
            if tag == b'NM':
                return None
            a = z + 1
        elif ty == ord('B'):
            sub = stream[a]
            cnt, = struct.unpack_from('<i', stream, a + 1)
            if tag == b'NM':
                return None
            a += 5 + cnt * _SIZE[sub]
        else:
            if tag == b'NM':
                return struct.unpack_from(_INT[ty], stream, a)[0] if ty in _INT else None
            a += _SIZE[ty]
    return None


def counters(path, all_reads=False, min_align=0.98, max_edit=0.02, min_qc=15):
    """(names, lengths, n_ref x 9 int64 counters in FIELDS order) of one BAM file."""
    stream = inflate(path)
    names, lens, p = parse_header(stream)
    cnt = np.zeros((len(names), 9), dtype=np.int64)
    n = len(stream)
    while p + 4 <= n:
        bs, ref, pos, l_name, mapq, _, n_cigar, flag, l_seq = struct.unpack_from('<iiiBBHHHi', stream, p)
        if ref == -1:
            break
        rec = p + 4
        cig = rec + 32 + l_name
        c = cnt[ref]
        c[0] += 1
        if flag & 0x4:
            pass
        elif flag & 0x400:
            c[1] += 1
        elif flag & 0x900:
            c[2] += 1
        elif flag & 0x200 or mapq < min_qc:
            c[3] += 1
        else:
            cigar = [(v >> 4, v & 15) for v in struct.unpack_from('<%dI' % n_cigar, stream, cig)]
            qal = query_alignment_length(cigar, l_seq)
            if qal < min_align * l_seq:
                c[4] += 1
            else:
                nm = nm_tag(stream, cig + 4 * n_cigar + (l_seq + 1) // 2 + l_seq, rec + bs)
                if nm is None:
                    raise ValueError('read %s has no integer NM tag' % stream[cig - l_name:cig - 1].decode())
                if nm > max_edit * l_seq:
                    c[5] += 1
                elif not all_reads and not flag & 0x2:
                    c[6] += 1
                else:
                    c[7] += 1
                    c[8] += qal
        p = rec + bs
    return names, lens, cnt


def _fasta_lengths(path):
    """{id: length} of a plain FASTA file, dict order = first appearance, the last record of a repeated id wins."""
    seqs, name = {}, None
    with open(path) as f:
        for line in f:
            if line.startswith('>'):
                name = line[1:].split(None, 1)[0]
                seqs[name] = 0
            elif name is not None:
                seqs[name] += len(line.rstrip('\r\n'))
    return seqs


def _stem(path):
    return os.path.splitext(os.path.basename(path))[0]


def coverage_tsv(binFiles, bamFiles, all_reads=False, min_align=0.98, max_edit=0.02, min_qc=15):
    """The text coverage.py:97-119 writes (threads=1 order)."""
    bin_of, length = {}, {}
    for bf in binFiles:
        for sid, ln in _fasta_lengths(bf).items():
            bin_of[sid] = _stem(bf)
            length[sid] = ln
    per_bam = []
    for bam in bamFiles:
        names, lens, cnt = counters(bam, all_reads, min_align, max_edit, min_qc)
        per_bam.append({nm: (ln, float(c[8]) / ln, int(c[7])) for nm, ln, c in zip(names, lens, cnt)})
    for info in per_bam:
        for sid, (ln, _, _) in info.items():
            length[sid] = ln
    lines = ['Sequence Id\tBin Id\tSequence length (bp)' + '\tBam Id\tCoverage\tMapped reads' * len(bamFiles)]
    for sid, ln in length.items():
        row = '%s\t%s\t%s' % (sid, bin_of.get(sid, 'unbinned'), ln)
        for bam, info in zip(bamFiles, per_bam):
            _, cov, mapped = info.get(sid, (0, 0, 0))
            row += '\t%s\t%f\t%d' % (_stem(bam), cov, mapped)
        lines.append(row)
    return '\n'.join(lines) + '\n'
