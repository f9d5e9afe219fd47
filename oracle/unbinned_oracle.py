"""Pure-Python restatement of `checkm unbinned` (checkm/unbinned.py:33-85 with util/seqUtils.py:180-211,279-286) over the
raw bytes of the files, with its own FASTA reader: the reference for tests that run where the reference is not installed.

run(bin_raws, seq_raw, min_len) -> (fasta bytes, stats bytes, INFO lines), or raises UnbinnedError naming the case."""
import io


class UnbinnedError(Exception):
    pass


def read_fasta(raw):
    """{id: sequence} as readFasta builds it: universal newlines, blank lines skipped, first position and last content of
    a repeated id, the last character of every sequence line dropped."""
    try:
        text = raw.decode('utf-8')
    except UnicodeDecodeError as e:
        raise UnbinnedError('not UTF-8: %s' % e)
    seqs, seqId = {}, None
    for line in io.StringIO(text, newline=None):
        if not line.strip():
            continue
        if line[0] == '>':
            parts = line[1:].split(None, 1)
            if not parts:
                raise UnbinnedError('header without an id')
            seqId = parts[0]
            seqs[seqId] = []
        else:
            if seqId is None:
                raise UnbinnedError('sequence before the first header')
            seqs[seqId].append(line[0:-1])
    return {k: ''.join(v) for k, v in seqs.items()}


def base_count(seq):
    s = seq.upper()
    return s.count('A'), s.count('C'), s.count('G'), s.count('T') + s.count('U')


def run(bin_raws, seq_raw, min_len):
    info = ['Reading binned sequences.']
    binned, binned_bases = {}, 0
    for raw in bin_raws:
        seqs = read_fasta(raw)
        binned.update(seqs)
        binned_bases += sum(len(s) for s in seqs.values())
    info.append('  Read %d (%.2f Mbp) binned sequences.' % (len(binned), float(binned_bases) / 1e6))
    info.append('Reading all sequences.')
    allSeqs = read_fasta(seq_raw)
    total = sum(len(s) for s in allSeqs.values())
    info.append('  Read %d (%.2f Mbp) sequences.' % (len(allSeqs), float(total) / 1e6))
    info.append('Identifying unbinned sequences >= %d bp.' % min_len)
    fasta, stats = [], ['Sequence Id\tLength\tGC\n']
    count = bases = 0
    for seqId, seq in allSeqs.items():
        if seqId in binned or len(seq) < min_len:
            continue
        a, c, g, t = base_count(seq)
        if a + c + g + t == 0:
            raise UnbinnedError('sequence %s has no A, C, G, T or U' % seqId)
        count += 1
        bases += len(seq)
        fasta.append('>' + seqId + '\n' + seq + '\n')
        stats.append('%s\t%d\t%.2f\n' % (seqId, len(seq), float(g + c) * 100 / (a + c + g + t)))
    info.append('  Identified %d (%.2f Mbp) unbinned sequences.' % (count, float(bases) / 1e6))
    if not allSeqs:
        raise UnbinnedError('no sequences')
    info.append('Percentage of unbinned sequences: %.2f%%' % (count * 100.0 / len(allSeqs)))
    if total == 0:
        raise UnbinnedError('no bases')
    info.append('Percentage of unbinned bases: %.2f%%' % (bases * 100.0 / total))
    return ''.join(fasta).encode('utf-8'), ''.join(stats).encode('utf-8'), info
