"""Fixtures for `checkm unbinned` and `checkm profile`, and what the REFERENCE's own Unbinned.run and Profile.run write for
them (checkm/unbinned.py, checkm/profile.py, imported read-only from /root/reference).  Run in the build container only:

    python tests/golden/make_unbinned_goldens.py

Writes tests/golden/unbinned/:
  inputs/asm.fna(.gz)        the assembly: CRLF line ends, a lone CR, blank lines, a last line without a newline (its last
                             base is dropped); lower case, U, IUPAC codes, N runs, a space inside a sequence line; an id
                             repeated in the assembly (first position, last content); headers with leading blanks or a tab,
                             and \\x1c, U+00A0, U+3000 and a tab as separators; a non-ASCII id character; a 0-length record
                             and a record of only N, both binned
  inputs/bin1.fna            bdup twice (a repeat inside one bin), bx, a 0-length record, an id absent from the assembly
  inputs/bin2.fna.gz         bx again (an id in two bins), the N-only record
  inputs/cov_*.tsv           synthetic coverage files for `profile`: one and three BAMs, bin ids sorting before and after
                             `unbinned`, no unbinned row, a bin without reads in one BAM, every binned bin without reads in
                             one BAM (the normalisation falls back to 0)
  expected/unbinned_<case>.fna / .tsv   Unbinned.run's two files per case; cases.json holds each case's bins, assembly,
                             minSeqLen and INFO lines
  expected/profile_<name>_{tab,table}.txt   Profile.run on every inputs/cov_*.tsv and on the four
                             tests/golden/coverage/coverage_*.tsv files, in both table styles"""
import gzip
import json
import logging
import os
import shutil
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, 'unbinned')
sys.path.insert(0, '/root/reference')

ASM = (b'>c1 desc one\r\n'
       b'ACGTACGTNNNNacgtu\r\n'
       b'\r\n'
       b'>  c2\tmore text\n'
       b'GGGCCCAAATTT\r\n'
       b'\n'
       b'   \n'
       b'RYKMSWBDHVN\n'
       b'ac gu\r\n'
       b'>c3\x1cx\n'
       b'ACGU\rACGT\r'
       b'>b1\n'
       b'ACGTACGTAC\n'
       b'>c4\xc2\xa0tail\n'
       b'NNNNNNNNNNACGTNNNNNNNNNNNNGGCC\n'
       b'>zero\n'
       b'>c5\xe3\x80\x80x y\n'
       + b'acgtacgtac' * 9 + b'\n'
       + b'>c\xc3\xa9\x1cd e\n'
       b'GATTACA\n'
       b'>nonly\n'
       b'NNNNNNNN\n'
       b'>bdup\n'
       b'ACGT\n'
       b'>c1 repeated\n'
       b'TTTTGGGGCCCCAAAT\n'
       b'>\tc7 x\n'
       b'ggccggccnnnnATATATATAT\n'
       b'>bx\n'
       b'CCCC\n'
       b'>clast\n'
       b'ACGTACGTTA')
BIN1 = (b'>bdup first\nACGTACGTACGT\n'
        b'>b1\nACGTACGTAC\n'
        b'>bx\r\nAAAAAA\r\n'
        b'>zero\n'
        b'>ghost not in the assembly\nGGGGGGGGGGGG\n'
        b'>bdup second\nACG\n')
BIN2 = b'>bx\nCCCCCCCCCCCCCCCCCCCC\n>nonly\nNNNNNNNN\n'
L = 28                                 # c2's length: 12 + 11 + 5
CASES = [('base', ['bin1.fna', 'bin2.fna.gz'], 'asm.fna', 0),
         ('negative', ['bin1.fna', 'bin2.fna.gz'], 'asm.fna', -5),
         ('below', ['bin1.fna', 'bin2.fna.gz'], 'asm.fna', L - 1),
         ('equal', ['bin1.fna', 'bin2.fna.gz'], 'asm.fna', L),
         ('above', ['bin1.fna', 'bin2.fna.gz'], 'asm.fna', L + 1),
         ('gzip', ['bin2.fna.gz', 'bin1.fna'], 'asm.fna.gz', 10)]

COV_HEADER = 'Sequence Id\tBin Id\tSequence length (bp)'


def coverage_file(bams, rows):
    """rows: (seq, bin, length, [mapped reads per BAM])"""
    lines = [COV_HEADER + ''.join('\tBam Id\tCoverage\tMapped reads' for _ in bams)]
    for seq, binId, length, reads in rows:
        lines.append('%s\t%s\t%d' % (seq, binId, length) + ''.join('\t%s\t%f\t%d' % (b, r * 150.0 / length, r)
                                                                     for b, r in zip(bams, reads)))
    return '\n'.join(lines) + '\n'


COVERAGE = {
    'one_bam': coverage_file(['s1'], [('a', 'bin1', 5000, [40]), ('b', 'unbinned', 800, [7]), ('c', 'Abin', 1200, [13]),
                                      ('d', 'bin1', 2500, [19]), ('e', 'zeta', 3100, [3])]),
    'three_bams': coverage_file(['s1', 's2', 's3'], [('a', 'bin1', 5000, [40, 0, 12]), ('b', 'unbinned', 800, [7, 5, 1]),
                                                     ('c', 'Abin', 1200, [13, 9, 0]), ('d', 'zeta', 3100, [3, 1, 8]),
                                                     ('e', 'unbinned', 333, [2, 0, 4]), ('f', 'Abin', 77, [1, 1, 1])]),
    'no_unbinned': coverage_file(['s1', 's2'], [('a', 'bin1', 5000, [40, 10]), ('c', 'bin2', 1200, [13, 0]),
                                                ('d', 'bin3', 3100, [3, 5])]),
    'norm_zero': coverage_file(['s1', 's2'], [('a', 'bin1', 5000, [40, 0]), ('b', 'unbinned', 800, [7, 11]),
                                              ('c', 'zz', 1200, [13, 0])]),
}


def main():
    from checkm.unbinned import Unbinned
    from checkm.profile import Profile

    inputs, expected = os.path.join(OUT, 'inputs'), os.path.join(OUT, 'expected')
    shutil.rmtree(inputs, ignore_errors=True)              # README.md beside them stays
    shutil.rmtree(expected, ignore_errors=True)
    os.makedirs(inputs)
    os.makedirs(expected)
    for name, raw in (('asm.fna', ASM), ('bin1.fna', BIN1)):
        with open(os.path.join(inputs, name), 'wb') as f:
            f.write(raw)
    for name, raw in (('asm.fna.gz', ASM), ('bin2.fna.gz', BIN2)):
        with gzip.GzipFile(os.path.join(inputs, name), 'wb', mtime=0) as f:
            f.write(raw)
    for name, text in COVERAGE.items():
        with open(os.path.join(inputs, 'cov_%s.tsv' % name), 'w') as f:
            f.write(text)

    logger = logging.getLogger('timestamp')
    logger.setLevel(logging.INFO)
    records = []

    class Keep(logging.Handler):
        def emit(self, record):
            records.append(record.getMessage())
    logger.addHandler(Keep())

    cases = {}
    with tempfile.TemporaryDirectory() as tmp:
        for name, bins, asm, min_len in CASES:
            del records[:]
            fna, tsv = os.path.join(tmp, name + '.fna'), os.path.join(tmp, name + '.tsv')
            Unbinned().run([os.path.join(inputs, b) for b in bins], os.path.join(inputs, asm), fna, tsv, min_len)
            shutil.copyfile(fna, os.path.join(expected, 'unbinned_%s.fna' % name))
            shutil.copyfile(tsv, os.path.join(expected, 'unbinned_%s.tsv' % name))
            cases[name] = {'bins': bins, 'seqFile': asm, 'minSeqLen': min_len, 'info': list(records)}
    with open(os.path.join(OUT, 'cases.json'), 'w') as f:
        json.dump(cases, f, indent=1, ensure_ascii=False)
        f.write('\n')

    covs = [os.path.join(inputs, 'cov_%s.tsv' % n) for n in COVERAGE]
    covs += [os.path.join(HERE, 'coverage', 'coverage_%s.tsv' % o) for o in ('all_reads', 'defaults', 'loose', 'strict')]
    for path in covs:
        stem = os.path.basename(path)[:-4]
        for style, tab in (('tab', True), ('table', False)):
            Profile().run(path, os.path.join(expected, 'profile_%s_%s.txt' % (stem, style)), tab)


if __name__ == '__main__':
    main()
