"""Fixture sequences for the genomic-signature row (`checkm tetra`) and what the REFERENCE's own GenomicSignatures computes
for them.

Run in the build container (needs /root/reference):  python tests/golden/make_tetra_goldens.py
Writes tests/golden/tetra/:
  fixture.fna             sequences of length 0..5, all-N, lower case, U, IUPAC codes and '*', the self-complementary
                          4-mers, a 6 kb homopolymer (one column 1.0), dinucleotide repeats, and random sequences with
                          invalid bytes placed around the 16-byte lane, 64-byte chunk, 512-byte block and 2 KB row edges
  <file>.tetra.tsv        GenomicSignatures(4, 1).calculate(<file>, ...) for fixture.fna and the three binstats fixture
                          bins (tests/golden/binstats/bins: gzip, CRLF, a repeated id, a last line without newline)
  signatures.json         {"order": {K: canonicalKmerOrder()}, "seqSignature": {K: [[seq, [repr(float(v)), ...]], ...]}}
                          for K = 1..4
At threads=1 the reference writes the sequences in file order."""
import json
import logging
import os
import shutil
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, 'tetra')
BINS = os.path.join(HERE, 'binstats', 'bins')
sys.path.insert(0, '/root/reference')

PALINDROMES = [a + b + {'A': 'T', 'C': 'G', 'G': 'C', 'T': 'A'}[b] + {'A': 'T', 'C': 'G', 'G': 'C', 'T': 'A'}[a] for a in 'ACGT' for b in 'ACGT']


def random_dna(rng, n, alphabet=b'ACGT'):
    return bytearray(rng.choice(np.frombuffer(alphabet, dtype=np.uint8), size=n).tobytes())


def fixture(rng):
    recs = []
    for n in range(0, 6):
        recs.append(('len%d' % n, random_dna(rng, n)))
    recs.append(('allN', bytearray(b'N' * 300)))
    recs.append(('alln_lower', bytearray(b'n' * 70)))
    recs.append(('lower', random_dna(rng, 500, b'acgtACGT')))
    recs.append(('with_U', random_dna(rng, 400, b'ACGTUu')))
    recs.append(('iupac', random_dna(rng, 600, b'ACGTRYKMSWBDHVN*-.X')))
    recs.append(('palindromes', bytearray(''.join(PALINDROMES).encode())))
    recs.append(('palindromes_split', bytearray('N'.join(PALINDROMES).encode())))
    recs.append(('ACGT', bytearray(b'ACGT')))
    recs.append(('homopolymer', bytearray(b'A' * 6000)))
    recs.append(('homopolymer_g', bytearray(b'g' * 3000)))
    recs.append(('dinucleotide', bytearray(b'AC' * 2500)))
    recs.append(('trinucleotide', bytearray(b'GAT' * 1500)))
    # invalid bytes around the edges the device scan works in: 16-byte lanes, 64-byte chunks, 512-byte blocks, 2 KB rows
    for name, n in (('edges_a', 9000), ('edges_b', 20000)):
        s = random_dna(rng, n, b'ACGTacgt')
        for edge in (16, 64, 512, 2048, 4096, 6144, 8192, 16384):
            if edge + 4 >= n:
                continue
            d = int(rng.integers(-4, 5))
            s[edge + d] = int(rng.choice(list(b'NUR*n')))
        recs.append((name, s))
    for n in (2047, 2048, 2049, 2051, 4095, 4096, 4097):
        recs.append(('row%d' % n, random_dna(rng, n)))
    recs.append(('long', random_dna(rng, 70000)))
    return recs


def write_fasta(path, recs, rng):
    with open(path, 'w') as fh:
        for name, s in recs:
            fh.write('>%s some description\n' % name)
            w = int(rng.choice([50, 60, 61, 80, 1000]))
            text = s.decode()
            for i in range(0, len(text), w):
                fh.write(text[i:i + w] + '\n')


def main():
    rng = np.random.default_rng(20261015)
    shutil.rmtree(OUT, ignore_errors=True)
    os.makedirs(OUT)
    recs = fixture(rng)
    write_fasta(os.path.join(OUT, 'fixture.fna'), recs, rng)

    os.environ['CHECKM_DATA_PATH'] = tempfile.mkdtemp()
    logging.getLogger('timestamp').setLevel(logging.WARNING)
    from checkm.genomicSignatures import GenomicSignatures
    files = {'fixture.fna': os.path.join(OUT, 'fixture.fna')}
    for f in ('bin1.fna', 'bin2.fna.gz', 'bin3.fna'):
        files[f] = os.path.join(BINS, f)
    for name, path in files.items():
        GenomicSignatures(4, 1).calculate(path, os.path.join(OUT, name.replace('.gz', '') + '.tetra.tsv'))

    chosen = [s.decode() for _, s in recs[:16]] + ['', 'A', 'ACGT', 'acgt', 'ACGU', 'NNNNACGTNNNN', 'TTTT', 'GATC' * 10,
                                                   'CCCCCCCCCCCCCCCCG', 'ATATATATATAT', 'aCgTnAcGtN']
    sigs, order = {}, {}
    for K in (1, 2, 3, 4):
        gs = GenomicSignatures(K, 1)
        order[K] = list(gs.canonicalKmerOrder())
        with np.errstate(invalid='ignore'):
            sigs[K] = [[s, [repr(float(v)) for v in gs.seqSignature(s)]] for s in chosen]
    with open(os.path.join(OUT, 'signatures.json'), 'w') as fh:
        json.dump({'order': order, 'seqSignature': sigs}, fh, indent=0)
    print(sum(os.path.getsize(os.path.join(OUT, f)) for f in os.listdir(OUT)), 'bytes in', OUT)


if __name__ == '__main__':
    main()
