"""Protein FASTA -> digitised residue stream (the `genes.faa` reader that sat inside hmmsearch; SURVEY.md 8f1).

One pass in the library (`ckm_fasta_parse`): residue codes, CSR offsets and the header lines; names and descriptions are
split out of the header lines here."""
import ctypes as C
import gzip

import numpy as np

from . import _lib


def read_fasta(path):
    """Returns names, descriptions (header text after the first blank), the digitised residues and the CSR offsets."""
    opener = gzip.open if path.endswith('.gz') else open
    with opener(path, 'rb') as f:
        raw = f.read()
    return parse_fasta(raw)


def parse_fasta(raw):
    n = len(raw)
    max_rec = int(np.count_nonzero(np.frombuffer(raw, dtype=np.uint8) == 62))     # '>' bytes: an upper bound on the records
    residues = np.empty(max(n, 1), dtype=np.uint8)
    offsets = np.zeros(max_rec + 1, dtype=np.int64)
    headers = C.create_string_buffer(max(n, 1))
    nrec, nres, hb = C.c_int32(), C.c_int64(), C.c_int64()
    _lib.check(_lib.lib().ckm_fasta_parse(raw, n, residues.ctypes.data, offsets.ctypes.data, max_rec, headers, max(n, 1),
                                          C.byref(nrec), C.byref(nres), C.byref(hb)))
    if nrec.value == 0:
        return [], [], np.zeros(0, dtype=np.uint8), np.zeros(1, dtype=np.int64)
    names, descs = [], []
    for line in headers.raw[:hb.value].decode('utf-8', 'replace').split('\n'):
        parts = line.split(None, 1)
        names.append(parts[0] if parts else '')
        descs.append(parts[1] if len(parts) > 1 else '')
    return names, descs, residues[:nres.value].copy(), offsets[:nrec.value + 1].copy()


def read_bytes(path):
    opener = gzip.open if path.endswith('.gz') else open
    with opener(path, 'rb') as f:
        return f.read()


def scan_nt_raw(raw):
    """ckm_fasta_scan_nt on one file's bytes: the header lines (text after '>', joined by '\\n', as bytes), the byte
    buffer, and the start (a multiple of 64) and length of every record, repeated ids included."""
    n = len(raw)
    max_rec = int(np.count_nonzero(np.frombuffer(raw, dtype=np.uint8) == 62))     # '>' bytes: an upper bound on the records
    data = np.empty(n + 64 * (max_rec + 1), dtype=np.uint8)
    starts = np.zeros(max(max_rec, 1), dtype=np.int64)
    lens = np.zeros(max(max_rec, 1), dtype=np.int64)
    headers = C.create_string_buffer(max(n, 1))
    nrec, used, hb = C.c_int32(), C.c_int64(), C.c_int64()
    _lib.check(_lib.lib().ckm_fasta_scan_nt(raw, n, data.ctypes.data, data.size, starts.ctypes.data, lens.ctypes.data, max_rec,
                                            headers, max(n, 1), C.byref(nrec), C.byref(used), C.byref(hb)))
    k = nrec.value
    return headers.raw[:hb.value], data[:used.value], starts[:k], lens[:k]


def scan_nt_fasta(raw):
    """A nucleotide FASTA file as the reference's readFasta sees it (checkm/util/seqUtils.py:180-211), laid out for the
    device scan: returns ids (first token of each header line), the byte buffer, and the start (a multiple of 64) and
    length of every record.  A record whose id repeats replaces the earlier one, as in the reference's dict."""
    hdr, data, starts, lens = scan_nt_raw(raw)
    k = len(lens)
    if k == 0:
        return [], data[:0], starts, lens
    ids = [line.split(None, 1)[0] for line in hdr.decode('utf-8', 'replace').split('\n')]   # IndexError: header without an id
    if len(set(ids)) != k:
        last = {}
        for i, name in enumerate(ids):
            last[name] = i                             # dict order = first appearance, content = last appearance
        keep = np.array(list(last.values()), dtype=np.int64)
        ids, starts, lens = list(last.keys()), starts[keep], lens[keep]
    return ids, data, starts, lens
