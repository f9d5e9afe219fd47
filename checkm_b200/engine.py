"""Thin Python object layer over the C ABI: Engine / Models / SeqDb.  All computation happens in libckm.so."""
import ctypes as C
import numpy as np

from . import _lib
from ._lib import check, Hit, Stats, ModelInfo

ALPHABET = "ACDEFGHIKLMNPQRSTVWY-BJZOUX*~"

HIT_DTYPE = np.dtype([(n, {C.c_int32: np.int32, C.c_float: np.float32, C.c_double: np.float64}[t]) for n, t in Hit._fields_],
                     align=True)
assert HIT_DTYPE.itemsize == C.sizeof(Hit)
MERGE_PAIR_DTYPE = np.dtype([('i', np.int32), ('j', np.int32), ('p', np.int32), ('s', np.int32)])   # ckm_merge_pair


def digitize(text):
    """ASCII protein text -> uint8 codes (unknown symbols become X), via the library."""
    b = text.encode() if isinstance(text, str) else bytes(text)
    out = np.empty(len(b), dtype=np.uint8)
    check(_lib.lib().ckm_digitize(b, len(b), out.ctypes.data))
    return out


class Signatures:
    """A profile matrix (n x 136 float64) resident on the device for the outlier calls of one run (ckm_sigs_create)."""

    def __init__(self, engine, values):
        values = np.ascontiguousarray(values, dtype=np.float64)
        if values.ndim != 2 or values.shape[1] != 136 or values.shape[0] < 1:
            raise ValueError("Signatures: values must be n x 136 with n >= 1")
        self.n = values.shape[0]
        self._h = C.c_void_p()
        check(_lib.lib().ckm_sigs_create(engine._h, values.ctypes.data, self.n, C.byref(self._h)))

    def close(self):
        if self._h:
            _lib.lib().ckm_sigs_free(self._h)
            self._h = C.c_void_p()


class Models:
    def __init__(self, engine, path):
        self.engine = engine
        self._h = C.c_void_p()
        check(_lib.lib().ckm_models_load(engine._h, path.encode(), C.byref(self._h)))
        self.path = path
        self.n = _lib.lib().ckm_models_count(self._h)
        self._info = None

    def info(self):
        if self._info is None:
            out = []
            for i in range(self.n):
                mi = ModelInfo()
                check(_lib.lib().ckm_models_info(self._h, i, C.byref(mi)))
                out.append(mi)
            self._info = out
        return self._info

    def find(self, key):
        return _lib.lib().ckm_models_find(self._h, key.encode())

    def select(self, keys):
        arr = (C.c_char_p * len(keys))(*[k.encode() for k in keys])
        idx = np.empty(max(self.n, 1), dtype=np.int32)
        n = C.c_int()
        check(_lib.lib().ckm_models_select(self._h, arr, len(keys), idx.ctypes.data, C.byref(n)))
        return idx[:n.value].copy()

    def write(self, idx, path):
        idx = np.ascontiguousarray(idx, dtype=np.int32)
        check(_lib.lib().ckm_models_write(self._h, idx.ctypes.data, len(idx), path.encode()))

    def close(self):
        if self._h:
            _lib.lib().ckm_models_free(self._h)
            self._h = C.c_void_p()


class SeqDb:
    def __init__(self, engine, residues, offsets, bin_of_seq=None, nbins=1):
        self.engine = engine
        self.residues = np.ascontiguousarray(residues, dtype=np.uint8)
        self.offsets = np.ascontiguousarray(offsets, dtype=np.int64)
        self.nseq = len(self.offsets) - 1
        self.nbins = int(nbins)
        self.bin_of_seq = None if bin_of_seq is None else np.ascontiguousarray(bin_of_seq, dtype=np.int32)
        self._h = C.c_void_p()
        check(_lib.lib().ckm_seqdb_create(engine._h, self.residues.ctypes.data, self.offsets.ctypes.data, self.nseq,
                                          None if self.bin_of_seq is None else self.bin_of_seq.ctypes.data,
                                          self.nbins, C.byref(self._h)))

    def close(self):
        if self._h:
            _lib.lib().ckm_seqdb_free(self._h)
            self._h = C.c_void_p()


def _batch_args(fn, comp, blocks, comp_base, segs=(), counters=None, n_ref=0):
    """The leading arguments of ckm_bgzf_inflate, ckm_bam_coverage and ckm_bam_windows for one BAM batch: comp, comp_base,
    the block table, then the segments (seg_start, seg_end) if given; each pointer keeps its array alive through the call.
    Given counters, checks them for the n_ref x 9 int64 sums the call adds to, in a message naming the method fn."""
    comp = np.ascontiguousarray(np.frombuffer(comp, dtype=np.uint8) if not isinstance(comp, np.ndarray) else comp)
    blocks = np.ascontiguousarray(blocks)
    segs = [np.ascontiguousarray(x, dtype=np.int64) for x in segs]
    if counters is not None and (counters.dtype != np.int64 or counters.shape != (n_ref, 9) or not counters.flags.c_contiguous):
        raise ValueError(fn + ": counters must be a C-contiguous n_ref x 9 int64 array")
    p = [a.ctypes.data_as(C.c_void_p) if a.size else None for a in [comp, blocks] + segs]
    args = [p[0], int(comp_base), comp.size, p[1], len(blocks)]
    return args + p[2:] + [len(segs[0])] if segs else args


class Engine:
    """One engine per process per GPU (a CUDA context cannot cross fork())."""

    def __init__(self, device=0):
        self._h = C.c_void_p()
        check(_lib.lib().ckm_init(int(device), C.byref(self._h)))
        self.device = int(device)

    def device_name(self):
        buf = C.create_string_buffer(256)
        check(_lib.lib().ckm_device_name(self._h, buf, 256))
        return buf.value.decode()

    def load_models(self, path):
        return Models(self, path)

    def seqdb(self, residues, offsets, bin_of_seq=None, nbins=1):
        return SeqDb(self, residues, offsets, bin_of_seq, nbins)

    def stats(self):
        s = Stats()
        check(_lib.lib().ckm_last_stats(self._h, C.byref(s)))
        return s

    def msv_scores(self, models, db, model_idx=None):
        """Dense [nmodels, nseq] int32: exact MSV xJ byte for SSV candidates (256 = overflow), -1 otherwise."""
        nm = models.n if model_idx is None else len(model_idx)
        out = np.empty((nm, db.nseq), dtype=np.int32)
        mi = None if model_idx is None else np.ascontiguousarray(model_idx, dtype=np.int32)
        check(_lib.lib().ckm_msv_scores(self._h, models._h, None if mi is None else mi.ctypes.data, nm, db._h,
                                        out.ctypes.data))
        return out

    def viterbi_scores(self, models, db, model_idx=None, int32_only=False, chunked_only=False):
        """Dense [nmodels, nseq] float32 ViterbiFilter scores of every pair (packed int16x2 kernel + int32 redo list, or the
        int32 kernels alone)."""
        nm = models.n if model_idx is None else len(model_idx)
        out = np.empty((nm, db.nseq), dtype=np.float32)
        mi = None if model_idx is None else np.ascontiguousarray(model_idx, dtype=np.int32)
        check(_lib.lib().ckm_viterbi_scores(self._h, models._h, None if mi is None else mi.ctypes.data, nm, db._h,
                                            2 if chunked_only else (1 if int32_only else 0), out.ctypes.data))
        return out

    def filter_scores(self, models, db, model_idx=None):
        """Dense [nmodels, nseq] arrays: bias-filter null score, Viterbi and Forward filter scores (NaN where a stage
        was not reached) and pass flags (bit0 MSV, bit1 bias, bit2 Viterbi, bit3 Forward)."""
        nm = models.n if model_idx is None else len(model_idx)
        fs = np.empty((nm, db.nseq), dtype=np.float32)
        vs = np.empty((nm, db.nseq), dtype=np.float32)
        fw = np.empty((nm, db.nseq), dtype=np.float32)
        ps = np.empty((nm, db.nseq), dtype=np.uint8)
        mi = None if model_idx is None else np.ascontiguousarray(model_idx, dtype=np.int32)
        check(_lib.lib().ckm_filter_scores(self._h, models._h, None if mi is None else mi.ctypes.data, nm, db._h,
                                           fs.ctypes.data, vs.ctypes.data, fw.ctypes.data, ps.ctypes.data))
        return fs, vs, fw, ps

    def search(self, models, db, model_idx=None, E=0.1, domE=0.1, bin_model_offsets=None):
        """Returns a numpy structured array of ckm_hit rows (domtblout rows)."""
        hits = C.POINTER(Hit)()
        n = C.c_int64()
        mi = None if model_idx is None else np.ascontiguousarray(model_idx, dtype=np.int32)
        if bin_model_offsets is None:
            nm = models.n if mi is None else len(mi)
            check(_lib.lib().ckm_search(self._h, models._h, None if mi is None else mi.ctypes.data, nm, db._h, E, domE,
                                        C.byref(hits), C.byref(n)))
        else:
            bo = np.ascontiguousarray(bin_model_offsets, dtype=np.int64)
            check(_lib.lib().ckm_search_per_bin(self._h, models._h, mi.ctypes.data, bo.ctypes.data, db._h, E, domE,
                                                C.byref(hits), C.byref(n)))
        if n.value == 0:
            arr = np.zeros(0, dtype=HIT_DTYPE)
        else:
            buf = (C.c_char * (n.value * C.sizeof(Hit))).from_address(C.addressof(hits.contents))
            arr = np.frombuffer(buf, dtype=HIT_DTYPE).copy()
        _lib.lib().ckm_hits_free(hits)
        return arr

    def align(self, models, db, model=0):
        """Optimal-accuracy alignment of every sequence of `db` to one model (ckm_align): per-residue states (+k match,
        -k insert, 0 flank) over the unpadded residue stream, and the optimal-accuracy score of every sequence."""
        state = np.zeros(len(db.residues), dtype=np.int32)
        oasc = np.zeros(db.nseq, dtype=np.float32)
        check(_lib.lib().ckm_align(self._h, models._h, int(model), db._h, state.ctypes.data, oasc.ctypes.data))
        return state, oasc

    def align_groups(self, models, db, group_model, group_seq_off):
        """`align` for many groups in one pass (ckm_align_groups): sequences group_seq_off[g]:group_seq_off[g + 1] of `db`
        aligned to model group_model[g].  Returns the per-residue states and the per-sequence scores, as `align` does."""
        gm = np.ascontiguousarray(group_model, dtype=np.int32)
        go = np.ascontiguousarray(group_seq_off, dtype=np.int64)
        if go.shape != (len(gm) + 1,):
            raise ValueError("align_groups: group_seq_off must hold one offset per group and one more")
        state = np.zeros(len(db.residues), dtype=np.int32)
        oasc = np.zeros(db.nseq, dtype=np.float32)
        check(_lib.lib().ckm_align_groups(self._h, models._h, gm.ctypes.data, go.ctypes.data, len(gm), db._h,
                                          state.ctypes.data, oasc.ctypes.data))
        return state, oasc

    def aai_pairs(self, rows, row_off, pairs):
        """Mismatches and compared length of every pair of masked alignment rows (ckm_aai_pairs).  rows: the rows' ASCII
        bytes back to back, row r = rows[row_off[r]:row_off[r + 1]]; pairs: npairs x 2 row indices of rows of equal width.
        Returns two int32 arrays of npairs values."""
        rows = np.ascontiguousarray(np.frombuffer(rows, dtype=np.uint8) if not isinstance(rows, np.ndarray) else rows, dtype=np.uint8)
        row_off = np.ascontiguousarray(row_off, dtype=np.int64)
        pairs = np.ascontiguousarray(pairs, dtype=np.int32).reshape(-1, 2)
        n = len(pairs)
        mis = np.zeros(n, dtype=np.int32)
        ln = np.zeros(n, dtype=np.int32)
        check(_lib.lib().ckm_aai_pairs(self._h, rows.ctypes.data if rows.size else None, row_off.ctypes.data, len(row_off) - 1,
                                       pairs.ctypes.data if n else None, n, mis.ctypes.data if n else None,
                                       ln.ctypes.data if n else None))
        return mis, ln

    def scaffold_stats(self, data, starts, lens):
        """Base counts and contigs of scaffolds laid out as `seqio.scan_nt_fasta` returns them (ckm_scaffold_stats).
        Returns stats (n x 8 int64: A C G T 'N' 'n' contigs contig-bases), the scaffold index and length of every contig
        (no particular order), and the scan kernel's duration in ms."""
        n = len(lens)
        stats = np.zeros((n, 8), dtype=np.int64)
        data = np.ascontiguousarray(data, dtype=np.uint8)
        starts = np.ascontiguousarray(starts, dtype=np.int64)
        lens = np.ascontiguousarray(lens, dtype=np.int64)
        cap = n + int(lens.sum()) // 2048 + 1024
        while True:
            cscaf = np.empty(cap, dtype=np.uint32)
            clen = np.empty(cap, dtype=np.uint32)
            found, ms = C.c_int64(), C.c_float()
            rc = _lib.lib().ckm_scaffold_stats(self._h, data.ctypes.data, data.size, starts.ctypes.data, lens.ctypes.data, n,
                                               stats.ctypes.data, cscaf.ctypes.data, clen.ctypes.data, cap, C.byref(found), C.byref(ms))
            if rc == 8 and found.value > cap:          # CKM_ECAPACITY: the count needed came back
                cap = found.value
                continue
            check(rc)
            return stats, cscaf[:found.value].astype(np.int64), clen[:found.value].astype(np.int64), float(ms.value)

    def kmer_counts(self, data, starts, lens, k=4):
        """Canonical k-mer counts of sequences laid out as `seqio.scan_nt_fasta` returns them (ckm_kmer_counts): n x C
        uint32, C = 2, 10, 32, 136 for k = 1..4, columns in GenomicSignatures.canonicalKmerOrder() order; and the scan
        kernel's duration in ms."""
        n = len(lens)
        ncols = {1: 2, 2: 10, 3: 32, 4: 136}.get(int(k), 1)
        counts = np.zeros((n, ncols), dtype=np.uint32)
        data = np.ascontiguousarray(data, dtype=np.uint8)
        starts = np.ascontiguousarray(starts, dtype=np.int64)
        lens = np.ascontiguousarray(lens, dtype=np.int64)
        ms = C.c_float()
        check(_lib.lib().ckm_kmer_counts(self._h, data.ctypes.data, data.size, starts.ctypes.data, lens.ctypes.data, n, int(k),
                                         counts.ctypes.data, C.byref(ms)))
        return counts, float(ms.value)

    def merge_pairs(self, counts, n_markers, min_delta_comp, max_delta_cont, min_merged_comp, max_merged_cont, capacity=None):
        """The bin pairs `checkm merge` reports (ckm_merge_pairs).  counts: nbins x nmarkers copy numbers, one row per bin
        in sorted() id order; n_markers: numMarkers() of each bin's marker set.  Returns the kept pairs as a
        MERGE_PAIR_DTYPE array (i ascending, then j) and the kernels' duration in ms.  When more pairs pass than `capacity`
        (default: 16 per bin) the call is repeated with room for exactly the number that came back."""
        counts = np.ascontiguousarray(counts, dtype=np.int32)
        n_markers = np.ascontiguousarray(n_markers, dtype=np.int32)
        if counts.ndim != 2 or n_markers.shape != (counts.shape[0],):
            raise ValueError("merge_pairs: counts must be nbins x nmarkers and n_markers hold one value per bin")
        nb, nm = counts.shape
        cap = min(nb * (nb - 1) // 2, 16 * nb + 1024) if capacity is None else int(capacity)
        while True:
            out = np.empty(cap, dtype=MERGE_PAIR_DTYPE)
            found, ms = C.c_int64(), C.c_float()
            rc = _lib.lib().ckm_merge_pairs(self._h, counts.ctypes.data if counts.size else None, nb, nm,
                                            n_markers.ctypes.data if nb else None, float(min_delta_comp), float(max_delta_cont),
                                            float(min_merged_comp), float(max_merged_cont), out.ctypes.data if cap else None,
                                            cap, C.byref(found), C.byref(ms))
            if rc == 8 and found.value > cap:          # CKM_ECAPACITY: the count needed came back
                cap = found.value
                continue
            check(rc)
            return out[:found.value], float(ms.value)

    def signatures(self, values):
        return Signatures(self, values)

    def outlier_scores(self, sigs, bin_off, lens, acgt, coding, sig_row, bin_gc_table, bin_cd_table, td_table, table_off,
                       table_key, table_lo, table_hi, binsig_in=None, want_binsig=False):
        """Every sequence of a batch of bins scored against its bin (ckm_outlier_scores; the arguments are the fields of
        ckm_outlier_in).  Returns bin_means (nbins x 3: meanGC, meanCD, meanTD), the bins' signatures (nbins x 136, or None
        unless want_binsig), seq_values (nseq x 9: GC, deltaGC, CD, deltaCD, TD, GC lower, GC upper, CD lower, TD upper),
        the outlying mask per sequence (1 GC, 2 CD, 4 TD) and the three kernels' durations in ms."""
        i64 = lambda a: np.ascontiguousarray(a, dtype=np.int64)       # noqa: E731
        f64 = lambda a: np.ascontiguousarray(a, dtype=np.float64)     # noqa: E731
        bin_off, lens, acgt, coding, sig_row, table_off = (i64(a) for a in (bin_off, lens, acgt, coding, sig_row, table_off))
        bin_gc_table = np.ascontiguousarray(bin_gc_table, dtype=np.int32)
        bin_cd_table = np.ascontiguousarray(bin_cd_table, dtype=np.int32)
        table_key, table_lo, table_hi = f64(table_key), f64(table_lo), f64(table_hi)
        nb, ns, nt = len(bin_off) - 1, len(lens), len(table_off) - 1
        if (acgt.shape != (ns, 4) or coding.shape != (ns,) or sig_row.shape != (ns,) or bin_gc_table.shape != (nb,) or
                bin_cd_table.shape != (nb,) or not (table_key.shape == table_lo.shape == table_hi.shape == (int(table_off[-1]),))):
            raise ValueError("outlier_scores: array shapes do not agree")
        if binsig_in is not None:
            binsig_in = f64(binsig_in)
            if binsig_in.shape != (nb, 136):
                raise ValueError("outlier_scores: binsig_in must be nbins x 136")
        means = np.empty((nb, 3), dtype=np.float64)
        binsig = np.empty((nb, 136), dtype=np.float64) if want_binsig else None
        values = np.empty((ns, 9), dtype=np.float64)
        mask = np.empty(ns, dtype=np.uint8)
        arg = _lib.OutlierIn(ns, nb, nt, bin_off.ctypes.data, lens.ctypes.data, acgt.ctypes.data, coding.ctypes.data,
                             sig_row.ctypes.data, bin_gc_table.ctypes.data, bin_cd_table.ctypes.data, int(td_table), 0,
                             table_off.ctypes.data, table_key.ctypes.data, table_lo.ctypes.data, table_hi.ctypes.data,
                             binsig_in.ctypes.data if binsig_in is not None else None)
        out = _lib.OutlierOut(means.ctypes.data, binsig.ctypes.data if want_binsig else None, values.ctypes.data, mask.ctypes.data)
        check(_lib.lib().ckm_outlier_scores(self._h, sigs._h, C.byref(arg), C.byref(out)))
        return means, binsig, values, mask, tuple(float(v) for v in out.kernel_ms)

    def id_join(self, text, bin_nrec, nasm):
        """The ids of the bins' and the assembly's records joined in one device call (ckm_id_join).  text: every header
        line followed by '\\n', the bins' (bin_nrec[b] per file) before the assembly's (nasm).  Returns id_start, id_len
        (per record, int64, byte spans in text), asm_flags (uint8: 1 = binned id, 2 = first record of its id), asm_last
        (int64: the last assembly record of its id), bin_keep (bool: the last record of its id in its own bin file), the
        number of distinct binned ids and the kernels' duration in ms.  A header without an id raises CkmError with the
        record's index as its `record` attribute (-1 for every other error)."""
        bin_nrec = np.ascontiguousarray(bin_nrec, dtype=np.int64)
        n = int(bin_nrec.sum()) + int(nasm)
        id_start = np.zeros(n, dtype=np.int64)
        id_len = np.zeros(n, dtype=np.int64)
        flags = np.zeros(nasm, dtype=np.uint8)
        last = np.zeros(nasm, dtype=np.int32)
        keep = np.zeros(n - nasm, dtype=np.uint8)
        nbinned, bad, ms = C.c_int64(), C.c_int64(), C.c_float()
        rc = _lib.lib().ckm_id_join(self._h, text, len(text), len(bin_nrec), bin_nrec.ctypes.data, int(nasm),
                                    id_start.ctypes.data, id_len.ctypes.data, flags.ctypes.data, last.ctypes.data,
                                    keep.ctypes.data, C.byref(nbinned), C.byref(bad), C.byref(ms))
        if rc:
            err = _lib.CkmError(rc, _lib.lib().ckm_last_error().decode(errors="replace"))
            err.record = int(bad.value)
            raise err
        return id_start, id_len, flags, last.astype(np.int64), keep.view(bool), int(nbinned.value), float(ms.value)

    def window_stats(self, data, starts, lens, window_size, win_off, bin_sig=None):
        """Per-window statistics of sequences laid out as `seqio.scan_nt_fasta` returns them (ckm_window_stats; sequence s
        owns windows win_off[s]:win_off[s + 1], coverageWindows.window_offsets).  Returns the A, C, G, T(+U) counts of every
        window (nwin x 4 int64), the tetranucleotide distance of every window to `bin_sig` (nwin float64, or None without
        a signature) and the kernels' duration in ms."""
        data = np.ascontiguousarray(data, dtype=np.uint8)
        starts = np.ascontiguousarray(starts, dtype=np.int64)
        lens = np.ascontiguousarray(lens, dtype=np.int64)
        win_off = np.ascontiguousarray(win_off, dtype=np.int64)
        if win_off.shape != (len(lens) + 1,):
            raise ValueError("window_stats: win_off must hold one offset per sequence and one more")
        nwin = int(win_off[-1])
        acgt = np.zeros((nwin, 4), dtype=np.int64)
        td = None
        if bin_sig is not None:
            bin_sig = np.ascontiguousarray(bin_sig, dtype=np.float64)
            if bin_sig.shape != (136,):
                raise ValueError("window_stats: bin_sig must hold 136 values")
            td = np.zeros(nwin, dtype=np.float64)
        ms = C.c_float()
        check(_lib.lib().ckm_window_stats(self._h, data.ctypes.data if data.size else None, data.size, starts.ctypes.data,
                                          lens.ctypes.data, len(lens), int(window_size), win_off.ctypes.data,
                                          None if bin_sig is None else bin_sig.ctypes.data, acgt.ctypes.data,
                                          None if td is None else td.ctypes.data, C.byref(ms)))
        return acgt, td, float(ms.value)

    def length_profile(self, lens, bin_off, x):
        """The length profile of many bins in one device call (ckm_length_profile; bin b = lens[bin_off[b]:bin_off[b + 1]],
        x ascending).  Returns per bin the total, the Nx list (nbins x len(x), -1 past the thresholds reached), the status
        (0 OK, 1 IndexError at the record of rank fail, 2 only fail thresholds reached), fail, the 10 length-class counts
        (nbins x 10); per record its rank in descending length order; and the kernel's duration in ms."""
        lens = np.ascontiguousarray(lens, dtype=np.int64)
        bin_off = np.ascontiguousarray(bin_off, dtype=np.int64)
        x = np.ascontiguousarray(x, dtype=np.float64)
        nbins, m = len(bin_off) - 1, len(x)
        if nbins < 0 or int(bin_off[-1]) != len(lens):
            raise ValueError("length_profile: bin_off must start at 0 and end at len(lens)")
        total = np.zeros(nbins, dtype=np.int64)
        nx = np.zeros((nbins, m), dtype=np.int64)
        status = np.zeros(nbins, dtype=np.int32)
        fail = np.zeros(nbins, dtype=np.int64)
        classes = np.zeros((nbins, 10), dtype=np.int64)
        rank = np.zeros(len(lens), dtype=np.int32)
        ms = C.c_float()
        check(_lib.lib().ckm_length_profile(self._h, lens.ctypes.data if lens.size else None, bin_off.ctypes.data, nbins,
                                            x.ctypes.data if m else None, m, total.ctypes.data, nx.ctypes.data,
                                            status.ctypes.data, fail.ctypes.data, classes.ctypes.data,
                                            rank.ctypes.data if rank.size else None, C.byref(ms)))
        return total, nx, status, fail, classes, rank, float(ms.value)

    def bgzf_inflate(self, comp, blocks, comp_base=0):
        """The payloads of BGZF `blocks` (a bam.BLOCK_DTYPE table of file offsets; comp[0] is the byte at file offset
        comp_base) inflated back to back on the device (ckm_bgzf_inflate), and the inflate kernel's duration in ms."""
        batch = _batch_args('bgzf_inflate', comp, blocks, comp_base)
        total = int(np.asarray(blocks)['isize'].sum())
        out = np.empty(max(total, 1), dtype=np.uint8)
        ms = C.c_float()
        check(_lib.lib().ckm_bgzf_inflate(self._h, *batch, out.ctypes.data, out.size, None, C.byref(ms)))
        return out[:total], float(ms.value)

    def bam_coverage(self, comp, blocks, seg_start, seg_end, n_ref, counters, comp_base=0, all_reads=False, min_qc=15,
                     min_align=0.98, max_edit=0.02):
        """One batch of a BAM (ckm_bam_coverage): blocks inflated, the segments walked, the nine counters of every
        reference added to `counters` (n_ref x 9 int64).  Returns the inflate and scan kernels' durations in ms."""
        batch = _batch_args('bam_coverage', comp, blocks, comp_base, (seg_start, seg_end), counters, n_ref)
        filt = _lib.BamFilter(int(bool(all_reads)), int(min_qc), float(min_align), float(max_edit))
        ms = (C.c_float * 2)()
        err = C.c_int64()
        check(_lib.lib().ckm_bam_coverage(self._h, *batch, int(n_ref), C.byref(filt), counters.ctypes.data if n_ref else None,
                                          ms, C.byref(err)))
        return float(ms[0]), float(ms[1])

    def bam_windows(self, comp, blocks, seg_start, seg_end, ref_len, window_size, win_off, counters, windows, comp_base=0,
                    all_reads=False, min_align=0.98, max_edit=0.02):
        """One batch of a BAM (ckm_bam_windows): blocks inflated, the segments walked with coverageWindows' rule, the nine
        counters of every reference added to `counters` (n_ref x 9 int64; the ninth is the covered bases) and each
        window's depth sum to `windows` (int64; reference r owns windows[win_off[r]:win_off[r + 1]]).  Returns the
        inflate and window kernels' durations in ms."""
        ref_len = np.ascontiguousarray(ref_len, dtype=np.int64)
        win_off = np.ascontiguousarray(win_off, dtype=np.int64)
        n_ref = len(ref_len)
        batch = _batch_args('bam_windows', comp, blocks, comp_base, (seg_start, seg_end), counters, n_ref)
        if win_off.shape != (n_ref + 1,):
            raise ValueError("bam_windows: win_off must hold n_ref + 1 offsets")
        if windows.dtype != np.int64 or windows.ndim != 1 or not windows.flags.c_contiguous or windows.size < win_off[-1]:
            raise ValueError("bam_windows: windows must be a C-contiguous int64 array of win_off[-1] values")
        filt = _lib.BamFilter(int(bool(all_reads)), 0, float(min_align), float(max_edit))
        ms = (C.c_float * 2)()
        err = C.c_int64()
        check(_lib.lib().ckm_bam_windows(self._h, *batch, n_ref, C.byref(filt), ref_len.ctypes.data if n_ref else None,
                                         int(window_size), win_off.ctypes.data, counters.ctypes.data if n_ref else None,
                                         windows.ctypes.data if windows.size else None, ms, C.byref(err)))
        return float(ms[0]), float(ms[1])

    def close(self):
        if self._h:
            _lib.lib().ckm_destroy(self._h)
            self._h = C.c_void_p()
