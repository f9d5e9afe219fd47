// idjoin.cu -- which assembly sequences lie in no bin (`checkm unbinned`; checkm/unbinned.py:33-85): the reference reads
// every bin and the assembly into dicts keyed by the first token of each header line and tests every assembly id against
// the binned ones.  Here every header line of one call -- the bins' first, then the assembly's -- is joined in one
// device pass:
//   1. find:   one thread per line finds the id as line.split(None, 1)[0] finds it (whitespace = str.isspace(), on the
//              UTF-8 bytes) and hashes it;
//   2. insert: one open-addressing table over all lines; a line either claims an empty slot or finds the slot of a line
//              with the same id.  A slot holds (upper 32 bits of the hash, line index); a tag match is only a candidate,
//              the ids' bytes decide.  The line that owns the slot represents its id (its "group");
//   3. group:  per group, the first and the last assembly line and the first bin line (atomic min / max on the
//              representative's entry); per (group, bin file) the last line, in a second table keyed by the pair;
//   4. emit:   per assembly line: binned, first of its id (a dict entry, in dict order), the last line of its id (the
//              dict's content); per bin line: whether it is the last of its id in its own file; the number of ids that
//              occur in any bin.
// Nothing here depends on the order in which threads win the slots, so the results are deterministic.
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <vector>
#include "engine.hpp"
#include "pool.hpp"

using namespace ckm;

namespace {

constexpr int IJ_THREADS = 256;
constexpr unsigned long long IJ_EMPTY = ~0ull;      // never a valid entry: line indices stay below 2^31
constexpr int32_t IJ_NONE = 0x7F7F7F7F;              // memset(0x7F) of an int32 min slot: above every line index

struct IjParams {
  const uint8_t *text;
  const int64_t *line_start;   // n + 1: line r is text[line_start[r], line_start[r + 1] - 1) (the '\n' excluded)
  const int32_t *bin_of;       // nb: the bin file of each bin line
  int64_t n, nb;               // lines in all; the first nb are bin lines
  int64_t *id_start;           // n
  int64_t *id_len;             // n
  unsigned long long *hash;    // n
  unsigned long long *table;   // cap entries (tag << 32 | line)
  unsigned long long mask;
  int32_t *rep;                // n: the line that represents the id of line r
  int32_t *first_asm, *last_asm, *first_bin;       // n, indexed by representative
  unsigned long long *table2;  // cap2 entries (rep << 32 | bin)
  int32_t *last2;              // cap2: last bin line of the (rep, bin) pair in the slot
  unsigned long long mask2;
  int32_t *slot2;              // nb: the slot of each bin line's pair
  uint8_t *asm_flags;          // n - nb
  int32_t *asm_last;           // n - nb
  uint8_t *bin_keep;           // nb
  unsigned long long *counters;   // [0] first line without an id (IJ_EMPTY: none), [1] ids that occur in a bin
};

// bytes of the str.isspace() character starting at p (0 if it is not one); the text is UTF-8
__device__ __forceinline__ int ws_len(const uint8_t *p, int64_t left) {
  const uint32_t b = p[0];
  if (b < 0x80u) return (b == 32u || (b >= 9u && b <= 13u) || (b >= 28u && b <= 31u)) ? 1 : 0;
  if (b == 0xC2u) return (left >= 2 && (p[1] == 0x85u || p[1] == 0xA0u)) ? 2 : 0;                     // U+0085 U+00A0
  if (left < 3) return 0;
  const uint32_t b1 = p[1], b2 = p[2];
  if (b == 0xE1u) return (b1 == 0x9Au && b2 == 0x80u) ? 3 : 0;                                          // U+1680
  if (b == 0xE2u) {
    if (b1 == 0x80u) return ((b2 >= 0x80u && b2 <= 0x8Au) || b2 == 0xA8u || b2 == 0xA9u || b2 == 0xAFu) ? 3 : 0;   // U+2000-200A 2028 2029 202F
    return (b1 == 0x81u && b2 == 0x9Fu) ? 3 : 0;                                                       // U+205F
  }
  if (b == 0xE3u) return (b1 == 0x80u && b2 == 0x80u) ? 3 : 0;                                          // U+3000
  return 0;
}

__device__ __forceinline__ unsigned long long fmix64(unsigned long long k) {
  k ^= k >> 33; k *= 0xff51afd7ed558ccdull; k ^= k >> 33; k *= 0xc4ceb9fe1a85ec53ull; k ^= k >> 33;
  return k;
}

__device__ __forceinline__ bool same_id(const IjParams &p, int64_t a, int64_t b) {
  const int64_t len = p.id_len[a];
  if (p.id_len[b] != len) return false;
  const uint8_t *x = p.text + p.id_start[a], *y = p.text + p.id_start[b];
  for (int64_t i = 0; i < len; ++i)
    if (x[i] != y[i]) return false;
  return true;
}

__global__ void __launch_bounds__(IJ_THREADS) idjoin_find_kernel(IjParams p) {
  const int64_t r = (int64_t)blockIdx.x * IJ_THREADS + threadIdx.x;
  if (r >= p.n) return;
  const int64_t lo = p.line_start[r], hi = p.line_start[r + 1] - 1;
  int64_t j = lo;
  for (int w; j < hi && (w = ws_len(p.text + j, hi - j)) > 0;) j += w;
  const int64_t s = j;
  unsigned long long h = 0xcbf29ce484222325ull;                    // FNV-1a over the id's bytes, then fmix64
  while (j < hi && ws_len(p.text + j, hi - j) == 0) { h = (h ^ p.text[j]) * 0x100000001b3ull; ++j; }
  p.id_start[r] = s;
  p.id_len[r] = j - s;
  p.hash[r] = fmix64(h ^ (unsigned long long)(j - s));
  if (j == s) atomicMin(&p.counters[0], (unsigned long long)r);
}

__global__ void __launch_bounds__(IJ_THREADS) idjoin_insert_kernel(IjParams p) {
  const int64_t r = (int64_t)blockIdx.x * IJ_THREADS + threadIdx.x;
  if (r >= p.n) return;
  const unsigned long long h = p.hash[r];
  const unsigned long long tag = h >> 32, mine = (tag << 32) | (unsigned long long)r;
  unsigned long long i = h & p.mask;
  // an entry never changes once written, so a plain read that sees one is final; an empty one is claimed by CAS
  for (;;) {
    unsigned long long cur = *(volatile unsigned long long *)&p.table[i];
    if (cur == IJ_EMPTY) {
      cur = atomicCAS(&p.table[i], IJ_EMPTY, mine);
      if (cur == IJ_EMPTY) { p.rep[r] = (int32_t)r; return; }
    }
    if ((cur >> 32) == tag) {
      const int64_t o = (int64_t)(cur & 0xFFFFFFFFull);
      if (same_id(p, o, r)) { p.rep[r] = (int32_t)o; return; }
    }
    i = (i + 1) & p.mask;
  }
}

__global__ void __launch_bounds__(IJ_THREADS) idjoin_group_kernel(IjParams p) {
  const int64_t r = (int64_t)blockIdx.x * IJ_THREADS + threadIdx.x;
  if (r >= p.n) return;
  const int32_t g = p.rep[r];
  if (r >= p.nb) {
    atomicMin(&p.first_asm[g], (int32_t)r);
    atomicMax(&p.last_asm[g], (int32_t)r);
    return;
  }
  atomicMin(&p.first_bin[g], (int32_t)r);
  const unsigned long long key = ((unsigned long long)g << 32) | (unsigned long long)(uint32_t)p.bin_of[r];
  unsigned long long i = fmix64(key) & p.mask2;
  for (;;) {
    unsigned long long cur = *(volatile unsigned long long *)&p.table2[i];
    if (cur == IJ_EMPTY) cur = atomicCAS(&p.table2[i], IJ_EMPTY, key);
    if (cur == IJ_EMPTY || cur == key) break;
    i = (i + 1) & p.mask2;
  }
  atomicMax(&p.last2[i], (int32_t)r);
  p.slot2[r] = (int32_t)i;
}

__global__ void __launch_bounds__(IJ_THREADS) idjoin_emit_kernel(IjParams p) {
  const int64_t r = (int64_t)blockIdx.x * IJ_THREADS + threadIdx.x;
  bool new_binned_id = false;
  if (r < p.n) {
    const int32_t g = p.rep[r];
    if (r >= p.nb) {
      const int64_t a = r - p.nb;
      p.asm_flags[a] = (uint8_t)((p.first_bin[g] != IJ_NONE ? 1u : 0u) | (p.first_asm[g] == (int32_t)r ? 2u : 0u));
      p.asm_last[a] = (int32_t)(p.last_asm[g] - p.nb);
    } else {
      p.bin_keep[r] = p.last2[p.slot2[r]] == (int32_t)r ? 1 : 0;
      new_binned_id = p.first_bin[g] == (int32_t)r;
    }
  }
  const unsigned int votes = __ballot_sync(0xffffffffu, new_binned_id);
  if ((threadIdx.x & 31) == 0 && votes) atomicAdd(&p.counters[1], (unsigned long long)__popc(votes));
}

unsigned long long table_size(int64_t n) {           // a power of two, at least twice the entries: probe chains stay short
  unsigned long long c = 1024;
  while (c < 2ull * (unsigned long long)n) c <<= 1;
  return c;
}

}  // namespace

extern "C" {

int ckm_id_join(ckm_engine *e, const char *text, int64_t nbytes, int32_t nbins, const int64_t *bin_nrec, int64_t nasm,
                int64_t *id_start_out, int64_t *id_len_out, uint8_t *asm_flags_out, int32_t *asm_last_out,
                uint8_t *bin_keep_out, int64_t *n_binned_ids_out, int64_t *bad_record_out, float *kernel_ms_out) {
  if (!e || nbytes < 0 || (nbytes > 0 && !text) || nbins < 0 || (nbins > 0 && !bin_nrec) || nasm < 0 ||
      !n_binned_ids_out || !bad_record_out) {
    set_error("ckm_id_join: bad argument"); return CKM_EINVAL;
  }
  int64_t nb = 0;
  for (int32_t b = 0; b < nbins; ++b) {
    if (bin_nrec[b] < 0) { set_error("ckm_id_join: bad argument"); return CKM_EINVAL; }
    nb += bin_nrec[b];
  }
  const int64_t n = nb + nasm;
  if (n >= IJ_NONE) { set_error("ckm_id_join: too many records for one call"); return CKM_EINVAL; }
  if (n > 0 && (!id_start_out || !id_len_out || (nasm > 0 && (!asm_flags_out || !asm_last_out)) || (nb > 0 && !bin_keep_out))) {
    set_error("ckm_id_join: bad argument"); return CKM_EINVAL;
  }
  *n_binned_ids_out = 0; *bad_record_out = -1;
  if (kernel_ms_out) *kernel_ms_out = 0.0f;
  // the lines: every one ends with '\n'
  std::vector<int64_t> line_start; line_start.reserve((size_t)n + 1);
  line_start.push_back(0);
  for (int64_t i = 0; i < nbytes;) {
    const char *nl = (const char *)std::memchr(text + i, '\n', (size_t)(nbytes - i));
    if (!nl) break;
    i = (nl - text) + 1;
    line_start.push_back(i);
  }
  if ((int64_t)line_start.size() != n + 1 || line_start.back() != nbytes) {
    set_error("ckm_id_join: the text must hold one '\\n'-terminated header line per record"); return CKM_EINVAL;
  }
  if (n == 0) return CKM_OK;
  std::vector<int32_t> bin_of((size_t)std::max<int64_t>(nb, 1));
  { int64_t r = 0; for (int32_t b = 0; b < nbins; ++b) for (int64_t k = 0; k < bin_nrec[b]; ++k) bin_of[(size_t)r++] = b; }

  const DeviceScope ws(e);
  const unsigned long long cap = table_size(n), cap2 = table_size(nb);
  const int64_t na = nasm;
  DevBuf dtext, dls, dbin, dis, dil, dh, dt, drep, dfa, dla, dfb, dt2, dl2, ds2, dflags, dlast, dkeep, dctr;
  CKM_TRY(dtext.put(text, (size_t)nbytes, ws.st));
  CKM_TRY(dls.put(line_start.data(), (size_t)n + 1, ws.st));
  CKM_TRY(dbin.put(bin_of.data(), (size_t)nb, ws.st));
  CKM_TRY(dt.fill(sizeof(unsigned long long) * cap, 0xFF, ws.st));
  CKM_TRY(dt2.fill(sizeof(unsigned long long) * cap2, 0xFF, ws.st));
  CKM_TRY(dl2.fill(sizeof(int32_t) * cap2, 0xFF, ws.st));
  CKM_TRY(dfa.fill(sizeof(int32_t) * n, 0x7F, ws.st));
  CKM_TRY(dfb.fill(sizeof(int32_t) * n, 0x7F, ws.st));
  CKM_TRY(dla.fill(sizeof(int32_t) * n, 0xFF, ws.st));
  CKM_TRY(dctr.fill(64, 0, ws.st));
  CKM_TRY(set_bytes(dctr.p, 0xFF, 8, ws.st));
  CKM_TRY(dis.alloc(sizeof(int64_t) * n));
  CKM_TRY(dil.alloc(sizeof(int64_t) * n));
  CKM_TRY(dh.alloc(sizeof(unsigned long long) * n));
  CKM_TRY(drep.alloc(sizeof(int32_t) * n));
  CKM_TRY(ds2.alloc(sizeof(int32_t) * nb));
  CKM_TRY(dflags.alloc((size_t)na));
  CKM_TRY(dlast.alloc(sizeof(int32_t) * na));
  CKM_TRY(dkeep.alloc((size_t)nb));
  IjParams p;
  p.text = dtext.as<uint8_t>(); p.line_start = dls.as<int64_t>(); p.bin_of = dbin.as<int32_t>(); p.n = n; p.nb = nb;
  p.id_start = dis.as<int64_t>(); p.id_len = dil.as<int64_t>(); p.hash = dh.as<unsigned long long>();
  p.table = dt.as<unsigned long long>(); p.mask = cap - 1; p.rep = drep.as<int32_t>();
  p.first_asm = dfa.as<int32_t>(); p.last_asm = dla.as<int32_t>(); p.first_bin = dfb.as<int32_t>();
  p.table2 = dt2.as<unsigned long long>(); p.last2 = dl2.as<int32_t>(); p.mask2 = cap2 - 1; p.slot2 = ds2.as<int32_t>();
  p.asm_flags = dflags.as<uint8_t>(); p.asm_last = dlast.as<int32_t>(); p.bin_keep = dkeep.as<uint8_t>();
  p.counters = dctr.as<unsigned long long>();
  const unsigned grid = (unsigned)((n + IJ_THREADS - 1) / IJ_THREADS);
  CKM_TRY(ev_record(e, 0));
  idjoin_find_kernel<<<grid, IJ_THREADS, 0, ws.st>>>(p);
  CKM_CUDA(cudaGetLastError());
  unsigned long long ctr[2] = {0, 0};
  CKM_TRY(dctr.get(ctr, 2, ws.st));
  CKM_TRY(stream_sync(ws.st));
  if (ctr[0] != IJ_EMPTY) {
    *bad_record_out = (int64_t)ctr[0];
    set_error("ckm_id_join: a header line without an id (record " + std::to_string((long long)ctr[0]) + ")");
    return CKM_EFORMAT;
  }
  idjoin_insert_kernel<<<grid, IJ_THREADS, 0, ws.st>>>(p);
  CKM_CUDA(cudaGetLastError());
  idjoin_group_kernel<<<grid, IJ_THREADS, 0, ws.st>>>(p);
  CKM_CUDA(cudaGetLastError());
  idjoin_emit_kernel<<<grid, IJ_THREADS, 0, ws.st>>>(p);
  CKM_CUDA(cudaGetLastError());
  CKM_TRY(ev_record(e, 1));
  CKM_TRY(dis.get(id_start_out, (size_t)n, ws.st));
  CKM_TRY(dil.get(id_len_out, (size_t)n, ws.st));
  CKM_TRY(dflags.get(asm_flags_out, (size_t)na, ws.st));
  CKM_TRY(dlast.get(asm_last_out, (size_t)na, ws.st));
  CKM_TRY(dkeep.get(bin_keep_out, (size_t)nb, ws.st));
  CKM_TRY(dctr.get(ctr, 2, ws.st));
  CKM_TRY(stream_sync(ws.st));
  CKM_TRY(ev_elapsed(e, kernel_ms_out, 0, 1));
  *n_binned_ids_out = (int64_t)ctr[1];
  return CKM_OK;
}

int ckm_format_unbinned(const char *ids, const int64_t *id_start, const int64_t *id_len, const uint8_t *bytes,
                        const int64_t *starts, const int64_t *lens, const int64_t *acgt, int64_t n, char *fasta_out,
                        int64_t fasta_cap, char *stats_out, int64_t stats_cap, int64_t *fasta_len_out, int64_t *stats_len_out) {
  if (n < 0 || !fasta_len_out || !stats_len_out || fasta_cap < 0 || stats_cap < 0 || (fasta_cap > 0 && !fasta_out) ||
      (stats_cap > 0 && !stats_out) || (n > 0 && (!id_start || !id_len || !starts || !lens || !acgt))) {
    set_error("ckm_format_unbinned: bad argument"); return CKM_EINVAL;
  }
  int64_t fw = 0, sw = 0;
  for (int64_t r = 0; r < n; ++r) {
    if (id_len[r] < 0 || lens[r] < 0 || (id_len[r] > 0 && !ids) || (lens[r] > 0 && !bytes)) {
      set_error("ckm_format_unbinned: bad argument"); return CKM_EINVAL;
    }
    fw += id_len[r] + lens[r] + 3;
    sw += id_len[r] + 48;             // "\t" + at most 20 digits + "\t" + at most "100.00" + "\n", with room to spare
  }
  *fasta_len_out = fw; *stats_len_out = sw;
  if (fw > fasta_cap || sw > stats_cap) {
    set_error("ckm_format_unbinned: output buffer too small (the sizes needed are returned)"); return CKM_ECAPACITY;
  }
  fw = 0; sw = 0;
  char line[64];
  for (int64_t r = 0; r < n; ++r) {
    const int64_t *c = acgt + 4 * r;
    const int64_t total = c[0] + c[1] + c[2] + c[3];
    if (total <= 0) { set_error("ckm_format_unbinned: a sequence without A, C, G, T or U (row " + std::to_string((long long)r) + ")"); return CKM_EINVAL; }
    const double gc = (double)(c[2] + c[1]) * 100.0 / (double)total;      // float(g + c) * 100 / (a + c + g + t)
    fasta_out[fw++] = '>';
    std::memcpy(fasta_out + fw, ids + id_start[r], (size_t)id_len[r]); fw += id_len[r];
    fasta_out[fw++] = '\n';
    std::memcpy(fasta_out + fw, bytes + starts[r], (size_t)lens[r]); fw += lens[r];
    fasta_out[fw++] = '\n';
    std::memcpy(stats_out + sw, ids + id_start[r], (size_t)id_len[r]); sw += id_len[r];
    const int k = std::snprintf(line, sizeof(line), "\t%lld\t%.2f\n", (long long)lens[r], gc);
    std::memcpy(stats_out + sw, line, (size_t)k); sw += k;
  }
  *fasta_len_out = fw; *stats_len_out = sw;
  return CKM_OK;
}

}  // extern "C"
