// outliers.cu -- `checkm outliers` (checkm/binTools.py:148-296): every sequence of every bin of a batch scored against its
// bin's GC, coding density and tetranucleotide signature in one device pass, and the host reader of the profile file.
//
// What the reference computes, restated.  Per bin, over its sequences s in dictionary order, with the integers
// a, c, g, t (A/C/G/T-or-U counts of the upper-cased sequence), len and coding (bases under a gene):
//   GC_s = double(g+c) / (a+c+g+t)         meanGC = double(sum(g+c)) / sum(a+c+g+t)       deltaGC_s = GC_s - meanGC
//   CD_s = double(coding) / len            meanCD = double(sum coding) / sum(len)         deltaCD_s = CD_s - meanCD
//   binSig = sig_0 * (double(len_0)/binSize), then binSig += sig_s * (double(len_s)/binSize) for s = 1, 2, ...  (136 columns,
//            product first, then the sum: the library builds with --fmad=false, so no FMA contracts the two)
//   TD_s   = np.sum(np.abs(sig_s - binSig))            meanTD = np.mean(TD)
// and per sequence the bounds of the length key nearest to len (first minimum of |key - len|) in the bin's GC table, the bin's
// CD table and the TD table; the sequence is outlying in GC when deltaGC < lower or deltaGC > upper, in CD when
// deltaCD < lower, in TD when TD > upper (all strict; a nan compares false).
//
// np.sum and np.mean of a contiguous float64 vector add in numpy's pairwise order, not left to right (pairwise.cuh).
//
// Which GC and CD table a bin uses, and which percentile columns, depends on the bin means (binTools.py:250-261).  The
// caller resolves that on the host from the same integer totals and passes each distinct (table, percentile columns) once as
// a list of (length key, lower, upper); a bin names its two lists by index.
//
// Device work.
//   outlier_bin_kernel   one block per bin.  The four integer totals by shared-memory atomics (exact, order-free), the two
//                        means from them; then thread c < 136 walks column c of the bin's signature rows in order, eight
//                        rows loaded ahead of the adds, so a row is one coalesced 1,088-byte read.
//   outlier_seq_kernel   half a warp per sequence.  136 = 64 + 72 terms: lanes 0-7 are the eight running sums of the first
//                        half (8 rounds), lanes 8-15 those of the second (9 rounds); three shuffles combine each eight in
//                        numpy's order and a fourth adds the halves.  Lane 0 then forms the ratios, finds the three length
//                        keys and writes the nine values and the mask.
//   outlier_mean_kernel  one block per bin: the pairwise tree over the bin's TDs.  The tree is stored as a binary heap
//                        (node i has children 2i+1, 2i+2); a node's range follows from the path its index spells, so every
//                        thread finds its own node.  Leaves (at most 128 elements) are summed first, then the levels are
//                        combined bottom-up.
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <thread>
#include <vector>
#include "engine.hpp"
#include "pool.hpp"
#include "pairwise.cuh"

using namespace ckm;

struct ckm_sigs {
  double *d = nullptr;
  int64_t nrows = 0;
  int device = 0;
};

namespace {

constexpr int OL_COLS = 136;                   // canonical tetranucleotides
constexpr int OL_SEQ_VALUES = 9;               // GC, deltaGC, CD, deltaCD, TD, GC lower, GC upper, CD lower, TD upper
constexpr int OL_AHEAD = 8;                    // signature rows in flight per column chain

struct OutlierParams {
  long long nseq; int nbins;
  const long long *bin_off;                    // nbins + 1
  const int *seq_bin;                          // nseq
  const long long *len, *acgt, *coding, *row;  // nseq (acgt: nseq x 4)
  const double *sig;                           // the profile matrix, nrows x 136
  const int *bin_gc, *bin_cd; int td_table;    // bound lists by index
  const long long *tab_off;                    // ntables + 1
  const double *tab_key, *tab_lo, *tab_hi;
  const double *binsig_in;                     // optional: bin signatures to use in place of the computed ones
  double *binsig;                              // nbins x 136
  double *means;                               // nbins x 3: meanGC, meanCD, meanTD
  double *seq;                                 // nseq x 9
  double *td;                                  // nseq, contiguous, for the mean
  unsigned char *mask;                         // nseq: 1 GC, 2 CD, 4 TD
  const long long *heap_off; const int *depth; // per bin: first heap slot, depth of the pairwise tree
  double *heap;
};

__global__ void __launch_bounds__(160) outlier_bin_kernel(OutlierParams q) {
  const int b = blockIdx.x, t = threadIdx.x;
  const long long s0 = q.bin_off[b], s1 = q.bin_off[b + 1];
  __shared__ unsigned long long tot[4];        // G+C, A+C+G+T, coding, length
  if (t < 4) tot[t] = 0;
  __syncthreads();
  unsigned long long gc = 0, all = 0, cod = 0, len = 0;
  for (long long s = s0 + t; s < s1; s += blockDim.x) {
    const long long *n = q.acgt + 4 * s;
    gc += n[1] + n[2]; all += n[0] + n[1] + n[2] + n[3]; cod += q.coding[s]; len += q.len[s];
  }
  atomicAdd(&tot[0], gc); atomicAdd(&tot[1], all); atomicAdd(&tot[2], cod); atomicAdd(&tot[3], len);
  __syncthreads();
  if (t == 0) {
    q.means[3 * b + 0] = (double)tot[0] / (double)tot[1];
    q.means[3 * b + 1] = (double)tot[2] / (double)tot[3];
  }
  if (t >= OL_COLS) return;
  double acc = 0.0;
  if (q.binsig_in) acc = q.binsig_in[(size_t)b * OL_COLS + t];
  else {
    const double size = (double)tot[3];
    for (long long s = s0; s < s1; s += OL_AHEAD) {
      const int m = (int)min((long long)OL_AHEAD, s1 - s);
      double v[OL_AHEAD], w[OL_AHEAD];
#pragma unroll
      for (int k = 0; k < OL_AHEAD; ++k)
        if (k < m) { v[k] = q.sig[(size_t)q.row[s + k] * OL_COLS + t]; w[k] = (double)q.len[s + k] / size; }
#pragma unroll
      for (int k = 0; k < OL_AHEAD; ++k)
        if (k < m) { const double x = v[k] * w[k]; acc = (s + k == s0) ? x : acc + x; }
    }
  }
  q.binsig[(size_t)b * OL_COLS + t] = acc;
}

__device__ __forceinline__ long long ol_nearest(const OutlierParams &q, int table, double len) {
  const long long lo = q.tab_off[table], hi = q.tab_off[table + 1];
  long long best = lo;
  double d0 = fabs(q.tab_key[lo] - len);
  for (long long i = lo + 1; i < hi; ++i) {
    const double d = fabs(q.tab_key[i] - len);
    if (d < d0) { d0 = d; best = i; }          // the first minimum wins, as np.argmin
  }
  return best;
}

__global__ void __launch_bounds__(256) outlier_seq_kernel(OutlierParams q) {
  const int hl = threadIdx.x & 15;
  const long long sraw = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 4;
  const bool live = sraw < q.nseq;
  const long long s = live ? sraw : q.nseq - 1;
  const int b = q.seq_bin[s];
  const double *x = q.sig + (size_t)q.row[s] * OL_COLS, *y = q.binsig + (size_t)b * OL_COLS;
  const int half = hl >> 3, j = hl & 7, base = half * 64, rounds = 8 + half;
  double r = fabs(x[base + j] - y[base + j]);
  for (int k = 1; k < rounds; ++k) { const int i = base + 8 * k + j; r += fabs(x[i] - y[i]); }
  r = r + __shfl_down_sync(0xFFFFFFFFu, r, 1, 16);
  r = r + __shfl_down_sync(0xFFFFFFFFu, r, 2, 16);
  r = r + __shfl_down_sync(0xFFFFFFFFu, r, 4, 16);
  const double td = r + __shfl_down_sync(0xFFFFFFFFu, r, 8, 16);
  if (!live || hl != 0) return;
  const long long *n = q.acgt + 4 * s;
  const double gc = (double)(n[1] + n[2]) / (double)(n[0] + n[1] + n[2] + n[3]);
  const double dgc = gc - q.means[3 * b + 0];
  const double len = (double)q.len[s];
  const double cd = (double)q.coding[s] / len;
  const double dcd = cd - q.means[3 * b + 1];
  const long long ig = ol_nearest(q, q.bin_gc[b], len), ic = ol_nearest(q, q.bin_cd[b], len), it = ol_nearest(q, q.td_table, len);
  const double gc_lo = q.tab_lo[ig], gc_hi = q.tab_hi[ig], cd_lo = q.tab_lo[ic], td_hi = q.tab_hi[it];
  double *o = q.seq + (size_t)s * OL_SEQ_VALUES;
  o[0] = gc; o[1] = dgc; o[2] = cd; o[3] = dcd; o[4] = td; o[5] = gc_lo; o[6] = gc_hi; o[7] = cd_lo; o[8] = td_hi;
  q.td[s] = td;
  q.mask[s] = (unsigned char)(((dgc < gc_lo || dgc > gc_hi) ? 1 : 0) | (dcd < cd_lo ? 2 : 0) | (td > td_hi ? 4 : 0));
}

// the range [off, off + cnt) of the node that `slot` spells at `depth` (bit depth-1 first; 0 = first half), or false when
// the path runs through a leaf
__device__ __forceinline__ bool ol_node(long long n, int depth, unsigned slot, long long &off, long long &cnt) {
  off = 0; cnt = n;
  for (int d = depth - 1; d >= 0; --d) {
    if (cnt <= PW_LEAF) return false;
    const long long n2 = pw_split(cnt);
    if ((slot >> d) & 1u) { off += n2; cnt -= n2; } else cnt = n2;
  }
  return true;
}

__global__ void __launch_bounds__(256) outlier_mean_kernel(OutlierParams q) {
  const int b = blockIdx.x;
  const long long s0 = q.bin_off[b], n = q.bin_off[b + 1] - s0;
  const int D = q.depth[b];
  double *heap = q.heap + q.heap_off[b];
  const double *a = q.td + s0;
  const unsigned slots = (2u << D) - 1u;
  for (unsigned i = threadIdx.x; i < slots; i += blockDim.x) {
    const int d = 31 - __clz(i + 1);
    long long off, cnt;
    if (ol_node(n, d, i + 1 - (1u << d), off, cnt) && cnt <= PW_LEAF) {
      const double *leaf = a + off;
      heap[i] = pw_leaf_sum([leaf](int k) { return leaf[k]; }, (int)cnt);
    }
  }
  for (int d = D - 1; d >= 0; --d) {
    __syncthreads();
    for (unsigned slot = threadIdx.x; slot < (1u << d); slot += blockDim.x) {
      const unsigned i = (1u << d) - 1u + slot;
      long long off, cnt;
      if (ol_node(n, d, slot, off, cnt) && cnt > PW_LEAF) heap[i] = heap[2 * i + 1] + heap[2 * i + 2];
    }
  }
  __syncthreads();
  if (threadIdx.x == 0) q.means[3 * b + 2] = heap[0] / (double)n;
}

// one line `id\tv1\t...\tvN` of the profile file; returns 0, or the 1-based column that does not parse (ncols + 2: too many)
int parse_profile_line(const char *p, const char *end, int ncols, int64_t *id_len, double *out) {
  const char *tab = (const char *)std::memchr(p, '\t', (size_t)(end - p));
  if (!tab) return 1;
  *id_len = tab - p;
  const char *f = tab + 1;
  char buf[64];
  for (int c = 0; c < ncols; ++c) {
    const char *stop = (const char *)std::memchr(f, '\t', (size_t)(end - f));
    const bool last = c == ncols - 1;
    if (last ? stop != nullptr : stop == nullptr) return last ? ncols + 2 : c + 2;
    if (!stop) stop = end;
    size_t n = (size_t)(stop - f);
    while (n > 0 && (f[n - 1] == '\r' || f[n - 1] == ' ')) --n;            // float() strips blanks
    if (n == 0 || n >= sizeof(buf)) return c + 2;
    std::memcpy(buf, f, n);
    buf[n] = 0;
    for (size_t k = 0; k < n; ++k)
      if (buf[k] == 'x' || buf[k] == 'X' || buf[k] == '(' || buf[k] == ',') return c + 2;   // strtod's hex floats, nan(...) and locale commas are not float()'s
    char *rest = nullptr;
    out[c] = std::strtod(buf, &rest);                                      // glibc: correctly rounded, as float()
    if (rest != buf + n) return c + 2;
    f = stop + 1;
  }
  return 0;
}

}  // namespace

extern "C" {

int ckm_parse_kmer_profiles(const char *text, int64_t n, int32_t ncols, int32_t nthreads, int64_t *id_start_out,
                            int32_t *id_len_out, double *values_out, int64_t row_cap, int64_t *nrows_out) {
  if (!text || n < 0 || ncols < 1 || !nrows_out || row_cap < 0 || (row_cap > 0 && (!id_start_out || !id_len_out || !values_out))) {
    set_error("ckm_parse_kmer_profiles: bad argument"); return CKM_EINVAL;
  }
  *nrows_out = 0;
  if (n == 0) { set_error("ckm_parse_kmer_profiles: the profile file is empty (line 1: no header)"); return CKM_EFORMAT; }
  const char *end = text + n;
  const char *nl = (const char *)std::memchr(text, '\n', (size_t)n);
  std::vector<int64_t> line_start;                                         // after the header
  for (const char *p = nl ? nl + 1 : end; p < end;) {
    line_start.push_back(p - text);
    const char *q = (const char *)std::memchr(p, '\n', (size_t)(end - p));
    p = q ? q + 1 : end;
  }
  const int64_t rows = (int64_t)line_start.size();
  *nrows_out = rows;
  if (rows > row_cap) { set_error("ckm_parse_kmer_profiles: more lines than the capacity (the number needed is returned)"); return CKM_ECAPACITY; }
  line_start.push_back(n);
  const int nt = (int)std::max<int64_t>(1, std::min<int64_t>(std::min(nthreads, 64), rows / 1024));
  std::vector<int64_t> bad_row(nt, -1);
  std::vector<int> bad_col(nt, 0);
  auto work = [&](int w) {
    for (int64_t r = rows * w / nt; r < rows * (w + 1) / nt; ++r) {
      const char *p = text + line_start[r], *e = text + line_start[r + 1];
      if (e > p && e[-1] == '\n') --e;
      int64_t idn = 0;
      const int col = parse_profile_line(p, e, ncols, &idn, values_out + (size_t)r * ncols);
      if (col || idn > 0x7FFFFFFF) { bad_row[w] = r; bad_col[w] = col; return; }
      id_start_out[r] = line_start[r];
      id_len_out[r] = (int32_t)idn;
    }
  };
  if (nt == 1) work(0);
  else {
    std::vector<std::thread> pool;
    for (int w = 0; w < nt; ++w) pool.emplace_back(work, w);
    for (auto &t : pool) t.join();
  }
  for (int w = 0; w < nt; ++w)
    if (bad_row[w] >= 0) {
      char msg[160];
      if (bad_col[w] == ncols + 2 || bad_col[w] == 1)
        std::snprintf(msg, sizeof(msg), "ckm_parse_kmer_profiles: line %lld does not have an id and %d values",
                      (long long)bad_row[w] + 2, ncols);
      else
        std::snprintf(msg, sizeof(msg), "ckm_parse_kmer_profiles: line %lld, column %d: not a number or a missing column",
                      (long long)bad_row[w] + 2, bad_col[w]);
      set_error(msg);
      return CKM_EFORMAT;
    }
  return CKM_OK;
}

int ckm_sigs_create(ckm_engine *e, const double *values, int64_t nrows, ckm_sigs **out) {
  if (!e || !out || nrows < 1 || !values) { set_error("ckm_sigs_create: bad argument"); return CKM_EINVAL; }
  *out = nullptr;
  cudaSetDevice(e->device);
  ckm_sigs *s = new ckm_sigs;
  s->nrows = nrows; s->device = e->device;
  const size_t bytes = sizeof(double) * (size_t)nrows * OL_COLS;
  cudaError_t err = cudaMalloc(&s->d, bytes);
  if (err == cudaSuccess) err = cudaMemcpy(s->d, values, bytes, cudaMemcpyHostToDevice);
  if (err != cudaSuccess) {
    if (s->d) cudaFree(s->d);
    delete s;
    return cuda_fail(err, "ckm_sigs_create");
  }
  *out = s;
  return CKM_OK;
}

void ckm_sigs_free(ckm_sigs *s) {
  if (!s) return;
  cudaSetDevice(s->device);
  cudaFree(s->d);
  delete s;
}

int ckm_outlier_scores(ckm_engine *e, const ckm_sigs *sigs, const ckm_outlier_in *in, ckm_outlier_out *out) {
  if (!e || !sigs || !in || !out || in->nbins < 1 || in->nseq < 1 || in->ntables < 1 || !in->bin_off || !in->len || !in->acgt ||
      !in->coding || !in->sig_row || !in->bin_gc_table || !in->bin_cd_table || !in->table_off || !in->table_key ||
      !in->table_lo || !in->table_hi || !out->bin_means || !out->seq_values || !out->seq_mask ||
      in->td_table < 0 || in->td_table >= in->ntables || sigs->device != e->device) {
    set_error("ckm_outlier_scores: bad argument"); return CKM_EINVAL;
  }
  const int nbins = in->nbins;
  const long long nseq = in->nseq;
  char msg[200];
  if (in->bin_off[0] != 0 || in->bin_off[nbins] != nseq) { set_error("ckm_outlier_scores: bin offsets must run from 0 to nseq"); return CKM_EINVAL; }
  for (int t = 0; t < in->ntables; ++t)
    if (in->table_off[t + 1] <= in->table_off[t] || in->table_off[0] != 0) { set_error("ckm_outlier_scores: every bound table needs at least one length key"); return CKM_EINVAL; }
  std::vector<int> seq_bin((size_t)nseq);
  std::vector<long long> heap_off((size_t)nbins + 1, 0);
  std::vector<int> depth((size_t)nbins);
  for (int b = 0; b < nbins; ++b) {
    const long long s0 = in->bin_off[b], s1 = in->bin_off[b + 1];
    if (s1 <= s0) { std::snprintf(msg, sizeof(msg), "ckm_outlier_scores: bin %d has no sequences", b); set_error(msg); return CKM_EINVAL; }
    if (in->bin_gc_table[b] < 0 || in->bin_gc_table[b] >= in->ntables || in->bin_cd_table[b] < 0 || in->bin_cd_table[b] >= in->ntables) {
      set_error("ckm_outlier_scores: bound table index out of range"); return CKM_EINVAL;
    }
    for (long long s = s0; s < s1; ++s) {
      seq_bin[(size_t)s] = b;
      const int64_t *c = in->acgt + 4 * s;
      const char *what = nullptr;
      if (in->len[s] < 1) what = "is empty";
      else if (c[0] < 0 || c[1] < 0 || c[2] < 0 || c[3] < 0 || c[0] + c[1] + c[2] + c[3] < 1) what = "has no A, C, G or T";
      else if (in->sig_row[s] < 0 || in->sig_row[s] >= sigs->nrows) what = "has no row in the signature matrix";
      else if (in->coding[s] < 0) what = "has a negative number of coding bases";
      if (what) {
        std::snprintf(msg, sizeof(msg), "ckm_outlier_scores: sequence %lld (the %lld-th of bin %d) %s", s, s - s0, b, what);
        set_error(msg); return CKM_EINVAL;
      }
    }
    depth[b] = pairwise_depth(s1 - s0);
    heap_off[b + 1] = heap_off[b] + ((2ll << depth[b]) - 1);
  }
  const long long nkeys = in->table_off[in->ntables];
  const DeviceScope ws(e);
  const size_t ns = (size_t)nseq, nb = (size_t)nbins;
  DevBuf dboff, dsbin, dlen, dacgt, dcod, drow, dbgc, dbcd, dtoff, dkey, dlo, dhi, dbsin, dbsig, dmeans, dseq, dtd, dmask, dhoff, ddepth, dheap;
  CKM_TRY(dboff.put(in->bin_off, nb + 1, ws.st));
  CKM_TRY(dsbin.put(seq_bin.data(), ns, ws.st));
  CKM_TRY(dlen.put(in->len, ns, ws.st));
  CKM_TRY(dacgt.put(in->acgt, 4 * ns, ws.st));
  CKM_TRY(dcod.put(in->coding, ns, ws.st));
  CKM_TRY(drow.put(in->sig_row, ns, ws.st));
  CKM_TRY(dbgc.put(in->bin_gc_table, nb, ws.st));
  CKM_TRY(dbcd.put(in->bin_cd_table, nb, ws.st));
  CKM_TRY(dtoff.put(in->table_off, (size_t)in->ntables + 1, ws.st));
  CKM_TRY(dkey.put(in->table_key, (size_t)nkeys, ws.st));
  CKM_TRY(dlo.put(in->table_lo, (size_t)nkeys, ws.st));
  CKM_TRY(dhi.put(in->table_hi, (size_t)nkeys, ws.st));
  CKM_TRY(dbsin.put(in->binsig_in, in->binsig_in ? nb * OL_COLS : 0, ws.st));
  CKM_TRY(dhoff.put(heap_off.data(), nb + 1, ws.st));
  CKM_TRY(ddepth.put(depth.data(), nb, ws.st));
  CKM_TRY(dbsig.alloc(8 * nb * OL_COLS));
  CKM_TRY(dmeans.alloc(8 * nb * 3));
  CKM_TRY(dseq.alloc(8 * ns * OL_SEQ_VALUES));
  CKM_TRY(dtd.alloc(8 * ns));
  CKM_TRY(dmask.alloc(ns));
  CKM_TRY(dheap.alloc(8 * (size_t)heap_off[nb]));
  OutlierParams q;
  std::memset(&q, 0, sizeof(q));
  q.nseq = nseq; q.nbins = nbins;
  q.bin_off = dboff.as<long long>(); q.seq_bin = dsbin.as<int>(); q.len = dlen.as<long long>(); q.acgt = dacgt.as<long long>();
  q.coding = dcod.as<long long>(); q.row = drow.as<long long>(); q.sig = sigs->d;
  q.bin_gc = dbgc.as<int>(); q.bin_cd = dbcd.as<int>(); q.td_table = in->td_table;
  q.tab_off = dtoff.as<long long>(); q.tab_key = dkey.as<double>(); q.tab_lo = dlo.as<double>(); q.tab_hi = dhi.as<double>();
  q.binsig_in = in->binsig_in ? dbsin.as<double>() : nullptr;
  q.binsig = dbsig.as<double>(); q.means = dmeans.as<double>(); q.seq = dseq.as<double>(); q.td = dtd.as<double>();
  q.mask = dmask.as<unsigned char>(); q.heap_off = dhoff.as<long long>(); q.depth = ddepth.as<int>(); q.heap = dheap.as<double>();
  CKM_TRY(ev_record(e, 0));
  outlier_bin_kernel<<<nbins, 160, 0, ws.st>>>(q);
  CKM_CUDA(cudaGetLastError());
  CKM_TRY(ev_record(e, 1));
  outlier_seq_kernel<<<(unsigned)((nseq + 15) / 16), 256, 0, ws.st>>>(q);
  CKM_CUDA(cudaGetLastError());
  CKM_TRY(ev_record(e, 2));
  outlier_mean_kernel<<<nbins, 256, 0, ws.st>>>(q);
  CKM_CUDA(cudaGetLastError());
  CKM_TRY(ev_record(e, 3));
  CKM_TRY(dmeans.get(out->bin_means, nb * 3, ws.st));
  CKM_TRY(dbsig.get(out->bin_sig, out->bin_sig ? nb * OL_COLS : 0, ws.st));
  CKM_TRY(dseq.get(out->seq_values, ns * OL_SEQ_VALUES, ws.st));
  CKM_TRY(dmask.get(out->seq_mask, ns, ws.st));
  CKM_TRY(stream_sync(ws.st));
  for (int k = 0; k < 3; ++k) CKM_TRY(ev_elapsed(e, &out->kernel_ms[k], k, k + 1));
  return CKM_OK;
}

}  // extern "C"
