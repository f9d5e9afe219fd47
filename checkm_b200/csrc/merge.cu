// merge.cu -- `checkm merge` (checkm/merger.py:34-110): every pair of bins with complementary marker genes, in one
// device pass, and the host writer of the merger.tsv rows.
//
// What the reference computes, restated.  The bins' most specific marker sets all share one marker union G
// (merger.py:43-47).  Per bin b, from its reduced hit dict and its own marker set ms_b:
//   c_b[g] = len(markerHits[g]) for g in G (0 when absent)
//   N_b    = ms_b.numMarkers(), the sum of the set sizes (larger than |G| when a marker is in two sets)
//   p_b    = #{g : c_b[g] >= 1},  s_b = sum_g c_b[g]
//   comp_b = 100 * double(p_b) / N_b,  cont_b = 100 * double(s_b - p_b) / N_b       (markerSets.py:208-217, individual mode)
// For every pair i < j of the bins in sorted() id order, the merged dict holds c_i[g] + c_j[g] hits per marker, and it is
// scored against bin J's marker set (merger.py:89):
//   x = #{g : c_i[g] >= 1 and c_j[g] >= 1},  p = p_i + p_j - x,  s = s_i + s_j
//   comp = 100 * double(p) / N_j,  cont = 100 * double(s - p) / N_j
// and the pair is written iff comp >= min_merged_comp, cont < max_merged_cont, comp - max(comp_i, comp_j) >= min_delta_comp
// and cont - max(cont_i, cont_j) < max_delta_cont (merger.py:92-100), in the order i ascending, then j ascending.
//
// Presence.  The reference counts a marker as present when its key is in the dict (markerSets.py:212); here it is c >= 1.
// The two agree because no reduction leaves an empty list under a key: the reference's addHit creates a key with one
// hit, filterHitsFromSameClan (util/pfam.py:86-147) appends to a key only when it keeps a hit, identifyAdjacentMarkerGenes
// replaces two hits by one; ckm_reduce creates a marker's entry with its first kept hit.
//
// Individual mode over the union.  genomeCheck iterates over G, so a marker in two sets of ms_b counts once in p and s,
// while N_b counts it twice.  ckm_genome_check's individual mode counts per entry of the sets instead; this file
// follows the reference.
//
// Device work.
//   merge_pack_kernel   one warp per bin: the presence bits of its row (one ballot per 32 markers), p_b and s_b.  The
//                       bits are stored word-major, bits[w * Bp + b], so a tile of 64 bins at one word is one 256-byte load.
//   merge_gram_kernel   x for the upper triangle of 64 x 64 tiles as a popcount Gram matrix: the tile's bit rows are
//                       staged through shared memory 8 words at a time, each thread keeps 4 x 4 accumulators in registers
//                       (LOP3 + POPC in place of the FMA of a GEMM).  The epilogue applies the filter in float64 with the
//                       operations above (the library builds with --fmad=false) and stores, per bin i and tile column,
//                       the 64-bit mask of the passing j, and adds its popcount to the count of row i.
//   (host)              the row counts come back; their sum is the number of pairs.  More than the caller's capacity ->
//                       CKM_ECAPACITY with the number needed.  Else an exclusive scan gives each row its first record.
//   merge_emit_kernel   one warp per row i: walks the row's masks in column order, lane l takes the l-th set bit, recomputes
//                       x for that pair from the bit rows (W words, the 64 j of a mask word are one 256-byte line per word)
//                       and writes (i, j, p, s) at its rank.  The records are in reference order without a sort.
// The Gram kernel is bound by POPC issue: B(B-1)/2 * W popcounts, where W is |G|/32 rounded up to 8.  The emit kernel
// costs W popcounts per passing pair.
#include <algorithm>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <vector>
#include "engine.hpp"
#include "pool.hpp"

using namespace ckm;

namespace {

constexpr int MG_TILE = 64;                    // bins per tile side
constexpr int MG_KC = 8;                       // 32-bit words per shared-memory stage
constexpr int MG_THREADS = 256;                // 16 x 16 threads, 4 x 4 pairs each
constexpr int MG_EMIT_WARPS = 8;

struct MergeParams {
  const int32_t *counts;                       // nbins x nmarkers
  const int32_t *nmk;                          // N_b
  int32_t nbins, nmarkers, W, Bp, nt;          // W: words per bit row (multiple of MG_KC); Bp: nbins rounded up to MG_TILE; nt: tiles per side
  uint32_t *bits;                              // W x Bp
  int32_t *p; long long *s;                    // per bin
  double *comp, *cont;                         // per bin
  unsigned long long *mask;                    // nbins x nt
  unsigned long long *rowcount;                // nbins, zeroed
  const long long *rowoff;                     // nbins: first record of row i
  int *bad;                                    // set when a copy number is negative or s_b is too large
  double min_delta_comp, max_delta_cont, min_merged_comp, max_merged_cont;
  int4 *out;                                   // (i, j, p, s)
};

__global__ void __launch_bounds__(256) merge_pack_kernel(MergeParams q) {
  const int lane = threadIdx.x & 31;
  const int b = blockIdx.x * 8 + (threadIdx.x >> 5);
  if (b >= q.nbins) return;
  const int32_t *row = q.counts + (size_t)b * q.nmarkers;
  int pres = 0; long long sum = 0; bool neg = false;
  for (int w = 0; w * 32 < q.nmarkers; ++w) {
    const int g = w * 32 + lane;
    const int c = g < q.nmarkers ? row[g] : 0;
    neg |= c < 0;
    sum += c;
    const uint32_t m = __ballot_sync(0xFFFFFFFFu, c > 0);
    if (lane == 0) q.bits[(size_t)w * q.Bp + b] = m;
    pres += __popc(m);
  }
  for (int o = 16; o; o >>= 1) sum += __shfl_xor_sync(0xFFFFFFFFu, sum, o);
  if (__any_sync(0xFFFFFFFFu, neg) || sum > 0x3FFFFFFFll) { if (lane == 0) atomicOr(q.bad, 1); }
  if (lane == 0) {
    q.p[b] = pres; q.s[b] = sum;
    const double n = (double)q.nmk[b];
    q.comp[b] = 100.0 * (double)pres / n;
    q.cont[b] = 100.0 * (double)(sum - pres) / n;
  }
}

__device__ __forceinline__ bool merge_passes(const MergeParams &q, int i, int j, int x) {
  const int p = q.p[i] + q.p[j] - x;
  const long long s = q.s[i] + q.s[j];
  const double n = (double)q.nmk[j];
  const double comp = 100.0 * (double)p / n;
  const double cont = 100.0 * (double)(s - p) / n;
  if (!(comp >= q.min_merged_comp && cont < q.max_merged_cont)) return false;
  const double ci = q.comp[i], cj = q.comp[j], ki = q.cont[i], kj = q.cont[j];
  const double dcomp = comp - (cj > ci ? cj : ci);              // Python's max(a, b): a unless b > a
  const double dcont = cont - (kj > ki ? kj : ki);
  return dcomp >= q.min_delta_comp && dcont < q.max_delta_cont;
}

__global__ void __launch_bounds__(MG_THREADS, 4) merge_gram_kernel(MergeParams q) {
  const int ti = blockIdx.y, tj = blockIdx.x;
  if (tj < ti) return;
  __shared__ __align__(16) uint32_t sa[MG_KC][MG_TILE];
  __shared__ __align__(16) uint32_t sb[MG_KC][MG_TILE];
  __shared__ int sx[MG_TILE][MG_TILE + 1];                      // x of the tile, for the epilogue
  const int t = threadIdx.x, tx = t & 15, ty = t >> 4;
  const int i0 = ti * MG_TILE, j0 = tj * MG_TILE;
  int acc[4][4];
#pragma unroll
  for (int a = 0; a < 4; ++a)
#pragma unroll
    for (int b = 0; b < 4; ++b) acc[a][b] = 0;
  // loaders: threads 0..127 stage A, 128..255 stage B; 8 words x 64 bins = 128 uint4 per side
  const int lt = t & 127, lk = lt >> 4, lc = (lt & 15) * 4;
  const uint32_t *src = q.bits + (size_t)lk * q.Bp + (t < 128 ? i0 : j0) + lc;
  uint32_t *dst = (t < 128 ? &sa[lk][lc] : &sb[lk][lc]);
  for (int k0 = 0; k0 < q.W; k0 += MG_KC) {
    *reinterpret_cast<uint4 *>(dst) = __ldg(reinterpret_cast<const uint4 *>(src + (size_t)k0 * q.Bp));
    __syncthreads();
#pragma unroll
    for (int k = 0; k < MG_KC; ++k) {
      const uint4 a = *reinterpret_cast<const uint4 *>(&sa[k][ty * 4]);
      const uint4 b = *reinterpret_cast<const uint4 *>(&sb[k][tx * 4]);
      const uint32_t av[4] = {a.x, a.y, a.z, a.w}, bv[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
      for (int r = 0; r < 4; ++r)
#pragma unroll
        for (int c = 0; c < 4; ++c) acc[r][c] += __popc(av[r] & bv[c]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int r = 0; r < 4; ++r)
#pragma unroll
    for (int c = 0; c < 4; ++c) sx[ty * 4 + r][tx * 4 + c] = acc[r][c];
  __syncthreads();
  // epilogue: warp w takes rows w, w + 8, ...; lane l columns l and l + 32, so one ballot gives each half of the row's mask
  const int lane = t & 31, warp = t >> 5;
#pragma unroll 1
  for (int r = warp; r < MG_TILE; r += MG_THREADS / 32) {
    const int i = i0 + r;
    if (i >= q.nbins) break;
    const int ja = j0 + lane, jb = ja + 32;
    const uint32_t lo = __ballot_sync(0xFFFFFFFFu, i < ja && ja < q.nbins && merge_passes(q, i, ja, sx[r][lane]));
    const uint32_t hi = __ballot_sync(0xFFFFFFFFu, i < jb && jb < q.nbins && merge_passes(q, i, jb, sx[r][lane + 32]));
    if (lane == 0) {
      const unsigned long long m = (unsigned long long)hi << 32 | lo;
      q.mask[(size_t)i * q.nt + tj] = m;
      if (m) atomicAdd(&q.rowcount[i], (unsigned long long)__popcll(m));
    }
  }
}

__global__ void __launch_bounds__(MG_EMIT_WARPS * 32) merge_emit_kernel(MergeParams q) {
  const int lane = threadIdx.x & 31;
  const int i = blockIdx.x * MG_EMIT_WARPS + (threadIdx.x >> 5);
  if (i >= q.nbins) return;
  long long at = q.rowoff[i];
  const int pi = q.p[i]; const long long si = q.s[i];
  for (int tj = i / MG_TILE; tj < q.nt; ++tj) {
    const unsigned long long m = q.mask[(size_t)i * q.nt + tj];
    if (!m) continue;
    const uint32_t lo = (uint32_t)m, hi = (uint32_t)(m >> 32);
    const int nlo = __popc(lo), n = nlo + __popc(hi);
    for (int base = 0; base < n; base += 32) {
      const int r = base + lane;
      if (r < n) {
        const int bit = r < nlo ? __fns(lo, 0, r + 1) : 32 + __fns(hi, 0, r - nlo + 1);
        const int j = tj * MG_TILE + bit;
        int x = 0;
        for (int w = 0; w < q.W; ++w) x += __popc(__ldg(q.bits + (size_t)w * q.Bp + i) & __ldg(q.bits + (size_t)w * q.Bp + j));
        q.out[at + r] = make_int4(i, j, pi + q.p[j] - x, (int)(si + q.s[j]));
      }
    }
    at += n;
  }
}

}  // namespace

extern "C" {

int ckm_merge_pairs(ckm_engine *e, const int32_t *counts, int32_t nbins, int32_t nmarkers, const int32_t *n_markers,
                    double min_delta_comp, double max_delta_cont, double min_merged_comp, double max_merged_cont,
                    ckm_merge_pair *pairs_out, int64_t pair_cap, int64_t *npairs_out, float *kernel_ms_out) {
  static_assert(sizeof(ckm_merge_pair) == sizeof(int4), "ckm_merge_pair is four int32");
  if (!e || nbins < 0 || nmarkers < 0 || !npairs_out || pair_cap < 0 || (pair_cap > 0 && !pairs_out) ||
      (nbins > 0 && (!n_markers || (nmarkers > 0 && !counts)))) {
    set_error("ckm_merge_pairs: bad argument"); return CKM_EINVAL;
  }
  *npairs_out = 0;
  if (kernel_ms_out) *kernel_ms_out = 0.0f;
  for (int32_t b = 0; b < nbins; ++b)
    if (n_markers[b] < 1) { set_error("ckm_merge_pairs: every bin needs a marker set of at least one marker"); return CKM_EINVAL; }
  if (nbins < 2) return CKM_OK;
  if (nbins > 65535 * MG_TILE) { set_error("ckm_merge_pairs: too many bins for one call"); return CKM_EINVAL; }
  MergeParams q;
  std::memset(&q, 0, sizeof(q));
  q.nbins = nbins; q.nmarkers = nmarkers;
  q.W = std::max(1, (nmarkers + 31) / 32);
  q.W = (q.W + MG_KC - 1) / MG_KC * MG_KC;
  q.nt = (nbins + MG_TILE - 1) / MG_TILE;
  q.Bp = q.nt * MG_TILE;
  q.min_delta_comp = min_delta_comp; q.max_delta_cont = max_delta_cont;
  q.min_merged_comp = min_merged_comp; q.max_merged_cont = max_merged_cont;
  const DeviceScope ws(e);
  const size_t nb = (size_t)nbins;
  DevBuf dcounts, dnmk, dbits, dp, ds, dcomp, dcont, dmask, drc, doff, dbad;
  CKM_TRY(dcounts.put(counts, nb * nmarkers, ws.st));
  CKM_TRY(dnmk.put(n_markers, nb, ws.st));
  CKM_TRY(dbits.fill(sizeof(uint32_t) * (size_t)q.W * q.Bp, 0, ws.st));
  CKM_TRY(drc.fill(sizeof(unsigned long long) * nb, 0, ws.st));
  CKM_TRY(dbad.fill(sizeof(int), 0, ws.st));
  CKM_TRY(dp.alloc(sizeof(int32_t) * nb));
  CKM_TRY(ds.alloc(sizeof(long long) * nb));
  CKM_TRY(dcomp.alloc(sizeof(double) * nb));
  CKM_TRY(dcont.alloc(sizeof(double) * nb));
  CKM_TRY(dmask.alloc(sizeof(unsigned long long) * nb * q.nt));
  CKM_TRY(doff.alloc(sizeof(long long) * nb));
  q.counts = dcounts.as<int32_t>(); q.nmk = dnmk.as<int32_t>(); q.bits = dbits.as<uint32_t>();
  q.p = dp.as<int32_t>(); q.s = ds.as<long long>(); q.comp = dcomp.as<double>(); q.cont = dcont.as<double>();
  q.mask = dmask.as<unsigned long long>(); q.rowcount = drc.as<unsigned long long>(); q.rowoff = doff.as<long long>();
  q.bad = dbad.as<int>();
  CKM_TRY(ev_record(e, 0));
  merge_pack_kernel<<<(nbins + 7) / 8, 256, 0, ws.st>>>(q);
  CKM_CUDA(cudaGetLastError());
  merge_gram_kernel<<<dim3(q.nt, q.nt), MG_THREADS, 0, ws.st>>>(q);
  CKM_CUDA(cudaGetLastError());
  CKM_TRY(ev_record(e, 1));
  std::vector<unsigned long long> rowcount(nb);
  int bad = 0;
  CKM_TRY(drc.get(rowcount.data(), nb, ws.st));
  CKM_TRY(dbad.get(&bad, 1, ws.st));
  CKM_TRY(stream_sync(ws.st));
  float ms_gram = 0.0f;
  CKM_TRY(ev_elapsed(e, &ms_gram, 0, 1));
  if (bad) {
    set_error("ckm_merge_pairs: copy numbers must be >= 0 and sum to less than 2^30 per bin");
    return CKM_EINVAL;
  }
  std::vector<long long> rowoff(nb);
  long long total = 0;
  for (size_t b = 0; b < nb; ++b) { rowoff[b] = total; total += (long long)rowcount[b]; }
  *npairs_out = total;
  if (kernel_ms_out) *kernel_ms_out = ms_gram;
  if (total > pair_cap) {
    set_error("ckm_merge_pairs: more passing pairs than the capacity (the number needed is returned)");
    return CKM_ECAPACITY;
  }
  if (total == 0) return CKM_OK;
  DevBuf dout;
  CKM_TRY(dout.alloc(sizeof(int4) * (size_t)total));
  q.out = dout.as<int4>();
  CKM_TRY(copy_in(doff.as<long long>(), rowoff.data(), nb, ws.st));
  CKM_TRY(ev_record(e, 0));
  merge_emit_kernel<<<(nbins + MG_EMIT_WARPS - 1) / MG_EMIT_WARPS, MG_EMIT_WARPS * 32, 0, ws.st>>>(q);
  CKM_CUDA(cudaGetLastError());
  CKM_TRY(ev_record(e, 1));
  CKM_TRY(dout.get(reinterpret_cast<int4 *>(pairs_out), (size_t)total, ws.st));
  CKM_TRY(stream_sync(ws.st));
  float ms_emit = 0.0f;
  CKM_TRY(ev_elapsed(e, &ms_emit, 0, 1));
  if (kernel_ms_out) *kernel_ms_out = ms_gram + ms_emit;
  return CKM_OK;
}

int ckm_format_merger_rows(const char *ids, const int64_t *id_offsets, int32_t nbins, const int32_t *p, const int32_t *s,
                           const int32_t *n_markers, const ckm_merge_pair *pairs, int64_t npairs, char *out, int64_t out_cap,
                           int64_t *out_len) {
  if (nbins < 0 || npairs < 0 || !out_len || out_cap < 0 || (out_cap > 0 && !out) ||
      (nbins > 0 && (!ids || !id_offsets || !p || !s || !n_markers)) || (npairs > 0 && !pairs)) {
    set_error("ckm_format_merger_rows: bad argument"); return CKM_EINVAL;
  }
  for (int32_t b = 0; b < nbins; ++b)
    if (n_markers[b] < 1 || id_offsets[b + 1] < id_offsets[b]) { set_error("ckm_format_merger_rows: bad bin table"); return CKM_EINVAL; }
  for (int64_t r = 0; r < npairs; ++r) {
    const ckm_merge_pair &m = pairs[r];
    if (m.i < 0 || m.j < 0 || m.i >= nbins || m.j >= nbins) { set_error("ckm_format_merger_rows: pair index out of range"); return CKM_EINVAL; }
  }
  int64_t w = 0;
  char line[512];
  for (int64_t r = 0; r < npairs; ++r) {
    const ckm_merge_pair &m = pairs[r];
    const double ni = (double)n_markers[m.i], nj = (double)n_markers[m.j];
    const double ci = 100.0 * (double)p[m.i] / ni, ki = 100.0 * (double)(s[m.i] - p[m.i]) / ni;
    const double cj = 100.0 * (double)p[m.j] / nj, kj = 100.0 * (double)(s[m.j] - p[m.j]) / nj;
    const double comp = 100.0 * (double)m.p / nj, cont = 100.0 * (double)((int64_t)m.s - m.p) / nj;
    const double dcomp = comp - (cj > ci ? cj : ci), dcont = cont - (kj > ki ? kj : ki);
    const int64_t li = id_offsets[m.i + 1] - id_offsets[m.i], lj = id_offsets[m.j + 1] - id_offsets[m.j];
    const int n = std::snprintf(line, sizeof(line), "\t%.2f\t%.2f\t%.2f\t%.2f\t%.2f\t%.2f\t%.2f\t%.2f\t%.2f\n",
                                ci, ki, cj, kj, dcomp, dcont, dcomp - dcont, comp, cont);
    const int64_t need = li + 1 + lj + n;
    if (w + need <= out_cap) {
      char *o = out + w;
      std::memcpy(o, ids + id_offsets[m.i], (size_t)li); o += li;
      *o++ = '\t';
      std::memcpy(o, ids + id_offsets[m.j], (size_t)lj); o += lj;
      std::memcpy(o, line, (size_t)n);
    }
    w += need;
  }
  *out_len = w;
  if (w > out_cap) { set_error("ckm_format_merger_rows: output buffer too small (the size needed is returned)"); return CKM_ECAPACITY; }
  return CKM_OK;
}

}  // extern "C"
