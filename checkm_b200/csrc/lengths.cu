// lengths.cu -- the length profile of every bin behind `checkm nx_plot`, `len_hist` and `marker_plot`
// (checkm/plot/nxPlot.py, lengthHistogram.py, markerGenePosPlot.py): one block per bin sorts the bin's record lengths,
// forms their prefix sums, and from them the Nx list, the status of the reference's Nx loop and the length classes.
//
// What the reference computes, restated for a bin of n records with lengths L (readFasta's dict: one per id):
//   total  = sum(L), an exact integer
//   order  = L sorted descending, equal lengths in record order (Python's stable sort(reverse=True)); rank[i] = the
//            position of record i in it; C[r] = L[order[0]] + ... + L[order[r]], exact
//   T[j]   = x[j] * float(total) in float64 (x ascending; one IEEE multiply, as numpy's x[j] * sum)
//   Nx     = calculateNx's loop: threshold j is reached at k_j, the first r with C[r] >= T[j] (int against float, exactly),
//            and nx[j] = L[order[k_j]]; k_j is non-decreasing because T is.  The loop's `break` leaves only the while, so
//            when the last threshold is reached at K = k_{m-1} < n - 1 the next record appends once more and raises
//            IndexError (status INDEX, at rank K + 1); when some threshold is never reached (an empty bin, x[-1] * total
//            above total) nx is shorter than x and the plot raises (status SHORT with the number reached); else OK.
//   class  = np.histogram(float(len) / 1e3, [0, 1, 2, 5, 10, 20, 50, 100, 200, 500, 1e12]): class c holds
//            e_c <= v < e_{c+1}, the last one also v == 1e12; v is one IEEE division in float64
//
// Device work: length_profile_kernel, one block of LP_THREADS per bin (grid-stride over bins).  The sort is a stable LSD
// radix sort on 8-bit digits of the descending key (255 - digit), only over the bytes the bin's largest length uses,
// between two global buffers: per pass a shared-memory digit histogram and its scan, then tiles of LP_THREADS records
// scattered in record order -- __match_any_sync ranks a record among its warp's equal digits, per-warp digit counts in
// shared memory rank it among the tile's earlier warps.  The inclusive prefix sum runs over the sorted keys tile by tile
// (warp shuffles, a carry between tiles) into the buffer the sort no longer needs; one thread per threshold binary-searches
// it.  A bin is read twice per pass and written once, so the kernel is bound by those passes over L2-resident buffers
// and by the block barriers of the tiles, not by HBM.
#include <cmath>
#include <cstdint>
#include <string>
#include "engine.hpp"
#include "pool.hpp"

using namespace ckm;

namespace {

constexpr int LP_THREADS = 512;
constexpr int LP_WARPS = LP_THREADS / 32;
constexpr int RADIX = 256;
constexpr int NCLASS = 10;
constexpr unsigned FULL = 0xffffffffu;

enum { LP_OK = 0, LP_INDEX = 1, LP_SHORT = 2 };

// c >= t for an integer c and a double t, exactly (t is never NaN here)
__device__ __forceinline__ bool int_ge(int64_t c, double t) {
  if (!(t > -9223372036854775808.0)) return true;
  if (t >= 9223372036854775808.0) return false;
  return c >= (int64_t)ceil(t);
}

// numpy's histogram class of float(len) / 1e3 over the reference's edges; -1 past 1e12
__device__ __forceinline__ int length_class(int64_t len) {
  const double v = (double)len / 1e3;
  const double edges[NCLASS] = {1.0, 2.0, 5.0, 10.0, 20.0, 50.0, 100.0, 200.0, 500.0, 1e12};
  int c = 0;
#pragma unroll
  for (int k = 0; k < NCLASS - 1; ++k) c += v >= edges[k];
  return v > edges[NCLASS - 1] ? -1 : c;
}

__device__ __forceinline__ unsigned digit_of(uint64_t key, int shift) { return 255u - (unsigned)((key >> shift) & 255u); }

__global__ void __launch_bounds__(LP_THREADS) length_profile_kernel(
    const int64_t *__restrict__ len, const int64_t *__restrict__ bin_off, int32_t nbins, const double *__restrict__ x, int32_t m,
    uint64_t *keys_a, uint64_t *keys_b, int32_t *idx_a, int32_t *idx_b, int64_t *__restrict__ total_out,
    int64_t *__restrict__ nx_out, int32_t *__restrict__ status_out, int64_t *__restrict__ fail_out,
    int64_t *__restrict__ class_out, int32_t *__restrict__ rank_out) {
  __shared__ unsigned hist[RADIX];
  __shared__ unsigned base[RADIX];
  __shared__ unsigned cnt[LP_WARPS][RADIX];
  __shared__ int64_t warp_sum[LP_WARPS];
  __shared__ unsigned long long key_or;
  __shared__ unsigned classes[NCLASS];
  __shared__ int reached;
  __shared__ int64_t last_k;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const unsigned lt_mask = (1u << lane) - 1u;

  for (int i = tid; i < LP_WARPS * RADIX; i += LP_THREADS) (&cnt[0][0])[i] = 0u;
  for (int32_t b = blockIdx.x; b < nbins; b += gridDim.x) {
    const int64_t lo = bin_off[b];
    const int32_t n = (int32_t)(bin_off[b + 1] - lo);
    if (tid == 0) { key_or = 0ull; reached = 0; last_k = -1; }
    if (tid < NCLASS) classes[tid] = 0u;
    __syncthreads();

    // load: keys, record order, the OR of the keys (how many bytes the sort needs), the length classes
    unsigned long long my_or = 0ull;
    for (int32_t i = tid; i < n; i += LP_THREADS) {
      const int64_t L = len[lo + i];
      keys_a[lo + i] = (uint64_t)L;
      idx_a[lo + i] = i;
      my_or |= (unsigned long long)L;
      const int c = length_class(L);
      if (c >= 0) atomicAdd(&classes[c], 1u);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) my_or |= __shfl_xor_sync(FULL, my_or, o);
    if (lane == 0 && my_or) atomicOr(&key_or, my_or);
    __syncthreads();
    int npass = 0;
    for (unsigned long long v = key_or; v; v >>= 8) ++npass;

    uint64_t *ks = keys_a, *kd = keys_b;
    int32_t *is = idx_a, *id = idx_b;
    for (int pass = 0; pass < npass; ++pass) {
      const int shift = 8 * pass;
      for (int d = tid; d < RADIX; d += LP_THREADS) hist[d] = 0u;
      __syncthreads();
      for (int32_t i = tid; i < n; i += LP_THREADS) atomicAdd(&hist[digit_of(ks[lo + i], shift)], 1u);
      __syncthreads();
      if (warp == 0) {                         // exclusive scan of the 256 counts: 8 per lane, then across the warp
        unsigned v[RADIX / 32], s = 0u;
#pragma unroll
        for (int k = 0; k < RADIX / 32; ++k) { v[k] = hist[lane * (RADIX / 32) + k]; s += v[k]; }
        unsigned inc = s;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { const unsigned t = __shfl_up_sync(FULL, inc, o); if (lane >= o) inc += t; }
        unsigned run = inc - s;
#pragma unroll
        for (int k = 0; k < RADIX / 32; ++k) { base[lane * (RADIX / 32) + k] = run; run += v[k]; }
      }
      __syncthreads();
      for (int32_t t0 = 0; t0 < n; t0 += LP_THREADS) {
        const int32_t i = t0 + tid;
        const bool valid = i < n;
        uint64_t key = 0;
        int32_t rec = 0;
        unsigned d = RADIX;                    // lanes past the end form a group of their own and write nothing
        if (valid) { key = ks[lo + i]; rec = is[lo + i]; d = digit_of(key, shift); }
        const unsigned peers = __match_any_sync(FULL, d);
        if (valid && (peers & lt_mask) == 0u) cnt[warp][d] = (unsigned)__popc(peers);
        __syncthreads();
        if (valid) {
          unsigned off = base[d] + (unsigned)__popc(peers & lt_mask);
          for (int w = 0; w < warp; ++w) off += cnt[w][d];
          kd[lo + off] = key;
          id[lo + off] = rec;
        }
        __syncthreads();
        for (int dd = tid; dd < RADIX; dd += LP_THREADS) {
          unsigned s = 0u;
#pragma unroll
          for (int w = 0; w < LP_WARPS; ++w) { s += cnt[w][dd]; cnt[w][dd] = 0u; }
          base[dd] += s;
        }
        __syncthreads();
      }
      uint64_t *kt = ks; ks = kd; kd = kt;
      int32_t *it = is; is = id; id = it;
    }

    // ranks, then the inclusive prefix sum of the sorted lengths into the buffer the sort left free
    int64_t *csum = reinterpret_cast<int64_t *>(kd);
    for (int32_t r = tid; r < n; r += LP_THREADS) rank_out[lo + is[lo + r]] = r;
    int64_t carry = 0;
    for (int32_t t0 = 0; t0 < n; t0 += LP_THREADS) {
      const int32_t r = t0 + tid;
      int64_t v = r < n ? (int64_t)ks[lo + r] : 0;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) { const int64_t t = __shfl_up_sync(FULL, v, o); if (lane >= o) v += t; }
      if (lane == 31) warp_sum[warp] = v;
      __syncthreads();
      int64_t before = carry, tile = 0;
      for (int w = 0; w < LP_WARPS; ++w) { const int64_t s = warp_sum[w]; if (w < warp) before += s; tile += s; }
      if (r < n) csum[lo + r] = before + v;
      carry += tile;
      __syncthreads();
    }
    const int64_t total = carry;

    // thresholds: k_j = first r with C[r] >= x[j] * total
    const double ftotal = (double)total;
    for (int j = tid; j < m; j += LP_THREADS) {
      const double T = x[j] * ftotal;
      int32_t a = 0, e = n;                    // first r in [a, e) with C[r] >= T; n if none
      while (a < e) {
        const int32_t mid = a + ((e - a) >> 1);
        if (int_ge(csum[lo + mid], T)) e = mid; else a = mid + 1;
      }
      nx_out[(int64_t)b * m + j] = a < n ? (int64_t)ks[lo + a] : -1;
      if (a < n) {
        atomicAdd(&reached, 1);
        if (j == m - 1) last_k = a;
      }
    }
    if (tid < NCLASS) class_out[(int64_t)b * NCLASS + tid] = (int64_t)classes[tid];
    __syncthreads();
    if (tid == 0) {
      total_out[b] = total;
      if (reached < m) { status_out[b] = LP_SHORT; fail_out[b] = reached; }
      else if (last_k < n - 1) { status_out[b] = LP_INDEX; fail_out[b] = last_k + 1; }
      else { status_out[b] = LP_OK; fail_out[b] = -1; }
    }
    __syncthreads();
  }
}

}  // namespace

extern "C" {

int ckm_length_profile(ckm_engine *e, const int64_t *lens, const int64_t *bin_off, int32_t nbins, const double *x, int32_t m,
                       int64_t *total_out, int64_t *nx_out, int32_t *status_out, int64_t *fail_out, int64_t *class_out,
                       int32_t *rank_out, float *kernel_ms_out) {
  if (!e || nbins < 0 || !bin_off || m < 1 || !x || (nbins > 0 && (!total_out || !nx_out || !status_out || !fail_out || !class_out))) {
    set_error("ckm_length_profile: bad argument"); return CKM_EINVAL;
  }
  if (bin_off[0] != 0) { set_error("ckm_length_profile: bin_off[0] must be 0"); return CKM_EINVAL; }
  for (int32_t b = 0; b < nbins; ++b) {
    const int64_t n = bin_off[b + 1] - bin_off[b];
    if (n < 0 || n > INT32_MAX) { set_error("ckm_length_profile: bin " + std::to_string(b) + " has a bad record count"); return CKM_EINVAL; }
  }
  const int64_t nrec = bin_off[nbins];
  if (nrec > 0 && (!lens || !rank_out)) { set_error("ckm_length_profile: bad argument"); return CKM_EINVAL; }
  for (int32_t b = 0; b < nbins; ++b) {
    int64_t sum = 0;
    for (int64_t i = bin_off[b]; i < bin_off[b + 1]; ++i) {
      if (lens[i] < 0 || __builtin_add_overflow(sum, lens[i], &sum)) {
        set_error("ckm_length_profile: record " + std::to_string(i) + " of bin " + std::to_string(b) +
                  (lens[i] < 0 ? " has a negative length" : " takes the bin's total past 2^63 - 1"));
        return CKM_EINVAL;
      }
    }
  }
  for (int32_t j = 0; j < m; ++j)
    if (std::isnan(x[j]) || (j > 0 && x[j] < x[j - 1])) {
      set_error("ckm_length_profile: x must be ascending and not NaN (x[" + std::to_string(j) + "])"); return CKM_EINVAL;
    }
  if (nbins == 0) { if (kernel_ms_out) *kernel_ms_out = 0.f; return CKM_OK; }

  const DeviceScope ws(e);
  DevBuf dlen, doff, dx, dka, dkb, dia, dib, dtotal, dnx, dstatus, dfail, dclass, drank;
  CKM_TRY(dlen.put(lens, (size_t)nrec, ws.st));
  CKM_TRY(doff.put(bin_off, (size_t)nbins + 1, ws.st));
  CKM_TRY(dx.put(x, (size_t)m, ws.st));
  CKM_TRY(dka.alloc(sizeof(uint64_t) * (size_t)nrec));
  CKM_TRY(dkb.alloc(sizeof(uint64_t) * (size_t)nrec));
  CKM_TRY(dia.alloc(sizeof(int32_t) * (size_t)nrec));
  CKM_TRY(dib.alloc(sizeof(int32_t) * (size_t)nrec));
  CKM_TRY(dtotal.alloc(sizeof(int64_t) * (size_t)nbins));
  CKM_TRY(dnx.alloc(sizeof(int64_t) * (size_t)nbins * (size_t)m));
  CKM_TRY(dstatus.alloc(sizeof(int32_t) * (size_t)nbins));
  CKM_TRY(dfail.alloc(sizeof(int64_t) * (size_t)nbins));
  CKM_TRY(dclass.alloc(sizeof(int64_t) * (size_t)nbins * NCLASS));
  CKM_TRY(drank.alloc(sizeof(int32_t) * (size_t)nrec));
  const unsigned blocks = (unsigned)std::min<int32_t>(nbins, 1 << 16);
  CKM_TRY(ev_record(e, 0));
  length_profile_kernel<<<blocks, LP_THREADS, 0, ws.st>>>(dlen.as<int64_t>(), doff.as<int64_t>(), nbins, dx.as<double>(), m,
                                                          dka.as<uint64_t>(), dkb.as<uint64_t>(), dia.as<int32_t>(), dib.as<int32_t>(),
                                                          dtotal.as<int64_t>(), dnx.as<int64_t>(), dstatus.as<int32_t>(),
                                                          dfail.as<int64_t>(), dclass.as<int64_t>(), drank.as<int32_t>());
  CKM_CUDA(cudaGetLastError());
  CKM_TRY(ev_record(e, 1));
  CKM_TRY(dtotal.get(total_out, (size_t)nbins, ws.st));
  CKM_TRY(dnx.get(nx_out, (size_t)nbins * (size_t)m, ws.st));
  CKM_TRY(dstatus.get(status_out, (size_t)nbins, ws.st));
  CKM_TRY(dfail.get(fail_out, (size_t)nbins, ws.st));
  CKM_TRY(dclass.get(class_out, (size_t)nbins * NCLASS, ws.st));
  CKM_TRY(drank.get(rank_out, (size_t)nrec, ws.st));
  CKM_TRY(stream_sync(ws.st));
  CKM_TRY(ev_elapsed(e, kernel_ms_out, 0, 1));
  return CKM_OK;
}

}  // extern "C"
