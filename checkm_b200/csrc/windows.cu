// windows.cu -- per-window statistics of a bin's sequences for the plots (`checkm gc_plot`, `coding_plot`, `tetra_plot`,
// `dist_plot` and the GC half of `gc_bias_plot`; checkm/plot/gcPlots.py:52-75, codingDensityPlots.py:70-89,
// tetraDistPlots.py:54-79, gcBiasPlots.py:48-66).
//
// Window k of a sequence of length L covers [kW, (k+1)W) and exists only while (k+1)W < L, so a sequence has (L-1)//W of
// them (the caller passes the offsets, coverageWindows.window_offsets).  Per window, restated from the reference:
//   * a, c, g, t: baseCount(seq[start:end]), case-insensitive, U counted with T (util/seqUtils.py:279-286), as ntstats.cu
//   * optionally the tetranucleotide distance to the bin signature: seqSignature(window) counts every 4-mer wholly inside
//     the window whose four bytes are A/C/G/T of either case (U is not T here, as kmers.cu) on its canonical column;
//     sig = counts / total (one float64 division per column; 0/0 = NaN), and the distance is np.sum(np.abs(sig - binSig))
//     over 136 terms in numpy's pairwise order (pairwise.cuh).
//
// Device work.
//   window_scan_kernel  the row stream of ntstats/kmers (ntrows.cuh): each warp streams a contiguous range of 2 KB rows
//                       through its TMA stage ring, a lane takes 64 bytes.  A byte, and a 4-mer by its first byte, belongs
//                       to the window its position in the sequence falls into; positions at or past nwin * W are dropped,
//                       and a 4-mer is counted only if its last byte is still inside its window (the 3 bytes after a lane's
//                       chunk are the next lane's, or the 16-byte halo after the row).
//                       Base counts: a lane's 64 bytes touch windows kf..kl.  A window wholly inside the chunk is that
//                       lane's alone and is stored; the first and last are shared with other lanes and warps and are added
//                       by atomics -- reduced over the warp first when every lane of the row is in the same window (the
//                       common case for W >= 2 KB).
//                       4-mer counts: 136 x uint32 per window in global memory.  For W >= 2 KB a row touches at most two
//                       windows, K and K + 1, so the warp counts into two shared-memory histograms (slot = window & 1)
//                       and adds a histogram to global memory when its window is left; below 2 KB every 4-mer is a global
//                       atomic.
//   window_dist_kernel  one warp per window: the 136 counts, their total, the 136 absolute differences into shared memory,
//                       then two lanes sum the halves (64 and 72 terms) in numpy's order and add them.
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <vector>
#include "engine.hpp"
#include "pool.hpp"
#include "device_utils.cuh"
#include "ntrows.cuh"
#include "pairwise.cuh"

using namespace ckm;

namespace {

constexpr int WN_THREADS = 256;
constexpr int WN_WARPS = WN_THREADS / 32;
constexpr int WN_STAGES = 3;                                   // rows in flight per warp
constexpr int WN_COLS = 136;                                   // canonical tetranucleotides
constexpr int WN_HIST_OFF = NtRing<WN_STAGES>::SMEM;           // per-warp shared memory: the ring, the histograms
constexpr int WN_WARP_SMEM = (WN_HIST_OFF + 2 * WN_COLS * 4 + 127) / 128 * 128;   // 7.4 KB per warp, 59 KB per CTA
constexpr int WN_CTAS_PER_SM = 2;                             // 3 would cap the scan at 80 registers and spill

struct WinParams {
  const uint8_t *bytes;                 // device copy of the caller's buffer
  const NtRow *rows;
  long long nrows;
  const long long *starts;              // nseq: where each sequence starts in `bytes`
  const long long *win_off;             // nseq + 1
  long long W;
  unsigned long long *acgt;             // nwin x 4, zeroed
  uint32_t *kmers;                      // nwin x 136, zeroed; null: no 4-mer work
  uint8_t col_of[256];                  // raw 4-mer code (A 0, C 1, G 2, T 3; first base highest) -> canonical column
};

// 2-bit code of a byte and whether it is one of ACGTacgt (bit 2 clear) -- 4 for anything else
__device__ __forceinline__ uint32_t wn_code(uint32_t b) {
  const uint32_t u = b & 0xDFu;
  return u == 'A' ? 0u : u == 'C' ? 1u : u == 'G' ? 2u : u == 'T' ? 3u : 4u;
}

// every lane: add the warp's shared histogram of `slot` to the global counters of window `win` and clear it
__device__ __forceinline__ void wn_flush(const WinParams &p, uint32_t *hist, long long win, int lane) {
  __syncwarp();
  if (win >= 0)
    for (int c = lane; c < WN_COLS; c += 32) {
      const uint32_t v = hist[c];
      if (v) { atomicAdd(&p.kmers[(size_t)win * WN_COLS + c], v); hist[c] = 0u; }
    }
  __syncwarp();
}

__global__ void __launch_bounds__(WN_THREADS, WN_CTAS_PER_SM) window_scan_kernel(WinParams p) {
  extern __shared__ __align__(128) uint8_t s_dyn[];             // WN_WARPS x WN_WARP_SMEM
  __shared__ uint8_t s_col[256];
  for (int i = threadIdx.x; i < 256; i += WN_THREADS) s_col[i] = p.col_of[i];
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const NtRange r = nt_warp_rows(p.nrows, (long long)blockIdx.x * WN_WARPS + warp, (long long)gridDim.x * WN_WARPS);
  if (r.lo >= r.hi) return;
  NtRing<WN_STAGES> ring(smem_u32(s_dyn) + warp * WN_WARP_SMEM, p.rows + r.lo, (int)(r.hi - r.lo), lane);
  uint32_t *hist = reinterpret_cast<uint32_t *>(s_dyn + warp * WN_WARP_SMEM + WN_HIST_OFF);   // 2 x 136
  for (int i = lane; i < 2 * WN_COLS; i += 32) hist[i] = 0u;
  long long hk0 = -1, hk1 = -1;                                  // window of each histogram slot (same in every lane)
  const long long W = p.W;
  const bool shared_hist = p.kmers != nullptr && W >= NT_ROW;
  ring.start();
  for (int k = 0; k < ring.n; ++k) {
    const auto [src, s, nbytes, first_row, last_row, body] = ring.wait();
    uint32_t w[17];
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const uint4 v = lds128(body + lane * NT_CHUNK + q * 16);
      w[4 * q] = v.x; w[4 * q + 1] = v.y; w[4 * q + 2] = v.z; w[4 * q + 3] = v.w;
    }
    w[16] = lds32(body + lane * NT_CHUNK + NT_CHUNK);             // the 3 bytes after the chunk
    __syncwarp();
    ring.release(k);

    const long long off = (long long)(src - (uint64_t)(uintptr_t)p.bytes) - p.starts[s] + (first_row ? 0 : NT_HALO);   // row in the sequence
    const long long woff = p.win_off[s], limit = (p.win_off[s + 1] - woff) * W;                      // bytes that have a window
    if (off >= limit) continue;                                                                     // same in every lane
    const long long c0 = off + lane * NT_CHUNK;
    const long long c1 = min(c0 + (long long)max(min(nbytes - lane * NT_CHUNK, NT_CHUNK), 0), limit);
    const bool active = c1 > c0;
    const long long kf = active ? c0 / W : -1, kl = active ? (c1 - 1) / W : -1;

    // ---- base counts ----
    unsigned long long mA = 0, mC = 0, mG = 0, mT = 0;
#pragma unroll
    for (int i = 0; i < 64; ++i) {
      const uint32_t u = (w[i >> 2] >> (8 * (i & 3))) & 0xDFu;
      mA |= (unsigned long long)(u == 'A') << i;
      mC |= (unsigned long long)(u == 'C') << i;
      mG |= (unsigned long long)(u == 'G') << i;
      mT |= (unsigned long long)(u == 'T' || u == 'U') << i;
    }
    const long long K0 = __shfl_sync(0xffffffffu, kf, 0);         // lane 0 is active: off < limit
    const bool uniform = __all_sync(0xffffffffu, !active || (kf == kl && kf == K0));
    if (uniform) {
      const unsigned long long rng = active ? (c1 - c0 >= 64 ? ~0ull : ((1ull << (c1 - c0)) - 1ull)) : 0ull;
      const uint32_t v[4] = {(uint32_t)__popcll(mA & rng), (uint32_t)__popcll(mC & rng), (uint32_t)__popcll(mG & rng), (uint32_t)__popcll(mT & rng)};
#pragma unroll
      for (int x = 0; x < 4; ++x) {
        const uint32_t t = __reduce_add_sync(0xffffffffu, v[x]);
        if (lane == x && t) atomicAdd(&p.acgt[(size_t)(woff + K0) * 4 + x], (unsigned long long)t);
      }
    } else if (active) {
      for (long long win = kf; win <= kl; ++win) {
        const long long a = max(c0, win * W), b = min(c1, (win + 1) * W);
        const int lo_bit = (int)(a - c0), nbit = (int)(b - a);
        const unsigned long long rng = (nbit >= 64 ? ~0ull : ((1ull << nbit) - 1ull)) << lo_bit;
        const unsigned long long v[4] = {(unsigned long long)__popcll(mA & rng), (unsigned long long)__popcll(mC & rng),
                                         (unsigned long long)__popcll(mG & rng), (unsigned long long)__popcll(mT & rng)};
        unsigned long long *o = p.acgt + (size_t)(woff + win) * 4;
        if (win * W >= c0 && (win + 1) * W <= c1) {                 // wholly inside this lane's chunk: no one else adds to it
          o[0] = v[0]; o[1] = v[1]; o[2] = v[2]; o[3] = v[3];
        } else {
#pragma unroll
          for (int x = 0; x < 4; ++x) if (v[x]) atomicAdd(&o[x], v[x]);
        }
      }
    }

    // ---- 4-mer counts ----
    if (p.kmers == nullptr) continue;
    if (shared_hist) {                                               // the row's windows K0 and K0 + 1 get a slot each
      const long long G = woff + K0;
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        long long &h = ((G + e) & 1) ? hk1 : hk0;
        if (h != G + e) { wn_flush(p, hist + ((G + e) & 1) * WN_COLS, h, lane); h = G + e; }
      }
    }
    if (active) {
      long long win = kf, r = c0 - kf * W;                          // window of the 4-mer starting at c0, and its place in it
      const int m = (int)(c1 - c0);
      uint32_t roll = 0, vroll = 0;
#pragma unroll
      for (int i = 0; i < 67; ++i) {
        const uint32_t code = wn_code((w[i >> 2] >> (8 * (i & 3))) & 0xFFu);
        roll = ((roll << 2) | (code & 3u)) & 0xFFu;
        vroll = ((vroll << 1) | (code < 4u ? 1u : 0u)) & 0xFu;
        if (i >= 3) {
          const int j = i - 3;                                       // the 4-mer starting at c0 + j
          if (j < m) {
            if (vroll == 0xFu && r + 3 < W) {
              const uint32_t col = s_col[roll];
              if (shared_hist) atomicAdd(&hist[(int)((woff + win) & 1) * WN_COLS + col], 1u);
              else atomicAdd(&p.kmers[(size_t)(woff + win) * WN_COLS + col], 1u);
            }
            if (++r == W) { r = 0; ++win; }
          }
        }
      }
    }
  }
  if (shared_hist) {
    wn_flush(p, hist, hk0, lane);
    wn_flush(p, hist + WN_COLS, hk1, lane);
  }
}

__global__ void __launch_bounds__(WN_THREADS) window_dist_kernel(const uint32_t *kmers, long long nwin, const double *binsig, double *td) {
  __shared__ double s_d[WN_WARPS][WN_COLS];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const long long win = (long long)blockIdx.x * WN_WARPS + warp;
  if (win >= nwin) return;                                       // the whole warp
  const uint32_t *c = kmers + (size_t)win * WN_COLS;
  uint32_t v[5], tot = 0;
#pragma unroll
  for (int j = 0; j < 5; ++j) { const int i = lane + 32 * j; v[j] = i < WN_COLS ? c[i] : 0u; tot += v[j]; }
  const double total = (double)__reduce_add_sync(0xffffffffu, tot);   // at most the window's length: exact
#pragma unroll
  for (int j = 0; j < 5; ++j) {
    const int i = lane + 32 * j;
    if (i < WN_COLS) s_d[warp][i] = fabs((double)v[j] / total - binsig[i]);
  }
  __syncwarp();
  const double *dd = s_d[warp];
  const int n2 = (int)pw_split(WN_COLS);                         // 64 and 72
  double half = 0.0;
  if (lane == 0) half = pw_leaf_sum([dd](int i) { return dd[i]; }, n2);
  if (lane == 1) half = pw_leaf_sum([dd, n2](int i) { return dd[n2 + i]; }, WN_COLS - n2);
  const double other = __shfl_down_sync(0xffffffffu, half, 1);
  if (lane == 0) td[win] = half + other;
}

}  // namespace

extern "C" {

int ckm_window_stats(ckm_engine *e, const uint8_t *bytes, int64_t nbytes, const int64_t *starts, const int64_t *lens,
                     int32_t nseq, int64_t window_size, const int64_t *win_off, const double *bin_sig, int64_t *acgt_out,
                     double *td_out, float *kernel_ms_out) {
  if (!e || nseq < 0 || nbytes < 0 || !win_off || (nseq > 0 && (!bytes || !starts || !lens)) || (bin_sig && !td_out)) {
    set_error("ckm_window_stats: bad argument"); return CKM_EINVAL;
  }
  char msg[200];
  if (window_size < 1) {
    std::snprintf(msg, sizeof msg, "ckm_window_stats: window size %lld; it must be at least 1", (long long)window_size);
    set_error(msg); return CKM_EINVAL;
  }
  if (kernel_ms_out) *kernel_ms_out = 0.0f;
  if (win_off[0] != 0) { set_error("ckm_window_stats: win_off[0] must be 0"); return CKM_EINVAL; }
  if (int rc = nt_check_layout("ckm_window_stats", "sequence", starts, lens, nseq, nbytes)) return rc;
  for (int32_t s = 0; s < nseq; ++s) {
    const int64_t want = std::max<int64_t>(lens[s] - 1, 0) / window_size;
    if (win_off[s + 1] - win_off[s] != want) {
      std::snprintf(msg, sizeof msg, "ckm_window_stats: sequence %d has %lld windows in win_off, (length - 1) / window size is %lld",
                    s, (long long)(win_off[s + 1] - win_off[s]), (long long)want);
      set_error(msg); return CKM_EINVAL;
    }
  }
  const int64_t nwin = win_off[nseq];
  if (nwin == 0) return CKM_OK;
  if (!acgt_out) { set_error("ckm_window_stats: bad argument"); return CKM_EINVAL; }
  const DeviceScope ws(e);
  const int dyn_smem = WN_WARPS * WN_WARP_SMEM;
  NtUpload u;
  CKM_TRY(nt_upload(e, "ckm_window_stats", bytes, nbytes, starts, lens, nseq, (const void *)window_scan_kernel, WN_WARPS,
                    WN_CTAS_PER_SM, dyn_smem, u));
  std::vector<long long> seq_info((size_t)2 * nseq + 1);           // starts, then win_off
  for (int32_t s = 0; s < nseq; ++s) seq_info[s] = starts[s];
  for (int32_t s = 0; s <= nseq; ++s) seq_info[(size_t)nseq + s] = win_off[s];
  DevBuf dinfo, dacgt, dkm, dsig, dtd;
  CKM_TRY(dinfo.put(seq_info.data(), seq_info.size(), ws.st));
  CKM_TRY(dacgt.fill(sizeof(int64_t) * 4 * (size_t)nwin, 0, ws.st));
  if (bin_sig) {
    CKM_TRY(dkm.fill(sizeof(uint32_t) * WN_COLS * (size_t)nwin, 0, ws.st));
    CKM_TRY(dsig.put(bin_sig, WN_COLS, ws.st));
    CKM_TRY(dtd.alloc(sizeof(double) * (size_t)nwin));
  }
  WinParams q;
  std::memset(&q, 0, sizeof(q));
  q.bytes = u.bytes.as<uint8_t>(); q.rows = u.rows.as<NtRow>(); q.nrows = u.nrows;
  q.starts = dinfo.as<long long>(); q.win_off = dinfo.as<long long>() + nseq; q.W = window_size;
  q.acgt = dacgt.as<unsigned long long>(); q.kmers = bin_sig ? dkm.as<uint32_t>() : nullptr;
  {
    uint8_t code[WN_COLS];                                        // a column and its code's reverse complement share it
    for (int c = 0, n = km_col_codes(4, code); c < n; ++c) q.col_of[code[c]] = q.col_of[km_revcomp(code[c], 4)] = (uint8_t)c;
  }
  CKM_TRY(ev_record(e, 0));
  if (u.nrows > 0) {
    window_scan_kernel<<<u.grid, WN_THREADS, dyn_smem, ws.st>>>(q);
    CKM_CUDA(cudaGetLastError());
  }
  if (bin_sig) {
    window_dist_kernel<<<(unsigned)((nwin + WN_WARPS - 1) / WN_WARPS), WN_THREADS, 0, ws.st>>>(dkm.as<uint32_t>(), nwin, dsig.as<double>(), dtd.as<double>());
    CKM_CUDA(cudaGetLastError());
  }
  CKM_TRY(ev_record(e, 1));
  CKM_TRY(dacgt.get(acgt_out, 4 * (size_t)nwin, ws.st));
  if (bin_sig) CKM_TRY(dtd.get(td_out, (size_t)nwin, ws.st));
  CKM_TRY(stream_sync(ws.st));
  CKM_TRY(ev_elapsed(e, kernel_ms_out, 0, 1));
  return CKM_OK;
}

}  // extern "C"
