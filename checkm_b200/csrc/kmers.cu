// kmers.cu -- canonical k-mer counts of every sequence, K = 1..4: the per-base half of CheckM's genomic signatures
// (checkm/genomicSignatures.py:44-84,131-149, `checkm tetra`; SURVEY.md 8), and the host writer of the profile lines.
//
// What the reference computes per sequence, restated: every window of K bytes of the upper-cased sequence that consists
// of A, C, G, T only adds one to the column of its canonical form (the lexicographically smaller of the k-mer and its
// reverse complement); every other window -- N, IUPAC codes, U, '*', anything -- is skipped.  The columns are the
// canonical k-mers in ascending lexicographic order (2, 10, 32, 136 of them).
//
// The scan streams the same 2 KB rows as ntstats_kernel (ntrows.cuh).  A k-mer belongs to the row that holds its last
// byte; the K-1 bytes it needs from before its row are in the 16-byte halo staged in front of the row, so warps never
// join anything.  Per row a warp takes four 512-byte blocks, a lane 16 consecutive bytes of each (one conflict-free
// LDS.128); the codes of the three bytes before a lane's 16 come from the lane before it by one shuffle.  Bases are
// encoded with the low-three-bit PRMT lookup of ntrows.cuh (A 1, C 3, T 4, G 7 -> 2-bit codes A 0, C 1, G 2, T 3), and every
// valid window adds one to a per-warp histogram over the 4^K raw window codes in shared memory (one ATOMS per window).
// At the last row of a sequence, and at the end of the warp's range, the histogram is folded onto the canonical columns
// (column c = code x plus its reverse complement) and written: by plain stores when the warp saw the whole sequence,
// by global atomics into the zeroed output when the sequence is split between warps.
#include <charconv>
#include <cmath>
#include <cstdint>
#include <cstdlib>
#include <cstring>
#include <vector>
#include "engine.hpp"
#include "pool.hpp"
#include "device_utils.cuh"
#include "ntrows.cuh"

using namespace ckm;

namespace {

constexpr int KM_THREADS = 256;
constexpr int KM_WARPS = KM_THREADS / 32;
constexpr int KM_STAGES = 3;                                   // rows in flight per warp
constexpr int KM_HIST_OFF = (NtRing<KM_STAGES>::SMEM + 127) / 128 * 128;   // per-warp shared memory: the ring, the histogram
constexpr int KM_WARP_SMEM = KM_HIST_OFF + 256 * 4;            // 7.4 KB per warp, 59 KB per CTA
constexpr int KM_CTAS_PER_SM = 3;
constexpr int KM_MAX_COLS = 136;

struct KmParams {
  const NtRow *rows;
  long long nrows;
  uint32_t *counts;                // nseq x ncols, zeroed
  uint8_t col_code[KM_MAX_COLS];   // raw code of the canonical k-mer of every column
};

__host__ __device__ constexpr int km_cols(int k) { return k == 1 ? 2 : k == 2 ? 10 : k == 3 ? 32 : 136; }

// 0x80 in every byte of x that is zero
__device__ __forceinline__ uint32_t zero4(uint32_t x) {
  const uint32_t t = (x & 0x7F7F7F7Fu) + 0x7F7F7F7Fu;
  return ~(t | x | 0x7F7F7F7Fu);
}

// One word of 4 bytes -> (valid nibble << 8) | packed codes: byte 0 (the earliest) in the top bits of both, so that
// appending a word to earlier codes is a shift by 8 (codes) or 4 (valid bits).  keep: bytes of the word in the sequence.
__device__ __forceinline__ uint32_t km_encode(uint32_t w, uint32_t keep) {
  const uint32_t sel = nt_sel(w);
  const uint32_t bad = (w & 0xDFDFDFDFu) ^ nt_letters(sel);                           // 'a' -> 'A'; 0 where the byte is ACGTacgt
  const uint32_t codes = prmt_b32(0x01000000u, 0x02000003u, sel);                     // A 0, C 1, G 2, T 3 per byte
  const uint32_t packed = (codes * 0x40100401u) >> 24;                                // byte b -> bits 6-2b, 7-2b
  const uint32_t valid = ((((zero4(bad) >> 7) * 0x08040201u) >> 24) & 0xFu) & ((0xFu << (4u - keep)) & 0xFu);   // byte b -> bit 3-b
  return (valid << 8) | packed;
}

template <int K>
__global__ void __launch_bounds__(KM_THREADS, KM_CTAS_PER_SM) kmer_kernel(KmParams p) {
  constexpr int C = km_cols(K);
  constexpr uint32_t KMASK = (1u << (2 * K)) - 1u;
  constexpr int NBINS = 1 << (2 * K);
  extern __shared__ __align__(128) uint8_t s_dyn[];             // KM_WARPS x KM_WARP_SMEM
  __shared__ uint8_t s_col[KM_MAX_COLS];
  for (int i = threadIdx.x; i < C; i += KM_THREADS) s_col[i] = p.col_code[i];
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const NtRange r = nt_warp_rows(p.nrows, (long long)blockIdx.x * KM_WARPS + warp, (long long)gridDim.x * KM_WARPS);
  if (r.lo >= r.hi) return;
  NtRing<KM_STAGES> ring(smem_u32(s_dyn) + warp * KM_WARP_SMEM, p.rows + r.lo, (int)(r.hi - r.lo), lane);
  uint32_t *hist = reinterpret_cast<uint32_t *>(s_dyn + warp * KM_WARP_SMEM + KM_HIST_OFF);
  for (int i = lane; i < NBINS; i += 32) hist[i] = 0u;
  ring.start();
  bool whole = false;                                            // the warp saw the first row of the sequence now open
  for (int k = 0; k < ring.n; ++k) {
    const auto [src, s, nbytes, first_row, last_row, body] = ring.wait();
    if (k == 0 || first_row) whole = first_row;
    // the three bytes before the row: the halo, except at a sequence's first row (whatever is there is not sequence)
    uint32_t carry = 0;
    if (lane == 0 && !first_row) carry = km_encode(lds32(body - 4), 4u);
    uint4 v[4];
#pragma unroll
    for (int q = 0; q < 4; ++q) v[q] = lds128(body + q * 512 + lane * 16);
    // every value read from the stage is in registers: it can take the row KM_STAGES further on
    __syncwarp();
    ring.release(k);
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int at = q * 512 + lane * 16;                        // where the lane's 16 bytes sit in the row
      const uint32_t w[4] = {v[q].x, v[q].y, v[q].z, v[q].w};
      uint32_t e[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) e[j] = km_encode(w[j], (uint32_t)min(max(nbytes - at - 4 * j, 0), 4));
      const uint32_t rolled = __shfl_sync(0xffffffffu, e[3], (lane + 31) & 31);
      uint32_t prev = lane ? rolled : carry;
      carry = rolled;                                            // lane 0: the last word of lane 31, for the next block
      if (at >= nbytes) continue;                            // nothing of the sequence in this lane's 16 bytes
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const uint32_t codes = ((prev & 0xFFu) << 8) | (e[j] & 0xFFu);             // 8 bases, the last one lowest
        uint32_t vb = (((prev >> 8) & 0xFu) << 4) | ((e[j] >> 8) & 0xFu);
        if (K > 1) vb &= vb >> 1;
        if (K > 2) vb &= vb >> 1;
        if (K > 3) vb &= vb >> 1;                                // bit 3-t: the window ending at byte t is all ACGT
#pragma unroll
        for (int t = 0; t < 4; ++t)
          if ((vb >> (3 - t)) & 1u) atomicAdd(&hist[(codes >> (2 * (3 - t))) & KMASK], 1u);
        prev = e[j];
      }
    }
    if (last_row || k + 1 == ring.n) {
      __syncwarp();
      uint32_t *out = p.counts + (size_t)s * C;
#pragma unroll
      for (int c0 = 0; c0 < C; c0 += 32) {
        const int c = c0 + lane;
        if (c < C) {
          const uint32_t x = s_col[c], r = km_revcomp(x, K);
          const uint32_t val = hist[x] + (r != x ? hist[r] : 0u);
          if (whole && last_row) out[c] = val;
          else if (val) atomicAdd(&out[c], val);
        }
      }
      __syncwarp();
      for (int i = lane; i < NBINS; i += 32) hist[i] = 0u;
      __syncwarp();
    }
  }
}

}  // namespace

namespace {

// str(np.float64(v)) for 0 <= v <= 1 or NaN: the shortest round-trip digits, laid out as Python's float repr does
// (positional for 1e-4 <= v < 1e16, else d.ddde-XX; '.0' after an integer).
int km_format_value(double v, char *o) {
  if (std::isnan(v)) { std::memcpy(o, "nan", 3); return 3; }
  char buf[40];
  const auto r = std::to_chars(buf, buf + sizeof(buf), v, std::chars_format::scientific);
  const int len = (int)(r.ptr - buf);
  buf[len] = '\0';
  const char *epos = (const char *)std::memchr(buf, 'e', (size_t)len);
  int exp = std::atoi(epos + 1);
  if (exp < -4 || exp >= 16) { std::memcpy(o, buf, (size_t)len); return len; }    // C++'s layout is Python's here
  char dig[24]; int nd = 0;
  for (const char *q = buf; q < epos; ++q) if (*q != '.') dig[nd++] = *q;
  int w = 0;
  if (exp < 0) {
    o[w++] = '0'; o[w++] = '.';
    for (int i = 0; i < -exp - 1; ++i) o[w++] = '0';
    for (int i = 0; i < nd; ++i) o[w++] = dig[i];
  } else {
    for (int i = 0; i <= exp; ++i) o[w++] = i < nd ? dig[i] : '0';
    o[w++] = '.';
    if (nd > exp + 1) for (int i = exp + 1; i < nd; ++i) o[w++] = dig[i];
    else o[w++] = '0';
  }
  return w;
}

}  // namespace

extern "C" {

int ckm_kmer_counts(ckm_engine *e, const uint8_t *bytes, int64_t nbytes, const int64_t *starts, const int64_t *lens,
                    int32_t nseq, int32_t k, uint32_t *counts_out, float *kernel_ms_out) {
  if (k < 1 || k > 4) { set_error("ckm_kmer_counts: k must lie in 1..4"); return CKM_EINVAL; }
  if (!e || nseq < 0 || nbytes < 0 || (nseq > 0 && (!bytes || !starts || !lens || !counts_out))) {
    set_error("ckm_kmer_counts: bad argument"); return CKM_EINVAL;
  }
  if (kernel_ms_out) *kernel_ms_out = 0.0f;
  if (nseq == 0) return CKM_OK;
  if (int rc = nt_check_layout("ckm_kmer_counts", "sequence", starts, lens, nseq, nbytes)) return rc;
  const int ncols = km_cols(k);
  const size_t out_bytes = sizeof(uint32_t) * (size_t)ncols * (size_t)nseq;
  const DeviceScope ws(e);
  const int dyn_smem = KM_WARPS * KM_WARP_SMEM;
  void (*kern)(KmParams) = k == 1 ? kmer_kernel<1> : k == 2 ? kmer_kernel<2> : k == 3 ? kmer_kernel<3> : kmer_kernel<4>;
  NtUpload u;
  CKM_TRY(nt_upload(e, "ckm_kmer_counts", bytes, nbytes, starts, lens, nseq, (const void *)kern, KM_WARPS, KM_CTAS_PER_SM, dyn_smem, u));
  if (u.nrows == 0) { std::memset(counts_out, 0, out_bytes); return CKM_OK; }
  DevBuf dcounts;
  CKM_TRY(dcounts.fill(out_bytes, 0, ws.st));
  KmParams p;
  std::memset(&p, 0, sizeof(p));
  p.rows = u.rows.as<NtRow>(); p.nrows = u.nrows; p.counts = dcounts.as<uint32_t>();
  km_col_codes(k, p.col_code);
  CKM_TRY(ev_record(e, 0));
  kern<<<u.grid, KM_THREADS, dyn_smem, ws.st>>>(p);
  CKM_CUDA(cudaGetLastError());
  CKM_TRY(ev_record(e, 1));
  CKM_TRY(dcounts.get(counts_out, (size_t)ncols * (size_t)nseq, ws.st));
  CKM_TRY(stream_sync(ws.st));
  CKM_TRY(ev_elapsed(e, kernel_ms_out, 0, 1));
  return CKM_OK;
}

int ckm_kmer_columns(int32_t k, char *out) {
  if (k < 1 || k > 4 || !out) { set_error("ckm_kmer_columns: k must lie in 1..4"); return CKM_EINVAL; }
  uint8_t codes[KM_MAX_COLS];
  const int n = km_col_codes(k, codes);
  for (int c = 0; c < n; ++c)
    for (int i = 0; i < k; ++i) out[c * k + i] = "ACGT"[(codes[c] >> (2 * (k - 1 - i))) & 3u];
  return CKM_OK;
}

int ckm_format_kmer_profiles(const uint32_t *counts, int32_t nseq, int32_t k, const char *ids, const int64_t *id_offsets,
                             char *out, int64_t out_cap, int64_t *out_len) {
  if (k < 1 || k > 4) { set_error("ckm_format_kmer_profiles: k must lie in 1..4"); return CKM_EINVAL; }
  if (nseq < 0 || !out_len || (nseq > 0 && (!counts || !ids || !id_offsets)) || out_cap < 0 || (out_cap > 0 && !out)) {
    set_error("ckm_format_kmer_profiles: bad argument"); return CKM_EINVAL;
  }
  const int ncols = km_cols(k);
  char val[40];
  int64_t w = 0;
  for (int32_t s = 0; s < nseq; ++s) {
    const uint32_t *c = counts + (size_t)s * ncols;
    uint64_t total = 0;
    for (int i = 0; i < ncols; ++i) total += c[i];
    const int64_t idn = id_offsets[s + 1] - id_offsets[s];
    if (w + idn <= out_cap) std::memcpy(out + w, ids + id_offsets[s], (size_t)idn);
    w += idn;
    for (int i = 0; i < ncols; ++i) {
      const double v = total ? (double)c[i] / (double)total : std::nan("");   // numpy: sig /= np.sum(sig), 0/0 = nan
      const int n = km_format_value(v, val);
      if (w + 1 + n <= out_cap) { out[w] = '\t'; std::memcpy(out + w + 1, val, (size_t)n); }
      w += 1 + n;
    }
    if (w + 1 <= out_cap) out[w] = '\n';
    w += 1;
  }
  *out_len = w;
  if (w > out_cap) { set_error("ckm_format_kmer_profiles: output buffer too small (the size needed is returned)"); return CKM_ECAPACITY; }
  return CKM_OK;
}

}  // extern "C"
