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
// encoded with the low-three-bit PRMT lookup of ntstats (A 1, C 3, T 4, G 7 -> 2-bit codes A 0, C 1, G 2, T 3), and every
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
constexpr int KM_DESC_OFF = KM_STAGES * NT_STAGE;              // per-warp shared memory: stages, descriptors, mbarriers, histogram
constexpr int KM_BAR_OFF = KM_DESC_OFF + KM_STAGES * 16;
constexpr int KM_HIST_OFF = (KM_BAR_OFF + KM_STAGES * 8 + 127) / 128 * 128;
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

// reverse complement of a K-mer code (2 bits per base, the last base lowest; A 0, C 1, G 2, T 3 so complement = xor 3)
__host__ __device__ __forceinline__ uint32_t km_revcomp(uint32_t x, int k) {
  uint32_t r = 0;
  for (int i = 0; i < k; ++i) { r = (r << 2) | ((x & 3u) ^ 3u); x >>= 2; }
  return r;
}

__device__ __forceinline__ uint32_t lds32(uint32_t addr) {
  uint32_t v;
  asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(addr));
  return v;
}

// 0x80 in every byte of x that is zero
__device__ __forceinline__ uint32_t zero4(uint32_t x) {
  const uint32_t t = (x & 0x7F7F7F7Fu) + 0x7F7F7F7Fu;
  return ~(t | x | 0x7F7F7F7Fu);
}

// One word of 4 bytes -> (valid nibble << 8) | packed codes: byte 0 (the earliest) in the top bits of both, so that
// appending a word to earlier codes is a shift by 8 (codes) or 4 (valid bits).  keep: bytes of the word in the sequence.
__device__ __forceinline__ uint32_t km_encode(uint32_t w, uint32_t keep) {
  uint32_t t = w & 0x07070707u;
  t |= t >> 4;
  const uint32_t sel = prmt_b32(t, 0u, 0x4420);                  // the four 3-bit indices as selector nibbles
  const uint32_t bad = (w & 0xDFDFDFDFu) ^ prmt_b32(0x43FF41FFu, 0x47FFFF54u, sel);   // 'a' -> 'A'; 0 where the byte is ACGTacgt
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
  const long long gw = (long long)blockIdx.x * KM_WARPS + warp, nw = (long long)gridDim.x * KM_WARPS;
  const long long lo = p.nrows * gw / nw, hi = p.nrows * (gw + 1) / nw;
  if (lo >= hi) return;
  const int n = (int)(hi - lo);
  const NtRow *mine = p.rows + lo;
  const uint32_t ring = smem_u32(s_dyn) + warp * KM_WARP_SMEM;
  uint32_t *hist = reinterpret_cast<uint32_t *>(s_dyn + warp * KM_WARP_SMEM + KM_HIST_OFF);
  for (int i = lane; i < NBINS; i += 32) hist[i] = 0u;
  NtRow upcoming = {0, 0u, 0u};
  if (lane == 0) {
    for (int i = 0; i < KM_STAGES; ++i) asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(ring + KM_BAR_OFF + i * 8) : "memory");
    fence_mbar_init();
    for (int i = 0; i < KM_STAGES && i < n; ++i) nt_issue(mine[i], ring + i * NT_STAGE, ring + KM_DESC_OFF + i * 16, ring + KM_BAR_OFF + i * 8);
    if (KM_STAGES < n) upcoming = mine[KM_STAGES];
  }
  __syncwarp();
  int st = 0; uint32_t phase = 0;
  bool whole = false;                                            // the warp saw the first row of the sequence now open
  for (int k = 0; k < n; ++k) {
    nt_wait(ring + KM_BAR_OFF + st * 8, phase);
    const uint4 d = lds128(ring + KM_DESC_OFF + st * 16);
    const uint32_t s = d.z;
    const int nbytes = (int)(d.w & 0xFFFu);
    const bool first_row = (d.w >> 30) & 1u, last_row = (d.w >> 31) != 0;
    if (k == 0 || first_row) whole = first_row;
    const uint32_t body = ring + st * NT_STAGE + NT_HALO;
    // the three bytes before the row: the halo, except at a sequence's first row (whatever is there is not sequence)
    uint32_t carry = 0;
    if (lane == 0 && !first_row) carry = km_encode(lds32(body - 4), 4u);
    uint4 v[4];
#pragma unroll
    for (int q = 0; q < 4; ++q) v[q] = lds128(body + q * 512 + lane * 16);
    // every value read from the stage is in registers: it can take the row KM_STAGES further on
    __syncwarp();
    if (lane == 0 && k + KM_STAGES < n) {
      nt_issue(upcoming, ring + st * NT_STAGE, ring + KM_DESC_OFF + st * 16, ring + KM_BAR_OFF + st * 8);
      if (k + KM_STAGES + 1 < n) upcoming = mine[k + KM_STAGES + 1];
    }
    if (++st == KM_STAGES) { st = 0; phase ^= 1u; }
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
    if (last_row || k + 1 == n) {
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

// The columns of K: canonical k-mer codes in ascending order (= lexicographic order of the strings, A < C < G < T).
int km_col_codes(int k, uint8_t *out) {
  int c = 0;
  for (uint32_t x = 0; x < (1u << (2 * k)); ++x)
    if (x <= km_revcomp(x, k)) out[c++] = (uint8_t)x;
  return c;
}

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
  for (int32_t s = 0; s < nseq; ++s) {
    if ((starts[s] & 63) || lens[s] < 0 || lens[s] > 0xFFFFFFFFll || starts[s] < 0 || (starts[s] + lens[s] + 63) / 64 * 64 > nbytes) {
      set_error("ckm_kmer_counts: every sequence must start at a multiple of 64 bytes and lie, padded to 64, inside the buffer");
      return CKM_EINVAL;
    }
  }
  const int ncols = km_cols(k);
  const size_t out_bytes = sizeof(uint32_t) * (size_t)ncols * (size_t)nseq;
  cudaSetDevice(e->device);
  PoolScope pool_scope(e);
  cudaStream_t st = e->stream;
  DevBuf dbytes;
  { int rc0 = dbytes.alloc((size_t)nbytes + 64); if (rc0) return rc0; }
  std::vector<NtRow> rows;
  nt_build_rows(dbytes.as<uint8_t>(), starts, lens, nseq, nbytes, rows);
  const int64_t nrows = (int64_t)rows.size();
  if (nrows == 0) { std::memset(counts_out, 0, out_bytes); return CKM_OK; }
  if (nrows > 0x7FFFFFFFll) { set_error("ckm_kmer_counts: too many bytes for one call"); return CKM_EINVAL; }
  DevBuf drows, dcounts;
  int rc;
  if ((rc = drows.alloc(sizeof(NtRow) * nrows)) || (rc = dcounts.alloc(out_bytes))) return rc;
  CKM_CUDA(cudaMemcpyAsync(dbytes.p, bytes, (size_t)nbytes, cudaMemcpyHostToDevice, st));
  CKM_CUDA(cudaMemcpyAsync(drows.p, rows.data(), sizeof(NtRow) * nrows, cudaMemcpyHostToDevice, st));
  CKM_CUDA(cudaMemsetAsync(dcounts.p, 0, out_bytes, st));
  KmParams p;
  std::memset(&p, 0, sizeof(p));
  p.rows = drows.as<NtRow>(); p.nrows = nrows; p.counts = dcounts.as<uint32_t>();
  km_col_codes(k, p.col_code);
  const int grid = (int)std::min<int64_t>((int64_t)e->prop.multiProcessorCount * KM_CTAS_PER_SM, (nrows + KM_WARPS - 1) / KM_WARPS);
  const int dyn_smem = KM_WARPS * KM_WARP_SMEM;
  void (*kern)(KmParams) = k == 1 ? kmer_kernel<1> : k == 2 ? kmer_kernel<2> : k == 3 ? kmer_kernel<3> : kmer_kernel<4>;
  CKM_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, dyn_smem));
  CKM_CUDA(cudaEventRecord(e->ev[0], st));
  kern<<<grid, KM_THREADS, dyn_smem, st>>>(p);
  CKM_CUDA(cudaGetLastError());
  CKM_CUDA(cudaEventRecord(e->ev[1], st));
  CKM_CUDA(cudaMemcpyAsync(counts_out, dcounts.p, out_bytes, cudaMemcpyDeviceToHost, st));
  CKM_CUDA(cudaStreamSynchronize(st));
  if (kernel_ms_out) CKM_CUDA(cudaEventElapsedTime(kernel_ms_out, e->ev[0], e->ev[1]));
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
