// aai.cu -- amino-acid identity between the copies of a multi-copy marker (checkm/aminoAcidIdentity.py:127-161): for
// every pair of equal-width masked alignment rows, the two integers the reference's aai() derives.
//
// What the reference computes, restated for rows a, b of width n ('-' = gap):
//   start = the first column where neither row has a gap; n if there is none
//   end   = 1 + the last column c in [1, n-1] where neither row has a gap; 1 if there is none; n if n < 2 (the backward
//           loop runs from n-1 down to 1 and never looks at column 0)
//   mismatches = #{c in [start, end) : a[c] != b[c]}            (a gap against a residue is a mismatch)
//   length     = mismatches + #{c in [start, end) : a[c] == b[c] != '-'}
// and AAI = 1.0 - double(mismatches) / length (0.0 when length is 0), which the caller computes in float64.
//
// Device work: aai_pairs_kernel, one warp per pair (grid-stride).  The host packs every row at a 16-byte boundary, so a
// lane reads 16 columns of each row with one 16-byte load; per byte quad, __vcmpeq4 gives gap and equality bytes that
// fold into three 16-bit lane masks (no gap in either row, bytes differ, not a gap in both).  The start scan walks
// 512-column steps forward and stops at the first step whose ballot is non-zero; the end scan walks backward the same
// way; the count step adds popcounts of the masks clipped to [start, end) and reduces them across the warp.  Rows of
// a few hundred columns make the boundary scans one step each, so a pair costs about one read of its two rows: the
// kernel is bound by those loads (2 * width bytes per pair) and by the host's packing and transfers around it.
#include <algorithm>
#include <cstdint>
#include <cstring>
#include <string>
#include <vector>
#include "engine.hpp"
#include "pool.hpp"

using namespace ckm;

namespace {

constexpr int AAI_WARPS = 8;                    // warps per block
constexpr int AAI_STEP = 32 * 16;               // columns per warp step
constexpr unsigned FULL = 0xffffffffu;

struct Cols { uint32_t ng, df, nbg; };          // bit i = column c0 + i: no gap in either row / bytes differ / not both gaps

__device__ __forceinline__ uint32_t byte_bits(uint32_t x) {     // 0xff / 0x00 per byte -> one bit per byte
  return ((x >> 7) & 1u) | ((x >> 14) & 2u) | ((x >> 21) & 4u) | ((x >> 28) & 8u);
}

// columns c0 .. c0+15 of rows A and B (width n; c0 is a multiple of 16 and the rows are padded to 16 bytes)
__device__ __forceinline__ Cols cols16(const uint8_t *__restrict__ A, const uint8_t *__restrict__ B, int c0, int n) {
  Cols r{0u, 0u, 0u};
  if (c0 >= n) return r;
  const uint4 va = __ldg(reinterpret_cast<const uint4 *>(A + c0)), vb = __ldg(reinterpret_cast<const uint4 *>(B + c0));
  const uint32_t wa[4] = {va.x, va.y, va.z, va.w}, wb[4] = {vb.x, vb.y, vb.z, vb.w};
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    const uint32_t ga = __vcmpeq4(wa[q], 0x2d2d2d2du), gb = __vcmpeq4(wb[q], 0x2d2d2d2du), eq = __vcmpeq4(wa[q], wb[q]);
    r.ng |= byte_bits(~ga & ~gb) << (4 * q);
    r.df |= byte_bits(~eq) << (4 * q);
    r.nbg |= byte_bits(~(ga & gb)) << (4 * q);
  }
  const int valid = n - c0;
  if (valid < 16) {
    const uint32_t vm = (1u << valid) - 1u;
    r.ng &= vm; r.df &= vm; r.nbg &= vm;
  }
  return r;
}

__global__ void __launch_bounds__(AAI_WARPS * 32) aai_pairs_kernel(const uint8_t *__restrict__ rows, const int64_t *__restrict__ start,
                                                                   const int32_t *__restrict__ width, const int2 *__restrict__ pairs,
                                                                   int64_t npairs, int32_t *__restrict__ mismatch_out,
                                                                   int32_t *__restrict__ len_out) {
  const int lane = threadIdx.x & 31;
  const int64_t nwarps = (int64_t)gridDim.x * AAI_WARPS;
  for (int64_t p = (int64_t)blockIdx.x * AAI_WARPS + (threadIdx.x >> 5); p < npairs; p += nwarps) {
    const int2 ab = pairs[p];
    const int n = width[ab.x];
    const uint8_t *A = rows + start[ab.x], *B = rows + start[ab.y];
    int s = n;
    for (int base = 0; base < n; base += AAI_STEP) {
      const uint32_t ng = cols16(A, B, base + lane * 16, n).ng;
      const unsigned bal = __ballot_sync(FULL, ng != 0u);
      if (bal) {
        const int l = __ffs(bal) - 1;
        s = base + l * 16 + __ffs(__shfl_sync(FULL, ng, l)) - 1;
        break;
      }
    }
    int e = n < 2 ? n : 1;
    if (n >= 2) {
      for (int base = ((n - 1) / AAI_STEP) * AAI_STEP; base >= 0; base -= AAI_STEP) {
        const int c0 = base + lane * 16;
        uint32_t ng = cols16(A, B, c0, n).ng;
        if (c0 == 0) ng &= ~1u;                  // column 0 is never looked at
        const unsigned bal = __ballot_sync(FULL, ng != 0u);
        if (bal) {
          const int l = 31 - __clz(bal);
          e = base + l * 16 + (31 - __clz(__shfl_sync(FULL, ng, l))) + 1;
          break;
        }
      }
    }
    int cm = 0, cl = 0;
    for (int base = (s / AAI_STEP) * AAI_STEP; base < e; base += AAI_STEP) {
      const int c0 = base + lane * 16;
      const Cols c = cols16(A, B, c0, n);
      const int lo = min(max(s - c0, 0), 16), hi = min(max(e - c0, 0), 16);
      const uint32_t rng = ((1u << hi) - 1u) & ~((1u << lo) - 1u);
      cm += __popc(c.df & rng);
      cl += __popc(c.nbg & rng);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      cm += __shfl_xor_sync(FULL, cm, o);
      cl += __shfl_xor_sync(FULL, cl, o);
    }
    if (lane == 0) { mismatch_out[p] = cm; len_out[p] = cl; }
  }
}

}  // namespace

extern "C" {

int ckm_aai_pairs(ckm_engine *e, const uint8_t *rows, const int64_t *row_off, int64_t nrows, const int32_t *pairs, int64_t npairs,
                  int32_t *mismatch_out, int32_t *len_out) {
  if (!e || nrows < 0 || npairs < 0 || !row_off || (npairs > 0 && (!pairs || !mismatch_out || !len_out))) {
    set_error("ckm_aai_pairs: bad argument"); return CKM_EINVAL;
  }
  if (row_off[0] != 0 || (row_off[nrows] > 0 && !rows)) { set_error("ckm_aai_pairs: bad argument"); return CKM_EINVAL; }
  std::vector<int64_t> start((size_t)std::max<int64_t>(nrows, 1));
  std::vector<int32_t> width((size_t)std::max<int64_t>(nrows, 1));
  int64_t packed_bytes = 0;
  for (int64_t r = 0; r < nrows; ++r) {
    const int64_t w = row_off[r + 1] - row_off[r];
    if (w < 0 || w > INT32_MAX - 16) { set_error("ckm_aai_pairs: row_off must be non-decreasing, rows narrower than 2^31 - 16"); return CKM_EINVAL; }
    start[(size_t)r] = packed_bytes; width[(size_t)r] = (int32_t)w;
    packed_bytes += (w + 15) & ~(int64_t)15;
  }
  for (int64_t p = 0; p < npairs; ++p) {
    const int32_t a = pairs[2 * p], b = pairs[2 * p + 1];
    if (a < 0 || b < 0 || a >= nrows || b >= nrows) {
      set_error("ckm_aai_pairs: pair " + std::to_string(p) + " names a row out of range"); return CKM_EINVAL;
    }
    if (width[(size_t)a] != width[(size_t)b]) {
      set_error("ckm_aai_pairs: pair " + std::to_string(p) + " joins rows of unequal width (" + std::to_string(width[(size_t)a]) + " and " +
                std::to_string(width[(size_t)b]) + ")");
      return CKM_EINVAL;
    }
  }
  if (npairs == 0) return CKM_OK;
  std::vector<uint8_t> packed((size_t)std::max<int64_t>(packed_bytes, 16), (uint8_t)'-');
  for (int64_t r = 0; r < nrows; ++r)
    if (width[(size_t)r]) std::memcpy(packed.data() + start[(size_t)r], rows + row_off[r], (size_t)width[(size_t)r]);

  const DeviceScope ws(e);
  DevBuf drows, dstart, dwidth, dpairs, dmis, dlen;
  CKM_TRY(drows.put(packed.data(), packed.size(), ws.st));
  CKM_TRY(dstart.put(start.data(), start.size(), ws.st));
  CKM_TRY(dwidth.put(width.data(), width.size(), ws.st));
  CKM_TRY(dpairs.put(reinterpret_cast<const int2 *>(pairs), (size_t)npairs, ws.st));
  CKM_TRY(dmis.alloc(sizeof(int32_t) * (size_t)npairs));
  CKM_TRY(dlen.alloc(sizeof(int32_t) * (size_t)npairs));
  const int64_t blocks = std::min<int64_t>((npairs + AAI_WARPS - 1) / AAI_WARPS, (int64_t)1 << 20);
  aai_pairs_kernel<<<(unsigned)blocks, AAI_WARPS * 32, 0, ws.st>>>(drows.as<uint8_t>(), dstart.as<int64_t>(), dwidth.as<int32_t>(),
                                                                  dpairs.as<int2>(), npairs, dmis.as<int32_t>(), dlen.as<int32_t>());
  CKM_CUDA(cudaGetLastError());
  CKM_TRY(dmis.get(mismatch_out, (size_t)npairs, ws.st));
  CKM_TRY(dlen.get(len_out, (size_t)npairs, ws.st));
  CKM_TRY(stream_sync(ws.st));
  return CKM_OK;
}

}  // extern "C"
