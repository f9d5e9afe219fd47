// ntrows.cuh -- the row list and stage ring that the nucleotide scans (ntstats.cu, kmers.cu, windows.cu) stream through
// shared memory, the host staging of a call, and the byte classification they share.
//
// Sequences lie in one byte buffer, each starting at a multiple of 64 and padded to the next one.  Every sequence is cut
// into 2 KB rows; the rows of all sequences of a call form one list, and each warp of a grid takes a contiguous range of
// it and streams its rows through its own ring of shared-memory stages, filled by TMA bulk copies (cp.async.bulk behind one
// mbarrier per stage) that lane 0 issues a few rows ahead.  A stage is NT_HALO + NT_ROW + NT_HALO bytes: the row's copy
// starts 16 bytes before the row (unless the row is its sequence's first) and ends 16 bytes after it (unless it is its
// last), so the bytes on either side of a row are at hand without another copy.
#pragma once
#include <algorithm>
#include <cstdint>
#include <string>
#include <vector>
#include "pool.hpp"
#include "device_utils.cuh"

namespace ckm {

constexpr int NT_CHUNK = 64;                         // bytes of one lane in one row
constexpr int NT_ROW = 32 * NT_CHUNK;                // 2 KB: what a warp takes at a time
constexpr int NT_HALO = 16;                          // bytes staged either side of a row
constexpr int NT_STAGE = NT_HALO + NT_ROW + NT_HALO;

// src: device address the row's copy starts at (16 bytes before the row unless it is the first of its sequence);
// info: valid bytes (1..2048) | 16-byte units of the copy << 12 | first row << 30 | last row << 31
struct NtRow { uint64_t src; uint32_t scaf; uint32_t info; };

// host: the row list of nseq sequences whose bytes start at device address `dev` (layout checked by nt_check_layout)
inline void nt_build_rows(const uint8_t *dev, const int64_t *starts, const int64_t *lens, int32_t nseq, int64_t nbytes,
                          std::vector<NtRow> &rows) {
  rows.clear();
  rows.reserve((size_t)(nbytes / NT_ROW) + nseq);
  for (int32_t s = 0; s < nseq; ++s)
    for (int64_t off = 0; off < lens[s]; off += NT_ROW) {
      const int64_t n = std::min<int64_t>(NT_ROW, lens[s] - off);
      const bool first = off == 0, last = off + NT_ROW >= lens[s];
      const int64_t left = first ? 0 : NT_HALO, copy = left + (n + 63) / 64 * 64 + (last ? 0 : NT_HALO);
      NtRow r; r.src = (uint64_t)(uintptr_t)(dev + starts[s] + off - left); r.scaf = (uint32_t)s;
      r.info = (uint32_t)n | ((uint32_t)(copy / 16) << 12) | (first ? 1u << 30 : 0u) | (last ? 1u << 31 : 0u);
      rows.push_back(r);
    }
}

// device: a staged row as nt_build_rows described it, and where its bytes begin in shared memory (body - NT_HALO is the
// halo before it, body + NT_ROW the halo after it)
struct NtStaged { uint64_t src; uint32_t seq; int nbytes; bool first, last; uint32_t body; };
__device__ __forceinline__ NtStaged nt_decode(uint4 d, uint32_t body) {
  return {(uint64_t)d.x | ((uint64_t)d.y << 32), d.z, (int)(d.w & 0xFFFu), ((d.w >> 30) & 1u) != 0, (d.w >> 31) != 0, body};
}

// lane 0: hand a stage to the copy engine.  Every value loaded from the stage has been used by now, so the loads are done.
__device__ __forceinline__ void nt_issue(const NtRow d, uint32_t stage, uint32_t desc, uint32_t bar) {
  asm volatile("st.shared.v4.u32 [%0], {%1,%2,%3,%4};" ::"r"(desc), "r"((uint32_t)d.src), "r"((uint32_t)(d.src >> 32)), "r"(d.scaf), "r"(d.info) : "memory");
  const uint32_t bytes = ((d.info >> 12) & 0xFFu) * 16u;
  fence_proxy_async();
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(stage + (((d.info >> 30) & 1u) ? (uint32_t)NT_HALO : 0u)),
               "l"(d.src), "r"(bytes), "r"(bar) : "memory");
}
__device__ __forceinline__ void nt_wait(uint32_t bar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "NT_WAIT:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra NT_DONE;\n"
      "bra NT_WAIT;\n"
      "NT_DONE:\n"
      "}\n" ::"r"(bar), "r"(parity) : "memory");
}

// The rows [lo, hi) of a call's nrows that warp gw of the grid's nw takes.  The host join of ckm_scaffold_stats walks the
// same ranges.
struct NtRange { long long lo, hi; };
__host__ __device__ __forceinline__ NtRange nt_warp_rows(long long nrows, long long gw, long long nw) {
  return {nrows * gw / nw, nrows * (gw + 1) / nw};
}

// One warp's ring of STAGES stages.  Its shared memory: the stages, their row descriptors (16 B each), their mbarriers
// (8 B each); the kernel's own per-warp data may begin at SMEM.  start() comes after the kernel has set up that data, so
// that its __syncwarp covers both.  Row k of the warp's range is waited for by the k-th wait(); release(k) hands its stage
// to row k + STAGES, so every lane must be done reading the stage by then.
template <int STAGES>
struct NtRing {
  static constexpr int DESC_OFF = STAGES * NT_STAGE;
  static constexpr int BAR_OFF = DESC_OFF + STAGES * 16;
  static constexpr int SMEM = (BAR_OFF + STAGES * 8 + 15) / 16 * 16;

  const uint32_t base;                 // shared address of the ring; stage i at base + i * NT_STAGE
  const NtRow *const rows;             // the warp's range of the row list
  const int n, lane;                   // n: rows in the range (the host keeps a call below 2^31 rows)
  int st = 0; uint32_t phase = 0;      // the stage the next row arrives in, and its mbarrier's parity
  NtRow upcoming;                      // lane 0: the row to issue next, fetched one row early (set before it is read)

  __device__ __forceinline__ NtRing(uint32_t base_, const NtRow *rows_, int n_, int lane_)
      : base(base_), rows(rows_), n(n_), lane(lane_) {}
  // the whole warp, once: lane 0 initialises the mbarriers and issues the first STAGES rows
  __device__ __forceinline__ void start() {
    if (lane == 0) {
      for (int i = 0; i < STAGES; ++i) asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(base + BAR_OFF + i * 8) : "memory");
      fence_mbar_init();
      for (int i = 0; i < STAGES && i < n; ++i) nt_issue(rows[i], base + i * NT_STAGE, base + DESC_OFF + i * 16, base + BAR_OFF + i * 8);
      if (STAGES < n) upcoming = rows[STAGES];
    }
    __syncwarp();
  }
  // the whole warp: the next row, once its copy has landed
  __device__ __forceinline__ NtStaged wait() const {
    nt_wait(base + BAR_OFF + st * 8, phase);
    return nt_decode(lds128(base + DESC_OFF + st * 16), base + st * NT_STAGE + NT_HALO);
  }
  // the whole warp, after its last read of row k's stage
  __device__ __forceinline__ void release(int k) {
    if (lane == 0 && k + STAGES < n) {
      nt_issue(upcoming, base + st * NT_STAGE, base + DESC_OFF + st * 16, base + BAR_OFF + st * 8);
      if (k + STAGES + 1 < n) upcoming = rows[k + STAGES + 1];
    }
    if (++st == STAGES) { st = 0; phase ^= 1u; }
  }
};

// The letter lookup of the byte classification (DESIGN §5c).  The low three bits of A, C, T, G differ (1, 3, 4, 7), so
// they make a PRMT selector per byte (nt_sel: the four 3-bit indices of a word as selector nibbles, all below 8); a
// permute of two 8-byte tables by it looks something up for each byte.  nt_letters: the upper-case letter each byte would
// have to be, 0xFF where no letter has its low bits.
__device__ __forceinline__ uint32_t nt_sel(uint32_t w) {
  uint32_t t = w & 0x07070707u;
  t |= t >> 4;
  return prmt_b32(t, 0u, 0x4420);
}
__device__ __forceinline__ uint32_t nt_letters(uint32_t sel) { return prmt_b32(0x43FF41FFu, 0x47FFFF54u, sel); }

// Reverse complement of a K-mer code (2 bits per base, the last base lowest; A 0, C 1, G 2, T 3 so complement = xor 3).
__host__ __device__ __forceinline__ uint32_t km_revcomp(uint32_t x, int k) {
  uint32_t r = 0;
  for (int i = 0; i < k; ++i) { r = (r << 2) | ((x & 3u) ^ 3u); x >>= 2; }
  return r;
}
// host: the columns of K, canonical k-mer codes in ascending order (= lexicographic order of the strings, A < C < G < T)
inline int km_col_codes(int k, uint8_t *out) {
  int c = 0;
  for (uint32_t x = 0; x < (1u << (2 * k)); ++x)
    if (x <= km_revcomp(x, k)) out[c++] = (uint8_t)x;
  return c;
}

// host: refuse a layout the row list cannot describe.  fn and what name the caller and its sequences in the message.
inline int nt_check_layout(const char *fn, const char *what, const int64_t *starts, const int64_t *lens, int32_t nseq, int64_t nbytes) {
  for (int32_t s = 0; s < nseq; ++s) {
    if ((starts[s] & 63) || lens[s] < 0 || lens[s] > 0xFFFFFFFFll || starts[s] < 0 || (starts[s] + lens[s] + 63) / 64 * 64 > nbytes) {
      set_error(std::string(fn) + ": every " + what + " must start at a multiple of 64 bytes and lie, padded to 64, inside the buffer");
      return CKM_EINVAL;
    }
  }
  return CKM_OK;
}

// host: a call's bytes and row list on the device, and its grid
struct NtUpload {
  DevBuf bytes, rows;                  // bytes: the caller's buffer and 64 bytes more
  std::vector<NtRow> host_rows;
  int64_t nrows = 0;
  int grid = 0;                        // ctas_per_sm CTAs per SM, but no more warps than rows
};
// Copies the bytes and the row list to the device on the engine's stream (inside the caller's DeviceScope) and lets `kernel`
// take dyn_smem bytes of dynamic shared memory.  With no rows, nothing is copied and u.nrows is 0.
inline int nt_upload(ckm_engine *e, const char *fn, const uint8_t *bytes, int64_t nbytes, const int64_t *starts, const int64_t *lens,
                     int32_t nseq, const void *kernel, int warps, int ctas_per_sm, int dyn_smem, NtUpload &u) {
  CKM_TRY(u.bytes.alloc((size_t)nbytes + 64));
  nt_build_rows(u.bytes.as<uint8_t>(), starts, lens, nseq, nbytes, u.host_rows);
  u.nrows = (int64_t)u.host_rows.size();
  if (u.nrows == 0) return CKM_OK;
  if (u.nrows > 0x7FFFFFFFll) { set_error(std::string(fn) + ": too many bytes for one call"); return CKM_EINVAL; }
  CKM_TRY(copy_in(u.bytes.as<uint8_t>(), bytes, (size_t)nbytes, e->stream));
  CKM_TRY(u.rows.put(u.host_rows.data(), (size_t)u.nrows, e->stream));
  u.grid = (int)std::min<int64_t>((int64_t)e->prop.multiProcessorCount * ctas_per_sm, (u.nrows + warps - 1) / warps);
  CKM_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, dyn_smem));
  return CKM_OK;
}

}  // namespace ckm
