// ntrows.cuh -- the row list that the nucleotide scans (ntstats.cu, kmers.cu) stream through shared memory.
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
#include <vector>
#include "device_utils.cuh"

namespace ckm {

constexpr int NT_CHUNK = 64;                         // bytes of one lane in one row
constexpr int NT_ROW = 32 * NT_CHUNK;                // 2 KB: what a warp takes at a time
constexpr int NT_HALO = 16;                          // bytes staged either side of a row
constexpr int NT_STAGE = NT_HALO + NT_ROW + NT_HALO;

// src: device address the row's copy starts at (16 bytes before the row unless it is the first of its sequence);
// info: valid bytes (1..2048) | 16-byte units of the copy << 12 | first row << 30 | last row << 31
struct NtRow { uint64_t src; uint32_t scaf; uint32_t info; };

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

// host: the row list of nseq sequences whose bytes start at device address `dev` (layout checked by the caller)
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

}  // namespace ckm
