// kernels_vitp.cu -- ViterbiFilter on packed int16x2 lanes (two model positions per 32-bit register, one DPX
// VIADDMNMX.S16x2 per add+max of both).  Stage 3 of the cascade behind checkm/hmmer.py:70-71; same result as the
// int32 kernels of kernels_filters.cu (the int16-saturating recurrence of SURVEY.md A.5 step 3), at ~4.5 ALU instructions per DP
// cell instead of ~11.
//
// Layout.  W = vq/2 words per lane, K = 64 W cells.  Word w of lane l holds position k0 = l*W + w + 1 in its low
// half and k1 = 32*W + k0 in its high half, so the (k-1) neighbour of BOTH halves is word w-1 of the same lane (no
// intra-register shift); word 0 takes it from lane l-1 by one SHFL per state, and lane 0 patches its two halves with
// one PRMT (low: the k = 0 boundary; high: the low half of lane 31, i.e. position 32*W).
//
// Arithmetic.  The reference filter saturates int16 adds at -32768; VIADDMNMX wraps.  We keep every DP value
// >= FLOOR = -10240 (third operand of the instruction) and clamp every table entry at -22528 when the tables are built
// (models.cu), so a + b >= -32768 always.  Raising low values changes nothing that can reach the final score when
//   C1:  |E->J| + |tmove(L)| + max_k |tBM(k)| + 64 <= 22528      C2:  |tmove(L)| + max_k |tBM(k)| + 64 <= 22240
// because then (a) a path that crossed a clamped ("-inf") entry sits >= 22528 below a value already banked in xJ, and
// re-entering the same cell through E->J->B->M costs less than that; (b) a path restarted from FLOOR is beaten by the
// plain B->M entry of the same cell (>= 12000 - |tmove| - |tBM| + e).  Rows whose every match cell sits below FLOOR
// report xE = FLOOR; if the final xC is not above FLOOR + E->C such a row may have set it and the pair is re-scored.
// Upper end: a row maximum >= 32767 - max emission could wrap on the next add -> re-scored (these are the strong
// hits, a few percent).  The full D->D evaluation floors block sums of tDD at -16384, which is only safe under
//   C1': |E->J| + |tmove(L)| + max_k |tBM(k)| + 64 <= 16384;
// pairs outside C1' are re-scored if the lazy-F test ever asks for the full evaluation.  "Re-scored" = appended to
// p.redo, which search.cu runs through the int32 kernels.  Pairs outside C1/C2 go there directly.
#include "engine.hpp"
#include "device_utils.cuh"
#include "stages.hpp"
#include "filter_common.cuh"

namespace ckm {

constexpr uint32_t VP_FLOORW = 0xD800D800u;      // -10240 | -10240
constexpr int      VP_FLOOR  = -10240;
constexpr uint32_t VP_TFLOORW = 0xC000C000u;     // -16384 | -16384 : floor of tDD block sums

__device__ __forceinline__ int vp_lo(uint32_t w) { return (int)(int16_t)(w & 0xffffu); }
__device__ __forceinline__ int vp_hi(uint32_t w) { return (int)w >> 16; }

// Grouping the survivor list by (class, model), in three passes over p.in.  Count: pairs that need no packed scoring leave
// here -- P already <= F2 to the pass list, models without a class to the redo list -- and the others are counted per model.
// Scan (one CTA): each model's first position in p.vit_idx and first chunk, classes in BLK_Q order, models in index order
// within a class.  Scatter: each pair's index into p.in at its model's next free position; the pair that opens a chunk writes
// the chunk.  The order within a model is whatever the atomics make it: every pair is scored on its own and the kernels append
// their results through atomics, so no result depends on it.
__global__ void vit_count_kernel(FilterParams p, int32_t *cnt) {
  const int n = min(*p.in_count, p.in_cap);
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const Candidate cd = p.in[i];
    if (!(cd.P > p.F2)) filter_pass(p, cd, 4);
    else if (p.ms[cd.model].vq == 0) vit_redo(p, cd);
    else atomicAdd(cnt + cd.model, 1);
  }
}

__global__ void __launch_bounds__(1024) vit_scan_kernel(FilterParams p, int32_t nmodels, const int32_t *cnt, int32_t *off, int32_t *choff) {
  __shared__ int ws[2][32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int run_pairs = 0, run_chunks = 0;
  for (int c = 0; c < N_BLK_CLASSES; ++c) {
    if (threadIdx.x == 0) p.vit_cls_chunks[c] = run_chunks;
    for (int b = 0; b < nmodels; b += 1024) {
      const int m = b + threadIdx.x;
      const int v = (m < nmodels && blk_class(p.ms[m].vq) == c) ? cnt[m] : 0, h = (v + VITP_CHUNK - 1) / VITP_CHUNK;
      int sv = v, sh = h;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int a = __shfl_up_sync(0xffffffffu, sv, o), d = __shfl_up_sync(0xffffffffu, sh, o);
        if (lane >= o) { sv += a; sh += d; }
      }
      if (lane == 31) { ws[0][warp] = sv; ws[1][warp] = sh; }
      __syncthreads();
      if (warp == 0) {
        int tv = ws[0][lane], th = ws[1][lane];
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
          const int a = __shfl_up_sync(0xffffffffu, tv, o), d = __shfl_up_sync(0xffffffffu, th, o);
          if (lane >= o) { tv += a; th += d; }
        }
        ws[0][lane] = tv; ws[1][lane] = th;
      }
      __syncthreads();
      if (v > 0) {
        off[m] = run_pairs + (warp ? ws[0][warp - 1] : 0) + sv - v;
        choff[m] = run_chunks + (warp ? ws[1][warp - 1] : 0) + sh - h;
      }
      run_pairs += ws[0][31]; run_chunks += ws[1][31];
      __syncthreads();
    }
  }
  if (threadIdx.x == 0) p.vit_cls_chunks[N_BLK_CLASSES] = run_chunks;
}

__global__ void vit_scatter_kernel(FilterParams p, const int32_t *cnt, int32_t *fill, const int32_t *off, const int32_t *choff) {
  const int n = min(*p.in_count, p.in_cap);
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const int m = p.in[i].model;
    if (!(p.in[i].P > p.F2) || p.ms[m].vq == 0) continue;
    const int r = atomicAdd(fill + m, 1), pos = off[m] + r;
    p.vit_idx[pos] = i;
    if (r % VITP_CHUNK == 0) p.vit_chunks[choff[m] + r / VITP_CHUNK] = make_int2(pos, off[m] + min(r + VITP_CHUNK, cnt[m]));
  }
}

int launch_vit_group(const FilterParams &p, int32_t nmodels, int32_t *ws, int grid, cudaStream_t st) {
  int32_t *cnt = ws, *fill = ws + nmodels, *off = ws + 2 * (size_t)nmodels, *choff = ws + 3 * (size_t)nmodels;
  cudaError_t e = cudaMemsetAsync(ws, 0, sizeof(int32_t) * 2 * (size_t)nmodels, st);
  if (e != cudaSuccess) return cuda_fail(e, "cudaMemsetAsync(vit groups)");
  vit_count_kernel<<<grid, 256, 0, st>>>(p, cnt);
  vit_scan_kernel<<<1, 1024, 0, st>>>(p, nmodels, cnt, off, choff);
  vit_scatter_kernel<<<grid, 256, 0, st>>>(p, cnt, fill, off, choff);
  e = cudaGetLastError();
  return e == cudaSuccess ? CKM_OK : cuda_fail(e, "vit grouping launch");
}

// Work distribution.  vit_group_pairs (below) first orders the survivor list by (class, model) into p.vit_idx and cuts each
// model's run into chunks of at most VITP_CHUNK pairs (p.vit_chunks; class c owns chunks [vit_cls_chunks[c],
// vit_cls_chunks[c+1])).  A CTA claims one chunk at a time from its class's cursor p.vit_work[cls], copies that model's
// emission words (KPAD x W x 32, 3.75 KB per W) -- and for W >= 6 its transitions (1 KB per W) -- into shared memory once,
// and its warps then take the chunk's pairs one by one from a shared cursor.  The row loop reads emissions with one
// conflict-free LDS.32 per word; for W <= 4 the transitions stay in registers, loaded once per chunk.
constexpr int VITP_THREADS = 128;

__host__ __device__ constexpr int vitp_smem_bytes(int W, bool tsmem) { return KPAD * W * 32 * 4 + (tsmem ? W * 64 * 16 : 0); }
// CTAs per SM the register budget must allow: 4 warps per scheduler for W <= 4, 3 for W <= 10, 2 beyond
__host__ __device__ constexpr int vitp_min_blocks(int W) { return W <= 4 ? 4 : (W <= 10 ? 3 : 2); }

template <int W, bool TSMEM>
__global__ void __launch_bounds__(VITP_THREADS, vitp_min_blocks(W)) vitp_kernel(FilterParams p, int cls) {
  extern __shared__ __align__(16) uint4 vsm[];
  __shared__ int s_chunk, s_next;
  __shared__ ModelScalars s_ms;                                    // the chunk's model: read where used, not held in registers
  uint32_t *esm = reinterpret_cast<uint32_t *>(vsm);              // [KPAD][W][32] emission words
  uint4 *tws = vsm + KPAD * W * 8;                                 // [half][w][lane] transitions (TSMEM): conflict-free LDS.128
  const int lane = threadIdx.x & 31;
  const uint32_t sel = (lane == 0) ? 0x1054u : 0x3210u;
  const int c0 = p.vit_cls_chunks[cls], nch = p.vit_cls_chunks[cls + 1] - c0;
  for (;;) {
    __syncthreads();                                               // every warp is done with the previous chunk's tables
    if (threadIdx.x == 0) {
      const int k = atomicAdd(p.vit_work + cls, 1);
      s_chunk = k;
      if (k < nch) {
        s_next = p.vit_chunks[c0 + k].x;
        s_ms = p.ms[p.in[p.vit_idx[s_next]].model];
      }
    }
    __syncthreads();
    const int k = s_chunk;
    if (k >= nch) break;
    const int2 ch = p.vit_chunks[c0 + k];
    const ModelScalars &ms = s_ms;
    {
      const uint4 *esrc = reinterpret_cast<const uint4 *>(p.rwp + ms.blk_off * 32 * (KPAD / 2));
      for (int z = threadIdx.x; z < KPAD * W * 8; z += VITP_THREADS) vsm[z] = __ldg(esrc + z);
      if (TSMEM) {
        const uint4 *tsrc = p.twp + ms.blk_off * 32;
        for (int z = threadIdx.x; z < W * 64; z += VITP_THREADS) tws[(z & 1) * (W * 32) + (z >> 1)] = __ldg(tsrc + z);
      }
    }
    uint4 tr0[TSMEM ? 1 : W], tr1[TSMEM ? 1 : W];
    if (!TSMEM) {
      const uint4 *tsrc = p.twp + ms.blk_off * 32;
#pragma unroll
      for (int w = 0; w < W; ++w) { tr0[TSMEM ? 0 : w] = __ldg(tsrc + (w * 32 + lane) * 2); tr1[TSMEM ? 0 : w] = __ldg(tsrc + (w * 32 + lane) * 2 + 1); }
    }
#define TR0(w) (TSMEM ? tws[(w) * 32 + lane] : tr0[TSMEM ? 0 : (w)])
#define TR1(w) (TSMEM ? tws[W * 32 + (w) * 32 + lane] : tr1[TSMEM ? 0 : (w)])
    __syncthreads();
    const uint32_t *erow = esm + lane;
    const int ddbound = ms.ddbound_w, cap = 32767 - (int)ms.vit_emax;
    const int e_move = ms.xw_e_move, e_loop = ms.xw_e_loop;
    for (;;) {
      int j = 0;
      if (lane == 0) j = atomicAdd(&s_next, 1);
      j = __shfl_sync(0xffffffffu, j, 0);
      if (j >= ch.y) break;
      const Candidate *cin = p.in + p.vit_idx[j];      // read again after the row loop rather than held through it
      const int s = cin->seq, L = p.len[s];
      bool redo = false;
      const int tmove = p.tmove_w[s];
      const int cost = -tmove - (int)ms.vit_tbm + 64;
      const bool c1 = (cost - (int)ms.xw_e_loop <= 22528) && (cost <= 22240);
      const bool c1p = (cost - (int)ms.xw_e_loop <= 16384);
      redo = !c1;
      float vsc = 0.0f;
      if (!redo) {
        uint32_t Mx[W], Ix[W], Dx[W];
#pragma unroll
        for (int w = 0; w < W; ++w) { Mx[w] = VP_FLOORW; Ix[w] = VP_FLOORW; Dx[w] = VP_FLOORW; }
        int xN = ms.base_w, xB = xN + tmove, xJ = -32768, xC = -32768;
        // residues 4 at a time, the next word requested one group of rows ahead
        const uint32_t *rp = reinterpret_cast<const uint32_t *>(p.res + p.off[s]);
        const int nw = (L + 3) >> 2;
        uint32_t wcur = (nw > 0) ? __ldg(rp) : 0u;
        bool stop = false;
        for (int q = 0; q < nw && !stop; ++q) {
          const uint32_t wnext = (q + 1 < nw) ? __ldg(rp + q + 1) : 0u;
#pragma unroll
          for (int rr = 0; rr < 4; ++rr) {
            if (q * 4 + rr >= L) { stop = true; break; }
            const uint32_t *ew = erow + ((wcur >> (8 * rr)) & 0xffu) * (W * 32);
            // row i-1 values of the position just below my block, both halves
            const uint32_t shM = __shfl_sync(0xffffffffu, Mx[W - 1], (lane + 31) & 31);
            const uint32_t shI = __shfl_sync(0xffffffffu, Ix[W - 1], (lane + 31) & 31);
            const uint32_t shD = __shfl_sync(0xffffffffu, Dx[W - 1], (lane + 31) & 31);
            const uint32_t pm0 = __byte_perm(shM, VP_FLOORW, sel), pi0 = __byte_perm(shI, VP_FLOORW, sel), pd0 = __byte_perm(shD, VP_FLOORW, sel);
            const uint32_t xBw = __byte_perm((uint32_t)xB, 0u, 0x1010u);
            uint32_t md[W];
            uint32_t xEw = VP_FLOORW, dmw = VP_FLOORW;
#pragma unroll
            for (int w = W - 1; w >= 0; --w) {
              const uint32_t pm = (w > 0) ? Mx[w - 1] : pm0, pi = (w > 0) ? Ix[w - 1] : pi0, pd = (w > 0) ? Dx[w - 1] : pd0;
              const uint4 t0 = TR0(w), t1 = TR1(w);
              uint32_t sv = __viaddmax_s16x2(xBw, t0.x, VP_FLOORW);
              sv = __viaddmax_s16x2(pm, t0.y, sv);
              sv = __viaddmax_s16x2(pi, t0.z, sv);
              sv = __viaddmax_s16x2(pd, t0.w, sv);
              sv = __viaddmax_s16x2(sv, ew[w * 32], VP_FLOORW);
              const uint32_t nI = __viaddmax_s16x2(Ix[w], t1.z, __viaddmax_s16x2(Mx[w], t1.y, VP_FLOORW));
              md[w] = __viaddmax_s16x2(sv, t1.x, VP_FLOORW);
              Mx[w] = sv; Ix[w] = nI;
            }
#pragma unroll
            for (int w = 0; w + 1 < W; w += 2) { xEw = __vimax3_s16x2(xEw, Mx[w], Mx[w + 1]); dmw = __vimax3_s16x2(dmw, md[w], md[w + 1]); }
            if (W & 1) { xEw = __vimax3_s16x2(xEw, Mx[W - 1], Mx[W - 1]); dmw = __vimax3_s16x2(dmw, md[W - 1], md[W - 1]); }
            const int xE = __reduce_max_sync(0xffffffffu, max(vp_lo(xEw), vp_hi(xEw)));
            if (xE >= cap) { redo = true; stop = true; break; }
            xC = max(xC, xE + e_move);
            xJ = max(xJ, xE + e_loop);
            xB = max(xJ + tmove, xN + tmove);
            const int Dmax = __reduce_max_sync(0xffffffffu, max(vp_lo(dmw), vp_hi(dmw)));
            if (Dmax + ddbound > xB) {
              if (!c1p) { redo = true; stop = true; break; }
              // full D->D.  Per lane and half: composite f(d) = max(Bb, d + Tb) of my W cells; inclusive max-plus scan over
              // the lanes (the two halves are two independent chains here); then the high chain takes the low chain's exit.
              uint32_t Bb = VP_FLOORW, Tb = 0u;
#pragma unroll
              for (int w = 0; w < W; ++w) { const uint32_t tdd = TR1(w).w; Bb = __viaddmax_s16x2(Bb, tdd, md[w]); Tb = __viaddmax_s16x2(Tb, __vimax3_s16x2(tdd, VP_TFLOORW, VP_TFLOORW), VP_TFLOORW); }
              uint32_t Bs = Bb, Ts = Tb;
#pragma unroll
              for (int o = 1; o < 32; o <<= 1) {
                const uint32_t Bl = __shfl_up_sync(0xffffffffu, Bs, o), Tl = __shfl_up_sync(0xffffffffu, Ts, o);
                if (lane >= o) { Bs = __viaddmax_s16x2(Bl, Ts, Bs); Ts = __viaddmax_s16x2(Ts, Tl, VP_TFLOORW); }
              }
              uint32_t din = __shfl_up_sync(0xffffffffu, Bs, 1), Tex = __shfl_up_sync(0xffffffffu, Ts, 1);
              if (lane == 0) { din = VP_FLOORW; Tex = 0u; }
              const uint32_t lowexit = __shfl_sync(0xffffffffu, Bs, 31);                 // low half: D(i, 32W+1)
              const uint32_t dmid = __byte_perm(lowexit, VP_FLOORW, 0x1054u);            // (low: FLOOR, high: that exit)
              din = __viaddmax_s16x2(dmid, Tex, din);
              uint32_t d = din;
#pragma unroll
              for (int w = 0; w < W; ++w) { Dx[w] = d; d = __viaddmax_s16x2(d, TR1(w).w, md[w]); }
            } else {
              // lazy F: no D->D path can beat entering from B; D(i,k) = M(i,k-1) + tMD(k-1)
              const uint32_t shd = __shfl_sync(0xffffffffu, md[W - 1], (lane + 31) & 31);
#pragma unroll
              for (int w = W - 1; w >= 1; --w) Dx[w] = md[w - 1];
              Dx[0] = __byte_perm(shd, VP_FLOORW, sel);
            }
          }
          wcur = wnext;
        }
        if (!redo && xC <= VP_FLOOR + e_move) redo = true;      // a floored row may have set xC (or nothing scored at all)
        if (!redo) vsc = vit_vsc(xC, tmove, ms);
      }
      Candidate cd = *cin;
      if (redo) {
        if (lane == 0) vit_redo(p, cd);
        continue;
      }
      if (vit_verdict(p, cd, vsc, ms, lane) && lane == 0) filter_pass(p, cd, 4);
    }   // pairs of this chunk
#undef TR0
#undef TR1
  }   // chunks
}

// every (model slot, sequence) pair as a candidate that still needs the Viterbi filter (parity entry point ckm_viterbi_scores)
__global__ void all_pairs_kernel(Candidate *out, int32_t *count, const int32_t *slot_model, int32_t nslots, int32_t nseq) {
  const int64_t n = (int64_t)nslots * nseq;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    Candidate cd;
    cd.seq = (int32_t)(i % nseq); cd.model = slot_model[i / nseq]; cd.usc = 0.0f; cd.filtersc = 0.0f; cd.vitsc = 0.0f; cd.fwdsc = 0.0f; cd.P = 1.0;
    out[i] = cd;
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) *count = (int32_t)n;
}
int launch_all_pairs(Candidate *out, int32_t *count, const int32_t *slot_model, int32_t nslots, int32_t nseq, cudaStream_t st) {
  return launch_kernel(all_pairs_kernel, "all_pairs_kernel", 592, 256, 0, st, out, count, slot_model, nslots, nseq);
}

int launch_vitp(const FilterParams &p, int cls, int grid, cudaStream_t st) {
  return with_class(cls, [&](auto Q, auto TSMEM) {
    return launch_kernel(vitp_kernel<Q / 2, TSMEM>, "vitp_kernel", grid, VITP_THREADS, vitp_smem_bytes(Q / 2, TSMEM), st, p, cls);
  });
}

}  // namespace ckm
