// kernels_filters.cu -- stages 2-4 of the cascade on the pairs that survive MSV: bias filter (thread per pair),
// ViterbiFilter (int16 semantics, warp per pair) and ForwardParser (fp32 scaled odds ratios, warp per pair).
// Replaces the corresponding stages inside the hmmsearch process (checkm/hmmer.py:70-71; SURVEY.md A.5 steps 2-4).
//
// Warp-per-pair layout: lane l owns model positions k = 32*c + l + 1 for chunk c = 0..; the previous DP row lives
// in shared memory, the (i-1,k-1) neighbour comes from the lane below by warp shuffle, and the within-row D->D
// chain is a warp scan (max-plus for Viterbi, linear for Forward) carried from chunk to chunk.
#include "engine.hpp"
#include "device_utils.cuh"
#include "stages.hpp"
#include "fwdback.cuh"
#include "filter_common.cuh"

namespace ckm {

// ------------------------------------------------------------------------------------------------
// Bias filter: 2-state HMM Forward over the sequence (state 0 background, state 1 model composition)
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(128) bias_kernel(FilterParams p) {
  const int n = min(*p.in_count, p.in_cap);
  for (int c = blockIdx.x * blockDim.x + threadIdx.x; c < n; c += gridDim.x * blockDim.x) {
    Candidate cd = p.in[c];
    const int s = cd.seq, m = cd.model, L = p.len[s];
    const ModelScalars ms = p.ms[m];
    const uint8_t *res = p.res + p.off[s];
    const float2 *eo = reinterpret_cast<const float2 *>(p.bias_eo) + (int64_t)m * KPAD;
    const float p1 = __fdiv_rn((float)L, (float)(L + 1));
    const float L1 = __fdiv_rn((float)ms.M, 8.0f);
    const float t00 = p1, t01 = __fsub_rn(1.0f, p1);
    const float t10 = __fdiv_rn(1.0f, __fadd_rn(L1, 1.0f)), t11 = __fdiv_rn(L1, __fadd_rn(L1, 1.0f));
    float2 e = __ldg(&eo[res[0]]);
    float dp0 = __fmul_rn(e.x, 0.999f), dp1 = __fmul_rn(e.y, 0.001f);
    float mx = fmaxf(dp0, dp1);
    if (mx < 0.0f) mx = 0.0f;
    dp0 = __fdiv_rn(dp0, mx); dp1 = __fdiv_rn(dp1, mx);
    float logsc = 0.0f;
    logsc = __fadd_rn(logsc, (float)log((double)mx));
    for (int i = 1; i < L; ++i) {
      e = __ldg(&eo[res[i]]);
      float n0 = 0.0f, n1 = 0.0f;
      n0 = __fadd_rn(n0, __fmul_rn(dp0, t00)); n0 = __fadd_rn(n0, __fmul_rn(dp1, t10)); n0 = __fmul_rn(n0, e.x);
      n1 = __fadd_rn(n1, __fmul_rn(dp0, t01)); n1 = __fadd_rn(n1, __fmul_rn(dp1, t11)); n1 = __fmul_rn(n1, e.y);
      mx = 0.0f;
      if (n0 > mx) mx = n0;
      if (n1 > mx) mx = n1;
      dp0 = __fdiv_rn(n0, mx); dp1 = __fdiv_rn(n1, mx);
      logsc = __fadd_rn(logsc, (float)log((double)mx));
    }
    float last = 0.0f;
    last = __fadd_rn(last, __fmul_rn(dp0, 1.0f));
    last = __fadd_rn(last, __fmul_rn(dp1, 1.0f));
    logsc = __fadd_rn(logsc, (float)log((double)last));
    const float filtersc = __fadd_rn(__fadd_rn(logsc, p.lenA[s]), p.lenB[s]);
    const float seq_score = __fdiv_rn(__fsub_rn(cd.usc, filtersc), 0.69314718055994529f);
    const double P = gumbel_surv((double)seq_score, (double)ms.evparam[0], (double)ms.evparam[1]);
    if (p.dense_filtersc != nullptr) p.dense_filtersc[(int64_t)p.model_slot[m] * p.nseq + s] = filtersc;
    if (P <= p.F1) {
      cd.filtersc = filtersc; cd.P = P;
      filter_pass(p, cd, 2);
    }
  }
}

// ------------------------------------------------------------------------------------------------
// ViterbiFilter
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ int sat16(int v) { return max(-32768, min(32767, v)); }

__global__ void __launch_bounds__(VIT_WARPS * 32) vit_kernel(FilterParams p) {
  extern __shared__ __align__(16) uint8_t smem[];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int16_t *rowM = reinterpret_cast<int16_t *>(smem) + (size_t)warp * 3 * p.row_elems;
  int16_t *rowI = rowM + p.row_elems, *rowD = rowI + p.row_elems;
  const int n = min(*p.in_count, p.in_cap);
  for (int c = blockIdx.x * VIT_WARPS + warp; c < n; c += gridDim.x * VIT_WARPS) {
    Candidate cd = p.in[c];
    const int s = cd.seq, m = cd.model, L = p.len[s];
    const ModelScalars ms = p.ms[m];
    if (p.use_blk && ms.vq != 0) continue;  // handled by vit2_kernel<Q> (CKM_BLK=0 sends every model here)
    bool pass = true;
    if (cd.P > p.F2) {
      const int M = ms.M, nchunk = (M + 31) >> 5;
      const uint8_t *res = p.res + p.off[s];
      const int16_t *rwv = p.rwv + (int64_t)ms.off_cells * KPAD;
      const uint4 *twv = reinterpret_cast<const uint4 *>(p.twv + (int64_t)ms.off_cells * T_N);
      for (int k = lane; k < nchunk * 32 + 1; k += 32) { rowM[k] = -32768; rowI[k] = -32768; rowD[k] = -32768; }
      __syncwarp();
      const int tmove = p.tmove_w[s];
      int xN = ms.base_w, xB = xN + tmove, xJ = -32768, xC = -32768;
      bool overflow = false;
      for (int i = 0; i < L && !overflow; ++i) {
        const int x = res[i];
        const int16_t *rsc = rwv + (int64_t)x * ms.Mpad;
        int xE = -32768;
        int cM = -32768, cI = -32768, cD = -32768;   // row i-1 values at the last position of the previous chunk
        int dcarry = -32768;                          // D(i, first k of this chunk)
        for (int ch = 0; ch < nchunk; ++ch) {
          const int k = ch * 32 + lane + 1;
          const int oM = rowM[k], oI = rowI[k], oD = rowD[k];
          int pm = __shfl_up_sync(0xffffffffu, oM, 1), pi = __shfl_up_sync(0xffffffffu, oI, 1), pd = __shfl_up_sync(0xffffffffu, oD, 1);
          if (lane == 0) { pm = cM; pi = cI; pd = cD; }
          cM = __shfl_sync(0xffffffffu, oM, 31); cI = __shfl_sync(0xffffffffu, oI, 31); cD = __shfl_sync(0xffffffffu, oD, 31);
          const uint4 tq = __ldg(twv + k);
          const int tBM = (int16_t)(tq.x & 0xffff), tMM = (int16_t)(tq.x >> 16), tIM = (int16_t)(tq.y & 0xffff), tDM = (int16_t)(tq.y >> 16);
          const int tMD = (int16_t)(tq.z & 0xffff), tMI = (int16_t)(tq.z >> 16), tII = (int16_t)(tq.w & 0xffff), tDD = (int16_t)(tq.w >> 16);
          int sv = sat16(xB + tBM);
          sv = max(sv, sat16(pm + tMM));
          sv = max(sv, sat16(pi + tIM));
          sv = max(sv, sat16(pd + tDM));
          sv = sat16(sv + (int)rsc[k]);
          if (k > M) sv = -32768;
          xE = max(xE, sv);
          const int nI = max(sat16(oM + tMI), sat16(oI + tII));
          // D chain: f_k(d) = max(a_k, d + t_k) gives D(i,k+1) from D(i,k); inclusive scan of the composites
          int B = (k <= M) ? sat16(sv + tMD) : -32768;
          int T = tDD;
#pragma unroll
          for (int o = 1; o < 32; o <<= 1) {
            const int Bl = __shfl_up_sync(0xffffffffu, B, o), Tl = __shfl_up_sync(0xffffffffu, T, o);
            if (lane >= o) { B = max(B, Bl + T); T = max(T + Tl, -(1 << 28)); }
          }
          const int dnext = max(max(B, dcarry + T), -32768);      // D(i, k+1)
          int dk = __shfl_up_sync(0xffffffffu, dnext, 1);           // D(i, k)
          if (lane == 0) dk = dcarry;
          dcarry = __shfl_sync(0xffffffffu, dnext, 31);
          rowM[k] = (int16_t)sv; rowI[k] = (int16_t)((k <= M) ? nI : -32768); rowD[k] = (int16_t)((k <= M) ? dk : -32768);
        }
        xE = warp_max_int(xE);
        if (xE >= 32767) { overflow = true; break; }
        xC = max(xC, xE + (int)ms.xw_e_move);
        xJ = max(xJ, xE + (int)ms.xw_e_loop);
        xB = max(xJ + tmove, xN + tmove);
        xC = max(xC, -32768); xJ = max(xJ, -32768); xB = max(xB, -32768);
        __syncwarp();
      }
      pass = vit_verdict(p, cd, vit_score(overflow, xC, tmove, ms), ms, lane);
    }
    if (lane == 0 && pass) filter_pass(p, cd, 4);
    __syncwarp();
  }
}

// ------------------------------------------------------------------------------------------------
// ViterbiFilter, lane-blocked: lane l keeps model positions l*Q+1 .. l*Q+Q of the current row in registers (M, I, D
// and the 8 transitions of each position), so a row costs two boundary shuffles, two warp reductions and -- only when
// the lazy-F test says a D->D path could matter -- one max-plus scan across the lanes.  Same int16 semantics as above.
// ------------------------------------------------------------------------------------------------
struct Tr8 { int bm, mm, im, dm, md, mi, ii, dd; };
__device__ __forceinline__ Tr8 unpack_tr(const uint4 t) {
  Tr8 r;
  r.bm = (int16_t)(t.x & 0xffff); r.mm = (int16_t)(t.x >> 16); r.im = (int16_t)(t.y & 0xffff); r.dm = (int16_t)(t.y >> 16);
  r.md = (int16_t)(t.z & 0xffff); r.mi = (int16_t)(t.z >> 16); r.ii = (int16_t)(t.w & 0xffff); r.dd = (int16_t)(t.w >> 16);
  return r;
}

// TSMEM: keep the (packed) transitions of the warp's model in shared memory instead of registers (Q = 32, M <= 1024)
template <int Q, bool TSMEM>
__global__ void __launch_bounds__(128) vit2_kernel(FilterParams p) {
  extern __shared__ __align__(16) uint8_t vsm[];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, wpb = blockDim.x >> 5;
  uint4 *tws = reinterpret_cast<uint4 *>(vsm) + (size_t)warp * Q * 32;
  const int n = min(*p.in_count, p.in_cap);
  for (int c = blockIdx.x * wpb + warp; c < n; c += gridDim.x * wpb) {
    Candidate cd = p.in[c];
    const int m = cd.model;
    const ModelScalars ms = p.ms[m];
    if (ms.vq != Q) continue;
    const int s = cd.seq, L = p.len[s];
    bool pass = true;
    if (cd.P > p.F2) {
      // transitions of my Q positions {BM, MM, IM, DM, MD, MI, II, DD}: registers, or shared memory for the widest class
      Tr8 trr[TSMEM ? 1 : Q];
      if (TSMEM) {
        __syncwarp();
        for (int q = 0; q < Q; ++q) tws[q * 32 + lane] = __ldg(p.twb + (ms.blk_off + q) * 32 + lane);
        __syncwarp();
      } else {
#pragma unroll
        for (int q = 0; q < Q; ++q) trr[q] = unpack_tr(__ldg(p.twb + (ms.blk_off + q) * 32 + lane));
      }
#define TRQ(q) (TSMEM ? unpack_tr(tws[(q) * 32 + lane]) : trr[TSMEM ? 0 : (q)])
      const uint32_t *rwb = p.rwb + ms.blk_off * 32 * (KPAD / 2) + lane;
      int Mx[Q], Ix[Q], Dx[Q];
#pragma unroll
      for (int q = 0; q < Q; ++q) { Mx[q] = -32768; Ix[q] = -32768; Dx[q] = -32768; }
      const int tmove = p.tmove_w[s], ddbound = ms.ddbound_w;
      int xN = ms.base_w, xB = xN + tmove, xJ = -32768, xC = -32768;
      bool overflow = false;
      const uint4 *rp = reinterpret_cast<const uint4 *>(p.res + p.off[s]);
      const int nblk = (L + 15) >> 4;
      for (int b = 0; b < nblk && !overflow; ++b) {
        const uint4 r16 = __ldg(rp + b);
        const uint32_t w4[4] = {r16.x, r16.y, r16.z, r16.w};
        const int rows = min(16, L - b * 16);
        for (int r = 0; r < rows; ++r) {
          const uint32_t x = (w4[r >> 2] >> (8 * (r & 3))) & 0xffu;
          uint32_t e2[Q / 2];
#pragma unroll
          for (int j = 0; j < Q / 2; ++j) e2[j] = __ldg(rwb + (x * (Q / 2) + j) * 32);
          // row i-1 values of the position just below my block
          const uint32_t packed = ((uint32_t)(uint16_t)Mx[Q - 1]) | ((uint32_t)(uint16_t)Ix[Q - 1] << 16);
          uint32_t bmi = __shfl_up_sync(0xffffffffu, packed, 1);
          int bd = __shfl_up_sync(0xffffffffu, Dx[Q - 1], 1);
          if (lane == 0) { bmi = 0x80008000u; bd = -32768; }
          const int pm_in = (int16_t)(bmi & 0xffff), pi_in = (int16_t)(bmi >> 16);
          int xEl = -32768, dml = -32768;
          int md[Q];
#pragma unroll
          for (int q = Q - 1; q >= 0; --q) {
            const int pm = (q > 0) ? Mx[q - 1] : pm_in, pi = (q > 0) ? Ix[q - 1] : pi_in, pd = (q > 0) ? Dx[q - 1] : bd;
            const Tr8 t = TRQ(q);
            int sv = __viaddmax_s32(xB, t.bm, -32768);
            sv = __viaddmax_s32(pm, t.mm, sv);
            sv = __viaddmax_s32(pi, t.im, sv);
            sv = __viaddmax_s32(pd, t.dm, sv);
            const int e = (q & 1) ? ((int)e2[q >> 1] >> 16) : (int)(int16_t)(e2[q >> 1] & 0xffffu);
            sv = min(__viaddmax_s32(sv, e, -32768), 32767);
            const int nI = __viaddmax_s32(Ix[q], t.ii, __viaddmax_s32(Mx[q], t.mi, -32768));
            md[q] = __viaddmax_s32(sv, t.md, -32768);
            xEl = max(xEl, sv); dml = max(dml, md[q]);
            Mx[q] = sv; Ix[q] = nI;
          }
          const int xE = __reduce_max_sync(0xffffffffu, xEl);
          if (xE >= 32767) { overflow = true; break; }
          xC = max(xC, xE + (int)ms.xw_e_move);
          xJ = max(xJ, xE + (int)ms.xw_e_loop);
          xB = max(xJ + tmove, xN + tmove);
          xC = max(xC, -32768); xJ = max(xJ, -32768); xB = max(xB, -32768);
          const int Dmax = __reduce_max_sync(0xffffffffu, dml);
          if (Dmax + ddbound > xB) {
            // full D->D: composite of my block f(d) = max(Bb, d + Tb), exclusive max-plus scan across lanes
            int Bb = -32768, Tb = 0;
#pragma unroll
            for (int q = 0; q < Q; ++q) { const int tdd = TRQ(q).dd; Bb = max(md[q], Bb + tdd); Bb = max(Bb, -32768); Tb = max(Tb + tdd, -(1 << 24)); }
            int Bs = Bb, Ts = Tb;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
              const int Bl = __shfl_up_sync(0xffffffffu, Bs, o), Tl = __shfl_up_sync(0xffffffffu, Ts, o);
              if (lane >= o) { Bs = max(Bs, Bl + Ts); Ts = max(Ts + Tl, -(1 << 24)); }
            }
            int din = __shfl_up_sync(0xffffffffu, max(Bs, -32768), 1);      // D(i, first k of my block)
            if (lane == 0) din = -32768;
            int d = din;
#pragma unroll
            for (int q = 0; q < Q; ++q) { Dx[q] = d; d = max(max(md[q], d + TRQ(q).dd), -32768); }
          } else {
            // lazy F: no D->D path can beat entering from B; keep the M->D partials only
            int din = __shfl_up_sync(0xffffffffu, md[Q - 1], 1);
            if (lane == 0) din = -32768;
#pragma unroll
            for (int q = Q - 1; q >= 1; --q) Dx[q] = md[q - 1];
            Dx[0] = din;
          }
        }
      }
      pass = vit_verdict(p, cd, vit_score(overflow, xC, tmove, ms), ms, lane);
    }
    if (lane == 0 && pass) filter_pass(p, cd, 4);
#undef TRQ
  }
}

// ------------------------------------------------------------------------------------------------
// Forward row engine (shared by the parser here and by the domain-definition stage)
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(FWD_WARPS * 32) fwd_kernel(FilterParams p) {
  extern __shared__ __align__(16) uint8_t smem[];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  float *rowM = reinterpret_cast<float *>(smem) + (size_t)warp * 3 * p.row_elems;
  float *rowI = rowM + p.row_elems, *rowD = rowI + p.row_elems;
  const int n = min(*p.in_count, p.in_cap);
  for (int c = blockIdx.x * FWD_WARPS + warp; c < n; c += gridDim.x * FWD_WARPS) {
    Candidate cd = p.in[c];
    const int s = cd.seq, m = cd.model, L = p.len[s];
    const ModelScalars ms = p.ms[m];
    if (p.use_blk && ms.vq != 0) continue;            // handled by fwd2_kernel<Q>
    const uint8_t *res = p.res + p.off[s];
    FwdModel fm;
    fm.M = ms.M; fm.Mpad = ms.Mpad;
    fm.rfv = p.rfv + (int64_t)ms.off_cells * KPAD;
    fm.tfv = reinterpret_cast<const float4 *>(p.tfv + (int64_t)ms.off_cells * T_N);
    const Specials sp = make_specials(L, true);
    float fsc;
    forward_rows<false>(fm, res, L, sp, rowM, rowI, rowD, lane, nullptr, nullptr, 0, &fsc);
    fwd_verdict(p, cd, fsc, ms, lane);
    __syncwarp();
  }
}

int launch_bias(const FilterParams &p, int grid, cudaStream_t st) { return launch_kernel(bias_kernel, "bias_kernel", grid, 128, 0, st, p); }
int launch_vit2(const FilterParams &p, int cls, int grid, cudaStream_t st) {
  return with_class(cls, [&](auto Q, auto TSMEM) {
    return launch_kernel(vit2_kernel<Q, TSMEM>, "vit2_kernel", grid, 128, TSMEM ? 4 * Q * 32 * sizeof(uint4) : 0, st, p);
  });
}
int launch_vit(const FilterParams &p, int grid, cudaStream_t st) {
  return launch_kernel(vit_kernel, "vit_kernel", grid, VIT_WARPS * 32, (size_t)VIT_WARPS * 3 * p.row_elems * sizeof(int16_t), st, p);
}
int launch_fwd(const FilterParams &p, int grid, cudaStream_t st) {
  return launch_kernel(fwd_kernel, "fwd_kernel", grid, FWD_WARPS * 32, (size_t)FWD_WARPS * 3 * p.row_elems * sizeof(float), st, p);
}

}  // namespace ckm
