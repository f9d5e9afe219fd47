// kernels_blk.cu -- lane-blocked (register-resident) versions of the Forward filter, the region finder and the
// envelope rescoring for models with M <= 1024 (the classes of BLK_Q in stages.hpp; from Q = 12 on the transitions sit in
// shared memory).  Same mathematics as kernels_filters.cu / kernels_domdef.cu, whose verdicts and envelope tail they share
// (filter_common.cuh, domdef_common.cuh); one row costs ~20 warp shuffles instead of ~20 per 32 model positions.  Longer
// models keep using the chunked kernels.
#include "engine.hpp"
#include "device_utils.cuh"
#include "stages.hpp"
#include "fwdback.cuh"
#include "fwdback_blk.cuh"
#include "domdef_common.cuh"
#include "filter_common.cuh"

namespace ckm {

constexpr int BLK_WARPS = 4;

__host__ __device__ constexpr size_t blk_tsm_bytes(int Q) { return (size_t)Q * 32 * 2 * sizeof(float4); }

// ------------------------------------------------------------------------------------------------
// Forward filter
// ------------------------------------------------------------------------------------------------
template <int Q, bool TSMEM>
__global__ void __launch_bounds__(BLK_WARPS * 32) fwd2_kernel(FilterParams p) {
  extern __shared__ __align__(16) uint8_t bsm[];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  float4 *tsm = reinterpret_cast<float4 *>(bsm) + (size_t)warp * Q * 32 * 2;
  const int n = min(*p.in_count, p.in_cap);
  for (int c = blockIdx.x * BLK_WARPS + warp; c < n; c += gridDim.x * BLK_WARPS) {
    Candidate cd = p.in[c];
    const ModelScalars ms = p.ms[cd.model];
    if (ms.vq != Q) continue;
    const int s = cd.seq, L = p.len[s];
    BlkModel<Q, TSMEM> bm;
    blk_model_load<Q, TSMEM>(bm, ms, p.tfb, p.rfb, tsm, lane);
    const float fsc = forward_blk<Q, TSMEM, false>(bm, p.res + p.off[s], L, make_specials(L, true), nullptr, nullptr);
    fwd_verdict(p, cd, fsc, ms, lane);
  }
}

// ------------------------------------------------------------------------------------------------
// Regions: Forward + Backward parsers with special-state columns, then the shared region walk
// ------------------------------------------------------------------------------------------------
template <int Q, bool TSMEM>
__global__ void __launch_bounds__(BLK_WARPS * 32) regions2_kernel(DomdefParams p) {
  extern __shared__ __align__(16) uint8_t bsm[];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  float4 *tsm = reinterpret_cast<float4 *>(bsm) + (size_t)warp * Q * 32 * 2;
  for (int idx = p.pair_begin + blockIdx.x * BLK_WARPS + warp; idx < p.pair_end; idx += gridDim.x * BLK_WARPS) {
    const int pi = p.pair_order[idx];
    const PairWork pw = p.pairs[pi];
    const ModelScalars ms = p.ms[pw.model];
    if (ms.vq != Q) continue;
    const int L = pw.L;
    BlkModel<Q, TSMEM> bm;
    blk_model_load<Q, TSMEM>(bm, ms, p.tfb, p.rfb, tsm, lane);
    const uint8_t *res = p.res + p.off[pw.seq];
    const Specials sp = make_specials(L, true);
    float *xf = p.xf + pw.row_off * X_NX, *xb = p.xb + pw.row_off * X_NX;
    forward_blk<Q, TSMEM, false>(bm, res, L, sp, xf, nullptr);
    __syncwarp();
    backward_blk<Q, TSMEM, 0>(bm, res, L, sp, xf, xb, nullptr);
    __syncwarp();
    regions_tail(p, pi, L, sp, xf, xb, p.btot + pw.row_off, p.etot + pw.row_off, p.mocc + pw.row_off, p.n2sc + pw.row_off, lane);
    __syncwarp();
  }
}

// ------------------------------------------------------------------------------------------------
// Envelope rescoring in the blocked layout
// ------------------------------------------------------------------------------------------------
// the traceback's view of the OA matrix: position k lives at q = (k-1) % Q of lane (k-1) / Q
template <int Q> struct BlockedLayout {
  const float *F; const float4 *tfb; int M;     // tfb: the model's lane-blocked transitions
  static __device__ __forceinline__ int at(int k) { return ((k - 1) % Q) * 32 + (k - 1) / Q; }
  __device__ __forceinline__ float cell(int row, int plane, int k) const { return F[((int64_t)row * 3 + plane) * (Q * 32) + at(k)]; }
  __device__ __forceinline__ float4 t0(int k) const { return __ldg(tfb + at(k) * 2); }
  __device__ __forceinline__ float4 t1(int k) const { return __ldg(tfb + at(k) * 2 + 1); }
  // The walk runs once per domain, but its shape steers the register allocation of the whole kernel: up to Q = 12 one fully
  // unrolled pass over M and D, beyond that two passes unrolled by 4 (ptxas -v: fewest registers and spill bytes per class).
  __device__ __forceinline__ void row_best(int row, int lane, float &bm, int &bk, float &bd, int &bdk) const {
    const float *dpc = F + (int64_t)row * 3 * (Q * 32) + lane;
    if constexpr (Q <= 12) {
#pragma unroll
      for (int q = 0; q < Q; ++q) {
        const int kk = lane * Q + q + 1;
        if (kk <= M) {
          const float v = dpc[q * 32]; if (v >= bm) { bm = v; bk = kk; }
          const float w = dpc[(Q + q) * 32]; if (w > bd) { bd = w; bdk = kk; }
        }
      }
    } else {
#pragma unroll 4
      for (int q = 0; q < Q; ++q) {
        const int kk = lane * Q + q + 1;
        if (kk <= M) { const float v = dpc[q * 32]; if (v >= bm) { bm = v; bk = kk; } }
      }
#pragma unroll 4
      for (int q = 0; q < Q; ++q) {
        const int kk = lane * Q + q + 1;
        if (kk <= M) { const float w = dpc[(Q + q) * 32]; if (w > bd) { bd = w; bdk = kk; } }
      }
    }
  }
};

template <int Q, bool TSMEM>
__global__ void __launch_bounds__(BLK_WARPS * 32) envelope2_kernel(DomdefParams p) {
  extern __shared__ __align__(16) uint8_t bsm[];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  float4 *tsm = reinterpret_cast<float4 *>(bsm) + (size_t)warp * Q * 32 * 2;
  float *null2 = reinterpret_cast<float *>(bsm + (TSMEM ? BLK_WARPS * blk_tsm_bytes(Q) : 0)) + warp * 32;
  constexpr int QW = Q * 32;
  for (int idx = p.env_begin + blockIdx.x * BLK_WARPS + warp; idx < p.env_end; idx += gridDim.x * BLK_WARPS) {
    const int ei = p.env_order[idx];
    const Envelope env = p.envs[ei];
    const PairWork pw = p.pairs[env.pair];
    const ModelScalars ms = p.ms[pw.model];
    if (ms.vq != Q) continue;
    BlkModel<Q, TSMEM> bm;
    blk_model_load<Q, TSMEM>(bm, ms, p.tfb, p.rfb, tsm, lane);
    const int M = ms.M, Ld = env.j - env.i + 1;
    const uint8_t *res = p.res + p.off[pw.seq] + (env.i - 1);
    const Specials sp = make_specials(pw.L, false);
    const int64_t mat = (int64_t)(Ld + 1) * 3 * QW;
    // ONE matrix of (Ld + 1) rows x 3 planes per envelope.  Forward fills planes 0 (M) and 2 (I); Backward replaces them in place by
    // F.B; the optimal-accuracy fill reads row r of F.B and then overwrites that very row with its own M / D / I cells (plane 1
    // was free until then), so the traceback finds the OA matrix where the Forward matrix used to be.
    float *F = p.scratch + env.scratch_off, *Bm = F;
    float *xf = F + mat, *xb = xf + (int64_t)(Ld + 1) * X_NX, *pps = xb + (int64_t)(Ld + 1) * X_NX;
    float *xo = xf;
    float *n2sc = p.n2sc + pw.row_off;
    const float envsc = forward_blk<Q, TSMEM, true, false>(bm, res, Ld, sp, xf, F);
    __syncwarp();
    backward_blk<Q, TSMEM, 2>(bm, res, Ld, sp, xf, xb, F);
    __syncwarp();
    // ---- posterior decoding: pp(r,k) = (F.B)(r,k) * totr; expected state usage for null2 (summed in row order) ----
    const float scaleproduct = __fdiv_rn(1.0f, xb[X_N]);
    float em[Q], ein[Q];
#pragma unroll
    for (int q = 0; q < Q; ++q) { em[q] = 0.0f; ein[q] = 0.0f; }
    for (int r = 1; r <= Ld; ++r) {
      if (r + 2 <= Ld && lane < Q) {
        const float *fn = F + (int64_t)(r + 2) * 3 * QW;
        prefetch_l2(fn + lane * 32); prefetch_l2(fn + (2 * Q + lane) * 32);
      }
      const float totr = scaleproduct * xf[(int64_t)r * X_NX + X_SCALE];
      const float *fr = F + (int64_t)r * 3 * QW + lane;
      float vm[Q], vi[Q];
#pragma unroll
      for (int q = 0; q < Q; ++q) { vm[q] = fr[q * 32]; vi[q] = fr[(2 * Q + q) * 32]; }
#pragma unroll
      for (int q = 0; q < Q; ++q) {
        const float pm = vm[q] * totr, pi = vi[q] * totr;
        em[q] = (r == 1) ? pm : em[q] + pm;
        ein[q] = (r == 1) ? pi : ein[q] + pi;
      }
    }
    special_posteriors(sp, xf, xb, scaleproduct, pps, Ld, lane);
    const bool range_err = isinf(scaleproduct);
    if (!range_err && !env.null2_done) {
      const float norm = __fdiv_rn(1.0f, (float)Ld);
      const float xfactor = special_xfactor(pps, Ld, norm, lane);
#pragma unroll
      for (int q = 0; q < Q; ++q) { em[q] *= norm; ein[q] *= norm; }
      for (int x = 0; x < K; ++x) {
        const float *rp = bm.rfb + (size_t)x * QW;
        float part = 0.0f;
#pragma unroll
        for (int q = 0; q < Q; ++q) { part += em[q] * __ldg(rp + q * 32); part += ein[q]; }
        part = warp_sum_float(part);
        if (lane == 0) null2[x] = part + xfactor;
      }
      null2_finish(null2, n2sc, res, env, lane);
    }
    // ---- optimal accuracy fill: OA matrix overwrites F, specials go to xo ----
    float oasc = 0.0f;
    const float NINF = -INFINITY;
    if (!range_err) {
      float oM[Q], oI[Q], oD[Q];
#pragma unroll
      for (int q = 0; q < Q; ++q) { oM[q] = NINF; oI[q] = NINF; oD[q] = NINF; }
#pragma unroll
      for (int z = 0; z < 3 * Q; ++z) Bm[z * 32 + lane] = NINF;
      OaSpecials os(sp);
      os.store(xo, lane);
      for (int r = 1; r <= Ld; ++r) {
        if (r + 2 <= Ld && lane < Q) {
          const float *fn = F + (int64_t)(r + 2) * 3 * QW;
          prefetch_l2(fn + lane * 32); prefetch_l2(fn + (2 * Q + lane) * 32);
        }
        const float totr = scaleproduct * xf[(int64_t)r * X_NX + X_SCALE];      // X_SCALE survives the xo writes below
        const float *ppr = F + (int64_t)r * 3 * QW + lane;
        float *orow = Bm + (int64_t)r * 3 * QW + lane;
        float ppm[Q], ppi[Q];
#pragma unroll
        for (int q = 0; q < Q; ++q) { ppm[q] = ppr[q * 32]; ppi[q] = ppr[(2 * Q + q) * 32]; }
        float pm_in = __shfl_up_sync(0xffffffffu, oM[Q - 1], 1), pi_in = __shfl_up_sync(0xffffffffu, oI[Q - 1], 1), pd_in = __shfl_up_sync(0xffffffffu, oD[Q - 1], 1);
        if (lane == 0) { pm_in = NINF; pi_in = NINF; pd_in = NINF; }
        float a[Q]; bool ps[Q];
        float emax = NINF;
#pragma unroll
        for (int q = Q - 1; q >= 0; --q) {
          const float4 t0 = bm.T0(q), t1 = bm.T1(q);
          const bool in = (lane * Q + q + 1) <= M;
          const float pm = (q > 0) ? oM[q - 1] : pm_in, pi = (q > 0) ? oI[q - 1] : pi_in, pd = (q > 0) ? oD[q - 1] : pd_in;
          float sv = (t0.x > 0.0f) ? os.B : 0.0f;
          sv = fmaxf(sv, (t0.y > 0.0f) ? pm : 0.0f);
          sv = fmaxf(sv, (t0.z > 0.0f) ? pi : 0.0f);
          sv = fmaxf(sv, (t0.w > 0.0f) ? pd : 0.0f);
          sv += ppm[q] * totr;
          if (!in) sv = NINF;
          const float nI = in ? fmaxf((t1.y > 0.0f) ? oM[q] : 0.0f, (t1.z > 0.0f) ? oI[q] : 0.0f) + ppi[q] * totr : NINF;
          a[q] = (t1.x > 0.0f) ? sv : 0.0f;
          ps[q] = (t1.w > 0.0f);
          if (!in) { a[q] = NINF; ps[q] = true; }
          if (!ps[q]) a[q] = fmaxf(a[q], 0.0f);
          oM[q] = sv; oI[q] = nI;
          emax = fmaxf(emax, sv);
        }
        // D(k+1) = pass_k ? max(a_k, D(k)) : a_k ; block composite, scan, replay
        float A = NINF; bool pass = true;
#pragma unroll
        for (int q = 0; q < Q; ++q) { if (ps[q]) { A = fmaxf(a[q], A); } else { A = a[q]; pass = false; } }
        float As = A; bool Ps = pass;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
          const float Al = __shfl_up_sync(0xffffffffu, As, o);
          const int pl = __shfl_up_sync(0xffffffffu, (int)Ps, o);
          if (lane >= o && Ps) { As = fmaxf(As, Al); Ps = (pl != 0); }
        }
        float d = __shfl_up_sync(0xffffffffu, As, 1);
        if (lane == 0) d = NINF;
#pragma unroll
        for (int q = 0; q < Q; ++q) {
          const bool in = (lane * Q + q + 1) <= M;
          oD[q] = in ? d : NINF;
          emax = fmaxf(emax, oD[q]);
          d = ps[q] ? fmaxf(a[q], d) : a[q];
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) emax = fmaxf(emax, __shfl_xor_sync(0xffffffffu, emax, o));
        os.row(sp, pps + r * 3, emax);
#pragma unroll
        for (int q = 0; q < Q; ++q) { orow[q * 32] = oM[q]; orow[(Q + q) * 32] = oD[q]; orow[(2 * Q + q) * 32] = oI[q]; }
        os.store(xo + (int64_t)r * X_NX, lane);
      }
      oasc = os.C;
    }
    __syncwarp();
    OaTrace tr;
    if (!range_err) tr = oa_traceback(BlockedLayout<Q>{Bm, p.tfb + ms.blk_off * 64, M}, p, pw, env, sp, xo, pps, Ld, M, lane);
    write_domain(p, env, n2sc, tr, envsc, oasc, lane);
    __syncwarp();
  }
}

// ------------------------------------------------------------------------------------------------
// launchers: one launch per class; every launch walks the whole list and picks its own models
// ------------------------------------------------------------------------------------------------
template <class P, class KF>
static int launch_blk(KF kern, const char *name, int Q, bool tsmem, const P &p, int grid, size_t extra, cudaStream_t st) {
  return launch_kernel(kern, name, grid, BLK_WARPS * 32, (tsmem ? BLK_WARPS * blk_tsm_bytes(Q) : 0) + extra, st, p);
}
int launch_fwd2(const FilterParams &p, int cls, int grid, cudaStream_t st) {
  return with_class(cls, [&](auto Q, auto TSMEM) { return launch_blk(fwd2_kernel<Q, TSMEM>, "fwd2_kernel", Q, TSMEM, p, grid, 0, st); });
}
int launch_regions2(const DomdefParams &p, int cls, int grid, cudaStream_t st) {
  return with_class(cls, [&](auto Q, auto TSMEM) { return launch_blk(regions2_kernel<Q, TSMEM>, "regions2_kernel", Q, TSMEM, p, grid, 0, st); });
}
int launch_envelopes2(const DomdefParams &p, int cls, int grid, cudaStream_t st) {
  return with_class(cls, [&](auto Q, auto TSMEM) {
    return launch_blk(envelope2_kernel<Q, TSMEM>, "envelope2_kernel", Q, TSMEM, p, grid, BLK_WARPS * 32 * sizeof(float), st);
  });
}

}  // namespace ckm
