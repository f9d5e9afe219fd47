// kernels_domdef.cu -- stage 5: domain definition by posterior heuristics on the pairs that pass the Forward filter,
// and the per-envelope rescoring (unihit Forward/Backward, posterior decoding, null2, optimal-accuracy alignment).
// Replaces the back half of the hmmsearch process (checkm/hmmer.py:70-71; SURVEY.md A.5 steps 5-6); its integer
// outputs are the hmm/ali/env coordinates CheckM consumes (checkm/resultsParser.py:351,431-437; util/pfam.py:117-133).
#include "engine.hpp"
#include "device_utils.cuh"
#include "stages.hpp"
#include "fwdback.cuh"
#include "domdef_common.cuh"

namespace ckm {

__device__ __forceinline__ FwdModel make_fwd_model(const DomdefParams &p, const ModelScalars &ms) {
  FwdModel fm;
  fm.M = ms.M; fm.Mpad = ms.Mpad;
  fm.rfv = p.rfv + (int64_t)ms.off_cells * KPAD;
  fm.tfv = reinterpret_cast<const float4 *>(p.tfv + (int64_t)ms.off_cells * T_N);
  return fm;
}

// ------------------------------------------------------------------------------------------------
// 5a: Forward/Backward parsers with special-state columns, domain decoding, region walk
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(FWD_WARPS * 32) regions_kernel(DomdefParams p) {
  extern __shared__ __align__(16) uint8_t smem[];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  float *rowM = reinterpret_cast<float *>(smem) + (size_t)warp * 3 * p.row_elems;
  float *rowI = rowM + p.row_elems, *rowD = rowI + p.row_elems;
  for (int idx = p.pair_begin + blockIdx.x * FWD_WARPS + warp; idx < p.pair_end; idx += gridDim.x * FWD_WARPS) {
    const int pi = p.pair_order[idx];                 // the host lists here only pairs without a lane-block class
    const PairWork pw = p.pairs[pi];
    const int L = pw.L;
    const ModelScalars ms = p.ms[pw.model];
    const FwdModel fm = make_fwd_model(p, ms);
    const uint8_t *res = p.res + p.off[pw.seq];
    const Specials sp = make_specials(L, true);
    float *xf = p.xf + pw.row_off * X_NX, *xb = p.xb + pw.row_off * X_NX;
    float *btot = p.btot + pw.row_off, *etot = p.etot + pw.row_off, *mocc = p.mocc + pw.row_off, *n2sc = p.n2sc + pw.row_off;
    forward_rows<false>(fm, res, L, sp, rowM, rowI, rowD, lane, xf, nullptr, 0, nullptr);
    __syncwarp();
    backward_rows<false>(fm, res, L, sp, rowM, rowI, rowD, lane, xf, xb, nullptr);
    __syncwarp();
    regions_tail(p, pi, L, sp, xf, xb, btot, etot, mocc, n2sc, lane);
    __syncwarp();
  }
}

// ------------------------------------------------------------------------------------------------
// 5b: rescore one envelope
// ------------------------------------------------------------------------------------------------
// the traceback's view of the OA matrix: planes of Mpad cells, position k at column k
struct ChunkedLayout {
  const float *F; const float4 *tfv; int M, Mpad;
  __device__ __forceinline__ float cell(int row, int plane, int k) const { return F[((int64_t)row * 3 + plane) * Mpad + k]; }
  __device__ __forceinline__ float4 t0(int k) const { return __ldg(tfv + 2 * k); }
  __device__ __forceinline__ float4 t1(int k) const { return __ldg(tfv + 2 * k + 1); }
  __device__ __forceinline__ void row_best(int row, int lane, float &bm, int &bk, float &bd, int &bdk) const {
    const float *dpc = F + (int64_t)row * 3 * Mpad;
    for (int kk = lane + 1; kk <= M; kk += 32) { const float v = dpc[kk]; if (v >= bm) { bm = v; bk = kk; } }
    for (int kk = lane + 1; kk <= M; kk += 32) { const float v = dpc[Mpad + kk]; if (v > bd) { bd = v; bdk = kk; } }
  }
};

__global__ void __launch_bounds__(FWD_WARPS * 32) envelope_kernel(DomdefParams p) {
  extern __shared__ __align__(16) uint8_t smem[];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  float *rowM = reinterpret_cast<float *>(smem) + (size_t)warp * 3 * p.row_elems;
  float *rowI = rowM + p.row_elems, *rowD = rowI + p.row_elems;
  for (int idx = p.env_begin + blockIdx.x * FWD_WARPS + warp; idx < p.env_end; idx += gridDim.x * FWD_WARPS) {
    const int ei = p.env_order[idx];                  // the host lists here only envelopes without a lane-block class
    const Envelope env = p.envs[ei];
    const PairWork pw = p.pairs[env.pair];
    const ModelScalars ms = p.ms[pw.model];
    const FwdModel fm = make_fwd_model(p, ms);
    const int M = fm.M, Mpad = fm.Mpad, Ld = env.j - env.i + 1, nchunk = (M + 31) >> 5;
    const uint8_t *res = p.res + p.off[pw.seq] + (env.i - 1);
    const Specials sp = make_specials(pw.L, false);
    const int64_t mat = (int64_t)(Ld + 1) * 3 * Mpad;
    float *F = p.scratch + env.scratch_off, *Bm = F + mat;
    float *xf = Bm + mat, *xb = xf + (int64_t)(Ld + 1) * X_NX, *pps = xb + (int64_t)(Ld + 1) * X_NX;   // pps: N,J,C posteriors per row
    float *xo = xf;                                                                                   // OA specials reuse xf
    float *n2sc = p.n2sc + pw.row_off;
    float envsc;
    forward_rows<true>(fm, res, Ld, sp, rowM, rowI, rowD, lane, xf, F, 0, &envsc);
    __syncwarp();
    backward_rows<true>(fm, res, Ld, sp, rowM, rowI, rowD, lane, xf, xb, Bm);
    __syncwarp();
    // ---- posterior decoding: pp overwrites the Backward matrix ----
    const float scaleproduct = __fdiv_rn(1.0f, xb[X_N]);
    for (int r = 1; r <= Ld; ++r) {
      const float totr = scaleproduct * xf[(int64_t)r * X_NX + X_SCALE];
      const float *fr = F + (int64_t)r * 3 * Mpad;
      float *br = Bm + (int64_t)r * 3 * Mpad;
      for (int k = lane + 1; k <= M; k += 32) {
        br[k] = fr[k] * br[k] * totr;
        br[Mpad + k] = 0.0f;
        br[2 * Mpad + k] = fr[2 * Mpad + k] * br[2 * Mpad + k] * totr;
      }
    }
    special_posteriors(sp, xf, xb, scaleproduct, pps, Ld, lane);
    const bool range_err = isinf(scaleproduct);
    // ---- null2 by expectation ----
    if (!range_err && !env.null2_done) {
      float *em = rowM, *ein = rowI;
      for (int k = lane + 1; k <= M; k += 32) {
        float a = Bm[(int64_t)1 * 3 * Mpad + k], b = Bm[(int64_t)1 * 3 * Mpad + 2 * Mpad + k];
        for (int r = 2; r <= Ld; ++r) { a += Bm[(int64_t)r * 3 * Mpad + k]; b += Bm[(int64_t)r * 3 * Mpad + 2 * Mpad + k]; }
        em[k] = a; ein[k] = b;
      }
      const float norm = __fdiv_rn(1.0f, (float)Ld);
      const float xfactor = special_xfactor(pps, Ld, norm, lane);
      for (int k = lane + 1; k <= M; k += 32) { em[k] *= norm; ein[k] *= norm; }
      __syncwarp();
      float *null2 = rowD;     // KP floats
      for (int x = 0; x < K; ++x) {
        const float *rp = fm.rfv + (int64_t)x * Mpad;
        float part = 0.0f;
        for (int k = lane + 1; k <= M; k += 32) { part += em[k] * __ldg(rp + k); part += ein[k]; }
        part = warp_sum_float(part);
        if (lane == 0) null2[x] = part + xfactor;
      }
      null2_finish(null2, n2sc, res, env, lane);
    }
    // ---- optimal accuracy fill: OA matrix overwrites the Forward matrix, specials go to xo ----
    float oasc = 0.0f;
    if (!range_err) {
      const float NINF = -INFINITY;
      for (int k = lane; k < 3 * Mpad; k += 32) F[k] = NINF;
      for (int k = lane; k < nchunk * 32 + 1; k += 32) { rowM[k] = NINF; rowI[k] = NINF; rowD[k] = NINF; }
      OaSpecials os(sp);
      os.store(xo, lane);
      __syncwarp();
      for (int r = 1; r <= Ld; ++r) {
        const float *ppr = Bm + (int64_t)r * 3 * Mpad;
        float *orow = F + (int64_t)r * 3 * Mpad;
        float emax = NINF, cM = NINF, cI = NINF, cD = NINF;
        float dcarry = NINF; bool dcarry_set = true;     // D(r,1) = -inf
        for (int ch = 0; ch < nchunk; ++ch) {
          const int k = ch * 32 + lane + 1;
          const float oM = rowM[k], oI = rowI[k], oD = rowD[k];
          float pm = __shfl_up_sync(0xffffffffu, oM, 1), pi2 = __shfl_up_sync(0xffffffffu, oI, 1), pd = __shfl_up_sync(0xffffffffu, oD, 1);
          if (lane == 0) { pm = cM; pi2 = cI; pd = cD; }
          cM = __shfl_sync(0xffffffffu, oM, 31); cI = __shfl_sync(0xffffffffu, oI, 31); cD = __shfl_sync(0xffffffffu, oD, 31);
          const float4 t0 = __ldg(fm.tfv + 2 * k), t1 = __ldg(fm.tfv + 2 * k + 1);
          float sv = (t0.x > 0.0f) ? os.B : 0.0f;
          sv = fmaxf(sv, (t0.y > 0.0f) ? pm : 0.0f);
          sv = fmaxf(sv, (t0.z > 0.0f) ? pi2 : 0.0f);
          sv = fmaxf(sv, (t0.w > 0.0f) ? pd : 0.0f);
          sv += ppr[k];
          const bool in = (k <= M);
          if (!in) sv = NINF;
          const float nI = in ? fmaxf((t1.y > 0.0f) ? oM : 0.0f, (t1.z > 0.0f) ? oI : 0.0f) + ppr[2 * Mpad + k] : NINF;
          // D(k+1) = max(a_k, pass_k ? D(k) : 0); state (A, pass): f(d) = pass ? max(A, d) : A
          float A = (t1.x > 0.0f) ? sv : 0.0f;
          bool pass = (t1.w > 0.0f);
          if (!in) { A = NINF; pass = true; }
          if (!pass) A = fmaxf(A, 0.0f);
#pragma unroll
          for (int o = 1; o < 32; o <<= 1) {
            const float Al = __shfl_up_sync(0xffffffffu, A, o);
            const int pl = __shfl_up_sync(0xffffffffu, (int)pass, o);
            if (lane >= o && pass) { A = fmaxf(A, Al); pass = (pl != 0); }
          }
          const float dnext = pass ? fmaxf(A, dcarry) : A;
          float dk = __shfl_up_sync(0xffffffffu, dnext, 1);
          if (lane == 0) dk = dcarry;
          dcarry = __shfl_sync(0xffffffffu, dnext, 31);
          if (!in) dk = NINF;
          emax = fmaxf(emax, fmaxf(sv, dk));
          rowM[k] = sv; rowI[k] = nI; rowD[k] = dk;
          orow[k] = sv; orow[Mpad + k] = dk; orow[2 * Mpad + k] = nI;
        }
        (void)dcarry_set;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) emax = fmaxf(emax, __shfl_xor_sync(0xffffffffu, emax, o));
        os.row(sp, pps + r * 3, emax);
        os.store(xo + (int64_t)r * X_NX, lane);
        __syncwarp();
      }
      oasc = os.C;
    }
    __syncwarp();
    OaTrace tr;
    if (!range_err) tr = oa_traceback(ChunkedLayout{F, fm.tfv, M, Mpad}, p, pw, env, sp, xo, pps, Ld, M, lane);
    write_domain(p, env, n2sc, tr, envsc, oasc, lane);
    __syncwarp();
  }
}

// ------------------------------------------------------------------------------------------------
// 5c: per-target and per-domain bit scores and P-values
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ float flogsum_dev(const float *tbl, float a, float b) {
  const float mx = fmaxf(a, b), mn = fminf(a, b);
  return (mn == -INFINITY || (mx - mn) >= 15.7f) ? mx : mx + tbl[(int)((mx - mn) * 1000.0f)];
}

__global__ void __launch_bounds__(128) scores_kernel(DomdefParams p) {
  for (int pi = blockIdx.x * blockDim.x + threadIdx.x; pi < p.npairs; pi += gridDim.x * blockDim.x) {
    const PairWork pw = p.pairs[pi];
    const ModelScalars ms = p.ms[pw.model];
    const int L = pw.L;
    HitOut h;
    h.ndom = 0; h.pre_score = h.score = h.sum_score = 0.f; h.lnP = 0.0; h.valid = 0;
    const float *n2sc = p.n2sc + pw.row_off;
    const float nullsc = p.nullsc[pw.seq], fwdsc = pw.fwdsc;
    const float logomega = -5.545177444479562f;      // log(1/256)
    const float LOG2F = 0.69314718055994529f;
    int ndom = 0;
    for (int d = pw.first_dom; d < pw.first_dom + pw.ndom_slots; ++d) if (p.doms[d].ok) ndom++;
    if (ndom > 0) {
      float seqbias = 0.0f;
      for (int i = 0; i <= L; ++i) seqbias += n2sc[i];
      seqbias = flogsum_dev(p.logsum_tbl, 0.0f, logomega + seqbias);
      float pre_score = __fdiv_rn(fwdsc - nullsc, LOG2F);
      float seq_score = __fdiv_rn(fwdsc - (nullsc + seqbias), LOG2F);
      float sum_score = 0.0f; int Ld = 0;
      seqbias = 0.0f;
      for (int d = pw.first_dom; d < pw.first_dom + pw.ndom_slots; ++d) {
        const DomainOut &dm = p.doms[d];
        if (!dm.ok) continue;
        if (dm.envsc - dm.domcorrection > 0.0f) { sum_score += dm.envsc; Ld += dm.jenv - dm.ienv + 1; seqbias += dm.domcorrection; }
      }
      seqbias = flogsum_dev(p.logsum_tbl, 0.0f, logomega + seqbias);
      const double lenterm = log((double)((float)L / (float)(L + 3)));
      sum_score = (float)((double)sum_score + (double)(L - Ld) * lenterm);
      const float pre2_score = __fdiv_rn(sum_score - nullsc, LOG2F);
      sum_score = __fdiv_rn(sum_score - (nullsc + seqbias), LOG2F);
      if (Ld > 0 && sum_score > seq_score) { seq_score = sum_score; pre_score = pre2_score; }
      h.pre_score = pre_score; h.score = seq_score; h.sum_score = sum_score;
      h.lnP = exp_logsurv((double)seq_score, (double)ms.evparam[4], (double)ms.evparam[5]);
      h.ndom = ndom; h.valid = 1;
      for (int d = pw.first_dom; d < pw.first_dom + pw.ndom_slots; ++d) {
        DomainOut &dm = p.doms[d];
        if (!dm.ok) continue;
        const int Ldd = dm.jenv - dm.ienv + 1;
        float bits = (float)((double)dm.envsc + (double)(L - Ldd) * lenterm);
        const float dombias = flogsum_dev(p.logsum_tbl, 0.0f, logomega + dm.domcorrection);
        bits = __fdiv_rn(bits - (nullsc + dombias), LOG2F);
        dm.bitscore = bits; dm.dombias = dombias;
        dm.lnP = exp_logsurv((double)bits, (double)ms.evparam[4], (double)ms.evparam[5]);
      }
    }
    p.hits[pi] = h;
  }
}

int launch_regions(const DomdefParams &p, int grid, cudaStream_t st) {
  return launch_kernel(regions_kernel, "regions_kernel", grid, FWD_WARPS * 32, (size_t)FWD_WARPS * 3 * p.row_elems * sizeof(float), st, p);
}
int launch_envelopes(const DomdefParams &p, int grid, cudaStream_t st) {
  return launch_kernel(envelope_kernel, "envelope_kernel", grid, FWD_WARPS * 32, (size_t)FWD_WARPS * 3 * p.row_elems * sizeof(float), st, p);
}
int launch_scores(const DomdefParams &p, int grid, cudaStream_t st) { return launch_kernel(scores_kernel, "scores_kernel", grid, 128, 0, st, p); }

}  // namespace ckm
