// domdef_common.cuh -- pieces shared by the chunked (kernels_domdef.cu) and lane-blocked (kernels_blk.cu) domain stages:
// the region walk, and everything of the envelope rescoring around its DP fills (posterior decoding of the special states,
// null2 completion, the optimal-accuracy special states, the traceback and the DomainOut record).
#pragma once
#include "device_utils.cuh"
#include "stages.hpp"
#include "fwdback.cuh"

namespace ckm {

enum { ST_M = 1, ST_D, ST_I, ST_S, ST_N, ST_B, ST_E, ST_C, ST_T, ST_J };

// domain decoding of the special-state columns + the region walk by posterior heuristics (SURVEY.md A.5 step 5)
__device__ __forceinline__ void regions_tail(const DomdefParams &p, int pi, int L, const Specials sp, const float *xf, const float *xb,
                                             float *btot, float *etot, float *mocc, float *n2sc, int lane) {
    const float scaleproduct = __fdiv_rn(1.0f, xb[X_N]);
    for (int i = lane; i <= L; i += 32) {
      n2sc[i] = 0.0f;
      if (i == 0) { btot[0] = 0.0f; etot[0] = 0.0f; mocc[0] = 0.0f; continue; }
      const float *f0 = xf + (int64_t)(i - 1) * X_NX, *f1 = xf + (int64_t)i * X_NX;
      const float *b0 = xb + (int64_t)(i - 1) * X_NX, *b1 = xb + (int64_t)i * X_NX;
      btot[i] = (f0[X_B] * b0[X_B]) * f0[X_SCALE] * scaleproduct;      // per-row terms; prefix-summed below
      etot[i] = (f1[X_E] * b1[X_E]) * f1[X_SCALE] * scaleproduct;
      float njcp;
      njcp = f0[X_N] * b1[X_N] * sp.nloop * scaleproduct;
      njcp += f0[X_J] * b1[X_J] * sp.nloop * scaleproduct;
      njcp += f0[X_C] * b1[X_C] * sp.nloop * scaleproduct;
      mocc[i] = 1.0f - njcp;
    }
    __syncwarp();
    if (lane == 0) {
      float bt = 0.0f, et = 0.0f;
      for (int i = 1; i <= L; ++i) { bt = bt + btot[i]; et = et + etot[i]; btot[i] = bt; etot[i] = et; }
      int i = -1; bool triggered = false;
      for (int j = 1; j <= L; ++j) {
        if (!triggered) {
          if (mocc[j] - (btot[j] - btot[j - 1]) < 0.10f) i = j;
          else if (i == -1) i = j;
          if (mocc[j] >= 0.25f) triggered = true;
        } else if (mocc[j] - (etot[j] - etot[j - 1]) < 0.10f) {
          float mx = -1.0f;
          for (int z = i; z <= j; ++z) {
            const float a = etot[z] - etot[i - 1], b = btot[j] - btot[z - 1];
            mx = fmaxf(mx, fminf(a, b));
          }
          const int pos = atomicAdd(p.region_count, 1);
          if (pos < p.region_cap) { Region r; r.pair = pi; r.i = i; r.j = j; r.multi = (mx >= 0.20f) ? 1 : 0; p.regions[pos] = r; }
          i = -1; triggered = false;
        }
      }
    }
}

// ---- envelope rescoring ----
// N, J, C posteriors of every row r (pps[3r .. 3r+2]; row 0 zero)
__device__ __forceinline__ void special_posteriors(const Specials &sp, const float *xf, const float *xb, float scaleproduct, float *pps,
                                                   int Ld, int lane) {
  for (int r = lane; r <= Ld; r += 32) {
    float pn = 0.f, pj = 0.f, pc = 0.f;
    if (r >= 1) {
      const float *f0 = xf + (int64_t)(r - 1) * X_NX, *b1 = xb + (int64_t)r * X_NX;
      pn = f0[X_N] * b1[X_N] * sp.nloop * scaleproduct;
      pj = f0[X_J] * b1[X_J] * sp.nloop * scaleproduct;
      pc = f0[X_C] * b1[X_C] * sp.nloop * scaleproduct;
    }
    pps[r * 3 + 0] = pn; pps[r * 3 + 1] = pj; pps[r * 3 + 2] = pc;
  }
  __syncwarp();
}
// null2's share of the special states: their posteriors summed in row order, each scaled by norm = 1/Ld, then added (every lane)
__device__ __forceinline__ float special_xfactor(const float *pps, int Ld, float norm, int lane) {
  float xn = 0.f, xc = 0.f, xj = 0.f;
  if (lane == 0) {
    xn = pps[3 + 0]; xj = pps[3 + 1]; xc = pps[3 + 2];
    for (int r = 2; r <= Ld; ++r) { xn += pps[r * 3 + 0]; xj += pps[r * 3 + 1]; xc += pps[r * 3 + 2]; }
  }
  xn = __shfl_sync(0xffffffffu, xn, 0) * norm; xc = __shfl_sync(0xffffffffu, xc, 0) * norm; xj = __shfl_sync(0xffffffffu, xj, 0) * norm;
  return xn + xc + xj;
}
// null2[0..K) holds the expected odds of the canonical residues (lane 0 wrote them): the degenerate residues, the logarithms,
// and the per-residue null2 scores of the envelope into n2sc
__device__ __forceinline__ void null2_finish(float *null2, float *n2sc, const uint8_t *res, const Envelope &env, int lane) {
  __syncwarp();
  if (lane == 0) {
    // degenerate residues: plain average of the odds over the set, summed in residue-index order; gap/'*'/'~' = 1
    { float r = 0.f; r += null2[2]; r += null2[11]; null2[21] = __fdiv_rn(r, 2.0f); }     // B = D|N
    { float r = 0.f; r += null2[7]; r += null2[9];  null2[22] = __fdiv_rn(r, 2.0f); }     // J = I|L
    { float r = 0.f; r += null2[3]; r += null2[13]; null2[23] = __fdiv_rn(r, 2.0f); }     // Z = E|Q
    null2[24] = null2[8];                                                                 // O -> K
    null2[25] = null2[1];                                                                 // U -> C
    float rx = 0.f;
    for (int x = 0; x < K; ++x) rx += null2[x];
    null2[26] = __fdiv_rn(rx, 20.0f);
    null2[20] = 1.0f; null2[27] = 1.0f; null2[28] = 1.0f; null2[29] = 1.0f;
  }
  __syncwarp();
  // per-residue log ratios: 30 table entries, logarithm in double and rounded once (the float value does not depend on
  // the libm at hand, so the oracle's host arithmetic reproduces it)
  if (lane < KPAD) null2[lane] = (float)log((double)null2[lane]);
  __syncwarp();
  for (int pos = env.i + lane; pos <= env.j; pos += 32) n2sc[pos] = null2[res[pos - env.i]];
  __syncwarp();
}

// optimal-accuracy special states of one row; lane 0 keeps every row's in xo for the traceback
struct OaSpecials {
  float E, N, J, C, B;
  __device__ __forceinline__ explicit OaSpecials(const Specials &sp)
      : E(-INFINITY), N(0.0f), J(-INFINITY), C(-INFINITY), B((sp.nmove > 0.0f) ? 0.0f : -INFINITY) {}
  __device__ __forceinline__ void store(float *xr, int lane) const {
    if (lane == 0) { xr[X_E] = E; xr[X_N] = N; xr[X_J] = J; xr[X_B] = B; xr[X_C] = C; }
  }
  // row r from its best match/delete value emax and its special posteriors ppr = pps + 3r
  __device__ __forceinline__ void row(const Specials &sp, const float *ppr, float emax) {
    E = emax;
    const float ppn = ppr[0], ppj = ppr[1], ppc = ppr[2];
    float t1s = (sp.nloop == 0.0f) ? FLT_MIN_F : 1.0f, t2s = (sp.eloop == 0.0f) ? FLT_MIN_F : 1.0f;
    J = fmaxf(t1s * (J + ppj), t2s * E);
    t2s = (sp.emove == 0.0f) ? FLT_MIN_F : 1.0f;
    C = fmaxf(t1s * (C + ppc), t2s * E);
    N = t1s * (N + ppn);
    t1s = (sp.nmove == 0.0f) ? FLT_MIN_F : 1.0f;
    B = fmaxf(t1s * N, t1s * J);
  }
};

// first and last match state of the (single) domain of the optimal-accuracy trace
struct OaTrace { int hmmfrom = 0, hmmto = 0, sqfrom = 0, sqto = 0; bool ok = false; };

// The optimal-accuracy traceback, a warp-uniform state machine (lane 0's reads are broadcast).  Lay gives the OA matrix
// and the transitions in the kernel's layout: cell(row, plane, k) with planes M = 0, D = 1, I = 2, t0(k) / t1(k) (the float4
// transition pairs of position k), and row_best(row, lane, ...), this lane's best M (last maximal k) and D (first strictly
// greater) cells of a row.  The M step reads column k - 1 only for k > 1: the chunked layout's column 0 holds 0.0, but the
// transitions from node 0 into k = 1 are 0 for every model (hmm_model.cpp), so that read could never win there either.
template <class Lay>
__device__ __forceinline__ OaTrace oa_traceback(const Lay &lay, const DomdefParams &p, const PairWork &pw, const Envelope &env,
                                                const Specials &sp, const float *xo, const float *pps, int Ld, int M, int lane) {
  OaTrace tr;
  bool ok = true;
  int i = Ld, k = 0, s0 = ST_C, s1 = -1;
  int firstMi = 0, firstMk = 0, lastMi = 0, lastMk = 0; bool have_last = false;
  int guard = 0;
  while (s0 != ST_S && ok) {
    if (++guard > 4 * (Ld + M) + 16) { ok = false; break; }
    const float *xc = xo + (int64_t)i * X_NX;
    if (s0 == ST_M) {
      const float4 t0 = lay.t0(k);
      float path[4];
      path[0] = (t0.y > 0.0f && k > 1) ? lay.cell(i - 1, 0, k - 1) : -INFINITY;
      path[1] = (t0.z > 0.0f && k > 1) ? lay.cell(i - 1, 2, k - 1) : -INFINITY;
      path[2] = (t0.w > 0.0f && k > 1) ? lay.cell(i - 1, 1, k - 1) : -INFINITY;
      path[3] = (t0.x > 0.0f) ? xo[(int64_t)(i - 1) * X_NX + X_B] : -INFINITY;
      int best = 0;
      for (int z = 1; z < 4; ++z) if (path[z] > path[best]) best = z;
      s1 = (best == 0) ? ST_M : (best == 1) ? ST_I : (best == 2) ? ST_D : ST_B;
      k--; i--;
    } else if (s0 == ST_D) {
      const float4 t1 = lay.t1(k - 1);
      const float a = (t1.x > 0.0f) ? lay.cell(i, 0, k - 1) : -INFINITY, b = (t1.w > 0.0f) ? lay.cell(i, 1, k - 1) : -INFINITY;
      s1 = (a >= b) ? ST_M : ST_D; k--;
    } else if (s0 == ST_I) {
      const float4 t1 = lay.t1(k);
      const float a = (t1.y > 0.0f) ? lay.cell(i - 1, 0, k) : -INFINITY, b = (t1.z > 0.0f) ? lay.cell(i - 1, 2, k) : -INFINITY;
      s1 = (a >= b) ? ST_M : ST_I; i--;
    } else if (s0 == ST_N) {
      s1 = (i == 0) ? ST_S : ST_N;
    } else if (s0 == ST_C) {
      const float t1s = (sp.nloop == 0.0f) ? FLT_MIN_F : 1.0f, t2s = (sp.emove == 0.0f) ? FLT_MIN_F : 1.0f;
      const float a = (i > 0) ? t1s * (xo[(int64_t)(i - 1) * X_NX + X_C] + pps[i * 3 + 2]) : -INFINITY, b = t2s * xc[X_E];
      s1 = (a > b) ? ST_C : ST_E;
    } else if (s0 == ST_J) {
      const float t1s = (sp.nloop == 0.0f) ? FLT_MIN_F : 1.0f, t2s = (sp.eloop == 0.0f) ? FLT_MIN_F : 1.0f;
      const float a = (i > 0) ? t1s * (xo[(int64_t)(i - 1) * X_NX + X_J] + pps[i * 3 + 1]) : -INFINITY, b = t2s * xc[X_E];
      s1 = (a > b) ? ST_J : ST_E;
    } else if (s0 == ST_E) {
      // argmax over k of M(i,k) (last maximal index wins ties); a D can only win if strictly greater than every M
      float bmv = -INFINITY, bd = -INFINITY; int bk = -1, bdk = -1;
      lay.row_best(i, lane, bmv, bk, bd, bdk);
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        const float om = __shfl_xor_sync(0xffffffffu, bmv, o); const int ok2 = __shfl_xor_sync(0xffffffffu, bk, o);
        if (om > bmv || (om == bmv && ok2 > bk)) { bmv = om; bk = ok2; }
        const float od = __shfl_xor_sync(0xffffffffu, bd, o); const int odk = __shfl_xor_sync(0xffffffffu, bdk, o);
        if (od > bd || (od == bd && odk >= 0 && (bdk < 0 || odk < bdk))) { bd = od; bdk = odk; }
      }
      if (bd > bmv) { s1 = ST_D; k = bdk; } else { s1 = ST_M; k = bk; }
      if (k < 1) { ok = false; break; }
    } else if (s0 == ST_B) {
      const float t1s = (sp.nmove == 0.0f) ? FLT_MIN_F : 1.0f;
      s1 = (t1s * xc[X_N] > t1s * xc[X_J]) ? ST_N : ST_J;
    } else { ok = false; break; }
    if (s1 == ST_M) {
      if (!have_last || s0 == ST_E) { lastMi = i; lastMk = k; have_last = true; }
      firstMi = i; firstMk = k;
      if (p.trace != nullptr && lane == 0) p.trace[pw.row_off + env.i - 1 + i] = k;
    } else if (s1 == ST_I) {
      if (p.trace != nullptr && lane == 0) p.trace[pw.row_off + env.i - 1 + i] = -k;
    }
    if ((s1 == ST_N || s1 == ST_J || s1 == ST_C) && s1 == s0) i--;
    s0 = s1;
  }
  if (!have_last) ok = false;
  tr.ok = ok;
  tr.hmmfrom = firstMk; tr.hmmto = lastMk; tr.sqfrom = firstMi + env.i - 1; tr.sqto = lastMi + env.i - 1;
  return tr;
}

// the envelope's DomainOut (lane 0): scores, null2 correction summed over the envelope, trace coordinates
__device__ __forceinline__ void write_domain(const DomdefParams &p, const Envelope &env, const float *n2sc, const OaTrace &tr,
                                             float envsc, float oasc, int lane) {
  if (lane == 0) {
    DomainOut out;
    out.pair = env.pair; out.ienv = env.i; out.jenv = env.j;
    float domcorrection = 0.0f;
    for (int pos = env.i; pos <= env.j; ++pos) domcorrection += n2sc[pos];
    out.ok = tr.ok ? 1 : 0;
    out.envsc = envsc; out.oasc = oasc; out.domcorrection = domcorrection;
    out.hmmfrom = tr.hmmfrom; out.hmmto = tr.hmmto; out.sqfrom = tr.sqfrom; out.sqto = tr.sqto;
    out.bitscore = 0.f; out.dombias = 0.f; out.pad = 0.f; out.lnP = 0.0;
    p.doms[env.slot] = out;
  }
}

}  // namespace ckm
