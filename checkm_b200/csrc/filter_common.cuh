// filter_common.cuh -- the verdicts of the filter stages, shared by every kernel variant of a stage (MSV: the SSV epilogue,
// msv_exact_kernel, msv2_kernel<Q>; Viterbi: vit_kernel, vit2_kernel<Q>, vitp_kernel<W>; Forward: fwd_kernel, fwd2_kernel<Q>):
// the score arithmetic, the P-value, the dense parity outputs and the way onto the next stage's list.
#pragma once
#include "device_utils.cuh"
#include "stages.hpp"

namespace ckm {

// ---- MSV ----
// filter score (nats) from the final xJ of the 8-bit recurrence
__device__ __forceinline__ float msv_usc(bool overflow, int xJ, int tjb, const ModelScalars &ms) {
  if (overflow) return INFINITY;
  float usc = ((float)(xJ - tjb) - (float)ms.base_b);
  usc = __fdiv_rn(usc, ms.scale_b);
  return __fsub_rn(usc, 3.0f);
}
// the dense xJ (parity output), the P-value against the null score, and the pass-list entry when P <= F1.
// Params: MsvParams or SsvParams (the same names for the dense output, the null scores and F1).
template <class Params>
__device__ __forceinline__ void msv_out(const Params &p, Candidate *out, int32_t *count, int32_t cap, int s, int m,
                                        const ModelScalars &ms, float usc, int xj_dense) {
  if (p.xj_dense != nullptr) p.xj_dense[(int64_t)p.model_slot[m] * p.nseq + s] = xj_dense;
  const float nullsc = p.nullsc[s];
  const float seq_score = __fdiv_rn(__fsub_rn(usc, nullsc), 0.69314718055994529f);
  const double P = gumbel_surv((double)seq_score, (double)ms.evparam[0], (double)ms.evparam[1]);
  if (P <= p.F1) {
    const int pos = atomicAdd(count, 1);
    if (pos < cap) {
      Candidate cd;
      cd.seq = s; cd.model = m; cd.usc = usc; cd.filtersc = nullsc; cd.vitsc = 0.f; cd.fwdsc = 0.f; cd.P = P;
      out[pos] = cd;
    }
  }
}

// ---- stages 2-4 ----
// onto the pass list of the stage; bit: the stage's flag in dense_passed (2 bias, 4 Viterbi, 8 Forward)
__device__ __forceinline__ void filter_pass(const FilterParams &p, const Candidate &cd, unsigned bit) {
  const int pos = atomicAdd(p.out_count, 1);
  if (pos < p.out_cap) p.out[pos] = cd;
  if (p.dense_passed != nullptr) atomicOr_u8(p.dense_passed, (int64_t)p.model_slot[cd.model] * p.nseq + cd.seq, bit);
}

// ---- ViterbiFilter ----
// filter score (nats) from the final xC of the int16 recurrence (a path was found and no row overflowed)
__device__ __forceinline__ float vit_vsc(int xC, int tmove, const ModelScalars &ms) {
  float vsc = __fsub_rn(__fadd_rn((float)xC, (float)tmove), (float)ms.base_w);
  vsc = __fdiv_rn(vsc, ms.scale_w);
  return __fsub_rn(vsc, 3.0f);
}
__device__ __forceinline__ float vit_score(bool overflow, int xC, int tmove, const ModelScalars &ms) {
  if (overflow) return INFINITY;
  return (xC > -32768) ? vit_vsc(xC, tmove, ms) : -INFINITY;
}
// score and P-value into cd, the dense score (parity output); true when the pair passes (P <= F2)
__device__ __forceinline__ bool vit_verdict(const FilterParams &p, Candidate &cd, float vsc, const ModelScalars &ms, int lane) {
  cd.vitsc = vsc;
  const float seq_score = __fdiv_rn(__fsub_rn(vsc, cd.filtersc), 0.69314718055994529f);
  const double P = gumbel_surv((double)seq_score, (double)ms.evparam[2], (double)ms.evparam[3]);
  cd.P = P;
  const bool pass = (P <= p.F2);
  if (lane == 0 && p.dense_vit != nullptr) p.dense_vit[(int64_t)p.model_slot[cd.model] * p.nseq + cd.seq] = vsc;
  return pass;
}
// the packed kernels' way out for the pairs they cannot score exactly: the int32 kernels' input list
__device__ __forceinline__ void vit_redo(const FilterParams &p, const Candidate &cd) {
  const int pos = atomicAdd(p.redo_count, 1);
  if (pos < p.redo_cap) p.redo[pos] = cd;
}

// ---- ForwardParser ----
// score and P-value into cd, the dense score (parity output), and the pass list when P <= F3
__device__ __forceinline__ void fwd_verdict(const FilterParams &p, Candidate &cd, float fsc, const ModelScalars &ms, int lane) {
  cd.fwdsc = fsc;
  const float seq_score = __fdiv_rn(__fsub_rn(fsc, cd.filtersc), 0.69314718055994529f);
  const double P = exp_surv((double)seq_score, (double)ms.evparam[4], (double)ms.evparam[5]);
  cd.P = P;
  if (lane == 0) {
    if (p.dense_fwd != nullptr) p.dense_fwd[(int64_t)p.model_slot[cd.model] * p.nseq + cd.seq] = fsc;
    if (P <= p.F3) filter_pass(p, cd, 8);
  }
}

}  // namespace ckm
