// insert_linear.cuh — the Λ mode of the fused insert loops (insert_loop_kernel in rewrite.cu,
// insert_wide_kernel in insert_wide.cu): the linear_insert edit of the reference
// (rewrite/ganrewrite.py:201-252), which runs Adam on Λ in  W = W0 + Λ d  instead of on W.
//
// Everything up to the weight gradient dW[o] is the projected loop's code.  What follows it is
// local to one output channel as well:
//   dΛ[o,r,t] = Σ_i dW[o,i,t] d[r,i]      (warp per (oc, r, t), as the gradient projection)
//   Adam on the rank·9 values of Λ[o]      (torch.optim.Adam's per-element arithmetic)
//   W[o,i,t]  = W0[o,i,t] + Σ_r Λ[o,r,t] d[r,i]
// The rebuild rounds the product and the sum separately (no FMA contraction), as the reference's
// `original_weight + einsum(...)` does, so a rank-1 rebuild is the reference's value bit for bit.
// Λ and its two Adam moments live in shared memory, [OC][kMaxRank*9] each, for the whole launch.
#pragma once
#include "rw_kernels.h"

namespace rw {
namespace linear_mode {

// Λ, exp_avg and exp_avg_sq of output channels o0 .. o0+OC-1 ([Cout][rank][9] in global memory)
// into shared memory; channels past Cout get zeros
template <int OC, int kStride, int kThreads>
__device__ __forceinline__ void load_state(const InsertLoopParams& p, int o0, int noc, float* lamS,
                                           float* lamMS, float* lamVS) {
  const int n = p.rank * 9;
  for (int e = threadIdx.x; e < OC * n; e += kThreads) {
    const int oc = e / n, rt = e - oc * n;
    const size_t g = static_cast<size_t>(o0) * n + e;
    const bool live = oc < noc;
    lamS[oc * kStride + rt] = live ? p.lam[g] : 0.f;
    lamMS[oc * kStride + rt] = live ? p.lam_m[g] : 0.f;
    lamVS[oc * kStride + rt] = live ? p.lam_v[g] : 0.f;
  }
}

template <int OC, int kStride, int kThreads>
__device__ __forceinline__ void store_state(const InsertLoopParams& p, int o0, int noc,
                                            const float* lamS, const float* lamMS,
                                            const float* lamVS) {
  const int n = p.rank * 9;
  for (int e = threadIdx.x; e < noc * n; e += kThreads) {
    const int oc = e / n, rt = e - oc * n;
    const size_t g = static_cast<size_t>(o0) * n + e;
    p.lam[g] = lamS[oc * kStride + rt];
    p.lam_m[g] = lamMS[oc * kStride + rt];
    p.lam_v[g] = lamVS[oc * kStride + rt];
  }
}

// Ws[oc][i*9+t] = W0[o][i*9+t] + Σ_r Λ[oc][r][t] d[r][i], r increasing, two roundings per term
template <int OC, int kStride, int kThreads>
__device__ __forceinline__ void rebuild_weights(const InsertLoopParams& p, int o0, int noc,
                                                const float* lamS, float* Ws) {
  const int Cin = p.Cin, nW = Cin * 9;
  for (int e = threadIdx.x; e < OC * nW; e += kThreads) {
    const int oc = e / nW, ei = e - oc * nW;
    const int i = ei / 9, t = ei - i * 9;
    if (oc >= noc) {
      Ws[e] = 0.f;
      continue;
    }
    const float* lr = lamS + oc * kStride + t;
    float s = __fmul_rn(lr[0], __ldg(p.d + i));
    for (int r = 1; r < p.rank; ++r) s = __fadd_rn(s, __fmul_rn(lr[r * 9], __ldg(p.d + r * Cin + i)));
    Ws[e] = __fadd_rn(__ldg(p.W0 + static_cast<size_t>(o0) * nW + e), s);
  }
}

// dΛ from the staged weight gradient dWS [OC][Cin*9], then one Adam step on Λ (torch.optim.Adam,
// amsgrad=False, weight_decay=0; the same expressions as the projected loop's Adam on W)
template <int OC, int kStride, int kWarps>
__device__ __forceinline__ void adam_step(const InsertLoopParams& p, int noc, const float* dWS,
                                          float* lamS, float* lamMS, float* lamVS, float step_size,
                                          float bc2_sqrt, float one_m_b1, float one_m_b2) {
  const int Cin = p.Cin, nW = Cin * 9, n = p.rank * 9;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int ort = warp; ort < noc * n; ort += kWarps) {
    const int oc = ort / n, rt = ort - oc * n;
    const int r = rt / 9, t = rt - r * 9;
    float a = 0.f;
    for (int i = lane; i < Cin; i += 32)
      a = fmaf(dWS[oc * nW + i * 9 + t], __ldg(p.d + r * Cin + i), a);
#pragma unroll
    for (int off = 16; off; off >>= 1) a += __shfl_xor_sync(0xffffffffu, a, off);
    if (lane == 0) {
      const int k = oc * kStride + rt;
      const float g = a;
      float mm = lamMS[k], vv = lamVS[k];
      mm = mm + (g - mm) * one_m_b1;                 // exp_avg.lerp_(grad, 1-beta1)
      vv = vv * p.beta2 + one_m_b2 * g * g;          // mul_(beta2).addcmul_(g, g, 1-beta2)
      lamMS[k] = mm;
      lamVS[k] = vv;
      const float denom = sqrtf(vv) / bc2_sqrt + p.eps;
      lamS[k] = lamS[k] - step_size * (mm / denom);
    }
  }
}

}  // namespace linear_mode
}  // namespace rw
