// insert_linear.cuh — what the fused insert loops (insert_loop_kernel in rewrite.cu,
// insert_wide_kernel in insert_wide.cu) share: their parameter block, its conversion from the
// C-ABI's rw_insert_args / rw_linear_insert_args, and the Λ mode.
//
// The Λ mode is the linear_insert edit of the reference (rewrite/ganrewrite.py:201-252), which runs
// Adam on Λ in  W = W0 + Λ d  instead of on W.
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
#include <cstring>

#include "../../include/rewriting_b200.h"
#include "rw_common.cuh"

namespace rw {

struct InsertLoopParams {
  float* W;             // [Cout, Cin, 3, 3] updated in place
  float* m;             // Adam first moment  (same shape)
  float* v;             // Adam second moment (same shape)
  const float* w_ortho; // W0 - P_d(W0), or null when low_rank_insert is off
  const float* d;       // [rank, Cin] orthonormal rows
  int rank;
  const float* key;     // key crop, zero-bordered channels-last [B][h+2][w+2][Cin]
  const float* style;   // [B, Cin]
  const float* target;  // [B, Cout, h, w] goal activations v*
  const float* noise;   // [B, h*w] or null
  float noise_w;
  const float* bias;    // [Cout]
  int B, Cin, Cout, h, w;
  int has_noise_act;    // 1: target ends after `activate`; 0: ends after dconv
  float lr, beta1, beta2, eps;
  int it0, niter_total, nsteps;  // run iterations it0 .. it0+nsteps-1
  int piter;
  int project_gradient; // low_rank_gradient
  float* loss_out;      // [nsteps, Cout] per-channel partial |v*-y| sums
  int plain_conv;       // 1: no demodulation, weight scale 1 (ProgGAN `layerN.conv`)
  float one_minus_beta1, one_minus_beta2;   // 1-beta as torch forms it (double, rounded once)
  double beta1_exact, beta2_exact;          // betas for the bias corrections (python doubles)
  // Λ mode only (linear_insert: W = W0 + Λ d, Adam on Λ; linear_mode below).  m, v, w_ortho,
  // piter and project_gradient are then unused.
  const float* W0;      // [Cout, Cin, 3, 3] original weight, read only (must not alias W)
  float* lam;           // [Cout, rank, 3, 3] Λ, updated in place
  float* lam_m;         // Adam exp_avg of Λ
  float* lam_v;         // Adam exp_avg_sq of Λ
};

inline int insert_params(const rw_insert_args* a, const char* who, InsertLoopParams& p,
                         bool need_moments = true) {
  if (!a || !a->W || (need_moments && (!a->m || !a->v)) || !a->d || !a->key_cl ||
      (!a->style && !a->plain_conv) ||
      !a->target || !a->loss_out || (a->has_noise_act && !a->bias)) {
    set_last_error("%s: bad argument", who);
    return RW_ERR_BAD_ARG;
  }
  memset(&p, 0, sizeof(p));
  p.W = a->W; p.m = a->m; p.v = a->v; p.w_ortho = a->w_ortho; p.d = a->d; p.rank = a->rank;
  p.key = a->key_cl; p.style = a->style; p.target = a->target; p.noise = a->noise;
  p.noise_w = a->noise_w; p.bias = a->bias;
  p.B = a->B; p.Cin = a->Cin; p.Cout = a->Cout; p.h = a->h; p.w = a->w;
  p.has_noise_act = a->has_noise_act;
  p.lr = a->lr; p.beta1 = a->beta1; p.beta2 = a->beta2; p.eps = a->eps;
  p.it0 = a->it0; p.niter_total = a->niter_total; p.nsteps = a->nsteps;
  p.piter = a->piter > 0 ? a->piter : 1;
  p.project_gradient = a->project_gradient;
  p.loss_out = a->loss_out;
  p.plain_conv = a->plain_conv;
  p.one_minus_beta1 = a->one_minus_beta1 != 0.f ? a->one_minus_beta1 : 1.0f - a->beta1;
  p.one_minus_beta2 = a->one_minus_beta2 != 0.f ? a->one_minus_beta2 : 1.0f - a->beta2;
  p.beta1_exact = a->beta1_exact != 0.0 ? a->beta1_exact : static_cast<double>(a->beta1);
  p.beta2_exact = a->beta2_exact != 0.0 ? a->beta2_exact : static_cast<double>(a->beta2);
  return 0;
}

// Λ mode: the base arguments without W's Adam moments, plus W0, Λ and Λ's moments.  The reference's
// linear_insert ignores low_rank_insert / low_rank_gradient and has no plain-conv (4-D weight) form.
inline int linear_insert_params(const rw_linear_insert_args* a, const char* who,
                                InsertLoopParams& p) {
  if (!a || a->struct_size != sizeof(rw_linear_insert_args)) {
    set_last_error("%s: struct_size %zu != %zu", who, a ? a->struct_size : static_cast<size_t>(0),
                   sizeof(rw_linear_insert_args));
    return RW_ERR_BAD_ARG;
  }
  if (!a->base || !a->W0 || !a->lam || !a->lam_m || !a->lam_v) {
    set_last_error("%s: NULL base, W0, lam or moment buffer", who);
    return RW_ERR_BAD_ARG;
  }
  const rw_insert_args* b = a->base;
  if (b->w_ortho != nullptr || b->project_gradient != 0 || b->plain_conv != 0) {
    set_last_error("%s: w_ortho, project_gradient and plain_conv must be unset for linear_insert", who);
    return RW_ERR_BAD_ARG;
  }
  int rc = insert_params(b, who, p, false);
  if (rc) return rc;
  p.m = p.v = nullptr;
  p.W0 = a->W0; p.lam = a->lam; p.lam_m = a->lam_m; p.lam_v = a->lam_v;
  return 0;
}

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
