// bwd.cu — HBM-bound CUDA-core kernels of the StyledConv BACKWARD pass.  Between the
// tensor-core kernels (dgrad row-GEMM, wgrad col-GEMM) the backward of
//   y = act( [blur]( conv(style*x, s*W) * demod ) + nw*noise + bias )
// (DemodulatedConv2dF / BlurF / NoiseInjectionF / FusedLeakyReLUF autograd,
//  utils/stylegan2/models.py:275-281,313-329,535-546 and op/fused_act.py:19-86)
// needs only elementwise work and per-(sample, channel) reductions over pixels.  Each kernel
// here makes ONE pass over its tensors and produces every reduction of that pass:
//
//   act_grad_reduce   (gy, y)        -> g_pre, sum g_pre, sum g_pre*pre, sum g_pre*noise
//   blur_adj_phase    g_pre          -> phase planes of demod * blur^T(g_pre)  (up layers)
//   dgrad_finish      (dk, x, style) -> gx = dk*style in place, sum dk*x
//   wgrad_finish      dWt, W, ...    -> gW incl. the demodulation term
//   style_grad_finish                -> g_style incl. the demodulation term
//
// All reductions are block-local trees (bit-reproducible, no atomics).
#include "../../include/rewriting_b200.h"
#include "rw_common.cuh"

namespace rw {

namespace {

constexpr float kSqrt2 = 1.4142135623730951f;
constexpr float kInvSqrt2 = 0.70710678118654752f;
constexpr float kSlope = 0.2f;

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int off = 16; off; off >>= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
  return v;
}

// sum of NV per-thread values over the block; the totals are valid in warp 0 (all lanes).
// blockDim.x must be a multiple of 32 (<= 1024); `red` holds 32*NV floats.
template <int NV>
__device__ __forceinline__ void block_sum(float (&v)[NV], float* red) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int nwarps = (blockDim.x + 31) >> 5;
#pragma unroll
  for (int j = 0; j < NV; ++j) v[j] = warp_sum(v[j]);
  if (lane == 0) {
#pragma unroll
    for (int j = 0; j < NV; ++j) red[warp * NV + j] = v[j];
  }
  __syncthreads();
  if (warp == 0) {
#pragma unroll
    for (int j = 0; j < NV; ++j) {
      const float a = (lane < nwarps) ? red[lane * NV + j] : 0.f;
      v[j] = warp_sum(a);
    }
  }
}

// ---------------------------------------------------------------------------
// act_grad_reduce: one block per (b, c) plane of HW pixels.
//   act:  g_pre = (y > 0 ? gy : 0.2*gy) * sqrt2          (fused_bias_act grad=1, ref = y:
//                                                          op/fused_bias_act_kernel.cu:30-47)
//         pre   = (y > 0 ? y : 5*y) / sqrt2 - bias[c]     (the pre-activation, recovered)
//   else: g_pre = gy, pre = y
//   t     = pre - nw*noise[b,p]       = demodulated (blurred) conv output
//   s_sum[b,c]   = sum_p g_pre        (-> bias gradient after summing over b)
//   s_dot[b,c]   = sum_p g_pre * t    (= dL/d demod * demod; blur^T is absorbed: <g, blur t_up>)
//   s_noise[b,c] = sum_p g_pre*noise  (-> noise-weight gradient after summing over b, c)
// ---------------------------------------------------------------------------
struct ActGradAcc {
  float s, d, n;
};

__device__ __forceinline__ float act_grad_one(float g, float yy, float nz, int act, float bv,
                                              float nw, ActGradAcc& a) {
  float gp, pre;
  if (act) {
    const bool pos = yy > 0.f;
    gp = (pos ? g : kSlope * g) * kSqrt2;
    pre = (pos ? yy : 5.f * yy) * kInvSqrt2 - bv;
  } else {
    gp = g;
    pre = yy;
  }
  pre = fmaf(-nw, nz, pre);
  a.s += gp;
  a.d = fmaf(gp, pre, a.d);
  a.n = fmaf(gp, nz, a.n);
  return gp;
}

__global__ void __launch_bounds__(256)
act_grad_reduce_kernel(const float* __restrict__ gy, const float* __restrict__ y,
                       const float* __restrict__ noise, long long noise_bstride,
                       const float* __restrict__ noise_w, const float* __restrict__ bias, int act,
                       int C, int HW, int vec, float* __restrict__ g_pre,
                       float* __restrict__ s_sum, float* __restrict__ s_dot,
                       float* __restrict__ s_noise) {
  __shared__ float red[32 * 3];
  const int bc = blockIdx.x;
  const int b = bc / C, c = bc - b * C;
  const size_t base = static_cast<size_t>(bc) * HW;
  const float nw = noise ? __ldg(noise_w) : 0.f;
  const float bv = (act && bias) ? __ldg(bias + c) : 0.f;
  const float* nzp = noise ? noise + static_cast<size_t>(b) * noise_bstride : nullptr;
  ActGradAcc a = {0.f, 0.f, 0.f};
  if (vec) {
    const float4* g4 = reinterpret_cast<const float4*>(gy + base);
    const float4* y4 = reinterpret_cast<const float4*>(y + base);
    const float4* n4 = reinterpret_cast<const float4*>(nzp);
    float4* o4 = g_pre ? reinterpret_cast<float4*>(g_pre + base) : nullptr;
    const int nq = HW >> 2;
    for (int i = threadIdx.x; i < nq; i += blockDim.x) {
      const float4 g = __ldg(g4 + i), yy = __ldg(y4 + i);
      const float4 nz = nzp ? __ldg(n4 + i) : make_float4(0.f, 0.f, 0.f, 0.f);
      float4 o;
      o.x = act_grad_one(g.x, yy.x, nz.x, act, bv, nw, a);
      o.y = act_grad_one(g.y, yy.y, nz.y, act, bv, nw, a);
      o.z = act_grad_one(g.z, yy.z, nz.z, act, bv, nw, a);
      o.w = act_grad_one(g.w, yy.w, nz.w, act, bv, nw, a);
      if (o4) o4[i] = o;
    }
  } else {
    for (int i = threadIdx.x; i < HW; i += blockDim.x) {
      const float nz = nzp ? __ldg(nzp + i) : 0.f;
      const float o = act_grad_one(__ldg(gy + base + i), __ldg(y + base + i), nz, act, bv, nw, a);
      if (g_pre) g_pre[base + i] = o;
    }
  }
  float v[3] = {a.s, a.d, a.n};
  block_sum<3>(v, red);
  if (threadIdx.x == 0) {
    s_sum[bc] = v[0];
    s_dot[bc] = v[1];
    s_noise[bc] = v[2];
  }
}

// ---------------------------------------------------------------------------
// blur_adj_phase: gradient phase planes of an upsampling StyledConv straight from g_pre.
//   g_t[ty,tx] = sum_{a,bb} kf[a][bb] * g_pre[ty-a+1, tx-bb+1]      (adjoint of BlurF pad (1,1);
//                kf = flipped 4x4 FIR, as blur_up_act applies it)     ty in [0,2H], tx in [0,2W]
//   planes[(b,m,n)][ph*C + c] = split_bf16(scale[b,c] * g_t[2m+pa, 2n+pb]),  ph = pa*2+pb
// (zero where 2m+pa > 2H or 2n+pb > 2W) — the layout rw_prep_phase_keys produces from a
// materialised g_t; here the [B,C,2H+1,2W+1] tensor never exists.  The 4 phases of one (m,n)
// share a 5x5 window of g_pre (25 loads for 4 outputs).
// grid: (ceil(Hp*Wp/32), C/64, B), block 256.
// ---------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
blur_adj_phase_kernel(const float* __restrict__ g, const float* __restrict__ scale,
                      const float* __restrict__ k4, int C, int H, int W,
                      __nv_bfloat16* __restrict__ hi, __nv_bfloat16* __restrict__ lo) {
  __shared__ float tile[4][64][33];
  const int Hp = H + 1, Wp = W + 1, Ho = 2 * H, Wo = 2 * W;
  const int img = Hp * Wp;
  const int p0 = blockIdx.x * 32;
  const int c0 = blockIdx.y * 64;
  const int b = blockIdx.z;
  const int t = threadIdx.x;
  float kf[16];
#pragma unroll
  for (int i = 0; i < 16; ++i) kf[i] = __ldg(k4 + 15 - i);
  {
    const int pl = t & 31;
    const int p = p0 + pl;
    const int m = p / Wp, n = p - m * Wp;
    const bool inimg = p < img;
    const int r0 = 2 * m - 2, q0 = 2 * n - 2;
#pragma unroll 1
    for (int i = 0; i < 8; ++i) {
      const int cl = (t >> 5) + 8 * i;
      float acc[4] = {0.f, 0.f, 0.f, 0.f};
      if (inimg) {
        const float* src = g + (static_cast<size_t>(b) * C + c0 + cl) * Ho * Wo;
        float win[5][5];
#pragma unroll
        for (int wr = 0; wr < 5; ++wr) {
          const int r = r0 + wr;
          const bool rok = (r >= 0) && (r < Ho);
#pragma unroll
          for (int wc = 0; wc < 5; ++wc) {
            const int q = q0 + wc;
            win[wr][wc] = (rok && q >= 0 && q < Wo) ? __ldg(src + static_cast<size_t>(r) * Wo + q) : 0.f;
          }
        }
#pragma unroll
        for (int pa = 0; pa < 2; ++pa)
#pragma unroll
          for (int pb = 0; pb < 2; ++pb)
#pragma unroll
            for (int wr = 0; wr < 5; ++wr)
#pragma unroll
              for (int wc = 0; wc < 5; ++wc) {
                const int a = pa + 3 - wr, bb = pb + 3 - wc;   // row r0+wr = (2m+pa) - a + 1
                if (a >= 0 && a < 4 && bb >= 0 && bb < 4)
                  acc[pa * 2 + pb] = fmaf(win[wr][wc], kf[a * 4 + bb], acc[pa * 2 + pb]);
              }
        const float s = scale ? __ldg(scale + static_cast<size_t>(b) * C + c0 + cl) : 1.f;
        // g_t has 2H+1 rows / 2W+1 columns: phase row 2m+1 with m == H (column 2n+1, n == W)
        // does not exist
        const bool row1 = m < H, col1 = n < W;
        acc[0] = s * acc[0];
        acc[1] = col1 ? s * acc[1] : 0.f;
        acc[2] = row1 ? s * acc[2] : 0.f;
        acc[3] = (row1 && col1) ? s * acc[3] : 0.f;
      }
#pragma unroll
      for (int ph = 0; ph < 4; ++ph) tile[ph][cl][pl] = acc[ph];
    }
  }
  __syncthreads();
  {
    const int pl = t >> 3;
    const int cg = (t & 7) * 8;
    const int p = p0 + pl;
    if (p < img) {
      const size_t row = static_cast<size_t>(b) * img + p;
#pragma unroll
      for (int ph = 0; ph < 4; ++ph) {
        __align__(16) __nv_bfloat16 h[8];
        __align__(16) __nv_bfloat16 l[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) split_bf16(tile[ph][cg + j][pl], h[j], l[j]);
        const size_t off = row * (4 * static_cast<size_t>(C)) + static_cast<size_t>(ph) * C + c0 + cg;
        *reinterpret_cast<uint4*>(hi + off) = *reinterpret_cast<const uint4*>(h);
        *reinterpret_cast<uint4*>(lo + off) = *reinterpret_cast<const uint4*>(l);
      }
    }
  }
}

// ---------------------------------------------------------------------------
// dgrad_finish: dk [B,Cin,H,W] is the gradient wrt the modulated key k = style*x
// (ApplyStyle, models.py:616-620).  One block per (b, i) plane:
//   gs_raw[b,i] = sum_p dk*x          (d/dstyle through the modulation)
//   dk         <- dk * style[b,i]     (= gradient wrt x, in place)
// ---------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
dgrad_finish_kernel(float* __restrict__ dk, const float* __restrict__ x,
                    const float* __restrict__ style, int HW, int vec, float* __restrict__ gs_raw) {
  __shared__ float red[32];
  const int bc = blockIdx.x;
  const size_t base = static_cast<size_t>(bc) * HW;
  const float s = __ldg(style + bc);
  float acc = 0.f;
  if (vec) {
    float4* d4 = reinterpret_cast<float4*>(dk + base);
    const float4* x4 = reinterpret_cast<const float4*>(x + base);
    const int nq = HW >> 2;
    for (int i = threadIdx.x; i < nq; i += blockDim.x) {
      float4 d = d4[i];
      const float4 xv = __ldg(x4 + i);
      acc = fmaf(d.x, xv.x, acc);
      acc = fmaf(d.y, xv.y, acc);
      acc = fmaf(d.z, xv.z, acc);
      acc = fmaf(d.w, xv.w, acc);
      d.x *= s; d.y *= s; d.z *= s; d.w *= s;
      d4[i] = d;
    }
  } else {
    for (int i = threadIdx.x; i < HW; i += blockDim.x) {
      const float d = dk[base + i];
      acc = fmaf(d, __ldg(x + base + i), acc);
      dk[base + i] = d * s;
    }
  }
  float v[1] = {acc};
  block_sum<1>(v, red);
  if (threadIdx.x == 0) gs_raw[bc] = v[0];
}

// ---------------------------------------------------------------------------
// wgrad_finish: the weight gradient in the Parameter's own layout, including the term through
// demod[b,o] = rsqrt(sum_i (s*W)^2 style^2 + eps)   (models.py:320-328):
//   gW[o,i,tap] = sc*dWt[o,tap,i] - sc^2 * W[o,i,tap] * sum_b (s_dot[b,o]*demod[b,o]^2) * style[b,i]^2
// one thread per (o, i).
// ---------------------------------------------------------------------------
__global__ void wgrad_finish_kernel(const float* __restrict__ dwt, const float* __restrict__ w,
                                    const float* __restrict__ s_dot, const float* __restrict__ dm,
                                    const float* __restrict__ style, int B, int Cout, int Cin,
                                    float sc, float* __restrict__ gw) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= Cout * Cin) return;
  const int o = idx / Cin, i = idx - o * Cin;
  float m = 0.f;
  if (s_dot) {
    for (int b = 0; b < B; ++b) {
      const float d = __ldg(dm + static_cast<size_t>(b) * Cout + o);
      const float s = __ldg(style + static_cast<size_t>(b) * Cin + i);
      m = fmaf(__ldg(s_dot + static_cast<size_t>(b) * Cout + o) * d * d, s * s, m);
    }
  }
  const float c2 = sc * sc * m;
  const float* src = dwt + static_cast<size_t>(o) * 9 * Cin + i;
  const float* wp = w + static_cast<size_t>(idx) * 9;
  float* dst = gw + static_cast<size_t>(idx) * 9;
#pragma unroll
  for (int tap = 0; tap < 9; ++tap)
    dst[tap] = sc * __ldg(src + static_cast<size_t>(tap) * Cin) - c2 * __ldg(wp + tap);
}

// ---------------------------------------------------------------------------
// style_grad_finish:  g_style[b,i] = gs_raw[b,i] - style[b,i] * sum_o (s_dot[b,o]*demod[b,o]^2) * wsq[o,i]
// (gs_raw may be null: pre-modulated input, only the demod term).  one thread per (b, i).
// ---------------------------------------------------------------------------
__global__ void style_grad_finish_kernel(const float* __restrict__ gs_raw,
                                         const float* __restrict__ style,
                                         const float* __restrict__ s_dot,
                                         const float* __restrict__ dm,
                                         const float* __restrict__ wsq, int B, int Cout, int Cin,
                                         float* __restrict__ g_style) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= B * Cin) return;
  const int b = idx / Cin, i = idx - b * Cin;
  float acc = 0.f;
  if (s_dot) {
    for (int o = 0; o < Cout; ++o) {
      const float d = __ldg(dm + static_cast<size_t>(b) * Cout + o);
      acc = fmaf(__ldg(s_dot + static_cast<size_t>(b) * Cout + o) * d * d,
                 __ldg(wsq + static_cast<size_t>(o) * Cin + i), acc);
    }
  }
  const float r = gs_raw ? gs_raw[idx] : 0.f;
  g_style[idx] = r - __ldg(style + idx) * acc;
}

inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

inline int plane_threads(int HW, int vec) {
  const int work = vec ? HW / 4 : HW;
  if (work <= 32) return 32;
  if (work <= 64) return 64;
  if (work <= 128) return 128;
  return 256;
}

}  // namespace

}  // namespace rw

using namespace rw;

extern "C" {

int rw_act_grad_reduce(const float* gy, const float* y, const float* noise,
                       long long noise_bstride, const float* noise_w, const float* bias, int act,
                       int B, int C, int HW, float* g_pre, float* s_sum, float* s_dot,
                       float* s_noise, rw_stream_t stream) {
  if (!gy || !y || !s_sum || !s_dot || !s_noise || B < 0 || C < 1 || HW < 0 ||
      (noise && !noise_w)) {
    set_last_error("rw_act_grad_reduce: bad argument");
    return RW_ERR_BAD_ARG;
  }
  const long long planes = static_cast<long long>(B) * C;
  if (planes <= 0 || HW <= 0) return RW_OK;
  if (planes > 0x7fffffffLL) {
    set_last_error("act_grad_reduce: B*C too large");
    return RW_ERR_BAD_ARG;
  }
  const int vec = ((HW & 3) == 0) && aligned16(gy) && aligned16(y) && (!g_pre || aligned16(g_pre)) &&
                  (!noise || (aligned16(noise) && (noise_bstride & 3) == 0));
  act_grad_reduce_kernel<<<static_cast<unsigned>(planes), plane_threads(HW, vec), 0, stream>>>(
      gy, y, noise, noise_bstride, noise_w, bias, act, C, HW, vec, g_pre, s_sum, s_dot, s_noise);
  return check_cuda(cudaGetLastError(), "act_grad_reduce launch");
}

int rw_blur_adj_phase_keys(const float* g_pre, const float* scale_bc, const float* k4, int B,
                           int C, int H, int W, void* hi, void* lo, rw_stream_t stream) {
  if (!g_pre || !k4 || !hi || !lo || B < 1 || H < 1 || W < 1) {
    set_last_error("rw_blur_adj_phase_keys: bad argument");
    return RW_ERR_BAD_ARG;
  }
  if (C % 64 != 0) {
    set_last_error("blur_adj_phase: C=%d must be a multiple of 64", C);
    return RW_ERR_BAD_ARG;
  }
  if (B > 65535) {
    set_last_error("blur_adj_phase: B=%d exceeds grid.z", B);
    return RW_ERR_BAD_ARG;
  }
  const int img = (H + 1) * (W + 1);
  dim3 grid((img + 31) / 32, C / 64, B);
  blur_adj_phase_kernel<<<grid, 256, 0, stream>>>(g_pre, scale_bc, k4, C, H, W,
                                                  static_cast<__nv_bfloat16*>(hi),
                                                  static_cast<__nv_bfloat16*>(lo));
  return check_cuda(cudaGetLastError(), "blur_adj_phase launch");
}

int rw_dgrad_finish(float* dk, const float* x, const float* style, int B, int C, int HW,
                    float* gs_raw, rw_stream_t stream) {
  if (!dk || !x || !style || !gs_raw || B < 0 || C < 1 || HW < 0) {
    set_last_error("rw_dgrad_finish: bad argument");
    return RW_ERR_BAD_ARG;
  }
  const long long planes = static_cast<long long>(B) * C;
  if (planes <= 0 || HW <= 0) return RW_OK;
  if (planes > 0x7fffffffLL) {
    set_last_error("dgrad_finish: B*C too large");
    return RW_ERR_BAD_ARG;
  }
  const int vec = ((HW & 3) == 0) && aligned16(dk) && aligned16(x);
  dgrad_finish_kernel<<<static_cast<unsigned>(planes), plane_threads(HW, vec), 0, stream>>>(
      dk, x, style, HW, vec, gs_raw);
  return check_cuda(cudaGetLastError(), "dgrad_finish launch");
}

int rw_wgrad_finish(const float* dwt, const float* w, const float* s_dot, const float* dm,
                    const float* style, int B, int Cout, int Cin, float sc, float* gw,
                    rw_stream_t stream) {
  if (!dwt || !w || !gw || Cout < 1 || Cin < 1 || (s_dot && (!dm || !style || B < 1))) {
    set_last_error("rw_wgrad_finish: bad argument");
    return RW_ERR_BAD_ARG;
  }
  const int n = Cout * Cin;
  wgrad_finish_kernel<<<(n + 127) / 128, 128, 0, stream>>>(dwt, w, s_dot, dm, style, B, Cout, Cin,
                                                           sc, gw);
  return check_cuda(cudaGetLastError(), "wgrad_finish launch");
}

int rw_style_grad_finish(const float* gs_raw, const float* style, const float* s_dot,
                         const float* dm, const float* wsq, int B, int Cout, int Cin,
                         float* g_style, rw_stream_t stream) {
  if (!style || !g_style || B < 1 || Cin < 1 || (s_dot && (!dm || !wsq || Cout < 1))) {
    set_last_error("rw_style_grad_finish: bad argument");
    return RW_ERR_BAD_ARG;
  }
  const int n = B * Cin;
  style_grad_finish_kernel<<<(n + 127) / 128, 128, 0, stream>>>(gs_raw, style, s_dot, dm, wsq, B,
                                                                Cout, Cin, g_style);
  return check_cuda(cudaGetLastError(), "style_grad_finish launch");
}

}  // extern "C"
