// gen_bwd.cu — backward of the StyleGAN2 generator's modulated 1x1 ToRGB conv under autograd (its
// forward is torgb_kernel of simt.cu).  fp32 on CUDA cores; every output is summed in a fixed order
// with no atomics, so two calls on the same input give the same bits.
#include "../../include/rewriting_b200.h"
#include "rw_common.cuh"

namespace rw {

namespace {

// ---------------------------------------------------------------------------
// Modulated ToRGB backward (Cout = 3), y[b,o,p] = sum_i scale W[o,i] s[b,i] x[b,i,p]:
//   gx[b,i,p] = scale s[b,i] sum_o W[o,i] gy[b,o,p]
//   R[b,o,i]  = sum_p gy[b,o,p] x[b,i,p]
//   gW[o,i]   = scale sum_b s[b,i] R[b,o,i]        gs[b,i] = scale sum_o W[o,i] R[b,o,i]
// Pass 1 (torgb_mod_bwd_kernel) is the one pass over x and gx: CTA (chunk, channel group, b)
// takes kRgbPix pixels of sample b and 32 channels; each thread keeps the gy of its 8 pixels in
// registers, writes gx for them and reduces its share of R over the chunk (warp shuffles, then the
// 8 warps in order) into part[b][chunk][o][i].  Pass 2 (torgb_mod_bwd_finish_kernel) sums the
// chunks of one sample in a fixed order (8 strided subsets, then the subsets in order), giving
// R, gs and t[b,o,i] = s[b,i] R[b,o,i]; pass 3 (torgb_mod_wsum_kernel) sums t over b in order.
// DRAM traffic per pixel: x and gx (4 C bytes each) and gy (12 bytes).
// ---------------------------------------------------------------------------
constexpr int kRgbPix = 2048;        // pixels per chunk: 256 threads x 8
constexpr int kRgbGroup = 32;        // channels per CTA

template <bool VEC>
__device__ __forceinline__ int rgb_pixel(int p0, int t) {
  // pixel of the thread's t-th value: 2 float4 groups (VEC) or 8 single pixels 256 apart
  return VEC ? p0 + ((t >> 2) * 256 + static_cast<int>(threadIdx.x)) * 4 + (t & 3)
             : p0 + t * 256 + static_cast<int>(threadIdx.x);
}

template <bool VEC>
__global__ void __launch_bounds__(256)
torgb_mod_bwd_kernel(const float* __restrict__ x, const float* __restrict__ style,
                     const float* __restrict__ w, const float* __restrict__ gy, int C, int HW,
                     float scale, int chunks, float* __restrict__ gx, float* __restrict__ part) {
  __shared__ float red[8][3][kRgbGroup];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int chunk = blockIdx.x, c0 = blockIdx.y * kRgbGroup, b = blockIdx.z;
  const int p0 = chunk * kRgbPix;
  const float* gyb = gy + static_cast<size_t>(b) * 3 * HW;
  float g[3][8];
  if (VEC) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int p = rgb_pixel<true>(p0, 4 * h);
#pragma unroll
      for (int o = 0; o < 3; ++o) {
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (p < HW) v = __ldg(reinterpret_cast<const float4*>(gyb + static_cast<size_t>(o) * HW + p));
        g[o][4 * h] = v.x; g[o][4 * h + 1] = v.y; g[o][4 * h + 2] = v.z; g[o][4 * h + 3] = v.w;
      }
    }
  } else {
#pragma unroll
    for (int t = 0; t < 8; ++t) {
      const int p = rgb_pixel<false>(p0, t);
#pragma unroll
      for (int o = 0; o < 3; ++o)
        g[o][t] = p < HW ? __ldg(gyb + static_cast<size_t>(o) * HW + p) : 0.f;
    }
  }
  const int cn = min(kRgbGroup, C - c0);
  for (int ci = 0; ci < cn; ++ci) {
    const int c = c0 + ci;
    const float w0 = __ldg(w + c), w1 = __ldg(w + C + c), w2 = __ldg(w + 2 * C + c);
    const float sc = scale * __ldg(style + static_cast<size_t>(b) * C + c);
    const size_t plane = (static_cast<size_t>(b) * C + c) * HW;
    float xv[8];
    if (VEC) {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int p = rgb_pixel<true>(p0, 4 * h);
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (p < HW) v = __ldg(reinterpret_cast<const float4*>(x + plane + p));
        xv[4 * h] = v.x; xv[4 * h + 1] = v.y; xv[4 * h + 2] = v.z; xv[4 * h + 3] = v.w;
      }
    } else {
#pragma unroll
      for (int t = 0; t < 8; ++t) {
        const int p = rgb_pixel<false>(p0, t);
        xv[t] = p < HW ? __ldg(x + plane + p) : 0.f;
      }
    }
    if (gx) {
      float gv[8];
#pragma unroll
      for (int t = 0; t < 8; ++t) gv[t] = sc * fmaf(w2, g[2][t], fmaf(w1, g[1][t], w0 * g[0][t]));
      if (VEC) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int p = rgb_pixel<true>(p0, 4 * h);
          if (p < HW)
            *reinterpret_cast<float4*>(gx + plane + p) =
                make_float4(gv[4 * h], gv[4 * h + 1], gv[4 * h + 2], gv[4 * h + 3]);
        }
      } else {
#pragma unroll
        for (int t = 0; t < 8; ++t) {
          const int p = rgb_pixel<false>(p0, t);
          if (p < HW) gx[plane + p] = gv[t];
        }
      }
    }
    float r[3];
#pragma unroll
    for (int o = 0; o < 3; ++o) {
      float a = 0.f;
#pragma unroll
      for (int t = 0; t < 8; ++t) a = fmaf(g[o][t], xv[t], a);
#pragma unroll
      for (int d = 16; d > 0; d >>= 1) a += __shfl_xor_sync(0xffffffffu, a, d);
      r[o] = a;
    }
    if (lane == 0) {
#pragma unroll
      for (int o = 0; o < 3; ++o) red[warp][o][ci] = r[o];
    }
  }
  __syncthreads();
  if (threadIdx.x < 3 * kRgbGroup) {
    const int o = threadIdx.x / kRgbGroup, ci = threadIdx.x % kRgbGroup;
    if (ci < cn) {
      float v = 0.f;
#pragma unroll
      for (int s = 0; s < 8; ++s) v += red[s][o][ci];
      part[((static_cast<size_t>(b) * chunks + chunk) * 3 + o) * C + c0 + ci] = v;
    }
  }
}

// CTA (channel group, b): lane = channel, warp = every 8th chunk
__global__ void __launch_bounds__(256)
torgb_mod_bwd_finish_kernel(const float* __restrict__ part, const float* __restrict__ style,
                            const float* __restrict__ w, int C, int chunks, float scale,
                            float* __restrict__ gs, float* __restrict__ t_out) {
  __shared__ float red[8][3][kRgbGroup];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int c = blockIdx.x * kRgbGroup + lane, b = blockIdx.y;
  float r[3] = {0.f, 0.f, 0.f};
  if (c < C) {
    for (int s = warp; s < chunks; s += 8) {
      const float* q = part + (static_cast<size_t>(b) * chunks + s) * 3 * C + c;
#pragma unroll
      for (int o = 0; o < 3; ++o) r[o] += __ldg(q + static_cast<size_t>(o) * C);
    }
  }
#pragma unroll
  for (int o = 0; o < 3; ++o) red[warp][o][lane] = r[o];
  __syncthreads();
  if (warp != 0 || c >= C) return;
  float R[3];
#pragma unroll
  for (int o = 0; o < 3; ++o) {
    float v = 0.f;
#pragma unroll
    for (int s = 0; s < 8; ++s) v += red[s][o][lane];
    R[o] = v;
  }
  if (gs)
    gs[static_cast<size_t>(b) * C + c] =
        scale * fmaf(__ldg(w + 2 * C + c), R[2], fmaf(__ldg(w + C + c), R[1], __ldg(w + c) * R[0]));
  const float sv = __ldg(style + static_cast<size_t>(b) * C + c);
#pragma unroll
  for (int o = 0; o < 3; ++o) t_out[(static_cast<size_t>(b) * 3 + o) * C + c] = sv * R[o];
}

// gW[o,i] = scale * sum_b t[b,o,i], b in order
__global__ void __launch_bounds__(256)
torgb_mod_wsum_kernel(const float* __restrict__ t, int B, int n, float scale, float* __restrict__ gw) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= n || !gw) return;
  float v = 0.f;
  for (int b = 0; b < B; ++b) v += __ldg(t + static_cast<size_t>(b) * n + e);
  gw[e] = v * scale;
}

inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

bool torgb_mod_shape_ok(int B, int C, int H, int W) {
  return B >= 1 && B <= 65535 && C >= 1 && C <= 65535 * kRgbGroup && H >= 1 && W >= 1 &&
         static_cast<long long>(H) * W <= 2147483647LL - kRgbPix;
}

int torgb_mod_chunks(int H, int W) {
  return static_cast<int>((static_cast<long long>(H) * W + kRgbPix - 1) / kRgbPix);
}

}  // namespace

}  // namespace rw

using namespace rw;

extern "C" {

size_t rw_torgb_mod_bwd_workspace_bytes(int B, int C, int H, int W) {
  if (!torgb_mod_shape_ok(B, C, H, W)) return 0;
  // part [B][chunks][3][C], then t [B][3][C]
  return (static_cast<size_t>(B) * (torgb_mod_chunks(H, W) + 1) * 3 * C) * sizeof(float);
}

int rw_torgb_mod_bwd(const float* x, const float* style, const float* w, const float* gy, int B,
                     int C, int H, int W, float scale, float* gx, float* gs, float* gw,
                     void* workspace, size_t workspace_bytes, rw_stream_t stream) {
  if (!x || !style || !w || !gy || !workspace || (!gx && !gs && !gw)) {
    set_last_error("rw_torgb_mod_bwd: bad argument");
    return RW_ERR_BAD_ARG;
  }
  const size_t need = rw_torgb_mod_bwd_workspace_bytes(B, C, H, W);
  if (need == 0 || workspace_bytes < need) {
    set_last_error("torgb_mod_bwd: bad shape or workspace %zu < %zu bytes (B=%d C=%d H=%d W=%d)",
                   workspace_bytes, need, B, C, H, W);
    return RW_ERR_BAD_ARG;
  }
  const int HW = H * W, chunks = torgb_mod_chunks(H, W);
  const int groups = (C + kRgbGroup - 1) / kRgbGroup;
  float* part = static_cast<float*>(workspace);
  float* t = part + static_cast<size_t>(B) * chunks * 3 * C;
  const bool vec = HW % 4 == 0 && aligned16(x) && aligned16(gy) && (!gx || aligned16(gx));
  dim3 grid(chunks, groups, B);
  if (vec)
    torgb_mod_bwd_kernel<true><<<grid, 256, 0, stream>>>(x, style, w, gy, C, HW, scale, chunks, gx,
                                                         part);
  else
    torgb_mod_bwd_kernel<false><<<grid, 256, 0, stream>>>(x, style, w, gy, C, HW, scale, chunks, gx,
                                                          part);
  int rc = check_cuda(cudaGetLastError(), "torgb_mod_bwd launch");
  if (rc) return rc;
  torgb_mod_bwd_finish_kernel<<<dim3(groups, B), 256, 0, stream>>>(part, style, w, C, chunks, scale,
                                                                   gs, t);
  rc = check_cuda(cudaGetLastError(), "torgb_mod_bwd finish launch");
  if (rc) return rc;
  const int n = 3 * C;
  torgb_mod_wsum_kernel<<<(n + 255) / 256, 256, 0, stream>>>(t, B, n, scale, gw);
  return check_cuda(cudaGetLastError(), "torgb_mod_wsum launch");
}

}  // extern "C"
