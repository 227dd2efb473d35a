// vgg.cu — the HBM-bound passes between the convolutions of a VGG feature stack (the perceptual
// network of all_weights_insert, reference ganrewrite.py:303-304): one read of a conv output a
// [B,C,H,W] fp32 applies the optional bias, ReLU and the optional 2x2 / stride-2 max pool (floor:
// an odd last row or column is dropped) and writes the next conv's bf16 hi/lo key planes (the
// padded-flat channels-last layout of prep_keys) and / or fp32 NCHW.  The backward re-derives every
// ReLU gate and pool argmax from the same a and bias with the same arithmetic, so the two passes
// cannot disagree, and follows torch's rules exactly:
//   relu        clamp_min(v, 0): a NaN passes through
//   max_pool2d  running max over the window in row-major order, replaced by a strictly greater
//               value or by a NaN (the first maximum wins ties, a NaN wins over numbers); the
//               gradient lands on that element as 0 + gy, every other element gets 0
//   threshold_backward  out <= 0 ? 0 : g   (so a NaN output passes its gradient)
#include "../../include/rewriting_b200.h"
#include "rw_common.cuh"

namespace rw {

namespace {

// relu(a[i] + bias) as torch forms it: the add rounds once, clamp_min keeps a NaN
__device__ __forceinline__ float relu_at(const float* __restrict__ ap, long long i, const float* bp) {
  float v = __ldg(ap + i);
  if (bp) v = __fadd_rn(v, __ldg(bp));
  return (v > 0.f || v != v) ? v : 0.f;
}

// the pooled window's value and its argmax k = dy * 2 + dx (torch's max_pool2d scan)
__device__ __forceinline__ float window_max(const float* __restrict__ ap, long long i0, int W,
                                            const float* bp, int& k) {
  float m = relu_at(ap, i0, bp);
  k = 0;
  const long long off[3] = {1, W, static_cast<long long>(W) + 1};
#pragma unroll
  for (int j = 0; j < 3; ++j) {
    const float v = relu_at(ap, i0 + off[j], bp);
    if (v > m || v != v) {
      m = v;
      k = j + 1;
    }
  }
  return m;
}

// forward value at output position (yo, xo) of one [H,W] plane
template <bool POOL>
__device__ __forceinline__ float fwd_value(const float* __restrict__ ap, const float* bp, int W, int yo,
                                           int xo) {
  if (!POOL) return relu_at(ap, static_cast<long long>(yo) * W + xo, bp);
  int k;
  return window_max(ap, static_cast<long long>(2 * yo) * W + 2 * xo, W, bp, k);
}

// gradient at input position (y, x) of one plane; gp is the plane of gy at output resolution
template <bool POOL>
__device__ __forceinline__ float bwd_value(const float* __restrict__ ap, const float* __restrict__ gp,
                                           const float* bp, int W, int Ho, int Wo, int y, int x) {
  const float r = relu_at(ap, static_cast<long long>(y) * W + x, bp);
  if (!POOL) return r <= 0.f ? 0.f : __ldg(gp + static_cast<long long>(y) * W + x);
  const int yo = y >> 1, xo = x >> 1;
  if (yo >= Ho || xo >= Wo) return 0.f;            // the dropped odd row / column
  int k;
  window_max(ap, static_cast<long long>(2 * yo) * W + 2 * xo, W, bp, k);
  if (k != ((y & 1) << 1) + (x & 1)) return 0.f;
  const float g = __fadd_rn(0.f, __ldg(gp + static_cast<long long>(yo) * Wo + xo));
  return r <= 0.f ? 0.f : g;
}

// value at position (y, x) of the result grid Hq x Wq (the output grid forward, the input grid
// backward) of plane (b, c)
template <bool BWD, bool POOL>
__device__ __forceinline__ float value_at(const float* __restrict__ a, const float* __restrict__ bias,
                                          const float* __restrict__ gy, long long plane, int c, int H,
                                          int W, int Ho, int Wo, int y, int x) {
  const float* ap = a + plane * H * W;
  const float* bp = bias ? bias + c : nullptr;
  if (BWD) return bwd_value<POOL>(ap, gy + plane * Ho * Wo, bp, W, Ho, Wo, y, x);
  return fwd_value<POOL>(ap, bp, W, y, x);
}

// Planes (and optional fp32 NCHW) of the Hq x Wq result: the smem transpose of prep_keys_kernel.
// grid: (ceil((Hq+1)*(Wq+1)/32), C/64, B), block 256
template <bool BWD, bool POOL>
__global__ void __launch_bounds__(256)
relu_pool_planes_kernel(const float* __restrict__ a, const float* __restrict__ bias,
                        const float* __restrict__ gy, int C, int H, int W, int Ho, int Wo, int Hq,
                        int Wq, __nv_bfloat16* __restrict__ hi, __nv_bfloat16* __restrict__ lo,
                        float* __restrict__ out) {
  __shared__ float tile[64][33];
  const int Hp = Hq + 1, Wp = Wq + 1;
  const int img = Hp * Wp;
  const int p0 = blockIdx.x * 32;
  const int c0 = blockIdx.y * 64;
  const int b = blockIdx.z;
  const int t = threadIdx.x;
  {
    const int pl = t & 31;
    const int p = p0 + pl;
    const int yy = p / Wp, xx = p - yy * Wp;
    const bool valid = (p < img) && (yy < Hq) && (xx < Wq);
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int c = c0 + (t >> 5) + 8 * i;
      float v = 0.f;
      if (valid) {
        const long long plane = static_cast<long long>(b) * C + c;
        v = value_at<BWD, POOL>(a, bias, gy, plane, c, H, W, Ho, Wo, yy, xx);
        if (out) out[(plane * Hq + yy) * Wq + xx] = v;
      }
      tile[c - c0][pl] = v;
    }
  }
  __syncthreads();
  {
    const int pl = t >> 3;
    const int cg = (t & 7) * 8;
    const int p = p0 + pl;
    if (p < img) {
      __align__(16) __nv_bfloat16 h[8];
      __align__(16) __nv_bfloat16 l[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) split_bf16(tile[cg + j][pl], h[j], l[j]);
      const size_t row = static_cast<size_t>(b) * img + p;
      *reinterpret_cast<uint4*>(hi + row * C + c0 + cg) = *reinterpret_cast<const uint4*>(h);
      *reinterpret_cast<uint4*>(lo + row * C + c0 + cg) = *reinterpret_cast<const uint4*>(l);
    }
  }
}

// fp32 NCHW only, any C: one thread per element of [B,C,Hq,Wq], grid-stride
template <bool BWD, bool POOL>
__global__ void __launch_bounds__(256)
relu_pool_nchw_kernel(const float* __restrict__ a, const float* __restrict__ bias,
                      const float* __restrict__ gy, int C, int H, int W, int Ho, int Wo, int Hq, int Wq,
                      long long n, float* __restrict__ out) {
  const long long hw = static_cast<long long>(Hq) * Wq;
  for (long long e = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; e < n;
       e += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long plane = e / hw;
    const long long r = e - plane * hw;
    const int y = static_cast<int>(r / Wq), x = static_cast<int>(r - static_cast<long long>(y) * Wq);
    out[e] = value_at<BWD, POOL>(a, bias, gy, plane, static_cast<int>(plane % C), H, W, Ho, Wo, y, x);
  }
}

template <bool BWD, bool POOL>
void launch(const float* a, const float* bias, const float* gy, int B, int C, int H, int W, int Ho,
            int Wo, void* hi, void* lo, float* out, cudaStream_t stream) {
  const int Hq = BWD ? H : Ho, Wq = BWD ? W : Wo;
  if (hi) {
    const int img = (Hq + 1) * (Wq + 1);
    dim3 grid((img + 31) / 32, C / 64, B);
    relu_pool_planes_kernel<BWD, POOL><<<grid, 256, 0, stream>>>(
        a, bias, gy, C, H, W, Ho, Wo, Hq, Wq, static_cast<__nv_bfloat16*>(hi),
        static_cast<__nv_bfloat16*>(lo), out);
  } else {
    const long long n = static_cast<long long>(B) * C * Hq * Wq;
    long long blocks = (n + 255) / 256;
    if (blocks > 132 * 32) blocks = 132 * 32;
    relu_pool_nchw_kernel<BWD, POOL><<<static_cast<unsigned>(blocks), 256, 0, stream>>>(
        a, bias, gy, C, H, W, Ho, Wo, Hq, Wq, n, out);
  }
}

inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

}  // namespace

// the forward (gy == null) and the backward of rw_relu_pool
static int relu_pool_launch(const float* a, const float* bias, const float* gy, int B, int C, int H,
                            int W, int pool, void* hi, void* lo, float* out, cudaStream_t stream) {
  const char* what = gy ? "relu_pool_bwd" : "relu_pool";
  if (B < 1 || C < 1 || H < 1 || W < 1 || B > 65535 ||
      static_cast<long long>(B) * C * (H + 1) * (W + 1) >= (1LL << 40)) {
    set_last_error("%s: bad shape B=%d C=%d H=%d W=%d", what, B, C, H, W);
    return RW_ERR_BAD_ARG;
  }
  if (pool && (H < 2 || W < 2)) {
    set_last_error("%s: a 2x2 pool needs H, W >= 2 (H=%d W=%d)", what, H, W);
    return RW_ERR_BAD_ARG;
  }
  if ((hi == nullptr) != (lo == nullptr) || (!hi && !out)) {
    set_last_error("%s: give both planes (hi and lo), an fp32 output, or both", what);
    return RW_ERR_BAD_ARG;
  }
  if (hi && (C % 64 != 0 || C / 64 > 65535 || !aligned16(hi) || !aligned16(lo))) {
    set_last_error("%s: planes need C %% 64 == 0 (C=%d) and 16-byte aligned hi / lo", what, C);
    return RW_ERR_BAD_ARG;
  }
  const int Ho = pool ? H / 2 : H, Wo = pool ? W / 2 : W;
  const bool bwd = gy != nullptr;
  if (bwd && pool) launch<true, true>(a, bias, gy, B, C, H, W, Ho, Wo, hi, lo, out, stream);
  else if (bwd) launch<true, false>(a, bias, gy, B, C, H, W, Ho, Wo, hi, lo, out, stream);
  else if (pool) launch<false, true>(a, bias, gy, B, C, H, W, Ho, Wo, hi, lo, out, stream);
  else launch<false, false>(a, bias, gy, B, C, H, W, Ho, Wo, hi, lo, out, stream);
  return check_cuda(cudaGetLastError(), what);
}

}  // namespace rw

using namespace rw;

extern "C" {

int rw_relu_pool(const float* a, const float* bias, int B, int C, int H, int W, int pool,
                 void* out_hi, void* out_lo, float* out, rw_stream_t stream) {
  if (!a) {
    set_last_error("rw_relu_pool: bad argument");
    return RW_ERR_BAD_ARG;
  }
  return relu_pool_launch(a, bias, nullptr, B, C, H, W, pool, out_hi, out_lo, out, stream);
}

int rw_relu_pool_bwd(const float* a, const float* bias, const float* gy, int B, int C, int H, int W,
                     int pool, void* g_hi, void* g_lo, float* g, rw_stream_t stream) {
  if (!a || !gy) {
    set_last_error("rw_relu_pool_bwd: bad argument");
    return RW_ERR_BAD_ARG;
  }
  return relu_pool_launch(a, bias, gy, B, C, H, W, pool, g_hi, g_lo, g, stream);
}

}  // extern "C"
