// lpips.cu — the edit distances of the paper's §5.1 (reference metrics/distances.py): spatial LPIPS
// v0.1 ("net-lin" on VGG-16) and the masked L1, around the package's VGG stack (perceptual.py).
// Three HBM-bound passes, each summing in a fixed order with no atomics:
//   input    both image sets (fp32 NCHW in [-1, 1], or uint8 NHWC decoded as x/255*2-1 the way
//            ToTensor + Normalize(0.5, 0.5) does) through LPIPS's scaling layer (x - shift) / scale,
//            into the one [2B,3,H,W] batch conv1_1 reads; every step rounds as torch's does
//   head     one read of a tap's pre-activation conv output a [2B,C,h,w] (first half im0, second
//            half im1): f = relu(a [+ bias]), and per pixel in float64 the five channel sums
//            S00 = sum f0^2, S11 = sum f1^2, P00 = sum w f0^2, P01 = sum w f0 f1, P11 = sum w f1^2,
//            so that with N = sqrt(S) + 1e-10
//              d = sum_c w (f0/N0 - f1/N1)^2 = P00/N0^2 - 2 P01/(N0 N1) + P11/N1^2
//            without a normalised copy of the features (float64 keeps the cancellation of the
//            expanded square far below the conv's own error)
//   combine  D = sum_l bilinear_up(d_l) (torch's align_corners=False with the output size given,
//            taps summed in order), written if asked for; or the masked L1 sum_c |im1 - im0| read
//            from the image sets directly; either way the per-image sums of D*w and w over
//            1024-pixel tiles into a workspace, then a fixed-order finish per image.
#include "../../include/rewriting_b200.h"
#include "rw_common.cuh"

namespace rw {

namespace {

constexpr int kMaxMaps = 8;
constexpr int kTile = 1024;          // pixels per combine block (256 threads x 4)

// torch.Tensor([-.030, -.088, -.188]) / ([.458, .448, .450]): the doubles rounded to float once
__constant__ float kShift[3] = {static_cast<float>(-.030), static_cast<float>(-.088),
                                static_cast<float>(-.188)};
__constant__ float kScale[3] = {static_cast<float>(.458), static_cast<float>(.448),
                                static_cast<float>(.450)};

// image value in [-1, 1] of channel c at pixel p of image b: fp32 NCHW, or uint8 NHWC as
// ToTensor (u / 255, a true division) then Normalize(0.5, 0.5) ((x - 0.5) / 0.5)
template <bool U8>
__device__ __forceinline__ float pixel_value(const void* im, int b, int c, long long p, long long hw) {
  if (U8) {
    const unsigned char u = static_cast<const unsigned char*>(im)[(static_cast<long long>(b) * hw + p) * 3 + c];
    const float x = __fdiv_rn(static_cast<float>(u), 255.f);
    return __fdiv_rn(__fsub_rn(x, 0.5f), 0.5f);
  }
  return __ldg(static_cast<const float*>(im) + (static_cast<long long>(b) * 3 + c) * hw + p);
}

// out [2B,3,H,W]: images 0..B-1 from im0, B..2B-1 from im1; one thread per pixel, grid-stride
template <bool U8>
__global__ void __launch_bounds__(256)
lpips_input_kernel(const void* __restrict__ im0, const void* __restrict__ im1, int B, long long hw,
                   float* __restrict__ out) {
  const long long n = 2LL * B * hw;
  for (long long e = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; e < n;
       e += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int img = static_cast<int>(e / hw);
    const long long p = e - static_cast<long long>(img) * hw;
    const bool second = img >= B;
    const int b = second ? img - B : img;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const float x = pixel_value<U8>(second ? im1 : im0, b, c, p, hw);
      out[(static_cast<long long>(img) * 3 + c) * hw + p] = __fdiv_rn(__fsub_rn(x, kShift[c]), kScale[c]);
    }
  }
}

__device__ __forceinline__ float relu_of(float v, const float* bp) {
  if (bp) v = __fadd_rn(v, __ldg(bp));
  return (v > 0.f || v != v) ? v : 0.f;
}

// d [B,h,w] from a [2B,C,h,w].  block 256 = 32 pixels x 8 channel slices; slice s takes channels
// s, s+8, s+16, ... in order, then warp 0 adds the eight slices in order.
// grid: (ceil(h*w / 32), B)
__global__ void __launch_bounds__(256)
lpips_head_kernel(const float* __restrict__ a, const float* __restrict__ bias,
                  const float* __restrict__ lin_w, int B, int C, long long hw, float* __restrict__ d) {
  __shared__ double part[5][8][33];
  const int lane = threadIdx.x & 31, s = threadIdx.x >> 5;
  const long long p = static_cast<long long>(blockIdx.x) * 32 + lane;
  const int b = blockIdx.y;
  double s00 = 0, s11 = 0, p00 = 0, p01 = 0, p11 = 0;
  if (p < hw) {
    const float* a0 = a + static_cast<long long>(b) * C * hw + p;
    const float* a1 = a + static_cast<long long>(b + B) * C * hw + p;
#pragma unroll 4
    for (int c = s; c < C; c += 8) {
      const float* bp = bias ? bias + c : nullptr;
      const double f0 = relu_of(__ldg(a0 + c * hw), bp);
      const double f1 = relu_of(__ldg(a1 + c * hw), bp);
      const double w = __ldg(lin_w + c);
      const double wf0 = w * f0, wf1 = w * f1;
      s00 = fma(f0, f0, s00);
      s11 = fma(f1, f1, s11);
      p00 = fma(wf0, f0, p00);
      p01 = fma(wf0, f1, p01);
      p11 = fma(wf1, f1, p11);
    }
  }
  part[0][s][lane] = s00;
  part[1][s][lane] = s11;
  part[2][s][lane] = p00;
  part[3][s][lane] = p01;
  part[4][s][lane] = p11;
  __syncthreads();
  if (s != 0 || p >= hw) return;
  double t[5];
#pragma unroll
  for (int k = 0; k < 5; ++k) {
    t[k] = part[k][0][lane];
#pragma unroll
    for (int j = 1; j < 8; ++j) t[k] += part[k][j][lane];
  }
  const double n0 = sqrt(t[0]) + 1e-10, n1 = sqrt(t[1]) + 1e-10;
  const double v = t[2] / (n0 * n0) - 2.0 * t[3] / (n0 * n1) + t[4] / (n1 * n1);
  d[static_cast<long long>(b) * hw + p] = static_cast<float>(v);
}

struct CombineParams {
  const float* maps[kMaxMaps];
  int mh[kMaxMaps], mw[kMaxMaps];
  int nmaps;
  const void* im0;
  const void* im1;
  int B, H, W;
  const float* mask;     // [mask_b,1,H,W] or null (weight 1)
  int mask_b;
  float* D;              // [B,1,H,W] or null
  double* part;          // [B][ntiles][2] or null
  int ntiles;
};

// torch's upsample_bilinear2d source coordinate (align_corners=False, output size given), in
// float64: index i0, neighbour step (0 at the last row / column) and weight of the second tap
__device__ __forceinline__ void bilinear_src(int o, int in, int out, int& i0, int& step, double& l1) {
  double src = (o + 0.5) * (static_cast<double>(in) / out) - 0.5;
  if (src < 0) src = 0;
  i0 = static_cast<int>(src);
  step = i0 < in - 1 ? 1 : 0;
  l1 = src - i0;
}

template <bool L1, bool U8>
__device__ __forceinline__ double pixel_distance(const CombineParams& P, int b, int y, int x) {
  const long long hw = static_cast<long long>(P.H) * P.W;
  const long long p = static_cast<long long>(y) * P.W + x;
  if (L1) {
    float s = 0.f;
#pragma unroll
    for (int c = 0; c < 3; ++c)
      s = __fadd_rn(s, fabsf(__fsub_rn(pixel_value<U8>(P.im1, b, c, p, hw), pixel_value<U8>(P.im0, b, c, p, hw))));
    return s;
  }
  double D = 0;
  for (int l = 0; l < P.nmaps; ++l) {
    const int h = P.mh[l], w = P.mw[l];
    int y0, sy, x0, sx;
    double ly, lx;
    bilinear_src(y, h, P.H, y0, sy, ly);
    bilinear_src(x, w, P.W, x0, sx, lx);
    const float* m = P.maps[l] + static_cast<long long>(b) * h * w;
    const float* r0 = m + static_cast<long long>(y0) * w + x0;
    const float* r1 = r0 + static_cast<long long>(sy) * w;
    const double v = (1.0 - ly) * ((1.0 - lx) * __ldg(r0) + lx * __ldg(r0 + sx)) +
                     ly * ((1.0 - lx) * __ldg(r1) + lx * __ldg(r1 + sx));
    D += v;
  }
  return D;
}

// grid: (ntiles, B), block 256; thread t takes pixels tile*1024 + t + 256 i, i = 0..3 in order,
// then a fixed tree over the block
template <bool L1, bool U8>
__global__ void __launch_bounds__(256) lpips_combine_kernel(const CombineParams P) {
  __shared__ double red[2][256];
  const int b = blockIdx.y;
  const long long hw = static_cast<long long>(P.H) * P.W;
  const float* mk = P.mask ? P.mask + (P.mask_b == 1 ? 0 : static_cast<long long>(b) * hw) : nullptr;
  double num = 0, den = 0;
#pragma unroll
  for (int i = 0; i < kTile / 256; ++i) {
    const long long p = static_cast<long long>(blockIdx.x) * kTile + i * 256 + threadIdx.x;
    if (p >= hw) break;
    const int y = static_cast<int>(p / P.W), x = static_cast<int>(p - static_cast<long long>(y) * P.W);
    const double D = pixel_distance<L1, U8>(P, b, y, x);
    if (P.D) P.D[static_cast<long long>(b) * hw + p] = static_cast<float>(D);
    const double w = mk ? static_cast<double>(__ldg(mk + p)) : 1.0;
    num += D * w;
    den += w;
  }
  if (!P.part) return;
  red[0][threadIdx.x] = num;
  red[1][threadIdx.x] = den;
  __syncthreads();
  for (int k = 128; k > 0; k >>= 1) {
    if (threadIdx.x < k) {
      red[0][threadIdx.x] += red[0][threadIdx.x + k];
      red[1][threadIdx.x] += red[1][threadIdx.x + k];
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    double* o = P.part + (static_cast<long long>(b) * P.ntiles + blockIdx.x) * 2;
    o[0] = red[0][0];
    o[1] = red[1][0];
  }
}

// num[b], den[b] = the sums of image b's tile partials: thread t takes tiles t, t+256, ... in
// order, then a fixed tree.  grid: B, block 256
__global__ void __launch_bounds__(256)
lpips_finish_kernel(const double* __restrict__ part, int ntiles, double* __restrict__ num,
                    double* __restrict__ den) {
  __shared__ double red[2][256];
  const double* pb = part + static_cast<long long>(blockIdx.x) * ntiles * 2;
  double n = 0, d = 0;
  for (int t = threadIdx.x; t < ntiles; t += 256) {
    n += pb[2 * t];
    d += pb[2 * t + 1];
  }
  red[0][threadIdx.x] = n;
  red[1][threadIdx.x] = d;
  __syncthreads();
  for (int k = 128; k > 0; k >>= 1) {
    if (threadIdx.x < k) {
      red[0][threadIdx.x] += red[0][threadIdx.x + k];
      red[1][threadIdx.x] += red[1][threadIdx.x + k];
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    num[blockIdx.x] = red[0][0];
    den[blockIdx.x] = red[1][0];
  }
}

bool bad_image_shape(int B, int H, int W) {
  return B < 1 || H < 1 || W < 1 || B > 65535 || static_cast<long long>(H) * W > (1LL << 31) ||
         2LL * B * H * W * 3 >= (1LL << 40);
}

int combine_run(CombineParams& P, bool l1, bool u8, double* num, double* den, void* workspace,
                size_t workspace_bytes, cudaStream_t stream, const char* what) {
  if (bad_image_shape(P.B, P.H, P.W)) {
    set_last_error("%s: bad shape B=%d H=%d W=%d", what, P.B, P.H, P.W);
    return RW_ERR_BAD_ARG;
  }
  if ((num == nullptr) != (den == nullptr) || (!num && !P.D)) {
    set_last_error("%s: give both num and den, the map D, or all three", what);
    return RW_ERR_BAD_ARG;
  }
  if (P.mask && P.mask_b != 1 && P.mask_b != P.B) {
    set_last_error("%s: the mask batch must be 1 or B (mask_b=%d B=%d)", what, P.mask_b, P.B);
    return RW_ERR_BAD_ARG;
  }
  const long long hw = static_cast<long long>(P.H) * P.W;
  P.ntiles = static_cast<int>((hw + kTile - 1) / kTile);
  P.part = nullptr;
  if (num) {
    const size_t need = rw_lpips_combine_workspace_bytes(P.B, P.H, P.W);
    if (!workspace || workspace_bytes < need || (reinterpret_cast<uintptr_t>(workspace) & 7u)) {
      set_last_error("%s: workspace %zu < %zu bytes or not 8-byte aligned", what, workspace_bytes, need);
      return RW_ERR_BAD_ARG;
    }
    P.part = static_cast<double*>(workspace);
  }
  const dim3 grid(P.ntiles, P.B);
  if (!l1) lpips_combine_kernel<false, false><<<grid, 256, 0, stream>>>(P);
  else if (u8) lpips_combine_kernel<true, true><<<grid, 256, 0, stream>>>(P);
  else lpips_combine_kernel<true, false><<<grid, 256, 0, stream>>>(P);
  if (num) lpips_finish_kernel<<<P.B, 256, 0, stream>>>(P.part, P.ntiles, num, den);
  return check_cuda(cudaGetLastError(), what);
}

}  // namespace

}  // namespace rw

using namespace rw;

extern "C" {

int rw_lpips_input(const void* im0, const void* im1, int u8, int B, int H, int W, float* out,
                   rw_stream_t stream) {
  if (!im0 || !im1 || !out) {
    set_last_error("rw_lpips_input: bad argument");
    return RW_ERR_BAD_ARG;
  }
  if (bad_image_shape(B, H, W) || (u8 != 0 && u8 != 1)) {
    set_last_error("lpips_input: bad shape or format B=%d H=%d W=%d u8=%d", B, H, W, u8);
    return RW_ERR_BAD_ARG;
  }
  const long long hw = static_cast<long long>(H) * W;
  long long blocks = (2LL * B * hw + 255) / 256;
  if (blocks > 132 * 32) blocks = 132 * 32;
  if (u8) lpips_input_kernel<true><<<static_cast<unsigned>(blocks), 256, 0, stream>>>(im0, im1, B, hw, out);
  else lpips_input_kernel<false><<<static_cast<unsigned>(blocks), 256, 0, stream>>>(im0, im1, B, hw, out);
  return check_cuda(cudaGetLastError(), "lpips_input");
}

int rw_lpips_head(const float* a, const float* bias, const float* lin_w, int B, int C, int h, int w,
                  float* d, rw_stream_t stream) {
  if (!a || !lin_w || !d) {
    set_last_error("rw_lpips_head: bad argument");
    return RW_ERR_BAD_ARG;
  }
  const long long hw = static_cast<long long>(h) * w;
  if (B < 1 || C < 1 || h < 1 || w < 1 || B > 65535 || (hw + 31) / 32 > 0x7fffffffLL ||
      C * hw >= (1LL << 40)) {
    set_last_error("lpips_head: bad shape B=%d C=%d h=%d w=%d", B, C, h, w);
    return RW_ERR_BAD_ARG;
  }
  const dim3 grid(static_cast<unsigned>((hw + 31) / 32), B);
  lpips_head_kernel<<<grid, 256, 0, stream>>>(a, bias, lin_w, B, C, hw, d);
  return check_cuda(cudaGetLastError(), "lpips_head");
}

size_t rw_lpips_combine_workspace_bytes(int B, int H, int W) {
  if (bad_image_shape(B, H, W)) return 0;
  const long long ntiles = (static_cast<long long>(H) * W + kTile - 1) / kTile;
  return static_cast<size_t>(B) * ntiles * 2 * sizeof(double);
}

int rw_lpips_combine(int nmaps, const float* const* maps, const int* map_hw, int B, int H, int W,
                     const float* mask, int mask_b, float* D, double* num, double* den,
                     void* workspace, size_t workspace_bytes, rw_stream_t stream) {
  if (!maps || !map_hw) {
    set_last_error("rw_lpips_combine: bad argument");
    return RW_ERR_BAD_ARG;
  }
  if (nmaps < 1 || nmaps > kMaxMaps) {
    set_last_error("lpips_combine: nmaps=%d outside 1..%d", nmaps, kMaxMaps);
    return RW_ERR_BAD_ARG;
  }
  CombineParams P = {};
  for (int l = 0; l < nmaps; ++l) {
    if (!maps[l] || map_hw[2 * l] < 1 || map_hw[2 * l + 1] < 1) {
      set_last_error("lpips_combine: map %d is null or has a size < 1", l);
      return RW_ERR_BAD_ARG;
    }
    P.maps[l] = maps[l];
    P.mh[l] = map_hw[2 * l];
    P.mw[l] = map_hw[2 * l + 1];
  }
  P.nmaps = nmaps;
  P.B = B; P.H = H; P.W = W;
  P.mask = mask; P.mask_b = mask_b; P.D = D;
  return combine_run(P, false, false, num, den, workspace, workspace_bytes, stream, "lpips_combine");
}

int rw_masked_l1(const void* im0, const void* im1, int u8, int B, int H, int W, const float* mask,
                 int mask_b, double* num, double* den, void* workspace, size_t workspace_bytes,
                 rw_stream_t stream) {
  if (!im0 || !im1) {
    set_last_error("rw_masked_l1: bad argument");
    return RW_ERR_BAD_ARG;
  }
  if ((u8 != 0 && u8 != 1) || !num) {
    set_last_error("masked_l1: u8 must be 0 or 1 and num, den given (u8=%d)", u8);
    return RW_ERR_BAD_ARG;
  }
  CombineParams P = {};
  P.im0 = im0; P.im1 = im1;
  P.B = B; P.H = H; P.W = W;
  P.mask = mask; P.mask_b = mask_b;
  return combine_run(P, true, u8 != 0, num, den, workspace, workspace_bytes, stream, "masked_l1");
}

}  // extern "C"
