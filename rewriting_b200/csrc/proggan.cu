// proggan.cu — fp32 CUDA-core kernels for the ProgGAN layers the tensor-core row-GEMM does not
// take (reference utils/proggan.py:143-199): the 4x4 "dense" input layer, 3x3 convolutions with a
// channel count that is not a multiple of 64 (the 64 -> 32 -> 16 channel tails of the 512² and
// 1024² generators) and the 1x1 ToRGB.  Every kernel reads and writes fp32 NCHW, sums in a fixed
// order (two calls on the same input are bit-identical), and takes no tensor-core path: these
// layers are narrow, so their cost is memory and the shared-memory operand reuse below.
#include "rw_common.cuh"
#include "rw_kernels.h"

namespace rw {

namespace {

// nn.LeakyReLU(0.2): x > 0 ? x : x * 0.2 (torch's leaky_relu kernel)
__device__ __forceinline__ float lrelu02(float v) { return v > 0.f ? v : v * 0.2f; }

// WScaleLayer then LeakyReLU with torch's two roundings (x * scale, then + b): the fused epilogue
// gives what the leaf path gives from the same conv output
__device__ __forceinline__ float wscale_lrelu(float acc, float wscale, float b) {
  return lrelu02(__fadd_rn(__fmul_rn(acc, wscale), b));
}

// ---------------------------------------------------------------------------
// Input layer: Conv2d(Z, C, 4, padding 3) on a 1x1 input is a GEMM,
//   out[b,o,y,x] = sum_i z[b,i] * w[o,i,3-y,3-x]     (w [C][Z][16], tap t = ky*4+kx -> pixel 15-t)
// One CTA per output channel and 16 samples: thread = (sample, tap), the 16 taps of w[o,i,:] are
// one coalesced 64-byte row shared by the CTA's samples.  bias != null: the fused block
// (acc * wscale + bias[o], LeakyReLU 0.2).
// ---------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
input_layer_fwd_kernel(const float* __restrict__ z, const float* __restrict__ w, int B, int Z, int C,
                       float wscale, const float* __restrict__ bias, float* __restrict__ out) {
  const int o = blockIdx.x;
  const int t = threadIdx.x & 15;
  const int b = blockIdx.y * 16 + (threadIdx.x >> 4);
  if (b >= B) return;
  const float* wp = w + static_cast<size_t>(o) * Z * 16 + t;
  const float* zp = z + static_cast<size_t>(b) * Z;
  float acc = 0.f;
  for (int i = 0; i < Z; ++i) acc = fmaf(__ldg(zp + i), __ldg(wp + static_cast<size_t>(i) * 16), acc);
  if (bias) acc = wscale_lrelu(acc, wscale, __ldg(bias + o));
  out[(static_cast<size_t>(b) * C + o) * 16 + (15 - t)] = acc;
}

// gz[b,i] = sum_o sum_t gy[b,o,15-t] * w[o,i,t]; thread = (i, 4 samples), o and t in order.
// gy and w rows are read as float4 (16-byte aligned).
constexpr int kInBwdB = 4;
__global__ void __launch_bounds__(128)
input_layer_dgrad_kernel(const float* __restrict__ gy, const float* __restrict__ w, int B, int Z, int C,
                         float* __restrict__ gz) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const int b0 = blockIdx.y * kInBwdB;
  if (i >= Z) return;
  float acc[kInBwdB];
#pragma unroll
  for (int k = 0; k < kInBwdB; ++k) acc[k] = 0.f;
  for (int o = 0; o < C; ++o) {
    const float4* wr = reinterpret_cast<const float4*>(w + (static_cast<size_t>(o) * Z + i) * 16);
    float wv[16];
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const float4 v = __ldg(wr + q);
      wv[4 * q] = v.x; wv[4 * q + 1] = v.y; wv[4 * q + 2] = v.z; wv[4 * q + 3] = v.w;
    }
#pragma unroll
    for (int k = 0; k < kInBwdB; ++k) {
      const int b = b0 + k < B ? b0 + k : B - 1;
      const float4* gr = reinterpret_cast<const float4*>(gy + (static_cast<size_t>(b) * C + o) * 16);
      float gv[16];
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const float4 v = __ldg(gr + q);
        gv[4 * q] = v.x; gv[4 * q + 1] = v.y; gv[4 * q + 2] = v.z; gv[4 * q + 3] = v.w;
      }
#pragma unroll
      for (int t = 0; t < 16; ++t) acc[k] = fmaf(gv[15 - t], wv[t], acc[k]);
    }
  }
#pragma unroll
  for (int k = 0; k < kInBwdB; ++k)
    if (b0 + k < B) gz[static_cast<size_t>(b0 + k) * Z + i] = acc[k];
}

// gw[o,i,t] = sum_b gy[b,o,15-t] * z[b,i], samples in order; thread = (o, i), 16 taps stored as
// four float4
__global__ void __launch_bounds__(256)
input_layer_wgrad_kernel(const float* __restrict__ gy, const float* __restrict__ z, int B, int Z, int C,
                         float* __restrict__ gw) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const int o = blockIdx.y;
  if (i >= Z) return;
  float acc[16];
#pragma unroll
  for (int t = 0; t < 16; ++t) acc[t] = 0.f;
  for (int b = 0; b < B; ++b) {
    const float zv = __ldg(z + static_cast<size_t>(b) * Z + i);
    const float4* gr = reinterpret_cast<const float4*>(gy + (static_cast<size_t>(b) * C + o) * 16);
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const float4 v = __ldg(gr + q);
      acc[15 - 4 * q] = fmaf(v.x, zv, acc[15 - 4 * q]);
      acc[14 - 4 * q] = fmaf(v.y, zv, acc[14 - 4 * q]);
      acc[13 - 4 * q] = fmaf(v.z, zv, acc[13 - 4 * q]);
      acc[12 - 4 * q] = fmaf(v.w, zv, acc[12 - 4 * q]);
    }
  }
  float4* dst = reinterpret_cast<float4*>(gw + (static_cast<size_t>(o) * Z + i) * 16);
#pragma unroll
  for (int q = 0; q < 4; ++q)
    dst[q] = make_float4(acc[4 * q], acc[4 * q + 1], acc[4 * q + 2], acc[4 * q + 3]);
}

// ---------------------------------------------------------------------------
// Narrow 3x3 conv (pad 1, no bias): out[b,o,y,x] = sum_i sum_{u,v} x[b,i,y+u-1,x+v-1] w[o,i,u,v]
// A CTA computes a 32 x 32 output tile for 16 output channels: thread = one column, 4 rows,
// 16 channels (64 accumulators).  Per step of 8 input channels the input tile with its halo and
// the 8 x 9 x 16 weights are staged in shared memory; each input value in registers feeds 16
// channels, each weight (a broadcast float4 read) 4 pixels.  FLIP: the dgrad, conv(gy, W') with
// W'[o][i][t] = W[i][o][8 - t] read straight from the forward's weight tensor.
// bias != null: the fused block epilogue (acc * wscale + bias[o], LeakyReLU 0.2).
// ---------------------------------------------------------------------------
constexpr int kNcTw = 32, kNcTh = 32, kNcPx = 4, kNcCo = 16, kNcCi = 8;

template <bool FLIP>
__global__ void __launch_bounds__(256, 2)
narrow_conv3x3_kernel(const float* __restrict__ x, const float* __restrict__ w, int Cin, int Cout,
                      int H, int W, int tiles_x, float wscale, const float* __restrict__ bias,
                      float* __restrict__ out) {
  __shared__ float xs[kNcCi][kNcTh + 2][kNcTw + 2];
  __shared__ __align__(16) float ws[kNcCi][9][kNcCo];
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const int x0 = (blockIdx.x % tiles_x) * kNcTw, y0 = (blockIdx.x / tiles_x) * kNcTh;
  const int co0 = blockIdx.y * kNcCo;
  const int b = blockIdx.z;
  const size_t hw = static_cast<size_t>(H) * W;
  const float* xb = x + static_cast<size_t>(b) * Cin * hw;
  float acc[kNcPx][kNcCo];
#pragma unroll
  for (int p = 0; p < kNcPx; ++p)
#pragma unroll
    for (int c = 0; c < kNcCo; ++c) acc[p][c] = 0.f;
  constexpr int kPlane = (kNcTh + 2) * (kNcTw + 2);
  for (int ci0 = 0; ci0 < Cin; ci0 += kNcCi) {
    for (int e = threadIdx.x; e < kNcCi * kPlane; e += 256) {
      const int c = e / kPlane, r = e - c * kPlane;
      const int yy = r / (kNcTw + 2), xx = r - yy * (kNcTw + 2);
      const int gy = y0 + yy - 1, gx = x0 + xx - 1, ci = ci0 + c;
      float v = 0.f;
      if (ci < Cin && gy >= 0 && gy < H && gx >= 0 && gx < W)
        v = __ldg(xb + ci * hw + static_cast<size_t>(gy) * W + gx);
      xs[c][yy][xx] = v;
    }
    for (int e = threadIdx.x; e < kNcCi * 9 * kNcCo; e += 256) {
      const int c = e / (9 * kNcCo), r = e - c * 9 * kNcCo;
      const int tap = r / kNcCo, co = r - tap * kNcCo;
      const int ci = ci0 + c, o = co0 + co;
      float v = 0.f;
      if (ci < Cin && o < Cout)
        v = FLIP ? __ldg(w + (static_cast<size_t>(ci) * Cout + o) * 9 + (8 - tap))
                 : __ldg(w + (static_cast<size_t>(o) * Cin + ci) * 9 + tap);
      ws[c][tap][co] = v;
    }
    __syncthreads();
#pragma unroll 1
    for (int c = 0; c < kNcCi; ++c) {
      float xv[kNcPx + 2][3];
#pragma unroll
      for (int r = 0; r < kNcPx + 2; ++r)
#pragma unroll
        for (int d = 0; d < 3; ++d) xv[r][d] = xs[c][ty * kNcPx + r][tx + d];
#pragma unroll
      for (int tap = 0; tap < 9; ++tap) {
        const int u = tap / 3, v = tap - u * 3;
        const float4* wr = reinterpret_cast<const float4*>(&ws[c][tap][0]);
        float wv[kNcCo];
#pragma unroll
        for (int q = 0; q < kNcCo / 4; ++q) {
          const float4 t4 = wr[q];
          wv[4 * q] = t4.x; wv[4 * q + 1] = t4.y; wv[4 * q + 2] = t4.z; wv[4 * q + 3] = t4.w;
        }
#pragma unroll
        for (int p = 0; p < kNcPx; ++p)
#pragma unroll
          for (int co = 0; co < kNcCo; ++co) acc[p][co] = fmaf(xv[p + u][v], wv[co], acc[p][co]);
      }
    }
    __syncthreads();
  }
  const int xo = x0 + tx;
  if (xo >= W) return;
#pragma unroll
  for (int p = 0; p < kNcPx; ++p) {
    const int yo = y0 + ty * kNcPx + p;
    if (yo >= H) continue;
#pragma unroll
    for (int co = 0; co < kNcCo; ++co) {
      const int o = co0 + co;
      if (o >= Cout) continue;
      float v = acc[p][co];
      if (bias) v = wscale_lrelu(v, wscale, __ldg(bias + o));
      out[(static_cast<size_t>(b) * Cout + o) * hw + static_cast<size_t>(yo) * W + xo] = v;
    }
  }
}

// Narrow 3x3 wgrad, split over the pixels: gw[o,i,u,v] = sum_{b,y,x} gy[b,o,y,x] x[b,i,y+u-1,x+v-1].
// CTA = (16 output x 16 input channels, split s); it walks the 8 x 32 pixel tiles s, s + S, ...
// (tiles over B x H x W) in order, with the tile of gy and the haloed tile of x in shared memory.
// Thread = one (o, i) pair with its 9 taps; along a row it slides a 3 x 3 register window, so a
// pixel costs 3 + 1 shared loads for 9 FMAs.  The partial of split s goes to part[s][o][i][9].
constexpr int kWgTh = 8, kWgTw = 32, kWgC = 16;
constexpr int kWgXs = (kWgTh + 2) * (kWgTw + 2) + 1;      // odd channel stride: no bank conflicts

__global__ void __launch_bounds__(256)
narrow_conv3x3_wgrad_kernel(const float* __restrict__ x, const float* __restrict__ gy, int B, int Cin,
                            int Cout, int H, int W, int tiles_x, int tiles_y, int splits,
                            float* __restrict__ part) {
  __shared__ float gs[kWgC][kWgTh * kWgTw];
  __shared__ float xs[kWgC * kWgXs];
  const int ol = threadIdx.x >> 4, il = threadIdx.x & 15;
  const int co_groups = (Cout + kWgC - 1) / kWgC;
  const int o0 = (blockIdx.y % co_groups) * kWgC, i0 = (blockIdx.y / co_groups) * kWgC;
  const int s = blockIdx.x;
  const long long ntiles = static_cast<long long>(B) * tiles_x * tiles_y;
  const size_t hw = static_cast<size_t>(H) * W;
  float acc[9];
#pragma unroll
  for (int t = 0; t < 9; ++t) acc[t] = 0.f;
  for (long long tile = s; tile < ntiles; tile += splits) {
    const int b = static_cast<int>(tile / (tiles_x * tiles_y));
    const int r = static_cast<int>(tile - static_cast<long long>(b) * tiles_x * tiles_y);
    const int y0 = (r / tiles_x) * kWgTh, x0 = (r % tiles_x) * kWgTw;
    for (int e = threadIdx.x; e < kWgC * kWgTh * kWgTw; e += 256) {
      const int c = e / (kWgTh * kWgTw), q = e - c * (kWgTh * kWgTw);
      const int yy = y0 + q / kWgTw, xx = x0 + q % kWgTw, o = o0 + c;
      gs[c][q] = (o < Cout && yy < H && xx < W)
                     ? __ldg(gy + (static_cast<size_t>(b) * Cout + o) * hw + static_cast<size_t>(yy) * W + xx)
                     : 0.f;
    }
    constexpr int kPlane = (kWgTh + 2) * (kWgTw + 2);
    for (int e = threadIdx.x; e < kWgC * kPlane; e += 256) {
      const int c = e / kPlane, q = e - c * kPlane;
      const int yy = y0 + q / (kWgTw + 2) - 1, xx = x0 + q % (kWgTw + 2) - 1, i = i0 + c;
      xs[c * kWgXs + q] = (i < Cin && yy >= 0 && yy < H && xx >= 0 && xx < W)
                              ? __ldg(x + (static_cast<size_t>(b) * Cin + i) * hw + static_cast<size_t>(yy) * W + xx)
                              : 0.f;
    }
    __syncthreads();
    const float* xi = xs + il * kWgXs;
    const float* go = gs[ol];
#pragma unroll 1
    for (int yr = 0; yr < kWgTh; ++yr) {
      float win[3][3];
#pragma unroll
      for (int u = 0; u < 3; ++u) {
        win[u][1] = xi[(yr + u) * (kWgTw + 2) + 0];
        win[u][2] = xi[(yr + u) * (kWgTw + 2) + 1];
      }
#pragma unroll 8
      for (int xc = 0; xc < kWgTw; ++xc) {
#pragma unroll
        for (int u = 0; u < 3; ++u) {
          win[u][0] = win[u][1];
          win[u][1] = win[u][2];
          win[u][2] = xi[(yr + u) * (kWgTw + 2) + xc + 2];
        }
        const float g = go[yr * kWgTw + xc];
#pragma unroll
        for (int u = 0; u < 3; ++u)
#pragma unroll
          for (int v = 0; v < 3; ++v) acc[u * 3 + v] = fmaf(g, win[u][v], acc[u * 3 + v]);
      }
    }
    __syncthreads();
  }
  const int o = o0 + ol, i = i0 + il;
  if (o < Cout && i < Cin) {
    float* dst = part + ((static_cast<size_t>(s) * Cout + o) * Cin + i) * 9;
#pragma unroll
    for (int t = 0; t < 9; ++t) dst[t] = acc[t];
  }
}

// out[e] = sum_{s < splits} part[s * n + e]: one warp per element, lane l takes s = l, l + 32, ...
// in order, then a fixed shuffle tree — the same sum on every call
__global__ void __launch_bounds__(256)
sum_splits_kernel(const float* __restrict__ part, int splits, long long n, float* __restrict__ out) {
  const long long e = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (e >= n) return;
  float acc = 0.f;
  for (int s = lane; s < splits; s += 32) acc += __ldg(part + static_cast<size_t>(s) * n + e);
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, d);
  if (lane == 0) out[e] = acc;
}

// ---------------------------------------------------------------------------
// ToRGB (OutputConvBlock: pixel norm -> 1x1 conv to Cout <= 4 channels -> WScale -> Hardtanh).
// Thread per pixel, input channels in order.  The fused kernel computes the norm exactly as
// pixel_norm_nchw_kernel does and the conv exactly as the leaf, so its image equals the
// leaf-by-leaf image bit for bit.
// ---------------------------------------------------------------------------
constexpr int kRgbMax = 4;

template <bool NORM>
__global__ void __launch_bounds__(256)
torgb1x1_kernel(const float* __restrict__ x, const float* __restrict__ w, int B, int Cin, int Cout,
                long long hw, float wscale, const float* __restrict__ bias, int clamp,
                float* __restrict__ out) {
  const long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (idx >= static_cast<long long>(B) * hw) return;
  const int b = static_cast<int>(idx / hw);
  const long long pix = idx - static_cast<long long>(b) * hw;
  const float* src = x + static_cast<long long>(b) * Cin * hw + pix;
  float den = 1.f;
  if (NORM) {
    float ss = 0.f;
    for (int c = 0; c < Cin; ++c) {
      const float v = __ldg(src + c * hw);
      ss = fmaf(v, v, ss);
    }
    den = sqrtf(ss / static_cast<float>(Cin) + 1e-8f);
  }
  float acc[kRgbMax] = {0.f, 0.f, 0.f, 0.f};
  for (int i = 0; i < Cin; ++i) {
    float v = __ldg(src + i * hw);
    if (NORM) v = v / den;
#pragma unroll
    for (int c = 0; c < kRgbMax; ++c)
      if (c < Cout) acc[c] = fmaf(__ldg(w + c * Cin + i), v, acc[c]);
  }
  float* dst = out + static_cast<long long>(b) * Cout * hw + pix;
#pragma unroll
  for (int c = 0; c < kRgbMax; ++c) {
    if (c >= Cout) continue;
    float v = acc[c];
    if (bias) {
      v = __fadd_rn(__fmul_rn(v, wscale), __ldg(bias + c));
      if (clamp) v = fminf(fmaxf(v, -1.f), 1.f);
    }
    dst[c * hw] = v;
  }
}

// gx[b,i,p] = sum_c w[c,i] gy[b,c,p]
__global__ void __launch_bounds__(256)
torgb1x1_dgrad_kernel(const float* __restrict__ gy, const float* __restrict__ w, int B, int Cin,
                      int Cout, long long hw, float* __restrict__ gx) {
  const long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (idx >= static_cast<long long>(B) * hw) return;
  const int b = static_cast<int>(idx / hw);
  const long long pix = idx - static_cast<long long>(b) * hw;
  float g[kRgbMax];
#pragma unroll
  for (int c = 0; c < kRgbMax; ++c)
    g[c] = c < Cout ? __ldg(gy + (static_cast<long long>(b) * Cout + c) * hw + pix) : 0.f;
  float* dst = gx + static_cast<long long>(b) * Cin * hw + pix;
  for (int i = 0; i < Cin; ++i) {
    float v = 0.f;
#pragma unroll
    for (int c = 0; c < kRgbMax; ++c)
      if (c < Cout) v = fmaf(__ldg(w + c * Cin + i), g[c], v);
    dst[i * hw] = v;
  }
}

// gw[c,i] = sum_{b,p} gy[b,c,p] x[b,i,p], split over pixels: CTA s takes the flat pixel chunk
// [s * kRgbChunk, (s + 1) * kRgbChunk) of B x HW, and for each input channel reduces its threads'
// sums in a fixed tree into part[s][c][i]
constexpr int kRgbChunk = 4096;

__global__ void __launch_bounds__(256)
torgb1x1_wgrad_kernel(const float* __restrict__ x, const float* __restrict__ gy, int B, int Cin,
                      int Cout, long long hw, float* __restrict__ part) {
  __shared__ float red[kRgbMax][8];
  const long long n = static_cast<long long>(B) * hw;
  const long long q0 = static_cast<long long>(blockIdx.x) * kRgbChunk;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int i = 0; i < Cin; ++i) {
    float acc[kRgbMax] = {0.f, 0.f, 0.f, 0.f};
    for (int k = threadIdx.x; k < kRgbChunk; k += 256) {
      const long long q = q0 + k;
      if (q >= n) break;
      const long long b = q / hw, pix = q - b * hw;
      const float xv = __ldg(x + (b * Cin + i) * hw + pix);
#pragma unroll
      for (int c = 0; c < kRgbMax; ++c)
        if (c < Cout) acc[c] = fmaf(__ldg(gy + (b * Cout + c) * hw + pix), xv, acc[c]);
    }
#pragma unroll
    for (int c = 0; c < kRgbMax; ++c)
#pragma unroll
      for (int d = 16; d > 0; d >>= 1) acc[c] += __shfl_xor_sync(0xffffffffu, acc[c], d);
    if (lane == 0)
#pragma unroll
      for (int c = 0; c < kRgbMax; ++c) red[c][warp] = acc[c];
    __syncthreads();
    if (threadIdx.x < Cout) {
      float v = 0.f;
#pragma unroll
      for (int k = 0; k < 8; ++k) v += red[threadIdx.x][k];
      part[(static_cast<size_t>(blockIdx.x) * Cout + threadIdx.x) * Cin + i] = v;
    }
    __syncthreads();
  }
}

inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

int narrow_wgrad_splits(int B, int Cin, int Cout, int H, int W) {
  const long long tiles = static_cast<long long>(B) * ((H + kWgTh - 1) / kWgTh) * ((W + kWgTw - 1) / kWgTw);
  const int groups = ((Cout + kWgC - 1) / kWgC) * ((Cin + kWgC - 1) / kWgC);
  long long s = (512 + groups - 1) / groups;   // ~512 CTAs in all: a fixed split, not per device
  if (s > tiles) s = tiles;
  return s < 1 ? 1 : static_cast<int>(s);
}

int torgb_wgrad_splits(int B, int H, int W) {
  return static_cast<int>((static_cast<long long>(B) * H * W + kRgbChunk - 1) / kRgbChunk);
}

int sum_splits(const float* part, int splits, long long n, float* out, cudaStream_t stream) {
  const long long blocks = (n * 32 + 255) / 256;
  sum_splits_kernel<<<static_cast<unsigned>(blocks), 256, 0, stream>>>(part, splits, n, out);
  return check_cuda(cudaGetLastError(), "sum_splits launch");
}

bool sizes_ok(long long B, long long a, long long b, long long H, long long W) {
  return B >= 1 && a >= 1 && b >= 1 && H >= 1 && W >= 1 && B <= 65535 &&
         B * a * H * W < (1LL << 40) && B * b * H * W < (1LL << 40);
}

}  // namespace

int proggan_input_fwd_launch(const float* z, const float* w, const float* bias, float wscale, int B,
                             int Z, int C, float* out, cudaStream_t stream) {
  if (B < 1 || Z < 1 || C < 1 || C > 2147483647 / 16) {
    set_last_error("proggan_input_fwd: bad shape B=%d Z=%d C=%d", B, Z, C);
    return RW_ERR_BAD_ARG;
  }
  dim3 grid(C, (B + 15) / 16);
  input_layer_fwd_kernel<<<grid, 256, 0, stream>>>(z, w, B, Z, C, wscale, bias, out);
  return check_cuda(cudaGetLastError(), "proggan_input_fwd launch");
}

int proggan_input_bwd_launch(const float* z, const float* w, const float* gy, int B, int Z, int C,
                             float* gz, float* gw, cudaStream_t stream) {
  if (B < 1 || Z < 1 || C < 1 || !aligned16(gy) || (gz && !aligned16(w)) || (gw && !aligned16(gw))) {
    set_last_error("proggan_input_bwd: bad shape or alignment (B=%d Z=%d C=%d; w, gy and gw need "
                   "16-byte alignment)", B, Z, C);
    return RW_ERR_BAD_ARG;
  }
  if (gz) {
    dim3 grid((Z + 127) / 128, (B + kInBwdB - 1) / kInBwdB);
    input_layer_dgrad_kernel<<<grid, 128, 0, stream>>>(gy, w, B, Z, C, gz);
    int rc = check_cuda(cudaGetLastError(), "proggan_input_bwd dgrad launch");
    if (rc) return rc;
  }
  if (gw) {
    dim3 grid((Z + 255) / 256, C);
    input_layer_wgrad_kernel<<<grid, 256, 0, stream>>>(gy, z, B, Z, C, gw);
    return check_cuda(cudaGetLastError(), "proggan_input_bwd wgrad launch");
  }
  return RW_OK;
}

int narrow_conv3x3_launch(const float* x, const float* w, const float* bias, float wscale, int B,
                          int Cin, int Cout, int H, int W, int flip, float* out, cudaStream_t stream) {
  if (!sizes_ok(B, Cin, Cout, H, W) || (Cout + kNcCo - 1) / kNcCo > 65535) {
    set_last_error("narrow_conv3x3: bad shape B=%d Cin=%d Cout=%d H=%d W=%d", B, Cin, Cout, H, W);
    return RW_ERR_BAD_ARG;
  }
  const int tiles_x = (W + kNcTw - 1) / kNcTw, tiles_y = (H + kNcTh - 1) / kNcTh;
  const long long tiles = static_cast<long long>(tiles_x) * tiles_y;
  if (tiles > 2147483647LL) {
    set_last_error("narrow_conv3x3: image too large (H=%d W=%d)", H, W);
    return RW_ERR_BAD_ARG;
  }
  dim3 grid(static_cast<unsigned>(tiles), (Cout + kNcCo - 1) / kNcCo, B);
  if (flip)
    narrow_conv3x3_kernel<true><<<grid, 256, 0, stream>>>(x, w, Cin, Cout, H, W, tiles_x, wscale,
                                                          bias, out);
  else
    narrow_conv3x3_kernel<false><<<grid, 256, 0, stream>>>(x, w, Cin, Cout, H, W, tiles_x, wscale,
                                                           bias, out);
  return check_cuda(cudaGetLastError(), "narrow_conv3x3 launch");
}

size_t narrow_conv3x3_wgrad_workspace_bytes(int B, int Cin, int Cout, int H, int W) {
  if (!sizes_ok(B, Cin, Cout, H, W)) return 0;
  return static_cast<size_t>(narrow_wgrad_splits(B, Cin, Cout, H, W)) * Cout * Cin * 9 * sizeof(float);
}

int narrow_conv3x3_wgrad_launch(const float* x, const float* gy, int B, int Cin, int Cout, int H,
                                int W, float* gw, void* workspace, size_t workspace_bytes,
                                cudaStream_t stream) {
  const size_t need = narrow_conv3x3_wgrad_workspace_bytes(B, Cin, Cout, H, W);
  if (need == 0 || workspace_bytes < need) {
    set_last_error("narrow_conv3x3_wgrad: bad shape or workspace %zu < %zu bytes (B=%d Cin=%d "
                   "Cout=%d H=%d W=%d)", workspace_bytes, need, B, Cin, Cout, H, W);
    return RW_ERR_BAD_ARG;
  }
  const int splits = narrow_wgrad_splits(B, Cin, Cout, H, W);
  const int tiles_x = (W + kWgTw - 1) / kWgTw, tiles_y = (H + kWgTh - 1) / kWgTh;
  const int groups = ((Cout + kWgC - 1) / kWgC) * ((Cin + kWgC - 1) / kWgC);
  float* part = static_cast<float*>(workspace);
  dim3 grid(splits, groups);
  narrow_conv3x3_wgrad_kernel<<<grid, 256, 0, stream>>>(x, gy, B, Cin, Cout, H, W, tiles_x, tiles_y,
                                                        splits, part);
  int rc = check_cuda(cudaGetLastError(), "narrow_conv3x3_wgrad launch");
  if (rc) return rc;
  return sum_splits(part, splits, static_cast<long long>(Cout) * Cin * 9, gw, stream);
}

int torgb1x1_launch(const float* x, const float* w, const float* bias, float wscale, int clamp,
                    int norm, int B, int Cin, int Cout, int H, int W, float* out,
                    cudaStream_t stream) {
  if (!sizes_ok(B, Cin, Cout, H, W) || Cout > kRgbMax) {
    set_last_error("torgb1x1: bad shape B=%d Cin=%d Cout=%d (1..%d) H=%d W=%d", B, Cin, Cout,
                   kRgbMax, H, W);
    return RW_ERR_BAD_ARG;
  }
  const long long hw = static_cast<long long>(H) * W;
  const long long blocks = (B * hw + 255) / 256;
  if (norm)
    torgb1x1_kernel<true><<<static_cast<unsigned>(blocks), 256, 0, stream>>>(x, w, B, Cin, Cout, hw,
                                                                             wscale, bias, clamp, out);
  else
    torgb1x1_kernel<false><<<static_cast<unsigned>(blocks), 256, 0, stream>>>(x, w, B, Cin, Cout, hw,
                                                                              wscale, bias, clamp, out);
  return check_cuda(cudaGetLastError(), "torgb1x1 launch");
}

int torgb1x1_dgrad_launch(const float* gy, const float* w, int B, int Cin, int Cout, int H, int W,
                          float* gx, cudaStream_t stream) {
  if (!sizes_ok(B, Cin, Cout, H, W) || Cout > kRgbMax) {
    set_last_error("torgb1x1_dgrad: bad shape B=%d Cin=%d Cout=%d H=%d W=%d", B, Cin, Cout, H, W);
    return RW_ERR_BAD_ARG;
  }
  const long long hw = static_cast<long long>(H) * W;
  const long long blocks = (B * hw + 255) / 256;
  torgb1x1_dgrad_kernel<<<static_cast<unsigned>(blocks), 256, 0, stream>>>(gy, w, B, Cin, Cout, hw, gx);
  return check_cuda(cudaGetLastError(), "torgb1x1_dgrad launch");
}

size_t torgb1x1_wgrad_workspace_bytes(int B, int Cin, int Cout, int H, int W) {
  if (!sizes_ok(B, Cin, Cout, H, W) || Cout > kRgbMax) return 0;
  return static_cast<size_t>(torgb_wgrad_splits(B, H, W)) * Cout * Cin * sizeof(float);
}

int torgb1x1_wgrad_launch(const float* x, const float* gy, int B, int Cin, int Cout, int H, int W,
                          float* gw, void* workspace, size_t workspace_bytes, cudaStream_t stream) {
  const size_t need = torgb1x1_wgrad_workspace_bytes(B, Cin, Cout, H, W);
  if (need == 0 || workspace_bytes < need) {
    set_last_error("torgb1x1_wgrad: bad shape or workspace %zu < %zu bytes (B=%d Cin=%d Cout=%d "
                   "H=%d W=%d)", workspace_bytes, need, B, Cin, Cout, H, W);
    return RW_ERR_BAD_ARG;
  }
  const int splits = torgb_wgrad_splits(B, H, W);
  float* part = static_cast<float*>(workspace);
  torgb1x1_wgrad_kernel<<<splits, 256, 0, stream>>>(x, gy, B, Cin, Cout,
                                                     static_cast<long long>(H) * W, part);
  int rc = check_cuda(cudaGetLastError(), "torgb1x1_wgrad launch");
  if (rc) return rc;
  return sum_splits(part, splits, static_cast<long long>(Cout) * Cin, gw, stream);
}

}  // namespace rw
