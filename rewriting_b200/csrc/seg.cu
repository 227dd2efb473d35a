// seg.cu — the passes of the unified-parsing segmenter (ResNet-50 deep stem + UPerNet, reference
// utils/segmenter.py:150-361, utils/upsegmodel/) between its convolutions.  The convolutions
// themselves run on the existing kernels (conv_tc for 3x3, the row-GEMM for 1x1, the narrow fp32
// conv for the 3-channel stem); what is here is HBM-bound and sums in a fixed order, no atomics:
//   input    (x + 1) / 2 * 255, RGB -> BGR, minus the model's mean, then an integer-factor average
//            pool when the segmentation size differs from the image (AdaptiveAvgPool2d)
//   map      one pass from a conv output (fp32 NCHW, or the row-GEMM's channels-last padded rows)
//            sampled directly, at every second pixel (a stride-2 conv computed at stride 1), or
//            bilinearly resized (align_corners=False); + bias + residual, optional ReLU; writes
//            the next conv's bf16 hi/lo planes into a channel slice of a wider plane set (so the
//            PPM and fusion concatenations are never built in fp32) and / or fp32 NCHW
//   maxpool  3x3 / stride 2 / pad 1 with -inf padding and torch's floor rule and scan order
//   prroi    PrRoI pooling of the whole map into s x s bins: the exact integral of the bilinear
//            surface (zero outside the map) over each bin, divided by the bin's area
//   classes  the heads' logits bilinearly up-sampled to the segmentation size, a softmax per
//            category / part group, summed over the segmentation sizes; written as probabilities
//            and / or as segment_batch's first three label channels (object argmax, material
//            argmax with its offset, the owning object's part translated), one pass per pixel
#include "rw_common.cuh"
#include "rw_kernels.h"

namespace rw {

namespace {

// torch.tensor([102.9801, 115.9465, 122.7717]): the doubles rounded to float once
__constant__ float kSegMean[3] = {static_cast<float>(102.9801), static_cast<float>(115.9465),
                                  static_cast<float>(122.7717)};

// out [B,3,S,S]: out[b,c] = mean over the fy x fx block of ((x + 1) / 2 * 255 - mean[c]) with x
// image channel 2 - c; one thread per output element, grid-stride
template <bool U8>
__global__ void __launch_bounds__(256)
seg_input_kernel(const void* __restrict__ im, int B, int H, int W, int S, int fy, int fx,
                 float* __restrict__ out) {
  const long long n = 3LL * B * S * S;
  const long long hw = static_cast<long long>(H) * W;
  for (long long e = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; e < n;
       e += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int x = static_cast<int>(e % S);
    const int y = static_cast<int>((e / S) % S);
    const int c = static_cast<int>((e / (static_cast<long long>(S) * S)) % 3);
    const int b = static_cast<int>(e / (3LL * S * S));
    const int ci = 2 - c;
    float s = 0.f;
    for (int dy = 0; dy < fy; ++dy) {
      for (int dx = 0; dx < fx; ++dx) {
        const long long p = static_cast<long long>(y * fy + dy) * W + (x * fx + dx);
        float v;
        if (U8) {
          const unsigned char u = static_cast<const unsigned char*>(im)[(b * hw + p) * 3 + ci];
          v = __fdiv_rn(__fsub_rn(__fdiv_rn(static_cast<float>(u), 255.f), 0.5f), 0.5f);
        } else {
          v = __ldg(static_cast<const float*>(im) + (static_cast<long long>(b) * 3 + ci) * hw + p);
        }
        v = __fmul_rn(__fdiv_rn(__fadd_rn(v, 1.f), 2.f), 255.f);
        s = __fadd_rn(s, __fsub_rn(v, kSegMean[c]));
      }
    }
    out[e] = (fy * fx == 1) ? s : __fdiv_rn(s, static_cast<float>(fy * fx));
  }
}

// torch's upsample_bilinear2d source index (align_corners=False, output size given), in float64
__device__ __forceinline__ void seg_bilinear_src(int o, int in, int out, int& i0, int& i1, double& l1) {
  double src = (o + 0.5) * (static_cast<double>(in) / out) - 0.5;
  if (src < 0) src = 0;
  i0 = static_cast<int>(src);
  i1 = i0 < in - 1 ? i0 + 1 : i0;
  l1 = src - i0;
}

struct MapParams {
  const float* a;
  int a_cl;              // 0: fp32 NCHW [B,C,Hin,Win]; 1: channels-last padded rows [B*(Hin+1)*(Win+1)][C]
  int C, Hin, Win, mode, Ho, Wo;
  const float* bias;     // [C] or null
  const float* res;      // [B,C,Ho,Wo] or null
  int relu;
  __nv_bfloat16* hi;     // [B*(Ho+1)*(Wo+1)][ldc], channels coff..coff+C-1, or null
  __nv_bfloat16* lo;
  int ldc, coff;
  float* out;            // [B,C,Ho,Wo] or null
};

__device__ __forceinline__ float map_at(const MapParams& P, int b, int c, int y, int x) {
  if (P.a_cl) {
    const long long row = (static_cast<long long>(b) * (P.Hin + 1) + y) * (P.Win + 1) + x;
    return __ldg(P.a + row * P.C + c);
  }
  return __ldg(P.a + ((static_cast<long long>(b) * P.C + c) * P.Hin + y) * P.Win + x);
}

// the source value of output (b, c, y, x) before bias / residual / ReLU
__device__ __forceinline__ float map_sample(const MapParams& P, int b, int c, int y, int x) {
  if (P.mode == 0) return map_at(P, b, c, y, x);
  if (P.mode == 1) return map_at(P, b, c, 2 * y, 2 * x);
  int y0, y1, x0, x1;
  double ly, lx;
  seg_bilinear_src(y, P.Hin, P.Ho, y0, y1, ly);
  seg_bilinear_src(x, P.Win, P.Wo, x0, x1, lx);
  const double v = (1.0 - ly) * ((1.0 - lx) * map_at(P, b, c, y0, x0) + lx * map_at(P, b, c, y0, x1)) +
                   ly * ((1.0 - lx) * map_at(P, b, c, y1, x0) + lx * map_at(P, b, c, y1, x1));
  return static_cast<float>(v);
}

// 32 padded-flat output positions x 64 channels per block: the source read in its own layout's
// coalesced order, then bias / residual / ReLU and the fp32 output pixel-fast, then the planes
// channel-fast (the smem transpose of relu_pool_planes_kernel).  grid: (ceil((Ho+1)*(Wo+1)/32),
// C/64, B), block 256
__global__ void __launch_bounds__(256) seg_map_kernel(const MapParams P) {
  __shared__ float tile[64][33];
  const int Hp = P.Ho + 1, Wp = P.Wo + 1;
  const int img = Hp * Wp;
  const int p0 = blockIdx.x * 32;
  const int c0 = blockIdx.y * 64;
  const int b = blockIdx.z;
  const int t = threadIdx.x;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    int pl, cl;
    if (P.a_cl) { cl = t & 63; pl = (t >> 6) + 4 * i; }
    else { pl = t & 31; cl = (t >> 5) + 8 * i; }
    const int p = p0 + pl;
    const int yy = p / Wp, xx = p - yy * Wp;
    float v = 0.f;
    if (p < img && yy < P.Ho && xx < P.Wo) v = map_sample(P, b, c0 + cl, yy, xx);
    tile[cl][pl] = v;
  }
  __syncthreads();
  {
    const int pl = t & 31;
    const int p = p0 + pl;
    const int yy = p / Wp, xx = p - yy * Wp;
    const bool valid = p < img && yy < P.Ho && xx < P.Wo;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int cl = (t >> 5) + 8 * i;
      const int c = c0 + cl;
      float v = 0.f;
      if (valid) {
        v = tile[cl][pl];
        const long long o = ((static_cast<long long>(b) * P.C + c) * P.Ho + yy) * P.Wo + xx;
        if (P.bias) v = __fadd_rn(v, __ldg(P.bias + c));
        if (P.res) v = __fadd_rn(v, __ldg(P.res + o));
        if (P.relu && !(v > 0.f || v != v)) v = 0.f;
        if (P.out) P.out[o] = v;
      }
      tile[cl][pl] = v;
    }
  }
  if (!P.hi) return;
  __syncthreads();
  const int pl = t >> 3;
  const int cg = (t & 7) * 8;
  const int p = p0 + pl;
  if (p < img) {
    __align__(16) __nv_bfloat16 h[8];
    __align__(16) __nv_bfloat16 l[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) split_bf16(tile[cg + j][pl], h[j], l[j]);
    const size_t row = static_cast<size_t>(b) * img + p;
    const size_t off = row * P.ldc + P.coff + c0 + cg;
    *reinterpret_cast<uint4*>(P.hi + off) = *reinterpret_cast<const uint4*>(h);
    *reinterpret_cast<uint4*>(P.lo + off) = *reinterpret_cast<const uint4*>(l);
  }
}

// out [B,C,Ho,Wo] = max over the 3x3 window at (2y - 1, 2x - 1), -inf outside the map; the
// window is scanned in row-major order and a strictly greater value or a NaN replaces the max
__global__ void __launch_bounds__(256)
seg_maxpool_kernel(const float* __restrict__ x, long long planes, int H, int W, int Ho, int Wo,
                   float* __restrict__ out) {
  const long long n = planes * Ho * Wo;
  for (long long e = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; e < n;
       e += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int xo = static_cast<int>(e % Wo);
    const int yo = static_cast<int>((e / Wo) % Ho);
    const float* xp = x + (e / (static_cast<long long>(Ho) * Wo)) * H * W;
    float m = -INFINITY;
    for (int y = 2 * yo - 1; y <= 2 * yo + 1; ++y) {
      if (y < 0 || y >= H) continue;
      for (int xx = 2 * xo - 1; xx <= 2 * xo + 1; ++xx) {
        if (xx < 0 || xx >= W) continue;
        const float v = __ldg(xp + static_cast<long long>(y) * W + xx);
        if (v > m || v != v) m = v;
      }
    }
    out[e] = m;
  }
}

// weight of grid point k in the integral over [s, e] of the hat function max(0, 1 - |t - k|)
__device__ __forceinline__ double hat_integral(int k, double s, double e) {
  double w = 0;
  const double a0 = fmax(s, k - 1.0), a1 = fmin(e, static_cast<double>(k));
  if (a1 > a0) w += 0.5 * ((a1 - k + 1) * (a1 - k + 1) - (a0 - k + 1) * (a0 - k + 1));
  const double b0 = fmax(s, static_cast<double>(k)), b1 = fmin(e, k + 1.0);
  if (b1 > b0) w += 0.5 * ((k + 1 - b0) * (k + 1 - b0) - (k + 1 - b1) * (k + 1 - b1));
  return w;
}

// out [B,C,s,s]: bin (py, px) covers [px W / s, (px + 1) W / s] x [py H / s, (py + 1) H / s];
// sum over the map's points of their two hat integrals times the value, in float64, rows then
// columns in order, over the bin's area.  One thread per output element, grid-stride
__global__ void __launch_bounds__(256)
seg_prroi_kernel(const float* __restrict__ x, long long planes, int H, int W, int s,
                 float* __restrict__ out) {
  const long long n = planes * s * s;
  const double bh = static_cast<double>(H) / s, bw = static_cast<double>(W) / s;
  for (long long e = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; e < n;
       e += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int px = static_cast<int>(e % s);
    const int py = static_cast<int>((e / s) % s);
    const float* xp = x + (e / (static_cast<long long>(s) * s)) * H * W;
    const double ys = py * bh, ye = ys + bh, xs = px * bw, xe = xs + bw;
    const int y0 = max(0, static_cast<int>(ceil(ys - 1.0))), y1 = min(H - 1, static_cast<int>(floor(ye + 1.0)));
    const int x0 = max(0, static_cast<int>(ceil(xs - 1.0))), x1 = min(W - 1, static_cast<int>(floor(xe + 1.0)));
    double acc = 0;
    for (int y = y0; y <= y1; ++y) {
      const double wy = hat_integral(y, ys, ye);
      double row = 0;
      for (int xx = x0; xx <= x1; ++xx) row += hat_integral(xx, xs, xe) * __ldg(xp + static_cast<long long>(y) * W + xx);
      acc += wy * row;
    }
    out[e] = static_cast<float>(acc / (bh * bw));
  }
}

constexpr int kMaxSizes = 4;
constexpr int kMaxGroups = 128;

struct ClassParams {
  const float* logits[kMaxSizes][3];   // per size and head (object, part, material): padded rows
  int lh[kMaxSizes], lw[kMaxSizes];
  int nsizes;
  const float* bias[3];
  int ld[3];
  int ngroups;
  int g_head[kMaxGroups], g_c0[kMaxGroups], g_n[kMaxGroups], g_owner[kMaxGroups], g_out[kMaxGroups];
  const long long* trans;              // part translation by part-head channel, or null
  long long mat_offset;
  int B, Ho, Wo;
  float* probs;                        // [B,Ctot,Ho,Wo] or null
  int ctot;
  long long* labels;                   // [B,3,Ho,Wo] or null
};

struct Taps {
  long long r[4];
  float w[4];
};

__device__ __forceinline__ float logit_at(const ClassParams& P, const Taps& T, int s, int hd, int c) {
  const float* L = P.logits[s][hd];
  const int ld = P.ld[hd];
  float v = T.w[0] * __ldg(L + T.r[0] * ld + c);
  v = fmaf(T.w[1], __ldg(L + T.r[1] * ld + c), v);
  v = fmaf(T.w[2], __ldg(L + T.r[2] * ld + c), v);
  v = fmaf(T.w[3], __ldg(L + T.r[3] * ld + c), v);
  return __fadd_rn(v, __ldg(P.bias[hd] + c));
}

// softmax of group g at every size, summed over the sizes; writes the group's probabilities when
// asked and returns its argmax (the first maximum)
__device__ int group_pass(const ClassParams& P, const Taps* T, int g, int b, long long pix, bool write) {
  const int hd = P.g_head[g], c0 = P.g_c0[g], n = P.g_n[g];
  float m[kMaxSizes], z[kMaxSizes];
  for (int s = 0; s < P.nsizes; ++s) {
    float mx = -INFINITY;
    for (int c = 0; c < n; ++c) mx = fmaxf(mx, logit_at(P, T[s], s, hd, c0 + c));
    float zs = 0.f;
    for (int c = 0; c < n; ++c) zs += expf(logit_at(P, T[s], s, hd, c0 + c) - mx);
    m[s] = mx;
    z[s] = zs;
  }
  const long long hw = static_cast<long long>(P.Ho) * P.Wo;
  int best = 0;
  float bp = -INFINITY;
  for (int c = 0; c < n; ++c) {
    float p = 0.f;
    for (int s = 0; s < P.nsizes; ++s)
      p = __fadd_rn(p, __fdiv_rn(expf(logit_at(P, T[s], s, hd, c0 + c) - m[s]), z[s]));
    if (write) P.probs[(static_cast<long long>(b) * P.ctot + P.g_out[g] + c) * hw + pix] = p;
    if (p > bp) { bp = p; best = c; }
  }
  return best;
}

// one thread per output pixel.  grid: (ceil(Ho*Wo/128), B), block 128
__global__ void __launch_bounds__(128) seg_classes_kernel(const ClassParams P) {
  const int b = blockIdx.y;
  const long long hw = static_cast<long long>(P.Ho) * P.Wo;
  const long long pix = static_cast<long long>(blockIdx.x) * 128 + threadIdx.x;
  if (pix >= hw) return;
  const int y = static_cast<int>(pix / P.Wo), x = static_cast<int>(pix - static_cast<long long>(y) * P.Wo);
  Taps T[kMaxSizes];
  for (int s = 0; s < P.nsizes; ++s) {
    int y0, y1, x0, x1;
    double ly, lx;
    seg_bilinear_src(y, P.lh[s], P.Ho, y0, y1, ly);
    seg_bilinear_src(x, P.lw[s], P.Wo, x0, x1, lx);
    const long long base = static_cast<long long>(b) * (P.lh[s] + 1);
    const int wp = P.lw[s] + 1;
    T[s].r[0] = (base + y0) * wp + x0;
    T[s].r[1] = (base + y0) * wp + x1;
    T[s].r[2] = (base + y1) * wp + x0;
    T[s].r[3] = (base + y1) * wp + x1;
    T[s].w[0] = static_cast<float>((1.0 - ly) * (1.0 - lx));
    T[s].w[1] = static_cast<float>((1.0 - ly) * lx);
    T[s].w[2] = static_cast<float>(ly * (1.0 - lx));
    T[s].w[3] = static_cast<float>(ly * lx);
  }
  // labels: object argmax (group 0), material argmax (group 1) with its offset, and the part of
  // the owning object (groups 2..): segment_batch's channels 0, 1, 2.  Without probabilities to
  // write, only the owning object's part group is evaluated.
  const bool write = P.probs != nullptr;
  int obj = 0, mat = 0;
  long long part = 0;
  for (int g = 0; g < P.ngroups; ++g) {
    if (!write && g >= 2 && P.g_owner[g] != obj) continue;
    const int a = group_pass(P, T, g, b, pix, write);
    if (g == 0) obj = a;
    else if (g == 1) mat = a;
    else if (P.labels && P.g_owner[g] == obj) part = __ldg(P.trans + P.g_c0[g] + a);
  }
  if (!P.labels) return;
  long long* lb = P.labels + static_cast<long long>(b) * 3 * hw + pix;
  lb[0] = obj;
  lb[hw] = mat == 0 ? 0 : mat + P.mat_offset;
  lb[2 * hw] = part;
}

unsigned grid_for(long long n) {
  long long blocks = (n + 255) / 256;
  if (blocks > 132 * 32) blocks = 132 * 32;
  return static_cast<unsigned>(blocks < 1 ? 1 : blocks);
}

inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

}  // namespace

int seg_input_launch(const void* im, int u8, int B, int H, int W, int S, float* out, cudaStream_t stream) {
  if (!im || !out || (u8 != 0 && u8 != 1) || B < 1 || H < 1 || W < 1 || S < 1 || B > 65535 ||
      H % S != 0 || W % S != 0 || 3LL * B * H * W >= (1LL << 40)) {
    set_last_error("seg_input: bad argument B=%d H=%d W=%d S=%d u8=%d (S must divide H and W)", B,
                   H, W, S, u8);
    return RW_ERR_BAD_ARG;
  }
  const unsigned g = grid_for(3LL * B * S * S);
  if (u8) seg_input_kernel<true><<<g, 256, 0, stream>>>(im, B, H, W, S, H / S, W / S, out);
  else seg_input_kernel<false><<<g, 256, 0, stream>>>(im, B, H, W, S, H / S, W / S, out);
  return check_cuda(cudaGetLastError(), "seg_input");
}

int seg_map_launch(const float* a, int a_cl, int B, int C, int Hin, int Win, int mode, int Ho, int Wo,
                   const float* bias, const float* res, int relu, void* hi, void* lo, int ldc,
                   int coff, float* out, cudaStream_t stream) {
  bool ok = a && B >= 1 && B <= 65535 && C >= 64 && C % 64 == 0 && C / 64 <= 65535 && Hin >= 1 &&
            Win >= 1 && Ho >= 1 && Wo >= 1 && (a_cl == 0 || a_cl == 1) && (relu == 0 || relu == 1) &&
            static_cast<long long>(B) * C * (Hin + 1) * (Win + 1) < (1LL << 40) &&
            static_cast<long long>(Ho + 1) * (Wo + 1) < (1LL << 30) &&
            ((hi == nullptr) == (lo == nullptr)) && (hi || out);
  if (ok && mode == 0) ok = Ho == Hin && Wo == Win;
  else if (ok && mode == 1) ok = Ho == (Hin + 1) / 2 && Wo == (Win + 1) / 2;
  else if (ok && mode != 2) ok = false;
  if (ok && hi)
    ok = ldc % 64 == 0 && coff % 64 == 0 && coff >= 0 && coff + C <= ldc && aligned16(hi) && aligned16(lo);
  if (!ok) {
    set_last_error("seg_map: bad argument B=%d C=%d %dx%d -> %dx%d mode=%d ldc=%d coff=%d", B, C, Hin,
                   Win, Ho, Wo, mode, ldc, coff);
    return RW_ERR_BAD_ARG;
  }
  MapParams P;
  P.a = a; P.a_cl = a_cl; P.C = C; P.Hin = Hin; P.Win = Win; P.mode = mode; P.Ho = Ho; P.Wo = Wo;
  P.bias = bias; P.res = res; P.relu = relu;
  P.hi = static_cast<__nv_bfloat16*>(hi); P.lo = static_cast<__nv_bfloat16*>(lo);
  P.ldc = ldc; P.coff = coff; P.out = out;
  const dim3 grid((static_cast<unsigned>((Ho + 1) * (Wo + 1)) + 31) / 32, C / 64, B);
  seg_map_kernel<<<grid, 256, 0, stream>>>(P);
  return check_cuda(cudaGetLastError(), "seg_map");
}

int seg_maxpool_launch(const float* x, int B, int C, int H, int W, float* out, cudaStream_t stream) {
  if (!x || !out || B < 1 || C < 1 || H < 1 || W < 1 || static_cast<long long>(B) * C * H * W >= (1LL << 40)) {
    set_last_error("seg_maxpool: bad argument B=%d C=%d H=%d W=%d", B, C, H, W);
    return RW_ERR_BAD_ARG;
  }
  const int Ho = (H - 1) / 2 + 1, Wo = (W - 1) / 2 + 1;
  const long long planes = static_cast<long long>(B) * C;
  seg_maxpool_kernel<<<grid_for(planes * Ho * Wo), 256, 0, stream>>>(x, planes, H, W, Ho, Wo, out);
  return check_cuda(cudaGetLastError(), "seg_maxpool");
}

int seg_prroi_launch(const float* x, int B, int C, int H, int W, int s, float* out, cudaStream_t stream) {
  if (!x || !out || B < 1 || C < 1 || H < 1 || W < 1 || s < 1 || s > 4096 ||
      static_cast<long long>(B) * C * H * W >= (1LL << 40)) {
    set_last_error("seg_prroi: bad argument B=%d C=%d H=%d W=%d s=%d", B, C, H, W, s);
    return RW_ERR_BAD_ARG;
  }
  const long long planes = static_cast<long long>(B) * C;
  seg_prroi_kernel<<<grid_for(planes * s * s), 256, 0, stream>>>(x, planes, H, W, s, out);
  return check_cuda(cudaGetLastError(), "seg_prroi");
}

int seg_classes_launch(int nsizes, const float* const* logits, const int* map_hw, const float* const* bias,
                       const int* ld, int ngroups, const int* groups, const long long* trans,
                       long long mat_offset, int B, int Ho, int Wo, float* probs, long long* labels,
                       cudaStream_t stream) {
  const char* what = "seg_classes";
  if (nsizes < 1 || nsizes > kMaxSizes || !logits || !map_hw || !bias || !ld || !groups ||
      ngroups < 1 || ngroups > kMaxGroups || B < 1 || B > 65535 || Ho < 1 || Wo < 1 ||
      static_cast<long long>(Ho) * Wo >= (1LL << 31) || (!probs && !labels) ||
      (labels && (ngroups < 2 || (ngroups > 2 && !trans)))) {
    set_last_error("%s: bad argument nsizes=%d ngroups=%d B=%d %dx%d", what, nsizes, ngroups, B, Ho, Wo);
    return RW_ERR_BAD_ARG;
  }
  ClassParams P = {};
  P.nsizes = nsizes;
  bool used[3] = {false, false, false};
  int ctot = 0;
  for (int g = 0; g < ngroups; ++g) {
    const int hd = groups[4 * g], c0 = groups[4 * g + 1], n = groups[4 * g + 2];
    if (hd < 0 || hd > 2 || c0 < 0 || n < 1 || c0 + n > ld[hd]) {
      set_last_error("%s: group %d (head %d, channels %d + %d) is outside its head", what, g, hd, c0, n);
      return RW_ERR_BAD_ARG;
    }
    used[hd] = true;
    P.g_head[g] = hd; P.g_c0[g] = c0; P.g_n[g] = n; P.g_owner[g] = groups[4 * g + 3];
    P.g_out[g] = ctot;
    ctot += n;
  }
  for (int hd = 0; hd < 3; ++hd) {
    if (!used[hd]) continue;
    if (!bias[hd] || ld[hd] < 1) {
      set_last_error("%s: head %d has no bias or a row length < 1", what, hd);
      return RW_ERR_BAD_ARG;
    }
    P.bias[hd] = bias[hd];
    P.ld[hd] = ld[hd];
  }
  for (int s = 0; s < nsizes; ++s) {
    P.lh[s] = map_hw[2 * s];
    P.lw[s] = map_hw[2 * s + 1];
    if (P.lh[s] < 1 || P.lw[s] < 1) {
      set_last_error("%s: logit map %d has a size < 1", what, s);
      return RW_ERR_BAD_ARG;
    }
    for (int hd = 0; hd < 3; ++hd) {
      P.logits[s][hd] = logits[3 * s + hd];
      if (used[hd] && !P.logits[s][hd]) {
        set_last_error("%s: logits of head %d at size %d are null", what, hd, s);
        return RW_ERR_BAD_ARG;
      }
    }
  }
  P.ngroups = ngroups; P.trans = trans; P.mat_offset = mat_offset;
  P.B = B; P.Ho = Ho; P.Wo = Wo; P.probs = probs; P.ctot = ctot; P.labels = labels;
  const long long hw = static_cast<long long>(Ho) * Wo;
  const dim3 grid(static_cast<unsigned>((hw + 127) / 128), B);
  seg_classes_kernel<<<grid, 128, 0, stream>>>(P);
  return check_cuda(cudaGetLastError(), what);
}

}  // namespace rw
