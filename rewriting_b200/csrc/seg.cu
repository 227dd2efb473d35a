// seg.cu — the passes of the two segmenters between their convolutions: the unified-parsing
// ResNet-50 deep stem + UPerNet (reference utils/segmenter.py:150-361, utils/upsegmodel/) and the
// semantic (colour) dilated ResNet-18 + PPM (utils/segmenter.py:392-574, utils/segmodel/).  The
// convolutions themselves run on the existing kernels (conv_tc for 3x3, the row-GEMM for 1x1, the
// narrow fp32 conv for the 3-channel stem); what is here is HBM-bound and sums in a fixed order, no
// atomics:
//   input    (x + 1) / 2 * mul, the channels optionally reversed, minus the mean, over the std, then
//            an integer-factor average pool when the segmentation size differs from the image
//            (AdaptiveAvgPool2d); mul 255 / std 1 / BGR for the unified model, the labels' own
//            imageformat for the semantic one
//   map      one pass from a conv output (fp32 NCHW, or the row-GEMM's channels-last padded rows)
//            sampled directly, at every second pixel (a stride-2 conv computed at stride 1), or
//            bilinearly resized (align_corners=False); + bias + residual, optional ReLU; writes
//            the next conv's bf16 hi/lo planes into a channel slice of a wider plane set (so the
//            PPM and fusion concatenations are never built in fp32) and / or fp32 NCHW.  Source and
//            destination may be phase-split: a dilation-d 3x3 conv is the plain 3x3 conv over the
//            d x d sub-grids, so its planes are written as d*d*B sub-images and conv_tc runs as is
//   maxpool  3x3 / stride 2 / pad 1 with -inf padding and torch's floor rule and scan order
//   prroi    PrRoI pooling of the whole map into s x s bins: the exact integral of the bilinear
//            surface (zero outside the map) over each bin, divided by the bin's area
//   avgpool  AdaptiveAvgPool2d(s) with torch's bin rule, summed row by row in order
//   classes  the heads' logits bilinearly up-sampled to the segmentation size, a softmax per
//            category / part group, summed over the segmentation sizes; written as probabilities
//            and / or as segment_batch's first three label channels (object argmax, material
//            argmax with its offset, the owning object's part translated), one pass per pixel
//   semseg   the semantic head's logits up-sampled, a softmax over all classes and then one per
//            category over those probabilities, summed over the sizes; probabilities and / or one
//            label channel per category (argmax mapped to a label, the mask rule, a merge offset)
#include "../../include/rewriting_b200.h"
#include "rw_common.cuh"

namespace rw {

namespace {

struct InputNorm {
  float mul;
  float mean[3], std[3];
  int flip;
};

// out [B,3,S,S]: out[b,c] = mean over the fy x fx block of (((x + 1) / 2 * mul - mean[c]) / std[c])
// with x image channel 2 - c when flip, else c; one thread per output element, grid-stride.  mul 1
// and std 1 are exact, so the unified model's (x + 1) / 2 * 255 - mean keeps its bits
template <bool U8>
__global__ void __launch_bounds__(256)
seg_input_kernel(const void* __restrict__ im, int B, int H, int W, int S, int fy, int fx,
                 const InputNorm N, float* __restrict__ out) {
  const long long n = 3LL * B * S * S;
  const long long hw = static_cast<long long>(H) * W;
  for (long long e = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; e < n;
       e += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int x = static_cast<int>(e % S);
    const int y = static_cast<int>((e / S) % S);
    const int c = static_cast<int>((e / (static_cast<long long>(S) * S)) % 3);
    const int b = static_cast<int>(e / (3LL * S * S));
    const int ci = N.flip ? 2 - c : c;
    const float mean = c == 0 ? N.mean[0] : (c == 1 ? N.mean[1] : N.mean[2]);
    const float sd = c == 0 ? N.std[0] : (c == 1 ? N.std[1] : N.std[2]);
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
        v = __fmul_rn(__fdiv_rn(__fadd_rn(v, 1.f), 2.f), N.mul);
        s = __fadd_rn(s, __fdiv_rn(__fsub_rn(v, mean), sd));
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
  int a_cl;              // 0: fp32 NCHW [sd*sd*B,C,Hs,Ws]; 1: channels-last padded rows
                         // [sd*sd*B*(Hs+1)*(Ws+1)][C]
  int B, C, Hin, Win, mode, Ho, Wo;
  int sd, Hs, Ws;        // source phase factor and sub-image size ceil(Hin/sd) x ceil(Win/sd)
  int dd, Hd, Wd;        // destination phase factor and sub-image size ceil(Ho/dd) x ceil(Wo/dd)
  const float* bias;     // [C] or null
  const float* res;      // [dd*dd*B,C,Hd,Wd] or null
  int relu;
  __nv_bfloat16* hi;     // [dd*dd*B*(Hd+1)*(Wd+1)][ldc], channels coff..coff+C-1, or null
  __nv_bfloat16* lo;
  int ldc, coff;
  float* out;            // [dd*dd*B,C,Hd,Wd] or null
};

// a at map pixel (y, x) of image b.  Phase-split by d, pixel (y, x) lives in sub-image
// ((y % d) * d + x % d) * B + b at (y / d, x / d)
__device__ __forceinline__ float map_at(const MapParams& P, int b, int c, int y, int x) {
  int H = P.Hin, W = P.Win;
  if (P.sd > 1) {
    b += ((y % P.sd) * P.sd + x % P.sd) * P.B;
    y /= P.sd; x /= P.sd; H = P.Hs; W = P.Ws;
  }
  if (P.a_cl) {
    const long long row = (static_cast<long long>(b) * (H + 1) + y) * (W + 1) + x;
    return __ldg(P.a + row * P.C + c);
  }
  return __ldg(P.a + ((static_cast<long long>(b) * P.C + c) * H + y) * W + x);
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
// channel-fast (the smem transpose of relu_pool_planes_kernel).  Output sub-image z holds map
// pixels (yy * dd + py, xx * dd + px) of image b, z = (py * dd + px) * B + b; its positions past the
// map are written as 0 (the zero padding of a dilated conv).  grid: (ceil((Hd+1)*(Wd+1)/32), C/64,
// dd*dd*B), block 256
__global__ void __launch_bounds__(256) seg_map_kernel(const MapParams P) {
  __shared__ float tile[64][33];
  const int Hp = P.Hd + 1, Wp = P.Wd + 1;
  const int img = Hp * Wp;
  const int p0 = blockIdx.x * 32;
  const int c0 = blockIdx.y * 64;
  const int z = blockIdx.z;
  const int b = z % P.B, ph = z / P.B;
  const int py = ph / P.dd, px = ph - py * P.dd;
  const int t = threadIdx.x;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    int pl, cl;
    if (P.a_cl) { cl = t & 63; pl = (t >> 6) + 4 * i; }
    else { pl = t & 31; cl = (t >> 5) + 8 * i; }
    const int p = p0 + pl;
    const int yy = p / Wp, xx = p - yy * Wp;
    const int y = yy * P.dd + py, x = xx * P.dd + px;
    float v = 0.f;
    if (p < img && yy < P.Hd && xx < P.Wd && y < P.Ho && x < P.Wo) v = map_sample(P, b, c0 + cl, y, x);
    tile[cl][pl] = v;
  }
  __syncthreads();
  {
    const int pl = t & 31;
    const int p = p0 + pl;
    const int yy = p / Wp, xx = p - yy * Wp;
    const int y = yy * P.dd + py, x = xx * P.dd + px;
    const bool inside = p < img && yy < P.Hd && xx < P.Wd;
    const bool valid = inside && y < P.Ho && x < P.Wo;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int cl = (t >> 5) + 8 * i;
      const int c = c0 + cl;
      float v = 0.f;
      const long long o = ((static_cast<long long>(z) * P.C + c) * P.Hd + yy) * P.Wd + xx;
      if (valid) {
        v = tile[cl][pl];
        if (P.bias) v = __fadd_rn(v, __ldg(P.bias + c));
        if (P.res) v = __fadd_rn(v, __ldg(P.res + o));
        if (P.relu && !(v > 0.f || v != v)) v = 0.f;
      }
      if (inside && P.out) P.out[o] = v;
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
    const size_t row = static_cast<size_t>(z) * img + p;
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

// out [B,C,s,s]: AdaptiveAvgPool2d(s), bin (i, j) rows floor(i H / s) .. ceil((i + 1) H / s) - 1 and
// likewise columns; the bin summed in float row by row, then divided by its height and its width
// (torch's order).  One thread per output element, grid-stride
__global__ void __launch_bounds__(256)
seg_avgpool_kernel(const float* __restrict__ x, long long planes, int H, int W, int s,
                   float* __restrict__ out) {
  const long long n = planes * s * s;
  for (long long e = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; e < n;
       e += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int px = static_cast<int>(e % s);
    const int py = static_cast<int>((e / s) % s);
    const float* xp = x + (e / (static_cast<long long>(s) * s)) * H * W;
    const int y0 = static_cast<int>(static_cast<long long>(py) * H / s);
    const int y1 = static_cast<int>((static_cast<long long>(py + 1) * H + s - 1) / s);
    const int x0 = static_cast<int>(static_cast<long long>(px) * W / s);
    const int x1 = static_cast<int>((static_cast<long long>(px + 1) * W + s - 1) / s);
    float acc = 0.f;
    for (int y = y0; y < y1; ++y)
      for (int xx = x0; xx < x1; ++xx) acc = __fadd_rn(acc, __ldg(xp + static_cast<long long>(y) * W + xx));
    out[e] = __fdiv_rn(__fdiv_rn(acc, static_cast<float>(y1 - y0)), static_cast<float>(x1 - x0));
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

// the bilinear taps of output pixel (y, x) of image b in an h x w map of padded rows, torch's
// align_corners=False rule, weights rounded to float once
__device__ __forceinline__ void make_taps(Taps& T, int b, int y, int x, int h, int w, int Ho, int Wo) {
  int y0, y1, x0, x1;
  double ly, lx;
  seg_bilinear_src(y, h, Ho, y0, y1, ly);
  seg_bilinear_src(x, w, Wo, x0, x1, lx);
  const long long base = static_cast<long long>(b) * (h + 1);
  const int wp = w + 1;
  T.r[0] = (base + y0) * wp + x0;
  T.r[1] = (base + y0) * wp + x1;
  T.r[2] = (base + y1) * wp + x0;
  T.r[3] = (base + y1) * wp + x1;
  T.w[0] = static_cast<float>((1.0 - ly) * (1.0 - lx));
  T.w[1] = static_cast<float>((1.0 - ly) * lx);
  T.w[2] = static_cast<float>(ly * (1.0 - lx));
  T.w[3] = static_cast<float>(ly * lx);
}

// channel c of padded rows L (row length ld) at the taps, plus its bias
__device__ __forceinline__ float tap_logit(const float* L, int ld, const float* bias, const Taps& T, int c) {
  float v = T.w[0] * __ldg(L + T.r[0] * ld + c);
  v = fmaf(T.w[1], __ldg(L + T.r[1] * ld + c), v);
  v = fmaf(T.w[2], __ldg(L + T.r[2] * ld + c), v);
  v = fmaf(T.w[3], __ldg(L + T.r[3] * ld + c), v);
  return __fadd_rn(v, __ldg(bias + c));
}

__device__ __forceinline__ float logit_at(const ClassParams& P, const Taps& T, int s, int hd, int c) {
  return tap_logit(P.logits[s][hd], P.ld[hd], P.bias[hd], T, c);
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
  for (int s = 0; s < P.nsizes; ++s) make_taps(T[s], b, y, x, P.lh[s], P.lw[s], P.Ho, P.Wo);
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

constexpr int kMaxSemClasses = 256;
constexpr int kMaxCats = 16;

struct SemClassParams {
  const float* logits[kMaxSizes];      // per size: the class conv's padded rows [B*(h+1)*(w+1)][ld]
  int lh[kMaxSizes], lw[kMaxSizes];
  int nsizes;
  const float* bias;                   // [ncls]
  int ld, ncls, ncat;
  short cat_start[kMaxCats + 1];       // category k's channels: chan[cat_start[k] .. cat_start[k+1])
  short chan[kMaxSemClasses];
  int label[kMaxSemClasses];           // the label of each entry of chan (category_map)
  int mask_cat[kMaxCats], mask_ind[kMaxCats];   // mask rule per category, mask_cat -1: none
  int B, Ho, Wo;
  float* probs;                        // [B,ncls,Ho,Wo] or null
  long long* labels;                   // [B,lchan,Ho,Wo], channels lcoff..lcoff+ncat-1, or null
  int lchan, lcoff;
  long long offset;
};

// one thread per output pixel.  Per size: the logits + bias up-sampled, p = softmax over all
// classes; per category, q = softmax of p over the category's channels; q summed over the sizes.
// grid: (ceil(Ho*Wo/128), B), block 128
__global__ void __launch_bounds__(128) semseg_classes_kernel(const SemClassParams P) {
  const int b = blockIdx.y;
  const long long hw = static_cast<long long>(P.Ho) * P.Wo;
  const long long pix = static_cast<long long>(blockIdx.x) * 128 + threadIdx.x;
  if (pix >= hw) return;
  const int y = static_cast<int>(pix / P.Wo), x = static_cast<int>(pix - static_cast<long long>(y) * P.Wo);
  Taps T[kMaxSizes];
  float m[kMaxSizes], z[kMaxSizes];
  for (int s = 0; s < P.nsizes; ++s) {
    make_taps(T[s], b, y, x, P.lh[s], P.lw[s], P.Ho, P.Wo);
    float mx = -INFINITY;
    for (int c = 0; c < P.ncls; ++c) mx = fmaxf(mx, tap_logit(P.logits[s], P.ld, P.bias, T[s], c));
    float zs = 0.f;
    for (int c = 0; c < P.ncls; ++c) zs += expf(tap_logit(P.logits[s], P.ld, P.bias, T[s], c) - mx);
    m[s] = mx;
    z[s] = zs;
  }
  int arg[kMaxCats];
  for (int k = 0; k < P.ncat; ++k) {
    const int j0 = P.cat_start[k], j1 = P.cat_start[k + 1];
    float mp[kMaxSizes], zp[kMaxSizes];
    for (int s = 0; s < P.nsizes; ++s) {
      float mx = -INFINITY;
      for (int j = j0; j < j1; ++j)
        mx = fmaxf(mx, __fdiv_rn(expf(tap_logit(P.logits[s], P.ld, P.bias, T[s], P.chan[j]) - m[s]), z[s]));
      float zs = 0.f;
      for (int j = j0; j < j1; ++j)
        zs += expf(__fdiv_rn(expf(tap_logit(P.logits[s], P.ld, P.bias, T[s], P.chan[j]) - m[s]), z[s]) - mx);
      mp[s] = mx;
      zp[s] = zs;
    }
    int best = 0;
    float bq = -INFINITY;
    for (int j = j0; j < j1; ++j) {
      float q = 0.f;
      for (int s = 0; s < P.nsizes; ++s) {
        const float p = __fdiv_rn(expf(tap_logit(P.logits[s], P.ld, P.bias, T[s], P.chan[j]) - m[s]), z[s]);
        q = __fadd_rn(q, __fdiv_rn(expf(p - mp[s]), zp[s]));
      }
      if (P.probs) P.probs[(static_cast<long long>(b) * P.ncls + P.chan[j]) * hw + pix] = q;
      if (q > bq) { bq = q; best = j - j0; }
    }
    arg[k] = best;
  }
  if (!P.labels) return;
  long long* lb = P.labels + (static_cast<long long>(b) * P.lchan + P.lcoff) * hw + pix;
  for (int k = 0; k < P.ncat; ++k) {
    long long v = P.label[P.cat_start[k] + arg[k]];
    if (P.mask_cat[k] >= 0 && arg[P.mask_cat[k]] != P.mask_ind[k]) v = 0;
    lb[k * hw] = v + P.offset;
  }
}

unsigned grid_for(long long n) {
  long long blocks = (n + 255) / 256;
  if (blocks > 132 * 32) blocks = 132 * 32;
  return static_cast<unsigned>(blocks < 1 ? 1 : blocks);
}

inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

}  // namespace

namespace {

int seg_input_common(const char* what, const void* im, int u8, int B, int H, int W, int S,
                     const InputNorm& N, float* out, cudaStream_t stream) {
  if (!im || !out || (u8 != 0 && u8 != 1) || B < 1 || H < 1 || W < 1 || S < 1 || B > 65535 ||
      H % S != 0 || W % S != 0 || 3LL * B * H * W >= (1LL << 40)) {
    set_last_error("%s: bad argument B=%d H=%d W=%d S=%d u8=%d (S must divide H and W)", what, B,
                   H, W, S, u8);
    return RW_ERR_BAD_ARG;
  }
  const unsigned g = grid_for(3LL * B * S * S);
  if (u8) seg_input_kernel<true><<<g, 256, 0, stream>>>(im, B, H, W, S, H / S, W / S, N, out);
  else seg_input_kernel<false><<<g, 256, 0, stream>>>(im, B, H, W, S, H / S, W / S, N, out);
  return check_cuda(cudaGetLastError(), what);
}

}  // namespace

}  // namespace rw

using namespace rw;

extern "C" {

int rw_seg_input(const void* im, int u8, int B, int H, int W, int S, float* out, rw_stream_t stream) {
  // torch.tensor([102.9801, 115.9465, 122.7717]): the doubles rounded to float once
  const InputNorm N = {255.f,
                       {static_cast<float>(102.9801), static_cast<float>(115.9465), static_cast<float>(122.7717)},
                       {1.f, 1.f, 1.f}, 1};
  return seg_input_common("seg_input", im, u8, B, H, W, S, N, out, stream);
}

int rw_seg_input_norm(const void* im, int u8, int B, int H, int W, int S, const float* mean,
                      const float* stdev, int bgr, float* out, rw_stream_t stream) {
  bool ok = mean && stdev && (bgr == 0 || bgr == 1);
  for (int c = 0; ok && c < 3; ++c)
    ok = isfinite(mean[c]) && isfinite(stdev[c]) && stdev[c] != 0.f;
  if (!ok) {
    set_last_error("seg_input_norm: mean / stdev missing, not finite or a zero stdev, or bgr not 0/1");
    return RW_ERR_BAD_ARG;
  }
  const InputNorm N = {1.f, {mean[0], mean[1], mean[2]}, {stdev[0], stdev[1], stdev[2]}, bgr};
  return seg_input_common("seg_input_norm", im, u8, B, H, W, S, N, out, stream);
}

int rw_seg_map(const float* a, int a_cl, int B, int C, int Hin, int Win, int mode, int Ho, int Wo,
               const float* bias, const float* res, int relu, void* hi, void* lo, int ldc,
               int coff, float* out, rw_stream_t stream) {
  return rw_seg_map_phase(a, a_cl, 1, B, C, Hin, Win, mode, Ho, Wo, bias, res, relu, 1, hi, lo, ldc,
                          coff, out, stream);
}

int rw_seg_map_phase(const float* a, int a_cl, int sd, int B, int C, int Hin, int Win, int mode,
                     int Ho, int Wo, const float* bias, const float* res, int relu, int dd,
                     void* hi, void* lo, int ldc, int coff, float* out, rw_stream_t stream) {
  bool ok = a && sd >= 1 && sd <= 8 && dd >= 1 && dd <= 8 && B >= 1 &&
            static_cast<long long>(dd) * dd * B <= 65535 && C >= 64 && C % 64 == 0 &&
            C / 64 <= 65535 && Hin >= 1 && Win >= 1 && Ho >= 1 && Wo >= 1 &&
            (a_cl == 0 || a_cl == 1) && (relu == 0 || relu == 1) &&
            ((hi == nullptr) == (lo == nullptr)) && (hi || out);
  const int Hs = ok ? (Hin + sd - 1) / sd : 0, Ws = ok ? (Win + sd - 1) / sd : 0;
  const int Hd = ok ? (Ho + dd - 1) / dd : 0, Wd = ok ? (Wo + dd - 1) / dd : 0;
  ok = ok && static_cast<long long>(sd) * sd * B * C * (Hs + 1) * (Ws + 1) < (1LL << 40) &&
       static_cast<long long>(Hd + 1) * (Wd + 1) < (1LL << 30) &&
       static_cast<long long>(dd) * dd * B * C * (Hd + 1) * (Wd + 1) < (1LL << 40);
  if (ok && mode == 0) ok = Ho == Hin && Wo == Win;
  else if (ok && mode == 1) ok = Ho == (Hin + 1) / 2 && Wo == (Win + 1) / 2;
  else if (ok && mode != 2) ok = false;
  if (ok && hi)
    ok = ldc % 64 == 0 && coff % 64 == 0 && coff >= 0 && coff + C <= ldc && aligned16(hi) && aligned16(lo);
  if (!ok) {
    set_last_error("seg_map: bad argument B=%d C=%d %dx%d -> %dx%d mode=%d ldc=%d coff=%d phases %d -> %d",
                   B, C, Hin, Win, Ho, Wo, mode, ldc, coff, sd, dd);
    return RW_ERR_BAD_ARG;
  }
  MapParams P;
  P.a = a; P.a_cl = a_cl; P.B = B; P.C = C; P.Hin = Hin; P.Win = Win; P.mode = mode; P.Ho = Ho; P.Wo = Wo;
  P.sd = sd; P.Hs = Hs; P.Ws = Ws; P.dd = dd; P.Hd = Hd; P.Wd = Wd;
  P.bias = bias; P.res = res; P.relu = relu;
  P.hi = static_cast<__nv_bfloat16*>(hi); P.lo = static_cast<__nv_bfloat16*>(lo);
  P.ldc = ldc; P.coff = coff; P.out = out;
  const dim3 grid((static_cast<unsigned>((Hd + 1) * (Wd + 1)) + 31) / 32, C / 64, dd * dd * B);
  seg_map_kernel<<<grid, 256, 0, stream>>>(P);
  return check_cuda(cudaGetLastError(), "seg_map");
}

int rw_seg_maxpool(const float* x, int B, int C, int H, int W, float* out, rw_stream_t stream) {
  if (!x || !out || B < 1 || C < 1 || H < 1 || W < 1 || static_cast<long long>(B) * C * H * W >= (1LL << 40)) {
    set_last_error("seg_maxpool: bad argument B=%d C=%d H=%d W=%d", B, C, H, W);
    return RW_ERR_BAD_ARG;
  }
  const int Ho = (H - 1) / 2 + 1, Wo = (W - 1) / 2 + 1;
  const long long planes = static_cast<long long>(B) * C;
  seg_maxpool_kernel<<<grid_for(planes * Ho * Wo), 256, 0, stream>>>(x, planes, H, W, Ho, Wo, out);
  return check_cuda(cudaGetLastError(), "seg_maxpool");
}

int rw_seg_prroi(const float* x, int B, int C, int H, int W, int s, float* out, rw_stream_t stream) {
  if (!x || !out || B < 1 || C < 1 || H < 1 || W < 1 || s < 1 || s > 4096 ||
      static_cast<long long>(B) * C * H * W >= (1LL << 40)) {
    set_last_error("seg_prroi: bad argument B=%d C=%d H=%d W=%d s=%d", B, C, H, W, s);
    return RW_ERR_BAD_ARG;
  }
  const long long planes = static_cast<long long>(B) * C;
  seg_prroi_kernel<<<grid_for(planes * s * s), 256, 0, stream>>>(x, planes, H, W, s, out);
  return check_cuda(cudaGetLastError(), "seg_prroi");
}

int rw_seg_avgpool(const float* x, int B, int C, int H, int W, int s, float* out, rw_stream_t stream) {
  if (!x || !out || B < 1 || C < 1 || H < 1 || W < 1 || s < 1 || s > 4096 ||
      static_cast<long long>(B) * C * H * W >= (1LL << 40) ||
      static_cast<long long>(B) * C * s * s >= (1LL << 40)) {
    set_last_error("seg_avgpool: bad argument B=%d C=%d H=%d W=%d s=%d", B, C, H, W, s);
    return RW_ERR_BAD_ARG;
  }
  const long long planes = static_cast<long long>(B) * C;
  seg_avgpool_kernel<<<grid_for(planes * s * s), 256, 0, stream>>>(x, planes, H, W, s, out);
  return check_cuda(cudaGetLastError(), "seg_avgpool");
}

int rw_seg_classes(int nsizes, const float* const* logits, const int* map_hw, const float* const* bias,
                   const int* ld, int ngroups, const int* groups, const long long* trans,
                   long long mat_offset, int B, int Ho, int Wo, float* probs, long long* labels,
                   rw_stream_t stream) {
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

int rw_semseg_classes(int nsizes, const float* const* logits, const int* map_hw, const float* bias,
                      int ld, int ncls, int ncat, const int* cat_start, const int* cat_chan,
                      const int* cat_label, const int* cat_mask, int B, int Ho, int Wo,
                      float* probs, long long* labels, int lchan, int lcoff, long long offset,
                      rw_stream_t stream) {
  const char* what = "semseg_classes";
  if (nsizes < 1 || nsizes > kMaxSizes || !logits || !map_hw || !bias || ncls < 1 ||
      ncls > kMaxSemClasses || ld < ncls || ncat < 1 || ncat > kMaxCats || !cat_start || !cat_chan ||
      !cat_label || !cat_mask || B < 1 || B > 65535 || Ho < 1 || Wo < 1 ||
      static_cast<long long>(Ho) * Wo >= (1LL << 31) || (!probs && !labels) ||
      (labels && (lcoff < 0 || lchan < lcoff + ncat || offset < 0))) {
    set_last_error("%s: bad argument nsizes=%d ncls=%d ld=%d ncat=%d B=%d %dx%d labels %d + %d of %d",
                   what, nsizes, ncls, ld, ncat, B, Ho, Wo, lcoff, ncat, lchan);
    return RW_ERR_BAD_ARG;
  }
  SemClassParams P = {};
  P.nsizes = nsizes; P.bias = bias; P.ld = ld; P.ncls = ncls; P.ncat = ncat;
  // every class in exactly one category, each category non-empty, masks inside their category
  bool seen[kMaxSemClasses] = {};
  if (cat_start[0] != 0 || cat_start[ncat] != ncls) {
    set_last_error("%s: the categories do not cover the %d classes", what, ncls);
    return RW_ERR_BAD_ARG;
  }
  for (int k = 0; k <= ncat; ++k) {
    if (k < ncat && cat_start[k + 1] <= cat_start[k]) {
      set_last_error("%s: category %d is empty or out of order", what, k);
      return RW_ERR_BAD_ARG;
    }
    P.cat_start[k] = static_cast<short>(cat_start[k]);
  }
  for (int j = 0; j < ncls; ++j) {
    const int c = cat_chan[j];
    if (c < 0 || c >= ncls || seen[c]) {
      set_last_error("%s: channel entry %d (%d) is outside 0..%d or repeated", what, j, c, ncls - 1);
      return RW_ERR_BAD_ARG;
    }
    seen[c] = true;
    P.chan[j] = static_cast<short>(c);
    P.label[j] = cat_label[j];
  }
  for (int k = 0; k < ncat; ++k) {
    const int mc = cat_mask[2 * k], mi = cat_mask[2 * k + 1];
    if (mc >= ncat || (mc >= 0 && (mi < 0 || mi >= cat_start[mc + 1] - cat_start[mc]))) {
      set_last_error("%s: category %d masks on category %d index %d, outside it", what, k, mc, mi);
      return RW_ERR_BAD_ARG;
    }
    P.mask_cat[k] = mc < 0 ? -1 : mc;
    P.mask_ind[k] = mi;
  }
  for (int s = 0; s < nsizes; ++s) {
    P.logits[s] = logits[s];
    P.lh[s] = map_hw[2 * s];
    P.lw[s] = map_hw[2 * s + 1];
    if (!P.logits[s] || P.lh[s] < 1 || P.lw[s] < 1) {
      set_last_error("%s: logit map %d is null or has a size < 1", what, s);
      return RW_ERR_BAD_ARG;
    }
  }
  P.B = B; P.Ho = Ho; P.Wo = Wo; P.probs = probs; P.labels = labels;
  P.lchan = lchan; P.lcoff = lcoff; P.offset = offset;
  const long long hw = static_cast<long long>(Ho) * Wo;
  const dim3 grid(static_cast<unsigned>((hw + 127) / 128), B);
  semseg_classes_kernel<<<grid, 128, 0, stream>>>(P);
  return check_cuda(cudaGetLastError(), what);
}

}  // extern "C"
