// faceparse.cu — the passes of the BiSeNet face parser (reference metrics/face-parsing.PyTorch,
// metrics/load_seg.py) that the segmenters' kernels do not already cover.  Its 3x3 convs run on
// conv_tc, its 1x1 convs on the row-GEMM, and bias / residual / ReLU / stride-2 subsampling and the
// max pool on seg.cu's passes; what is here is fp32 on CUDA cores, sums in a fixed order and uses
// no atomics:
//   stem       the images nearest-resized to S x S on the read (torch's index rule), then the 7x7 /
//              stride-2 / pad-3 conv 3 -> 64 with the folded batch norm's bias and ReLU
//   attention  a global average pool (sum, then divide) and one or two small GEMVs, each with an
//              optional bias and none / ReLU / sigmoid: the context path's conv_avg, the attention
//              refinement modules' attention vectors and the feature fusion module's
//   fuse       v = a * s[b,c] (+ a) (+ a [B,C] vector or a map), one IEEE operation per step, written
//              nearest-resized as fp32 NCHW and / or the next conv's bf16 planes in a channel slice
//   labels     the class logits bilinearly up-sampled (align_corners=True) to S x S, evaluated only at
//              the pixels that the nearest resize back to the image size picks, and their first argmax
#include "../../include/rewriting_b200.h"
#include "rw_common.cuh"

namespace rw {

namespace {

constexpr int kStemCout = 64;
constexpr int kStemK = 7;
constexpr int kStemTy = 8, kStemTx = 16;                       // output pixels per block
constexpr int kStemIy = 2 * kStemTy + kStemK - 2;              // input rows per block (21)
constexpr int kStemIx = 2 * kStemTx + kStemK - 2;              // input columns per block (37)
constexpr int kAttMax = 1024;

// torch's nearest source index (upsample_nearest2d without scales): the scale in -> out rounded to
// fp32, then min(floor(dst * scale), in - 1) with the product in fp32
__device__ __forceinline__ int nearest_src(int dst, int in, int out) {
  const float scale = __fdiv_rn(static_cast<float>(in), static_cast<float>(out));
  const int s = static_cast<int>(floorf(__fmul_rn(static_cast<float>(dst), scale)));
  return s < in - 1 ? s : in - 1;
}

// out [B,64,Ho,Wo], Ho = ceil(S/2): relu(bias + sum over (ci, ky, kx) in order of w * x), x the image
// nearest-resized to S x S and zero-padded by 3.  Block: an 8 x 16 output tile, 256 threads, thread
// t computes pixel t % 128 for channels 32 * (t / 128) .. + 31; weights and the input patch in smem.
// grid: (ceil(Wo/16), ceil(Ho/8), B)
template <bool U8>
__global__ void __launch_bounds__(256)
face_stem_kernel(const void* __restrict__ im, int H, int W, int S, int Ho, int Wo,
                 const float* __restrict__ w, const float* __restrict__ bias, float* __restrict__ out) {
  __shared__ float ws[kStemCout * 3 * kStemK * kStemK];
  __shared__ float xs[3][kStemIy][kStemIx];
  const int t = threadIdx.x;
  const int b = blockIdx.z;
  const int oy0 = blockIdx.y * kStemTy, ox0 = blockIdx.x * kStemTx;
  const int iy0 = 2 * oy0 - 3, ix0 = 2 * ox0 - 3;
  for (int i = t; i < kStemCout * 3 * kStemK * kStemK; i += 256) ws[i] = __ldg(w + i);
  const long long hw = static_cast<long long>(H) * W;
  for (int i = t; i < 3 * kStemIy * kStemIx; i += 256) {
    const int c = i / (kStemIy * kStemIx);
    const int r = (i / kStemIx) % kStemIy;
    const int q = i % kStemIx;
    const int y = iy0 + r, x = ix0 + q;
    float v = 0.f;
    if (y >= 0 && y < S && x >= 0 && x < S) {
      const long long p = static_cast<long long>(nearest_src(y, H, S)) * W + nearest_src(x, W, S);
      if (U8) {
        const unsigned char u = static_cast<const unsigned char*>(im)[(b * hw + p) * 3 + c];
        v = __fdiv_rn(__fsub_rn(__fdiv_rn(static_cast<float>(u), 255.f), 0.5f), 0.5f);
      } else {
        v = __ldg(static_cast<const float*>(im) + (static_cast<long long>(b) * 3 + c) * hw + p);
      }
    }
    xs[c][r][q] = v;
  }
  __syncthreads();
  const int pl = t & 127, co0 = (t >> 7) * 32;
  const int ty = pl / kStemTx, tx = pl % kStemTx;
  const int oy = oy0 + ty, ox = ox0 + tx;
  float acc[32];
#pragma unroll
  for (int j = 0; j < 32; ++j) acc[j] = 0.f;
  for (int c = 0; c < 3; ++c) {
    for (int ky = 0; ky < kStemK; ++ky) {
#pragma unroll
      for (int kx = 0; kx < kStemK; ++kx) {
        const float xv = xs[c][2 * ty + ky][2 * tx + kx];
        const int k = (c * kStemK + ky) * kStemK + kx;
#pragma unroll
        for (int j = 0; j < 32; ++j) acc[j] = fmaf(ws[(co0 + j) * 3 * kStemK * kStemK + k], xv, acc[j]);
      }
    }
  }
  if (oy >= Ho || ox >= Wo) return;
  const long long plane = static_cast<long long>(Ho) * Wo;
  float* o = out + (static_cast<long long>(b) * kStemCout + co0) * plane + static_cast<long long>(oy) * Wo + ox;
#pragma unroll
  for (int j = 0; j < 32; ++j) {
    float v = __fadd_rn(acc[j], __ldg(bias + co0 + j));
    if (!(v > 0.f || v != v)) v = 0.f;
    o[j * plane] = v;
  }
}

__device__ __forceinline__ float activate(float v, int act) {
  if (act == 1) return (v > 0.f || v != v) ? v : 0.f;
  if (act == 2) return __fdiv_rn(1.f, __fadd_rn(1.f, expf(-v)));
  return v;
}

// the fixed-order sum of 32 lanes' partials (xor butterfly: every lane ends with the same bits)
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = __fadd_rn(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

struct AttParams {
  const float* x;
  int C, HW;
  const float* w[2];
  const float* bias[2];
  int n[2], act[2], nlayers;
  float* out;
};

// one block per image, 512 threads (16 warps).  Warp-per-channel pooling: lane l sums positions
// l, l + 32, ... in order, the 32 partials are added in a butterfly, then divided by H*W; each GEMV
// output is a warp's dot product over its input, split by lanes the same way.
// grid: B
__global__ void __launch_bounds__(512) face_attention_kernel(const AttParams P) {
  __shared__ float v0[kAttMax], v1[kAttMax];
  const int b = blockIdx.x;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const float* xb = P.x + static_cast<long long>(b) * P.C * P.HW;
  for (int c = warp; c < P.C; c += 16) {
    const float* xc = xb + static_cast<long long>(c) * P.HW;
    float s = 0.f;
    for (int i = lane; i < P.HW; i += 32) s = __fadd_rn(s, __ldg(xc + i));
    s = warp_sum(s);
    if (lane == 0) v0[c] = __fdiv_rn(s, static_cast<float>(P.HW));
  }
  __syncthreads();
  float* in = v0;
  float* res = v1;
  int k = P.C;
  for (int l = 0; l < P.nlayers; ++l) {
    const int n = P.n[l];
    for (int o = warp; o < n; o += 16) {
      const float* wr = P.w[l] + static_cast<long long>(o) * k;
      float s = 0.f;
      for (int i = lane; i < k; i += 32) s = fmaf(__ldg(wr + i), in[i], s);
      s = warp_sum(s);
      if (P.bias[l]) s = __fadd_rn(s, __ldg(P.bias[l] + o));
      s = activate(s, P.act[l]);
      if (lane == 0) {
        if (l == P.nlayers - 1) P.out[static_cast<long long>(b) * n + o] = s;
        else res[o] = s;
      }
    }
    __syncthreads();
    float* tmp = in; in = res; res = tmp;
    k = n;
  }
}

struct FuseParams {
  const float* a;        // [B,C,H,W]
  const float* s;        // [B,C]
  int plus_a;
  const float* add;      // null, [B,C] (add_mode 1) or [B,C,H,W] (add_mode 2)
  int add_mode;
  int B, C, H, W, Ho, Wo;
  float* out;            // [B,C,Ho,Wo] or null
  __nv_bfloat16* hi;     // [B*(Ho+1)*(Wo+1)][ldc], channels coff..coff+C-1, or null
  __nv_bfloat16* lo;
  int ldc, coff;
};

// the fused value at output pixel (y, x), source pixel (nearest_src(y), nearest_src(x))
__device__ __forceinline__ float fuse_at(const FuseParams& P, int b, int c, int y, int x) {
  const int sy = nearest_src(y, P.H, P.Ho), sx = nearest_src(x, P.W, P.Wo);
  const long long bc = static_cast<long long>(b) * P.C + c;
  const long long e = (bc * P.H + sy) * P.W + sx;
  const float a = __ldg(P.a + e);
  float v = __fmul_rn(a, __ldg(P.s + bc));
  if (P.plus_a) v = __fadd_rn(v, a);
  if (P.add_mode == 1) v = __fadd_rn(v, __ldg(P.add + bc));
  else if (P.add_mode == 2) v = __fadd_rn(v, __ldg(P.add + e));
  return v;
}

// seg_map_kernel's tiling: 32 padded-flat output positions x 64 channels per block, the values
// pixel-fast into smem and the fp32 output, then the planes channel-fast.
// grid: (ceil((Ho+1)*(Wo+1)/32), C/64, B), block 256
__global__ void __launch_bounds__(256) face_fuse_kernel(const FuseParams P) {
  __shared__ float tile[64][33];
  const int Hp = P.Ho + 1, Wp = P.Wo + 1;
  const int img = Hp * Wp;
  const int p0 = blockIdx.x * 32;
  const int c0 = blockIdx.y * 64;
  const int b = blockIdx.z;
  const int t = threadIdx.x;
  {
    const int pl = t & 31;
    const int p = p0 + pl;
    const int y = p / Wp, x = p - y * Wp;
    const bool valid = p < img && y < P.Ho && x < P.Wo;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int cl = (t >> 5) + 8 * i;
      const int c = c0 + cl;
      float v = 0.f;
      if (valid) {
        v = fuse_at(P, b, c, y, x);
        if (P.out) P.out[((static_cast<long long>(b) * P.C + c) * P.Ho + y) * P.Wo + x] = v;
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

// torch's upsample_bilinear2d source position with align_corners=True, in fp32: the scale
// (in - 1) / (out - 1) (0 for out = 1), then the index, its successor inside the map and the weight
__device__ __forceinline__ void bilinear_ac(int o, int in, int out, int& i0, int& i1, float& l1) {
  const float scale = out > 1 ? __fdiv_rn(static_cast<float>(in - 1), static_cast<float>(out - 1)) : 0.f;
  const float r = __fmul_rn(scale, static_cast<float>(o));
  i0 = static_cast<int>(r);
  i1 = i0 < in - 1 ? i0 + 1 : i0;
  l1 = __fsub_rn(r, static_cast<float>(i0));
}

// one thread per output pixel: the S x S grid pixel the nearest resize picks, the bilinear value of
// every class there, (1 - ly)((1 - lx) v00 + lx v01) + ly((1 - lx) v10 + lx v11), and the first
// maximum (a NaN wins, as numpy's argmax takes it).  grid: (ceil(Ho*Wo/128), B), block 128
__global__ void __launch_bounds__(128)
face_labels_kernel(const float* __restrict__ L, int h, int w, int ld, int ncls, int S, int Ho, int Wo,
                   long long* __restrict__ labels, float* __restrict__ up) {
  const int b = blockIdx.y;
  const long long hw = static_cast<long long>(Ho) * Wo;
  const long long pix = static_cast<long long>(blockIdx.x) * 128 + threadIdx.x;
  if (pix >= hw) return;
  const int y = static_cast<int>(pix / Wo), x = static_cast<int>(pix - static_cast<long long>(y) * Wo);
  const int gy = nearest_src(y, S, Ho), gx = nearest_src(x, S, Wo);
  int y0, y1, x0, x1;
  float ly, lx;
  bilinear_ac(gy, h, S, y0, y1, ly);
  bilinear_ac(gx, w, S, x0, x1, lx);
  const float hy = __fsub_rn(1.f, ly), hx = __fsub_rn(1.f, lx);
  const long long base = static_cast<long long>(b) * (h + 1);
  const float* r00 = L + ((base + y0) * (w + 1) + x0) * ld;
  const float* r01 = L + ((base + y0) * (w + 1) + x1) * ld;
  const float* r10 = L + ((base + y1) * (w + 1) + x0) * ld;
  const float* r11 = L + ((base + y1) * (w + 1) + x1) * ld;
  int best = 0;
  float bv = 0.f;
  for (int c = 0; c < ncls; ++c) {
    const float top = __fadd_rn(__fmul_rn(hx, __ldg(r00 + c)), __fmul_rn(lx, __ldg(r01 + c)));
    const float bot = __fadd_rn(__fmul_rn(hx, __ldg(r10 + c)), __fmul_rn(lx, __ldg(r11 + c)));
    const float v = __fadd_rn(__fmul_rn(hy, top), __fmul_rn(ly, bot));
    if (up) up[(static_cast<long long>(b) * ncls + c) * hw + pix] = v;
    if (c == 0 || (bv == bv && (v > bv || v != v))) { bv = v; best = c; }
  }
  labels[static_cast<long long>(b) * hw + pix] = best;
}

inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

}  // namespace

}  // namespace rw

using namespace rw;

extern "C" {

int rw_face_stem(const void* im, int u8, int B, int H, int W, int S, const float* w,
                 const float* bias, float* out, rw_stream_t stream) {
  if (!im || !w || !bias || !out || (u8 != 0 && u8 != 1) || B < 1 || B > 65535 || H < 1 ||
      W < 1 || S < 2 || S > 8192 || 3LL * B * H * W >= (1LL << 40) ||
      static_cast<long long>(B) * kStemCout * ((S + 1) / 2) * ((S + 1) / 2) >= (1LL << 40)) {
    set_last_error("face_stem: bad argument B=%d H=%d W=%d S=%d u8=%d", B, H, W, S, u8);
    return RW_ERR_BAD_ARG;
  }
  const int Ho = (S + 1) / 2, Wo = Ho;
  const dim3 grid((Wo + kStemTx - 1) / kStemTx, (Ho + kStemTy - 1) / kStemTy, B);
  if (u8) face_stem_kernel<true><<<grid, 256, 0, stream>>>(im, H, W, S, Ho, Wo, w, bias, out);
  else face_stem_kernel<false><<<grid, 256, 0, stream>>>(im, H, W, S, Ho, Wo, w, bias, out);
  return check_cuda(cudaGetLastError(), "face_stem");
}

int rw_face_attention(const float* x, int B, int C, int H, int W, const float* w1, const float* b1,
                      int n1, int act1, const float* w2, const float* b2, int n2, int act2,
                      float* out, rw_stream_t stream) {
  const int nl = w2 ? 2 : 1;
  if (!x || !w1 || !out || B < 1 || B > 65535 || C < 1 || C > kAttMax || H < 1 || W < 1 ||
      static_cast<long long>(H) * W >= (1LL << 31) ||
      static_cast<long long>(B) * C * H * W >= (1LL << 40) || n1 < 1 || n1 > kAttMax ||
      act1 < 0 || act1 > 2 || (nl == 2 && (n2 < 1 || n2 > kAttMax || act2 < 0 || act2 > 2)) ||
      (nl == 1 && b2)) {
    set_last_error("face_attention: bad argument B=%d C=%d %dx%d n1=%d act1=%d n2=%d act2=%d%s", B, C,
                   H, W, n1, act1, n2, act2, (nl == 1 && b2) ? " (a second bias without a weight)" : "");
    return RW_ERR_BAD_ARG;
  }
  AttParams P;
  P.x = x; P.C = C; P.HW = H * W;
  P.w[0] = w1; P.bias[0] = b1; P.n[0] = n1; P.act[0] = act1;
  P.w[1] = w2; P.bias[1] = b2; P.n[1] = nl == 2 ? n2 : 0; P.act[1] = nl == 2 ? act2 : 0;
  P.nlayers = nl; P.out = out;
  face_attention_kernel<<<B, 512, 0, stream>>>(P);
  return check_cuda(cudaGetLastError(), "face_attention");
}

int rw_face_fuse(const float* a, const float* s, int plus_a, const float* add, int add_mode, int B,
                 int C, int H, int W, int Ho, int Wo, float* out, void* hi, void* lo, int ldc,
                 int coff, rw_stream_t stream) {
  bool ok = a && s && (plus_a == 0 || plus_a == 1) && add_mode >= 0 && add_mode <= 2 &&
            ((add != nullptr) == (add_mode != 0)) && B >= 1 && B <= 65535 && C >= 64 &&
            C % 64 == 0 && C / 64 <= 65535 && H >= 1 && W >= 1 && Ho >= 1 && Wo >= 1 &&
            ((hi == nullptr) == (lo == nullptr)) && (hi || out) &&
            static_cast<long long>(B) * C * H * W < (1LL << 40) &&
            static_cast<long long>(Ho + 1) * (Wo + 1) < (1LL << 30) &&
            static_cast<long long>(B) * C * (Ho + 1) * (Wo + 1) < (1LL << 40);
  if (ok && hi)
    ok = ldc % 64 == 0 && coff % 64 == 0 && coff >= 0 && coff + C <= ldc && aligned16(hi) && aligned16(lo);
  if (!ok) {
    set_last_error("face_fuse: bad argument B=%d C=%d %dx%d -> %dx%d add_mode=%d plus_a=%d ldc=%d coff=%d",
                   B, C, H, W, Ho, Wo, add_mode, plus_a, ldc, coff);
    return RW_ERR_BAD_ARG;
  }
  FuseParams P;
  P.a = a; P.s = s; P.plus_a = plus_a; P.add = add; P.add_mode = add_mode;
  P.B = B; P.C = C; P.H = H; P.W = W; P.Ho = Ho; P.Wo = Wo; P.out = out;
  P.hi = static_cast<__nv_bfloat16*>(hi); P.lo = static_cast<__nv_bfloat16*>(lo);
  P.ldc = ldc; P.coff = coff;
  const dim3 grid((static_cast<unsigned>((Ho + 1) * (Wo + 1)) + 31) / 32, C / 64, B);
  face_fuse_kernel<<<grid, 256, 0, stream>>>(P);
  return check_cuda(cudaGetLastError(), "face_fuse");
}

int rw_face_labels(const float* logits, int B, int h, int w, int ld, int ncls, int S, int Ho, int Wo,
                   long long* labels, float* up, rw_stream_t stream) {
  if (!logits || !labels || B < 1 || B > 65535 || h < 1 || w < 1 || ncls < 1 || ncls > 64 ||
      ld < ncls || S < 1 || Ho < 1 || Wo < 1 || static_cast<long long>(Ho) * Wo >= (1LL << 31) ||
      static_cast<long long>(B) * (h + 1) * (w + 1) * ld >= (1LL << 40)) {
    set_last_error("face_labels: bad argument B=%d %dx%d ld=%d ncls=%d S=%d -> %dx%d", B, h, w, ld,
                   ncls, S, Ho, Wo);
    return RW_ERR_BAD_ARG;
  }
  const long long hw = static_cast<long long>(Ho) * Wo;
  const dim3 grid(static_cast<unsigned>((hw + 127) / 128), B);
  face_labels_kernel<<<grid, 128, 0, stream>>>(logits, h, w, ld, ncls, S, Ho, Wo, labels, up);
  return check_cuda(cudaGetLastError(), "face_labels");
}

}  // extern "C"
