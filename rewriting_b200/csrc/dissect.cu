// dissect.cu — GAN dissection's unit / label statistics (reference utils/quickdissect.py,
// utils/upsample.py, utils/tally.py:218-249, 483-511):
//   upsample  a layer's activations [B,U,h,w] bilinearly to the segmentation size, written as
//             sample rows [B*H*W][U] for the quantile tally.  torch's grid_sample with
//             align_corners=True and zero padding over upsample_grid's grid, whose source
//             coordinate is affine per axis: src = t * scale + offset.  Taps outside the map are
//             zero, so the border rows and columns fade toward 0.
//   counts    one pass per batch: the activations upsampled in registers by the same device code
//             (so a compared value has the bits of the row rw_upsample_bilinear writes), compared
//             with the per-unit levels, and counted against the label maps [B,K,H,W]:
//             I[c,u] = #pixels with label c in some channel and unit u above its level, A[u], G[c]
//             and the pixel count.  Integer atomics: exact, independent of order and batching.
// Counting design: a tile of 512 pixels holds few distinct labels (C is ~1700, at most K are set
// per pixel), so the labels present are compacted in shared memory (a slot per label number) and
// each present label and each unit becomes a 512-bit plane over the tile's pixels; I is the
// popcount of their AND — a binary GEMM over the labels present only, never over all C.
#include <cmath>

#include "../../include/rewriting_b200.h"
#include "rw_common.cuh"

namespace rw {

namespace {

constexpr int kThreads = 256;
constexpr int kWords = 16;                 // 32-bit words per tile plane
constexpr int kTile = 32 * kWords;         // pixels per tile
constexpr int kLabChunk = 128;             // label planes held at once
constexpr int kUnitChunk = 128;            // unit planes held at once
constexpr unsigned short kEmpty = 0xFFFF;
constexpr unsigned short kPending = 0xFFFE;

struct Grid {
  double sy, oy, sx, ox;
};

// the two taps of one axis: first index and weights; src = t * s + o
struct UpTaps {
  int y0, x0;
  double wy0, wy1, wx0, wx1;
};

__device__ __forceinline__ UpTaps up_taps(int y, int x, const Grid& g) {
  UpTaps t;
  const double sy = __fma_rn(static_cast<double>(y), g.sy, g.oy);
  const double sx = __fma_rn(static_cast<double>(x), g.sx, g.ox);
  const double fy = floor(sy), fx = floor(sx);
  t.y0 = static_cast<int>(fy);
  t.x0 = static_cast<int>(fx);
  t.wy1 = __dsub_rn(sy, fy);
  t.wy0 = __dsub_rn(1.0, t.wy1);
  t.wx1 = __dsub_rn(sx, fx);
  t.wx0 = __dsub_rn(1.0, t.wx1);
  return t;
}

// the upsampled value at taps t of one [h,w] plane, in float64, rounded once to float.  Every
// operation is an explicit intrinsic so that both kernels execute the same sequence.
__device__ __forceinline__ float up_value(const float* __restrict__ plane, int h, int w, const UpTaps& t) {
  const bool vy0 = t.y0 >= 0 && t.y0 < h, vy1 = t.y0 + 1 >= 0 && t.y0 + 1 < h;
  const bool vx0 = t.x0 >= 0 && t.x0 < w, vx1 = t.x0 + 1 >= 0 && t.x0 + 1 < w;
  const float* r0 = plane + static_cast<long long>(t.y0) * w;
  const float* r1 = r0 + w;
  const double a00 = (vy0 && vx0) ? static_cast<double>(__ldg(r0 + t.x0)) : 0.0;
  const double a01 = (vy0 && vx1) ? static_cast<double>(__ldg(r0 + t.x0 + 1)) : 0.0;
  const double a10 = (vy1 && vx0) ? static_cast<double>(__ldg(r1 + t.x0)) : 0.0;
  const double a11 = (vy1 && vx1) ? static_cast<double>(__ldg(r1 + t.x0 + 1)) : 0.0;
  const double top = __fma_rn(t.wx1, a01, __dmul_rn(t.wx0, a00));
  const double bot = __fma_rn(t.wx1, a11, __dmul_rn(t.wx0, a10));
  return __double2float_rn(__fma_rn(t.wy1, bot, __dmul_rn(t.wy0, top)));
}

// rows [B*H*W][U]: 32 pixels x 64 units per block, computed pixel-fast and written unit-fast
// through a shared-memory transpose.  grid: (ceil(B*H*W / 32), ceil(U / 64)), block 256
__global__ void __launch_bounds__(kThreads)
upsample_rows_kernel(const float* __restrict__ act, int U, int h, int w, int H, int W, long long P,
                     Grid g, float* __restrict__ rows) {
  __shared__ float tile[64][33];
  const long long p0 = static_cast<long long>(blockIdx.x) * 32;
  const int u0 = blockIdx.y * 64;
  const int pl = threadIdx.x & 31;
  const long long p = p0 + pl;
  const int hw = H * W;
  if (p < P) {
    const int b = static_cast<int>(p / hw);
    const int pix = static_cast<int>(p - static_cast<long long>(b) * hw);
    const UpTaps t = up_taps(pix / W, pix % W, g);
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int ul = (threadIdx.x >> 5) + 8 * i;
      const int u = u0 + ul;
      if (u < U) tile[ul][pl] = up_value(act + (static_cast<long long>(b) * U + u) * h * w, h, w, t);
    }
  }
  __syncthreads();
  const int ul = threadIdx.x & 63;
  const int u = u0 + ul;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int q = (threadIdx.x >> 6) + 4 * i;
    if (u < U && p0 + q < P) rows[(p0 + q) * U + u] = tile[ul][q];
  }
}

struct CountParams {
  const float* act;
  const float* level;
  const long long* labels;
  int B, U, h, w, H, W, K, C;
  long long P;
  Grid g;
  long long* isect;        // [C,U]
  long long* unit_total;   // [U]
  long long* label_total;  // [C]
  long long* count;        // [1]
};

__device__ __forceinline__ void atomic_add_ll(long long* p, long long v) {
  atomicAdd(reinterpret_cast<unsigned long long*>(p), static_cast<unsigned long long>(v));
}

// one tile of kTile consecutive pixels (of [B*H*W]) per iteration, grid-stride.
// dynamic shared memory: slot[C] (ushort, the label's index in the tile's list or kEmpty),
// list[min(C, K*kTile)] (the labels present), lab[kLabChunk][kWords], unit[kUnitChunk][kWords+1]
__global__ void __launch_bounds__(kThreads, 2) dissect_counts_kernel(const CountParams P, int list_cap) {
  extern __shared__ __align__(16) unsigned char smem[];
  uint32_t* lab = reinterpret_cast<uint32_t*>(smem);
  uint32_t* unit = lab + kLabChunk * kWords;
  int* list = reinterpret_cast<int*>(unit + kUnitChunk * (kWords + 1));
  unsigned short* slot = reinterpret_cast<unsigned short*>(list + list_cap);
  __shared__ int nlab;

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int hw = P.H * P.W;
  for (int c = tid; c < P.C; c += kThreads) slot[c] = kEmpty;
  if (blockIdx.x == 0 && tid == 0) atomic_add_ll(P.count, P.P);
  const long long ntiles = (P.P + kTile - 1) / kTile;

  for (long long tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const long long t0 = tile * kTile;
    if (tid == 0) nlab = 0;
    __syncthreads();
    // collect the distinct labels of the tile (label 0 is never a condition)
    for (int i = tid; i < kTile * P.K; i += kThreads) {
      const int q = i % kTile, k = i / kTile;
      const long long p = t0 + q;
      if (p >= P.P) continue;
      const long long b = p / hw;
      const long long c = __ldg(P.labels + (b * P.K + k) * hw + (p - b * hw));
      if (c <= 0 || c >= P.C) continue;
      if (slot[c] == kEmpty && atomicCAS(slot + c, kEmpty, kPending) == kEmpty)
        list[atomicAdd(&nlab, 1)] = static_cast<int>(c);
    }
    __syncthreads();
    const int n = nlab;
    for (int s = tid; s < n; s += kThreads) slot[list[s]] = static_cast<unsigned short>(s);
    __syncthreads();

    // each thread's two pixels' taps, for the unit planes: warp w builds words w and w + 8
    UpTaps taps[kWords / 8];
    long long pbase[kWords / 8];
    bool valid[kWords / 8];
#pragma unroll
    for (int j = 0; j < kWords / 8; ++j) {
      const long long p = t0 + (warp + 8 * j) * 32 + lane;
      valid[j] = p < P.P;
      const long long b = valid[j] ? p / hw : 0;
      const int pix = valid[j] ? static_cast<int>(p - b * hw) : 0;
      taps[j] = up_taps(pix / P.W, pix % P.W, P.g);
      pbase[j] = b * P.U;
    }

    // label chunks: more than kLabChunk labels in one tile only happens for scattered labels
    for (int l0 = 0; l0 < (n > 0 ? n : 1); l0 += kLabChunk) {
      const int nl = min(kLabChunk, n - l0);
      for (int i = tid; i < kLabChunk * kWords; i += kThreads) lab[i] = 0u;
      __syncthreads();
      for (int i = tid; i < kTile * P.K; i += kThreads) {
        const int q = i % kTile, k = i / kTile;
        const long long p = t0 + q;
        if (p >= P.P) continue;
        const long long b = p / hw;
        const long long c = __ldg(P.labels + (b * P.K + k) * hw + (p - b * hw));
        if (c <= 0 || c >= P.C) continue;
        const int s = slot[c] - l0;
        if (s >= 0 && s < nl) atomicOr(lab + s * kWords + (q >> 5), 1u << (q & 31));
      }
      __syncthreads();
      for (int s = tid; s < nl; s += kThreads) {
        int g = 0;
#pragma unroll
        for (int wd = 0; wd < kWords; ++wd) g += __popc(lab[s * kWords + wd]);
        if (g) atomic_add_ll(P.label_total + list[l0 + s], g);
      }
      for (int u0 = 0; u0 < P.U; u0 += kUnitChunk) {
        const int nu = min(kUnitChunk, P.U - u0);
        // unit planes: bit q of unit u is (upsampled value > level[u]); NaN compares false
        for (int ul = 0; ul < nu; ++ul) {
          const int u = u0 + ul;
          const float lv = __ldg(P.level + u);
#pragma unroll
          for (int j = 0; j < kWords / 8; ++j) {
            bool above = false;
            if (valid[j]) above = up_value(P.act + (pbase[j] + u) * P.h * P.w, P.h, P.w, taps[j]) > lv;
            const uint32_t bits = __ballot_sync(0xffffffffu, above);
            if (lane == 0) unit[ul * (kWords + 1) + warp + 8 * j] = bits;
          }
        }
        __syncthreads();
        if (l0 == 0) {
          for (int ul = tid; ul < nu; ul += kThreads) {
            int a = 0;
#pragma unroll
            for (int wd = 0; wd < kWords; ++wd) a += __popc(unit[ul * (kWords + 1) + wd]);
            if (a) atomic_add_ll(P.unit_total + u0 + ul, a);
          }
        }
        for (int i = tid; i < nl * nu; i += kThreads) {
          const int s = i / nu, ul = i - s * nu;
          int cnt = 0;
#pragma unroll
          for (int wd = 0; wd < kWords; ++wd)
            cnt += __popc(lab[s * kWords + wd] & unit[ul * (kWords + 1) + wd]);
          if (cnt) atomic_add_ll(P.isect + static_cast<long long>(list[l0 + s]) * P.U + u0 + ul, cnt);
        }
        __syncthreads();
      }
    }
    for (int s = tid; s < n; s += kThreads) slot[list[s]] = kEmpty;
    __syncthreads();
  }
}

bool grid_ok(double s, double o, int n) {
  const double lim = 1 << 20;
  return std::isfinite(s) && std::isfinite(o) && fabs(o) <= lim && fabs(o + (n - 1) * s) <= lim;
}

bool sizes_ok(int B, int U, int h, int w, int H, int W, const Grid& g) {
  return B >= 1 && U >= 1 && U <= 65535 && h >= 1 && w >= 1 && H >= 1 && W >= 1 && h <= 1024 &&
         w <= 1024 && H <= 1024 && W <= 1024 && static_cast<long long>(B) * H * W < (1LL << 31) &&
         static_cast<long long>(B) * U * h * w < (1LL << 40) &&
         static_cast<long long>(B) * H * W * U < (1LL << 40) && grid_ok(g.sy, g.oy, H) &&
         grid_ok(g.sx, g.ox, W);
}

}  // namespace

}  // namespace rw

using namespace rw;

extern "C" {

int rw_upsample_bilinear(const float* act, int B, int U, int h, int w, int H, int W, double sy,
                         double oy, double sx, double ox, float* rows, rw_stream_t stream) {
  const Grid g{sy, oy, sx, ox};
  if (!act || !rows || !sizes_ok(B, U, h, w, H, W, g)) {
    set_last_error("upsample_bilinear: bad argument B=%d U=%d %dx%d -> %dx%d (sizes 1..1024, grid "
                   "within 2^20)", B, U, h, w, H, W);
    return RW_ERR_BAD_ARG;
  }
  const long long P = static_cast<long long>(B) * H * W;
  const dim3 grid(static_cast<unsigned>((P + 31) / 32), (U + 63) / 64);
  upsample_rows_kernel<<<grid, kThreads, 0, stream>>>(act, U, h, w, H, W, P, g, rows);
  return check_cuda(cudaGetLastError(), "upsample_bilinear");
}

int rw_dissect_counts(const float* act, const float* level, const long long* labels, int B, int U,
                      int h, int w, int H, int W, int K, int C, double sy, double oy, double sx,
                      double ox, long long* isect, long long* unit_total, long long* label_total,
                      long long* count, rw_stream_t stream) {
  const Grid g{sy, oy, sx, ox};
  if (!act || !level || !labels || !isect || !unit_total || !label_total || !count ||
      !sizes_ok(B, U, h, w, H, W, g) || K < 1 || K > 8 || C < 2 || C > 32768 ||
      static_cast<long long>(B) * K * H * W >= (1LL << 40)) {
    set_last_error("dissect_counts: bad argument B=%d U=%d %dx%d -> %dx%d K=%d C=%d (K 1..8, C "
                   "2..32768)", B, U, h, w, H, W, K, C);
    return RW_ERR_BAD_ARG;
  }
  CountParams P;
  P.act = act; P.level = level; P.labels = labels;
  P.B = B; P.U = U; P.h = h; P.w = w; P.H = H; P.W = W; P.K = K; P.C = C;
  P.P = static_cast<long long>(B) * H * W;
  P.g = g;
  P.isect = isect; P.unit_total = unit_total; P.label_total = label_total; P.count = count;
  const int list_cap = min(C, K * kTile);
  const size_t smem = sizeof(uint32_t) * (kLabChunk * kWords + kUnitChunk * (kWords + 1)) +
                      sizeof(int) * list_cap + sizeof(unsigned short) * C;
  if (smem > 48 * 1024) {
    const cudaError_t e = cudaFuncSetAttribute(dissect_counts_kernel,
                                               cudaFuncAttributeMaxDynamicSharedMemorySize,
                                               static_cast<int>(smem));
    if (e != cudaSuccess) return check_cuda(e, "dissect_counts");
  }
  const long long ntiles = (P.P + kTile - 1) / kTile;
  const long long cap = 4LL * device_sm_count();
  const unsigned grid = static_cast<unsigned>(ntiles < cap ? ntiles : cap);
  dissect_counts_kernel<<<grid, kThreads, smem, stream>>>(P, list_cap);
  return check_cuda(cudaGetLastError(), "dissect_counts");
}

}  // extern "C"
