// gram_tc.cu — wgmma "col-GEMM": contraction over pixel rows.
//
//   out[m, n] = sum_r A[r + shift_a, m] * B[r + shift_b, n]
//
// With A == B == key planes this is the key second moment  mom2 += sum_n a_n a_n^T
// that the reference accumulates with one rank-1 addbmm per row
// (utils/runningstats.py:1086-1097, 1181-1190 — 10 240 batched 512x1 @ 1x512
// products per call).  With A = output-gradient planes and B = shifted key
// planes it is the conv weight gradient (autograd of models.py:313-329).
//
// Operands are the bf16 hi/lo planes [rows][C] (channels contiguous), i.e. the
// contraction index is the *slow* one: both operands are MN-major for the
// tensor core.  TMA boxes of 64 channels x 64 rows land as 128-byte swizzled
// rows; the wgmma descriptor walks 8-row groups with SBO = 1024 B and 64-channel
// blocks with LBO = one box (kBlockBytes).  Three MMAs per k-step (hi*hi + lo*hi
// + hi*lo), fp32 accumulate in registers.  Row ranges are split across CTAs;
// partial tiles go to a workspace that a second kernel reduces in a fixed order
// (bit-reproducible, unlike atomics).
#include <cstring>

#include "../../include/rewriting_b200.h"
#include "rw_common.cuh"

namespace rw {

struct GramTcParams {
  int rows;            // contraction length (rows r in [0, rows))
  int rows_a, rows_b;  // allocated rows of the A / B planes (for the TMA bounds)
  int Cm, Cn;          // channels of A (-> M) and B (-> N)
  int shift_a, shift_b;
  int ntaps;              // >= 1; grid.z
  int tap_shift_a[9];     // extra row shift of the A operand per tap
  int tap_acol[9];        // column offset inside the A planes per tap
  int a_cols;             // total columns of the A planes (0 -> Cm)
  int tap_shift_b[9];     // extra row shift of the B operand per tap
  int tap_col_ofs[9];     // column offset of this tap's block inside a partial row
  int splits;          // row-range splits (partials reduced deterministically afterwards)
  float* partial;      // [splits][Cm][ldp] fp32 workspace
  long long ldp;       // leading dimension (elements) of one partial matrix row
  int upper_only;      // 1: skip tiles strictly below the diagonal (symmetric A==B)
};

// the col-GEMM's tile extent along a channel dimension of C (C % 64 == 0): 128 where it divides C
inline int gram_tile_width(int C) { return C % 128 == 0 ? 128 : 64; }
inline int gram_tiles(int Cm, int Cn) {
  return (Cm / gram_tile_width(Cm)) * (Cn / gram_tile_width(Cn));
}

namespace {

// The output tile is TM x TN, each 128 or 64 (gram_tile_width: 64 only where the channel count is
// not a multiple of 128, as at the 64-channel layers of the 512² generator).
constexpr int RB = 64;            // rows (contraction) per pipeline stage
constexpr int MMA_K = 16;
constexpr int kStages = 3;
// fp32 accumulation in the tensor core truncates (see conv_tc.cu): the wgmma accumulator holds
// at most kChunkRB row-blocks (1024 rows = 192 accumulations); chunks are summed in fp32
// registers (round-to-nearest).  Measured on an H100 at 135 200 rows (DESIGN.md §4): a shrinkage
// of 2.7e-6..4.2e-6, 1.0-1.5x the chunk model's n/2 * 2^-25 over each split's chunks.
constexpr int kChunkRB = 16;
constexpr int kBlockBytes = 64 * RB * 2;       // one 64-channel x RB-row box
template <int TM, int TN>
struct GramCfg {
  // one consumer warpgroup per 64 rows of M (wgmma + epilogue), then one TMA warp
  static constexpr int kConsumers = TM / 64;
  static constexpr int kNumThreads = kConsumers * 128 + 32;
  static constexpr int kTmaWarp = kConsumers * 4;
  static constexpr int kAPlaneBytes = (TM / 64) * kBlockBytes;
  static constexpr int kBPlaneBytes = (TN / 64) * kBlockBytes;
  static constexpr int kStageBytes = 2 * kAPlaneBytes + 2 * kBPlaneBytes;  // A_hi, A_lo, B_hi, B_lo
  static constexpr int kSmemTotal = kStages * kStageBytes + 1024 + 256;
};

struct Barriers {
  uint64_t full[kStages];
  uint64_t empty[kStages];
};

template <int TM, int TN>
__global__ void __launch_bounds__(GramCfg<TM, TN>::kNumThreads, 1)
gram_tc_kernel(const __grid_constant__ CUtensorMap map_a_hi,
               const __grid_constant__ CUtensorMap map_a_lo,
               const __grid_constant__ CUtensorMap map_b_hi,
               const __grid_constant__ CUtensorMap map_b_lo, const GramTcParams p) {
  using G = GramCfg<TM, TN>;
  constexpr int kTmaWarp = G::kTmaWarp, kStageBytes = G::kStageBytes;
  constexpr int kAPlane = G::kAPlaneBytes, kBPlane = G::kBPlaneBytes;
  constexpr int NR = TN / 2;    // accumulator registers per thread
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                             ~static_cast<uintptr_t>(1023));
  Barriers* bars = reinterpret_cast<Barriers*>(smem + kStages * kStageBytes);

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  // tile decode (optionally upper-triangular tiles only)
  const int nt_count = p.Cn / TN;
  int mt, nt;
  if (p.upper_only) {
    int t = blockIdx.x;
    mt = 0;
    while (t >= nt_count - mt) { t -= nt_count - mt; ++mt; }
    nt = mt + t;
  } else {
    mt = blockIdx.x / nt_count;
    nt = blockIdx.x % nt_count;
  }
  const int m0 = mt * TM;
  const int n0 = nt * TN;
  const int tap = blockIdx.z;
  const int shift_b = p.shift_b + p.tap_shift_b[tap];
  const int shift_a = p.shift_a + p.tap_shift_a[tap];
  const int acol = p.tap_acol[tap];
  const int col_ofs = p.tap_col_ofs[tap];

  const int total_rb = (p.rows + RB - 1) / RB;
  const int split = blockIdx.y;
  const int rb_per = (total_rb + p.splits - 1) / p.splits;
  const int rb_begin = split * rb_per;
  int rb_end = rb_begin + rb_per;
  if (rb_end > total_rb) rb_end = total_rb;
  const int num_rb = rb_end > rb_begin ? rb_end - rb_begin : 0;

  if (warp == kTmaWarp && lane == 0) {
    tma_prefetch_desc(&map_a_hi);
    tma_prefetch_desc(&map_a_lo);
    tma_prefetch_desc(&map_b_hi);
    tma_prefetch_desc(&map_b_lo);
    for (int s = 0; s < kStages; ++s) {
      mbar_init(&bars->full[s], 1);
      mbar_init(&bars->empty[s], G::kConsumers);   // one arrival per consumer warpgroup
    }
    fence_mbar_init();
  }
  __syncthreads();

  if (warp == kTmaWarp) {
    if (lane == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (int rb = rb_begin; rb < rb_begin + num_rb; ++rb) {
        mbar_wait(&bars->empty[stage], phase ^ 1u);
        uint8_t* st = smem + stage * kStageBytes;
        mbar_expect_tx(&bars->full[stage], kStageBytes);
        const int ra = rb * RB + shift_a;
        const int rbb = rb * RB + shift_b;
#pragma unroll
        for (int j = 0; j < (TM > TN ? TM : TN) / 64; ++j) {
          if (j < TM / 64) {
            tma_load_2d(st + j * kBlockBytes, &map_a_hi, &bars->full[stage], acol + m0 + j * 64, ra);
            tma_load_2d(st + kAPlane + j * kBlockBytes, &map_a_lo, &bars->full[stage],
                        acol + m0 + j * 64, ra);
          }
          if (j < TN / 64) {
            tma_load_2d(st + 2 * kAPlane + j * kBlockBytes, &map_b_hi, &bars->full[stage],
                        n0 + j * 64, rbb);
            tma_load_2d(st + 2 * kAPlane + kBPlane + j * kBlockBytes, &map_b_lo, &bars->full[stage],
                        n0 + j * 64, rbb);
          }
        }
        if (++stage == kStages) { stage = 0; phase ^= 1u; }
      }
    }
    return;
  }

  // warpgroup wg owns the 64 output rows m0 + 64 wg .. : its A operand is the wg-th 64-channel box
  const int wg = threadIdx.x >> 7;
  float acc[NR], d[NR];
#pragma unroll
  for (int j = 0; j < NR; ++j) acc[j] = 0.f;
  int stage = 0;
  uint32_t phase = 0;
  for (int i0 = 0; i0 < num_rb; i0 += kChunkRB) {
    const int i_end = (i0 + kChunkRB < num_rb) ? i0 + kChunkRB : num_rb;
    for (int i = i0; i < i_end; ++i) {
      mbar_wait(&bars->full[stage], phase);
      const uint32_t sa = smem_u32(smem + stage * kStageBytes);
      const uint64_t da_hi = make_smem_desc(sa + wg * kBlockBytes, kBlockBytes, 1024);
      const uint64_t da_lo = make_smem_desc(sa + kAPlane + wg * kBlockBytes, kBlockBytes, 1024);
      const uint64_t db_hi = make_smem_desc(sa + 2 * kAPlane, kBlockBytes, 1024);
      const uint64_t db_lo = make_smem_desc(sa + 2 * kAPlane + kBPlane, kBlockBytes, 1024);
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < RB / MMA_K; ++kk) {
        // 16 rows = two 8-row swizzle groups of 1024 B
        const uint64_t adv = static_cast<uint64_t>((kk * MMA_K * 128) >> 4);
        wgmma_m64nN<1, 1>(d, da_lo + adv, db_hi + adv, ((i - i0) | kk) != 0);
        wgmma_m64nN<1, 1>(d, da_hi + adv, db_lo + adv, 1u);
        wgmma_m64nN<1, 1>(d, da_hi + adv, db_hi + adv, 1u);
      }
      wgmma_commit();
      wgmma_wait<0>();
      if ((threadIdx.x & 127) == 0) mbar_arrive(&bars->empty[stage]);
      if (++stage == kStages) { stage = 0; phase ^= 1u; }
    }
#pragma unroll
    for (int j = 0; j < NR; ++j) acc[j] += d[j];
  }
  // rows m0 + 64 wg + 16 (warp % 4) + lane / 4 (+ 8), columns 8 j + 2 (lane % 4) (+ 1)
  const int row = m0 + wg * 64 + (warp & 3) * 16 + (lane >> 2);
  float* dst = p.partial + (static_cast<size_t>(split) * p.Cm + row) * p.ldp + col_ofs + n0 + 2 * (lane & 3);
#pragma unroll
  for (int i = 0; i < 2; ++i)
#pragma unroll
    for (int j = 0; j < TN / 8; ++j)
      *reinterpret_cast<float2*>(dst + static_cast<size_t>(8 * i) * p.ldp + 8 * j) =
          make_float2(acc[4 * j + 2 * i], acc[4 * j + 2 * i + 1]);
}

// out[m, n] (= | +=) sum_s partial[s][m][n], 32 x 32 tiles, float reads along n (coalesced).
// mirror_upper: only tiles on or above the diagonal are computed; an off-diagonal tile is also
// stored transposed through shared memory, so both the reads and the two stores are full
// 128-byte rows (the first version read the lower triangle column-wise: 32 lines per load).
__global__ void __launch_bounds__(256)
reduce_partials_kernel(const float* __restrict__ partial, int splits, int M, int N, long long ldp,
                       float* __restrict__ out, long long ldo, int accumulate, int mirror_upper) {
  __shared__ float tile[32][33];
  const int tn = blockIdx.x, tm = blockIdx.y;
  if (mirror_upper && tm > tn) return;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;      // 32 x 8 threads
  const size_t plane = static_cast<size_t>(M) * ldp;
  const bool diag = mirror_upper && tm == tn;
#pragma unroll
  for (int r = 0; r < 4; ++r) {
    const int lm = ty + r * 8;
    const int m = tm * 32 + lm, n = tn * 32 + tx;
    float acc = 0.f;
    if (m < M && n < N && !(diag && lm > tx)) {
      const float* src = partial + static_cast<size_t>(m) * ldp + n;
      for (int s = 0; s < splits; ++s) acc += src[s * plane];
      float* o = out + static_cast<size_t>(m) * ldo + n;
      *o = accumulate ? (*o + acc) : acc;
    }
    tile[lm][tx] = acc;
  }
  if (!mirror_upper) return;
  if (diag) {
    // diagonal tile: the strictly-lower entries are the transposed upper ones (bit-identical,
    // so the accumulated matrix stays exactly symmetric)
    __syncthreads();
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      const int lm = ty + r * 8;
      const int m = tm * 32 + lm, n = tn * 32 + tx;
      if (lm > tx && m < M && n < N) {
        const float v = tile[tx][lm];
        float* o = out + static_cast<size_t>(m) * ldo + n;
        *o = accumulate ? (*o + v) : v;
      }
    }
    return;
  }
  __syncthreads();
#pragma unroll
  for (int r = 0; r < 4; ++r) {
    const int ln = ty + r * 8;                  // row of the mirrored tile = column of this one
    const int m2 = tn * 32 + ln, n2 = tm * 32 + tx;
    if (m2 < N && n2 < M) {
      float* o = out + static_cast<size_t>(m2) * ldo + n2;
      const float v = tile[tx][ln];
      *o = accumulate ? (*o + v) : v;
    }
  }
}

}  // namespace

template <int TM, int TN>
static int gram_tc_launch_tile(const GramTcParams& p, const CUtensorMap& ma_hi,
                               const CUtensorMap& ma_lo, const CUtensorMap& mb_hi,
                               const CUtensorMap& mb_lo, cudaStream_t stream) {
  using G = GramCfg<TM, TN>;
  static bool attr_set = false;
  if (!attr_set) {
    int rc = check_cuda(cudaFuncSetAttribute(gram_tc_kernel<TM, TN>,
                                             cudaFuncAttributeMaxDynamicSharedMemorySize,
                                             G::kSmemTotal),
                        "gram_tc smem attr");
    if (rc) return rc;
    attr_set = true;
  }
  const int mt = p.Cm / TM, nt = p.Cn / TN;
  const int tiles = p.upper_only ? mt * (mt + 1) / 2 : mt * nt;
  dim3 grid(tiles, p.splits, p.ntaps);
  gram_tc_kernel<TM, TN><<<grid, G::kNumThreads, G::kSmemTotal, stream>>>(
      ma_hi, ma_lo, mb_hi, mb_lo, p);
  return check_cuda(cudaGetLastError(), "gram_tc launch");
}

static int gram_tc_launch(const GramTcParams& p, const void* a_hi, const void* a_lo,
                          const void* b_hi, const void* b_lo, cudaStream_t stream) {
  if (p.Cm % 64 != 0 || p.Cn % 64 != 0 || p.Cm < 64 || p.Cn < 64 || p.rows <= 0 || p.splits < 1 ||
      p.ntaps < 1 || p.ntaps > 9) {
    set_last_error("gram_tc: unsupported shape Cm=%d Cn=%d rows=%d splits=%d", p.Cm, p.Cn, p.rows,
                   p.splits);
    return RW_ERR_BAD_ARG;
  }
  if (p.upper_only && (p.Cm != p.Cn)) {
    set_last_error("gram_tc: upper_only needs a square output");
    return RW_ERR_BAD_ARG;
  }
  // rows r >= p.rows must contribute zero: clip the A operand's row extent at the
  // contraction range so the TMA zero-fills past it (B may then hold anything).
  int max_sa = p.tap_shift_a[0];
  for (int t = 1; t < p.ntaps; ++t) max_sa = p.tap_shift_a[t] > max_sa ? p.tap_shift_a[t] : max_sa;
  long long a_extent = static_cast<long long>(p.rows) + p.shift_a + max_sa;
  if (a_extent > p.rows_a) a_extent = p.rows_a;
  if (a_extent < 1) a_extent = 1;
  const int a_cols = p.a_cols > 0 ? p.a_cols : p.Cm;
  const long long b_extent = p.rows_b;
  CUtensorMap ma_hi, ma_lo, mb_hi, mb_lo;
  int rc;
  if ((rc = make_tmap_2d_bf16(&ma_hi, a_hi, a_cols, a_extent, (uint64_t)a_cols * 2, 64, RB))) return rc;
  if ((rc = make_tmap_2d_bf16(&ma_lo, a_lo, a_cols, a_extent, (uint64_t)a_cols * 2, 64, RB))) return rc;
  if ((rc = make_tmap_2d_bf16(&mb_hi, b_hi, p.Cn, b_extent, (uint64_t)p.Cn * 2, 64, RB))) return rc;
  if ((rc = make_tmap_2d_bf16(&mb_lo, b_lo, p.Cn, b_extent, (uint64_t)p.Cn * 2, 64, RB))) return rc;
  const bool m128 = gram_tile_width(p.Cm) == 128, n128 = gram_tile_width(p.Cn) == 128;
  if (m128 && n128) return gram_tc_launch_tile<128, 128>(p, ma_hi, ma_lo, mb_hi, mb_lo, stream);
  if (m128) return gram_tc_launch_tile<128, 64>(p, ma_hi, ma_lo, mb_hi, mb_lo, stream);
  if (n128) return gram_tc_launch_tile<64, 128>(p, ma_hi, ma_lo, mb_hi, mb_lo, stream);
  return gram_tc_launch_tile<64, 64>(p, ma_hi, ma_lo, mb_hi, mb_lo, stream);
}

// out[m*ldo+n] (= or +=) sum_s partial[s][m][n]; optional symmetric mirror of the
// upper triangle into the lower one.
static int reduce_partials_launch(const float* partial, int splits, int M, int N, long long ldp,
                                  float* out, long long ldo, int accumulate, int mirror_upper,
                                  cudaStream_t stream) {
  dim3 grid((N + 31) / 32, (M + 31) / 32);
  reduce_partials_kernel<<<grid, 256, 0, stream>>>(partial, splits, M, N, ldp, out, ldo, accumulate,
                                                   mirror_upper);
  return check_cuda(cudaGetLastError(), "reduce_partials launch");
}

// split heuristic shared by the workspace query and the launches; upper_only (symmetric output)
// runs only the tiles on and above the diagonal
static int gram_splits(int Cm, int Cn, long long rows, int ntaps, bool upper_only) {
  const int mt = Cm / gram_tile_width(Cm);
  const int tiles = upper_only ? mt * (mt + 1) / 2 : gram_tiles(Cm, Cn);
  const long long total_rb = (rows + 63) / 64;
  const int sms = device_sm_count();
  long long s = (sms + static_cast<long long>(tiles) * ntaps - 1) / (static_cast<long long>(tiles) * ntaps);
  if (s > total_rb) s = total_rb;
  if (s < 1) s = 1;
  if (s > 64) s = 64;
  return static_cast<int>(s);
}

// The col-GEMM behind every gram entry point.  p holds the shape (Cm, Cn, ntaps, upper_only,
// a_cols) and the tap tables; this sets the row range, the splits and the partials' layout, checks
// the workspace, launches, and reduces the partials into out [Cm][ntaps * Cn] (+= when accumulate,
// mirrored into the lower triangle when upper_only).
static int gram_run(const char* who, GramTcParams& p, long long rows, const void* a_hi,
                    const void* a_lo, const void* b_hi, const void* b_lo, float* out, int accumulate,
                    void* workspace, size_t workspace_bytes, cudaStream_t stream) {
  p.rows = p.rows_a = p.rows_b = static_cast<int>(rows);
  p.splits = gram_splits(p.Cm, p.Cn, rows, p.ntaps, p.upper_only != 0);
  p.ldp = static_cast<long long>(p.ntaps) * p.Cn;
  p.partial = static_cast<float*>(workspace);
  const size_t need = static_cast<size_t>(p.splits) * p.Cm * p.ldp * sizeof(float);
  if (workspace_bytes < need) {
    set_last_error("%s: workspace %zu < %zu bytes", who, workspace_bytes, need);
    return RW_ERR_BAD_ARG;
  }
  int rc = gram_tc_launch(p, a_hi, a_lo, b_hi, b_lo, stream);
  if (rc) return rc;
  return reduce_partials_launch(p.partial, p.splits, p.Cm, static_cast<int>(p.ldp), p.ldp, out,
                                p.ldp, accumulate, p.upper_only, stream);
}

}  // namespace rw

using namespace rw;

extern "C" {

size_t rw_gram_workspace_bytes(int Cm, int Cn, long long rows, int ntaps) {
  if (Cm < 64 || Cn < 64 || Cm % 64 != 0 || Cn % 64 != 0 || ntaps < 1) return 0;
  // the symmetric path uses fewer tiles -> more splits; size for the larger of the two
  const int s1 = gram_splits(Cm, Cn, rows, ntaps, false);
  const int s2 = gram_splits(Cm, Cn, rows, ntaps, Cm == Cn);
  const int s = s1 > s2 ? s1 : s2;
  return static_cast<size_t>(s) * Cm * static_cast<size_t>(Cn) * ntaps * sizeof(float);
}

int rw_second_moment_accum(const void* hi, const void* lo, long long rows, int C, float* mom2,
                           void* workspace, size_t workspace_bytes, rw_stream_t stream) {
  if (rows == 0) return RW_OK;
  if (!hi || !lo || !mom2 || !workspace || rows < 0 || rows > 0x7fffffffLL || C < 64 || C % 64 != 0) {
    set_last_error("rw_second_moment_accum: bad argument (rows=%lld C=%d)", rows, C);
    return RW_ERR_BAD_ARG;
  }
  GramTcParams p;
  memset(&p, 0, sizeof(p));
  p.Cm = p.Cn = C;
  p.ntaps = 1;
  p.upper_only = 1;
  return gram_run("rw_second_moment_accum", p, rows, hi, lo, hi, lo, mom2, /*accumulate=*/1,
                  workspace, workspace_bytes, stream);
}

int rw_conv_wgrad(const void* g_hi, const void* g_lo, const void* kp_hi, const void* kp_lo,
                  long long rows, int Cout, int Cin, int Wp, float* dw_toi, void* workspace,
                  size_t workspace_bytes, rw_stream_t stream) {
  if (!g_hi || !g_lo || !kp_hi || !kp_lo || !dw_toi || !workspace || rows <= 0 ||
      rows > 0x7fffffffLL) {
    set_last_error("rw_conv_wgrad: bad argument");
    return RW_ERR_BAD_ARG;
  }
  GramTcParams p;
  memset(&p, 0, sizeof(p));
  p.Cm = Cout;
  p.Cn = Cin;
  p.ntaps = 9;
  for (int u = 0; u < 3; ++u)
    for (int v = 0; v < 3; ++v) {
      p.tap_shift_b[u * 3 + v] = (u - 1) * Wp + (v - 1);
      p.tap_col_ofs[u * 3 + v] = (u * 3 + v) * Cin;
    }
  return gram_run("rw_conv_wgrad", p, rows, g_hi, g_lo, kp_hi, kp_lo, dw_toi, /*accumulate=*/0,
                  workspace, workspace_bytes, stream);
}

int rw_conv_up_wgrad(const void* gph_hi, const void* gph_lo, const void* kp_hi, const void* kp_lo,
                     long long rows, int Cout, int Cin, int Wp, float* dw_toi, void* workspace,
                     size_t workspace_bytes, rw_stream_t stream) {
  if (!gph_hi || !gph_lo || !kp_hi || !kp_lo || !dw_toi || !workspace || rows <= 0 ||
      rows > 0x7fffffffLL) {
    set_last_error("rw_conv_up_wgrad: bad argument");
    return RW_ERR_BAD_ARG;
  }
  GramTcParams p;
  memset(&p, 0, sizeof(p));
  p.Cm = Cout;
  p.Cn = Cin;
  p.a_cols = 4 * Cout;
  p.ntaps = 9;
  for (int u = 0; u < 3; ++u)
    for (int v = 0; v < 3; ++v) {
      const int t = u * 3 + v;
      p.tap_shift_a[t] = (u >> 1) * Wp + (v >> 1);
      p.tap_acol[t] = ((u & 1) * 2 + (v & 1)) * Cout;
      p.tap_col_ofs[t] = t * Cin;
    }
  return gram_run("rw_conv_up_wgrad", p, rows, gph_hi, gph_lo, kp_hi, kp_lo, dw_toi,
                  /*accumulate=*/0, workspace, workspace_bytes, stream);
}

}  // extern "C"
