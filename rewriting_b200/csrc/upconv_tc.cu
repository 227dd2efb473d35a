// upconv_tc.cu — the upsampling StyledConv of the generation fast path as ONE kernel:
//
//   conv_transpose2d(k, scale*W, stride 2)  ->  blur 4x4 (pad 1,1)  ->  * demod  ->
//   + noise_w * noise + bias  ->  leaky-ReLU * sqrt(2)  ->  * next style  ->  bf16 hi/lo planes
//
// (reference chain: DemodulatedConv2dF models.py:313-329 -> BlurF :275-281 / upfirdn2d_kernel.cu
//  :52-137 -> NoiseInjectionF :535-546 -> FusedLeakyReLUF, fused_bias_act_kernel.cu:27-47 ->
//  the next layer's ApplyStyle :616-620).  The fp32 conv_transpose output `t` (1.04 GB at layer
//  13, batch 32) is never written: round 1 wrote it channels-last and read it back in a separate
//  SIMT blur kernel (2.3x the algorithmic DRAM traffic of the layer pair).
//
// Formulation ("scatter" polyphase).  For an INPUT pixel p and tap (u, v) let
//     P_uv[p, o] = sum_i k[p, i] * (scale*W)[o, i, u, v]
// (no shifted operands at all: one A tile serves all nine taps).  The conv_transpose output is
//     t[2y+u, 2x+v] += P_uv[(y, x)]
// so a GEMM tile is M = 128 input pixels x N = 144 = 9 taps x 16 output channels, K = Cin, issued
// as wgmma m64n144k16 by two warpgroups (64 rows each).  Every accumulation chain is only
// Cin/16 * 3 long (the 3-term bf16 split), so no chunk promotion is needed against the tensor
// core's truncating fp32 accumulate (see conv_tc.cu).
//
// A tile is ONE image row per image: 128 / W images of width W <= 128 (a power of two).  A CTA
// marches down the rows of its images; the 4x4 FIR needs t rows 2y-3 .. 2y+1 to emit output rows
// 2y-2, 2y-1 after step y, all of which depend on P at rows <= y of the SAME pixel (vertical
// direction) and of the two neighbouring pixels (horizontal direction).
//
// Epilogue data mapping.  The tile's rows are PERMUTED inside every 32-pixel quarter — tile row
// 8 j + g holds pixel 4 g + j — which costs nothing: the tensor map lists the key planes'
// dimensions in the order (channel, x/4 % 8, x % 4, x/32, row) and TMA fills shared memory in that
// order.  A wgmma accumulator gives lane (g = lane / 4, c = lane % 4) rows g and g + 8 of its
// warp's 16, so the two warps of a quarter together hold, per lane, the FOUR ADJACENT pixels
// 4g .. 4g+3; they trade channel halves through shared memory, after which each thread owns four
// pixels and two output channels: three of every four horizontal neighbours are in the thread's
// own registers, the fourth comes from lane +-4 or, at a quarter boundary, from a shared-memory
// mailbox.  Vertical state (three horizontally filtered rows + the u = 2 taps of the previous row)
// stays in registers; nothing is recomputed except two warm-up rows per row band.  Output: bf16
// hi/lo words staged with stmatrix ([image][X % 8][X / 8][16 channels], 32-byte swizzle:
// conflict-free) and written by 5-d TMA stores (as LSU stores the 32-byte pieces of 64 pixels hit
// 64 different lines per instruction).
//
// Warp roles (384 threads): warps 0..7 = wgmma + epilogue — lane quarter q = warp / 2, channel
// half h = warp % 2 (8 of the tile's 16 output channels); warpgroup 2 = producer, which hands its
// registers to the two consumer warpgroups (setmaxnreg) and whose warp 8 issues the TMA loads.
#include <cstring>

#include "../../include/rewriting_b200.h"
#include "rw_common.cuh"

namespace rw {

struct UpFusedParams {
  int B, Cin, Cout, H, W;      // input resolution H x W (W a power of two, 4..128)
  const float* demod;          // [B, Cout]
  const float* bias;           // [Cout]
  const float* noise;          // [B, noise_bstride], indexed Y * 2W + X at OUTPUT resolution
  long long noise_bstride;
  const float* noise_w;        // device scalar
  const float* k4;             // 4x4 blur kernel (rank one)
  const float* next_scale;     // [B, Cout] style of the consuming layer
  void* next_hi;               // [B][2H+1][2W+1][Cout] bf16 planes (pad row / column zeroed)
  void* next_lo;
  // layer-level mode (the autograd op's forward): y_out != null writes the layer's own output
  // y [B][Cout][2H][2W] fp32 instead of the next layer's planes; demod / noise / noise_w may then
  // be null (= 1 / no noise) and act = 0 skips bias + leaky-ReLU
  float* y_out;
  int act;
  int ncg, nbands, nitems;     // filled by the launcher
  long long* debug_prof;       // per (CTA, epilogue warp) cycle counters [grid][8][16], or null
                               // (rw_debug_upconv_profile)
};

namespace {

constexpr int UM = 128;                 // input pixels per tile
constexpr int UNC = 16;                 // output channels per tile
constexpr int UN = 9 * UNC;             // GEMM N = 144
// k-block of 32 channels = one 64-byte swizzle row: a 34 KB stage, so that five fit next to the
// epilogue's buffers and the producer runs up to four k-blocks ahead of the MMAs
constexpr int UBK = 32;
constexpr int UK = 16;
constexpr int kUStages = 5;
constexpr int kUThreads = 384;       // warps 0-7: wgmma + epilogue, warpgroup 2: producer
constexpr int kUTmaWarp = 8;
// register split after setmaxnreg: 128 x 40 + 256 x 232 = 384 x 168, the launch allocation
constexpr uint32_t kUProducerRegs = 40;
constexpr uint32_t kUConsumerRegs = 232;
constexpr int kUABytes = UM * UBK * 2;  // one plane of A: 8 KB
constexpr int kUBBytes = UN * UBK * 2;  // one plane of B: 9 KB
constexpr int kUStageBytes = 2 * kUABytes + 2 * kUBBytes;    // 34 KB
constexpr int kUMailFloats = 2 * 2 * 4 * 2 * 32;             // [buf][half][quarter][side][32]
constexpr int kUOutSlotBytes = 64 * 32;                      // 64 output pixels x 16 channels, one plane
constexpr int kUOutQuarterBytes = 2 * kUOutSlotBytes;        // hi + lo slot of a lane quarter
constexpr int kUOutStageBytes = 4 * kUOutQuarterBytes;       // 16 KB
// accumulator exchange between the two warps of a lane quarter: [warp][tap][row half][lane] float2
constexpr int kUXchgFloat2 = 9 * 2 * 32;
constexpr int kUXchgBytes = 8 * kUXchgFloat2 * 8;
constexpr int kUSmemTotal =
    kUStages * kUStageBytes + kUMailFloats * 4 + kUOutStageBytes + kUXchgBytes + 512 + 256;
// 512-byte alignment serves the 64-byte swizzle atoms of the ring and the 32-byte swizzle of the
// output staging; the total must stay within the 227 KB a block may opt in to
static_assert(kUSmemTotal <= 232448, "upconv_fused: shared memory over the per-block limit");

struct UBarriers {
  uint64_t full[kUStages];
  uint64_t empty[kUStages];
};

__device__ __forceinline__ void tma_load_5d(void* smem_dst, const CUtensorMap* m, uint64_t* bar,
                                            int32_t c0, int32_t c1, int32_t c2, int32_t c3,
                                            int32_t c4) {
  asm volatile(
      "cp.async.bulk.tensor.5d.shared::cluster.global.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4, %5, %6, %7}], [%2];\n" ::"r"(smem_u32(smem_dst)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3),
      "r"(c4)
      : "memory");
}

// channel-pair arithmetic, one rounding per operation (the same results as the scalar operations)
__device__ __forceinline__ float2 f2add(float2 a, float2 b) {
  return make_float2(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y));
}
__device__ __forceinline__ float2 f2mul(float2 a, float2 b) {
  return make_float2(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y));
}
__device__ __forceinline__ float2 f2fma(float2 a, float2 b, float2 c) {
  return make_float2(__fmaf_rn(a.x, b.x, c.x), __fmaf_rn(a.y, b.y, c.y));
}
// producer-side wait: back off between polls so the spin does not take issue slots from the
// epilogue warps that share the scheduler
__device__ __forceinline__ void mbar_wait_relaxed(uint64_t* bar, uint32_t parity) {
  uint32_t spins = 0;
  while (!mbar_try_wait(bar, parity)) {
    __nanosleep(40);
    if (++spins > RW_SPIN_LIMIT) __trap();
  }
}

// vector accesses to the mailbox by 32-bit shared-window address
__device__ __forceinline__ void sts_v4(uint32_t a, float x, float y, float z, float w) {
  asm volatile("st.shared.v4.f32 [%0], {%1, %2, %3, %4};\n" ::"r"(a), "f"(x), "f"(y), "f"(z), "f"(w)
               : "memory");
}
__device__ __forceinline__ void lds_v4(uint32_t a, float& x, float& y, float& z, float& w) {
  asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];\n"
               : "=f"(x), "=f"(y), "=f"(z), "=f"(w)
               : "r"(a)
               : "memory");
}

// named barriers: 1, 2 = mailbox of a channel half; 3 + q = the two warps of lane quarter q
constexpr int kBarPair = 3;

struct UpItem {
  int bg, band, cg;
  int y_first, y_emit, y_end;   // steps y_first .. y_end-1; rows are emitted for y >= y_emit
};

__device__ __forceinline__ UpItem decode_item(int item, const UpFusedParams& p) {
  UpItem it;
  it.cg = item % p.ncg;
  const int r = item / p.ncg;
  it.band = r % p.nbands;
  it.bg = r / p.nbands;
  // bands partition the emitting steps [1, H + 1)
  const int ya = 1 + (it.band * p.H) / p.nbands;
  const int yb = 1 + ((it.band + 1) * p.H) / p.nbands;
  it.y_emit = ya;
  it.y_first = ya - 2 < 0 ? 0 : ya - 2;
  it.y_end = yb;
  return it;
}

// PROF = true: bring-up variant that accumulates, per epilogue warp, the cycles spent in each phase
// of a step (tools/prof_upconv.py) into p.debug_prof; the product launches PROF = false.
// NCHW = true: the layer-level op — writes y (fp32 NCHW, this layer's activation) instead of the
// next layer's operand planes (no staging, no TMA stores, no next-style scaling).
template <bool PROF, bool NCHW>
__global__ void __launch_bounds__(kUThreads, 1)
upconv_fused_kernel(const __grid_constant__ CUtensorMap map_a_hi,
                    const __grid_constant__ CUtensorMap map_a_lo,
                    const __grid_constant__ CUtensorMap map_w_hi,
                    const __grid_constant__ CUtensorMap map_w_lo,
                    const __grid_constant__ CUtensorMap map_o_hi,
                    const __grid_constant__ CUtensorMap map_o_lo, const UpFusedParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 511) &
                                             ~static_cast<uintptr_t>(511));
  float* mail = reinterpret_cast<float*>(smem + kUStages * kUStageBytes);
  uint8_t* out_stage = smem + kUStages * kUStageBytes + kUMailFloats * 4;
  float2* xchg = reinterpret_cast<float2*>(out_stage + kUOutStageBytes);
  UBarriers* bars = reinterpret_cast<UBarriers*>(out_stage + kUOutStageBytes + kUXchgBytes);

  // broadcast from lane 0: the compiler then knows the role branches are warp-uniform, which it
  // needs to give the consumer code the registers setmaxnreg grants
  const int warp = __shfl_sync(0xffffffffu, static_cast<int>(threadIdx.x >> 5), 0);
  const int lane = threadIdx.x & 31;
  const int kb_count = p.Cin / UBK;
  const int G = UM / p.W;                 // images per tile

  if (warp == kUTmaWarp && lane == 0) {
    tma_prefetch_desc(&map_a_hi);
    tma_prefetch_desc(&map_a_lo);
    tma_prefetch_desc(&map_w_hi);
    tma_prefetch_desc(&map_w_lo);
    tma_prefetch_desc(&map_o_hi);
    tma_prefetch_desc(&map_o_lo);
    for (int s = 0; s < kUStages; ++s) {
      mbar_init(&bars->full[s], 1);
      mbar_init(&bars->empty[s], 2);      // one arrival per consumer warpgroup
    }
    fence_mbar_init();
  }
  __syncthreads();

  // the consumer branch comes first: with the producer first, ptxas kept the consumer code at the
  // 168-register launch bound and spilled 480 B per thread
  if (warp < kUTmaWarp) {
    // ------------------------------ MMA + epilogue ----------------------------
    // warp w (0..7) issues, with its warpgroup, the wgmma rows 16 w .. 16 w + 15 of the tile = the
    // pixels j = 2 (w % 2) + i (i = 0, 1) of lane quarter q = w / 2, for all 144 columns; it keeps
    // channel half h = w % 2 and trades the other half with warp w ^ 1 through shared memory.
    // Then thread (g = lane / 4, c = lane % 4) of warp (q, h) owns the four adjacent pixels
    // 32 q + 4 g + j of the tile and the two output channels 8 h + 2 c + e of the item's sixteen:
    // "unit" u = 2 j + e indexes its eight (pixel, channel) pairs.
    setmaxnreg_inc<kUConsumerRegs>();
    const int wg = warp >> 2;
    const int q = warp >> 1;
    const int h = warp & 1;
    int stage = 0;
    uint32_t phase = 0;
    const int g = lane >> 2, c = lane & 3;
    const int W = p.W;
    const int T0 = q * 32 + 4 * g;             // tile index of the first of the four pixels
    const int x0 = T0 & (W - 1);
    const int img_in_tile = T0 / W;
    const int Ho = 2 * p.H, Wo = 2 * W;
    const bool first_x = (x0 == 0), last_x = (x0 + 4 == W);
    const bool cross = W > 32;                 // x-neighbours can live in another warp
    const bool mail_l = cross && g == 0 && !first_x, mail_r = cross && g == 7 && !last_x;
    // flipped blur kernel (upfirdn2d correlates with the flipped kernel), rank one:
    //   kf[a][b] = kv[a] * kh[b],  kv[a] = kf[a][0],  kh[b] = kf[0][b] / kf[0][0]
    float kv[4], kh[4];
    {
      const float k00 = __ldg(p.k4 + 15);
#pragma unroll
      for (int a = 0; a < 4; ++a) {
        kv[a] = __ldg(p.k4 + 15 - a * 4);
        kh[a] = __ldg(p.k4 + 15 - a) / k00;
      }
    }
    const float nw = (!NCHW || (p.noise != nullptr && p.noise_w != nullptr)) ? __ldg(p.noise_w) : 0.f;
    uint32_t step = 0;
    // mailbox across quarter boundaries (W > 32): slot (h, q, side) = 4 lanes (c) x 8 floats
    // [t row E/O][ro|le e0, e1, od e0, e1]; double buffered by step parity
    constexpr uint32_t kMailBufBytes = 2 * 4 * 2 * 32 * 4;
    const uint32_t mail_s = smem_u32(mail) + h * (4 * 2 * 32 * 4) + c * 32;
    const uint32_t post_r = mail_s + (q * 2 + 1) * 128, post_l = mail_s + (q * 2 + 0) * 128;
    const uint32_t read_l = mail_s + ((q - 1) * 2 + 1) * 128, read_r = mail_s + ((q + 1) * 2 + 0) * 128;
    // output staging of this quarter: slot 0 = `hi` plane, slot 1 = `lo` plane of ONE output row
    // segment (64 pixels x 16 channels), in the order the 5-d store map reads it,
    // [image][pixel % 8][pixel / 8][16 channels], 32-byte swizzle.  stmatrix row addresses: lane
    // supplies row g' = lane % 8 of matrix m = lane / 8 (= pixel 4 g' + m of the quarter).
    const uint32_t slot_s = smem_u32(out_stage) + q * kUOutQuarterBytes;
    uint32_t st_addr[2];
    {
      const int m = lane >> 3, gp = lane & 7;
      const int Wm = W < 32 ? W : 32;
      const int tl = 4 * gp + m;
      const int il = tl / W;                          // image inside the quarter (W < 32)
      const int xg = ((4 * gp) & (Wm - 1)) >> 2;
#pragma unroll
      for (int xi = 0; xi < 2; ++xi) {
        uint32_t a = slot_s + (((il * 8 + 2 * m + xi) * (Wm >> 2) + xg) << 5) + (h << 4);
        a ^= ((a >> 7) & 1u) << 4;
        st_addr[xi] = a;
      }
    }
    const CUtensorMap* omap = h ? &map_o_lo : &map_o_hi;   // warp (q, h) issues plane h's stores
    const uint32_t my_slot = slot_s + h * kUOutSlotBytes;
    const int o_xg = ((32 * q) & (W - 1)) >> 2;
    const int o_img = (32 * q) / W;
    long long prof_acc[16] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0};   // wait, tmem, combine+post+barrier, shuffles, fixups, hf, emit, steps, [emit split:] pack, slot wait, stage, issue

    for (int item = blockIdx.x; item < p.nitems; item += gridDim.x) {
      const UpItem it = decode_item(item, p);
      const int b0 = it.bg * G;
      const int b = b0 + img_in_tile;
      const bool img_ok = b < p.B;
      const int c0 = it.cg * UNC + h * 8 + 2 * c;     // first of this thread's 2 output channels
      const size_t chan_o = static_cast<size_t>(img_ok ? b : 0) * p.Cout + c0;
      float2 dm = make_float2(1.f, 1.f), bs = make_float2(0.f, 0.f), ns = make_float2(1.f, 1.f);
      if (!NCHW || p.demod != nullptr) dm = __ldg(reinterpret_cast<const float2*>(p.demod + chan_o));
      if (!NCHW || (p.act && p.bias != nullptr)) bs = __ldg(reinterpret_cast<const float2*>(p.bias + c0));
      if (!NCHW) ns = __ldg(reinterpret_cast<const float2*>(p.next_scale + chan_o));
      const bool has_noise = !NCHW || (p.noise != nullptr && p.noise_w != nullptr);
      // vertical state: u = 2 taps of the previous input row, and the horizontally filtered
      // t rows 2y-3 (w0), 2y-2 (w1), 2y-1 (w2); each [2 output columns][8 units]
      // (all per-pixel quantities are float2 = the thread's channel pair: the FIRs and the
      // activation run on packed FFMA2 / FADD2 / FMUL2, bit-identical to the scalar operations)
      float2 c20[4], c21[4], c22[4];
      float2 w0[2][4], w1[2][4], w2[2][4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        c20[j] = c21[j] = c22[j] = make_float2(0.f, 0.f);
        w0[0][j] = w0[1][j] = w1[0][j] = w1[1][j] = w2[0][j] = w2[1][j] = make_float2(0.f, 0.f);
      }
      const float* nrow_base = p.noise + static_cast<size_t>(img_ok ? b : 0) * p.noise_bstride + 2 * x0;
      __nv_bfloat16* out_hi = static_cast<__nv_bfloat16*>(p.next_hi);
      __nv_bfloat16* out_lo = static_cast<__nv_bfloat16*>(p.next_lo);
      const size_t img_row0 = static_cast<size_t>(img_ok ? b : 0) * (Ho + 1);

      for (int y = it.y_first; y < it.y_end; ++y, ++step) {
        const bool rows_out = (y >= it.y_emit);   // warp-, pair- and CTA-uniform
        const bool emit = rows_out && img_ok;
        if (emit && c < 2 && has_noise) {          // noise of the two output rows -> L1
          const float* np = nrow_base + static_cast<size_t>(2 * y - 2 + c) * Wo;
          asm volatile("prefetch.global.L1 [%0];\n" ::"l"(np));
        }
        long long tq[8];
        if constexpr (PROF) tq[0] = clock64();
        float2 P[9][4];                                              // [tap][pixel j] (e0, e1)
        {
          float d[72];
          // one wgmma group stays in flight: a stage is released once the group after it has
          // been issued and the group that read it has completed
          int held = -1;
          for (int kb = 0; kb < kb_count; ++kb) {
            mbar_wait(&bars->full[stage], phase);
            const uint32_t sa = smem_u32(smem + stage * kUStageBytes);
            const uint64_t da_hi = make_smem_desc(sa + wg * (kUABytes / 2), 16, 512, 2);
            const uint64_t da_lo = make_smem_desc(sa + kUABytes + wg * (kUABytes / 2), 16, 512, 2);
            const uint64_t db_hi = make_smem_desc(sa + 2 * kUABytes, 16, 512, 2);
            const uint64_t db_lo = make_smem_desc(sa + 2 * kUABytes + kUBBytes, 16, 512, 2);
            wgmma_fence();
#pragma unroll
            for (int kk = 0; kk < UBK / UK; ++kk) {
              const uint64_t adv = static_cast<uint64_t>((kk * UK * 2) >> 4);
              wgmma_m64n144<0, 0>(d, da_lo + adv, db_hi + adv, (kb | kk) != 0);
              wgmma_m64n144<0, 0>(d, da_hi + adv, db_lo + adv, 1u);
              wgmma_m64n144<0, 0>(d, da_hi + adv, db_hi + adv, 1u);
            }
            wgmma_commit();
            wgmma_wait<1>();
            if (held >= 0 && (threadIdx.x & 127) == 0) mbar_arrive(&bars->empty[held]);
            held = stage;
            if (++stage == kUStages) { stage = 0; phase ^= 1u; }
          }
          wgmma_wait<0>();
          if ((threadIdx.x & 127) == 0) mbar_arrive(&bars->empty[held]);
          if constexpr (PROF) tq[1] = clock64();
          // accumulator columns: [channel half][tap][8 channels] (prep_weights, transpose_io = 2);
          // every register index is a compile-time constant (a run-time one puts d in local memory)
          float2* to = xchg + (warp ^ 1) * kUXchgFloat2 + lane;
#pragma unroll
          for (int t = 0; t < 9; ++t)
#pragma unroll
            for (int i = 0; i < 2; ++i)
              to[(t * 2 + i) * 32] = h ? make_float2(d[4 * t + 2 * i], d[4 * t + 2 * i + 1])
                                       : make_float2(d[4 * (9 + t) + 2 * i], d[4 * (9 + t) + 2 * i + 1]);
          named_bar_sync(kBarPair + q, 64);
          const float2* from = xchg + warp * kUXchgFloat2 + lane;
#pragma unroll
          for (int t = 0; t < 9; ++t)
#pragma unroll
            for (int i = 0; i < 2; ++i) {
              const float2 own = h ? make_float2(d[4 * (9 + t) + 2 * i], d[4 * (9 + t) + 2 * i + 1])
                                   : make_float2(d[4 * t + 2 * i], d[4 * t + 2 * i + 1]);
              const float2 other = from[(t * 2 + i) * 32];
              P[t][i] = h ? other : own;               // pixels j = 0, 1 come from the h = 0 warp
              P[t][2 + i] = h ? own : other;           // pixels j = 2, 3 from the h = 1 warp
            }
          named_bar_sync(kBarPair + q, 64);          // the slot is free for the next step
        }
        if constexpr (PROF) tq[2] = clock64();

        // t rows E = 2y, O = 2y+1 in pixel-local pieces (see the header comment):
        //   E.e[x] = leE[x] + rE[x-1], E.o[x] = oE[x];   O.e[x] = leO[x] + rO[x-1], O.o[x] = oO[x]
        float2 le[2][4], ro[2][4], od[2][4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          le[0][j] = f2add(P[0][j], c20[j]);
          od[0][j] = f2add(P[1][j], c21[j]);
          ro[0][j] = f2add(P[2][j], c22[j]);
          le[1][j] = P[3][j];
          od[1][j] = P[4][j];
          ro[1][j] = P[5][j];
          c20[j] = P[6][j];
          c21[j] = P[7][j];
          c22[j] = P[8][j];
        }
        // mailbox across quarter boundaries: the g = 7 lanes post (ro, od) of their last pixel for
        // the right-hand quarter, the g = 0 lanes post (le, od) of their first pixel
        const uint32_t mbo = (step & 1u) * kMailBufBytes;
        if (cross) {
          if (g == 7) {
            sts_v4(post_r + mbo, ro[0][3].x, ro[0][3].y, od[0][3].x, od[0][3].y);
            sts_v4(post_r + mbo + 16, ro[1][3].x, ro[1][3].y, od[1][3].x, od[1][3].y);
          }
          if (g == 0) {
            sts_v4(post_l + mbo, le[0][0].x, le[0][0].y, od[0][0].x, od[0][0].y);
            sts_v4(post_l + mbo + 16, le[1][0].x, le[1][0].y, od[1][0].x, od[1][0].y);
          }
        }
        if constexpr (PROF) tq[3] = clock64();
        // the only pieces that come from other threads: left (ro, od) of pixel 4g-1 (lane - 4),
        // right (le, od) of pixel 4g+4 (lane + 4); [t row]
        float2 Lro[2], Lod[2], Rle[2], Rod[2];
#pragma unroll
        for (int r = 0; r < 2; ++r) {
          Lro[r].x = __shfl_up_sync(0xffffffffu, ro[r][3].x, 4);
          Lro[r].y = __shfl_up_sync(0xffffffffu, ro[r][3].y, 4);
          Lod[r].x = __shfl_up_sync(0xffffffffu, od[r][3].x, 4);
          Lod[r].y = __shfl_up_sync(0xffffffffu, od[r][3].y, 4);
          Rle[r].x = __shfl_down_sync(0xffffffffu, le[r][0].x, 4);
          Rle[r].y = __shfl_down_sync(0xffffffffu, le[r][0].y, 4);
          Rod[r].x = __shfl_down_sync(0xffffffffu, od[r][0].x, 4);
          Rod[r].y = __shfl_down_sync(0xffffffffu, od[r][0].y, 4);
        }
        if constexpr (PROF) tq[6] = clock64();
        // horizontal FIR; pixels j = 1, 2 need nothing from outside the thread and are filtered
        // BEFORE the mailbox barrier (its wait is skew between the four quarter warps)
        const float2 kh0 = make_float2(kh[0], kh[0]), kh1 = make_float2(kh[1], kh[1]),
                     kh2 = make_float2(kh[2], kh[2]), kh3 = make_float2(kh[3], kh[3]);
        float2 hf[2][2][4];                      // [t row E/O][output column 2x / 2x+1][pixel j]
        auto hfir = [&](int r, int j, float2 l_ro, float2 l_od, float2 r_le, float2 r_od) {
          const float2 e0 = f2add(le[r][j], l_ro);    // t col 2x
          const float2 e1 = f2add(r_le, ro[r][j]);    // t col 2x+2
          const float2 o0 = od[r][j];                      // t col 2x+1
          hf[r][0][j] = f2fma(kh3, e1, f2fma(kh2, o0, f2fma(kh1, e0, f2mul(kh0, l_od))));
          hf[r][1][j] = f2fma(kh3, r_od, f2fma(kh2, e1, f2fma(kh1, o0, f2mul(kh0, e0))));
        };
#pragma unroll
        for (int r = 0; r < 2; ++r) {
          hfir(r, 1, ro[r][0], od[r][0], le[r][2], od[r][2]);
          hfir(r, 2, ro[r][1], od[r][1], le[r][3], od[r][3]);
        }
        if (cross) named_bar_sync(1 + h, 128);
        if (first_x) {                            // image edge: nothing to the left
#pragma unroll
          for (int r = 0; r < 2; ++r) Lro[r] = Lod[r] = make_float2(0.f, 0.f);
        } else if (mail_l) {                      // left neighbour lives in the previous quarter
          lds_v4(read_l + mbo, Lro[0].x, Lro[0].y, Lod[0].x, Lod[0].y);
          lds_v4(read_l + mbo + 16, Lro[1].x, Lro[1].y, Lod[1].x, Lod[1].y);
        }
        if (last_x) {
#pragma unroll
          for (int r = 0; r < 2; ++r) Rle[r] = Rod[r] = make_float2(0.f, 0.f);
        } else if (mail_r) {
          lds_v4(read_r + mbo, Rle[0].x, Rle[0].y, Rod[0].x, Rod[0].y);
          lds_v4(read_r + mbo + 16, Rle[1].x, Rle[1].y, Rod[1].x, Rod[1].y);
        }
        if constexpr (PROF) tq[7] = clock64();
#pragma unroll
        for (int r = 0; r < 2; ++r) {
          hfir(r, 0, Lro[r], Lod[r], le[r][1], od[r][1]);
          hfir(r, 3, ro[r][2], od[r][2], Rle[r], Rod[r]);
        }
        if constexpr (PROF) tq[4] = clock64();
        if (rows_out) {
          // output rows Y0 = 2y-2 (t rows 2y-3..2y) and Y1 = 2y-1 (t rows 2y-2..2y+1): each is
          // packed to bf16 hi/lo words, staged with stmatrix and stored by TMA (the 32-byte pieces
          // of 64 pixels scatter over 64 lines: as LSU stores they cost a third of the step)
#pragma unroll
          for (int yi = 0; yi < 2; ++yi) {
            const int Y = 2 * y - 2 + yi;
            float nz[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
            if (has_noise) {
              const float4* np = reinterpret_cast<const float4*>(nrow_base + static_cast<size_t>(Y) * Wo);
              const float4 a4 = __ldg(np), b4 = __ldg(np + 1);
              nz[0] = a4.x; nz[1] = a4.y; nz[2] = a4.z; nz[3] = a4.w;
              nz[4] = b4.x; nz[5] = b4.y; nz[6] = b4.z; nz[7] = b4.w;
            }
            uint32_t hw[2][4], lw[2][4];
            float2 yv[2][4];                      // NCHW mode: [xi][j] activation of the channel pair
            long long te[7];
            if constexpr (PROF) te[0] = clock64();
            const float2 kv0 = make_float2(kv[0], kv[0]), kv1 = make_float2(kv[1], kv[1]),
                         kv2 = make_float2(kv[2], kv[2]), kv3 = make_float2(kv[3], kv[3]);
#pragma unroll
            for (int xi = 0; xi < 2; ++xi) {
#pragma unroll
              for (int j = 0; j < 4; ++j) {
                const float nzv = nw * nz[2 * j + xi];
                float2 v;
                if (yi == 0)
                  v = f2fma(kv3, hf[0][xi][j],
                                 f2fma(kv2, w2[xi][j], f2fma(kv1, w1[xi][j], f2mul(kv0, w0[xi][j]))));
                else
                  v = f2fma(kv3, hf[1][xi][j],
                                 f2fma(kv2, hf[0][xi][j], f2fma(kv1, w2[xi][j], f2mul(kv0, w1[xi][j]))));
                v = f2add(f2fma(v, dm, make_float2(nzv, nzv)), bs);
                if (!NCHW || p.act) {
                  const float2 t02 = f2mul(v, make_float2(0.2f, 0.2f));
                  v = f2mul(make_float2(fmaxf(v.x, t02.x), fmaxf(v.y, t02.y)),
                                 make_float2(1.4142135623730951f, 1.4142135623730951f));
                }
                if constexpr (NCHW) {
                  yv[xi][j] = v;
                } else {
                  const float2 kk = f2mul(ns, v);
                  const __nv_bfloat162 hh = __floats2bfloat162_rn(kk.x, kk.y);
                  const uint32_t hu = *reinterpret_cast<const uint32_t*>(&hh);
                  const __nv_bfloat162 ll = __floats2bfloat162_rn(
                      kk.x - __uint_as_float(hu << 16), kk.y - __uint_as_float(hu & 0xffff0000u));
                  hw[xi][j] = hu;
                  lw[xi][j] = *reinterpret_cast<const uint32_t*>(&ll);
                }
              }
            }
            if constexpr (NCHW) {
              // 8 consecutive output pixels (X = 2 x0 + 2 j + xi) of each channel: 32 contiguous
              // bytes per (row, channel); the eight g lanes of a channel pair cover 256 bytes
              if (img_ok) {
                float* yrow = p.y_out + ((static_cast<size_t>(b) * p.Cout + c0) * Ho + Y) * Wo + 2 * x0;
                const size_t cstride = static_cast<size_t>(Ho) * Wo;
                *reinterpret_cast<float4*>(yrow) = make_float4(yv[0][0].x, yv[1][0].x, yv[0][1].x, yv[1][1].x);
                *reinterpret_cast<float4*>(yrow + 4) = make_float4(yv[0][2].x, yv[1][2].x, yv[0][3].x, yv[1][3].x);
                *reinterpret_cast<float4*>(yrow + cstride) = make_float4(yv[0][0].y, yv[1][0].y, yv[0][1].y, yv[1][1].y);
                *reinterpret_cast<float4*>(yrow + cstride + 4) =
                    make_float4(yv[0][2].y, yv[1][2].y, yv[0][3].y, yv[1][3].y);
              }
              continue;
            }
            // the slots are free once the previous row's stores have read them
            if constexpr (PROF) te[1] = clock64();
            if (lane == 0) tma_store_wait_read_n<0>();
            named_bar_sync(kBarPair + q, 64);
            if constexpr (PROF) te[2] = clock64();
#pragma unroll
            for (int xi = 0; xi < 2; ++xi) {
              stmatrix_x4(st_addr[xi], hw[xi]);
              stmatrix_x4(st_addr[xi] + kUOutSlotBytes, lw[xi]);
            }
            if constexpr (PROF) te[5] = clock64();
            fence_proxy_async_smem();
            if constexpr (PROF) te[6] = clock64();
            named_bar_sync(kBarPair + q, 64);
            if constexpr (PROF) te[3] = clock64();
            // warp (q, h) issues plane h's store.  (Two dedicated store warps instead, fed through
            // arrive/sync barrier pairs, were slower: 922 vs 830 us at layer 13.)
            if (lane == 0) tma_store_5d(omap, my_slot, it.cg * UNC, o_xg, 0, Y, b0 + o_img);
            if constexpr (PROF) {
              te[4] = clock64();
#pragma unroll
              for (int i = 0; i < 4; ++i) prof_acc[8 + i] += te[i + 1] - te[i];
              prof_acc[12] += te[5] - te[2];
              prof_acc[13] += te[6] - te[5];
              prof_acc[14] += te[3] - te[6];
            }
            if (img_ok && last_x && c == 0) {       // zero pad column of the output grid
              const size_t off = ((img_row0 + Y) * (Wo + 1) + Wo) * p.Cout + it.cg * UNC + h * 8;
              *reinterpret_cast<uint4*>(out_hi + off) = make_uint4(0u, 0u, 0u, 0u);
              *reinterpret_cast<uint4*>(out_lo + off) = make_uint4(0u, 0u, 0u, 0u);
            }
          }
        }
        if (!NCHW && emit && y == p.H) {           // last step of the image: zero pad row
          const size_t prow = (img_row0 + Ho) * (Wo + 1);
#pragma unroll
          for (int i = 0; i < 3; ++i) {
            // lane c covers output pixels 2 x0 + 2c, +1; the last lane also the pad corner
            if (i < 2 || (last_x && c == 3)) {
              const size_t off = (prow + 2 * x0 + 2 * c + i) * p.Cout + it.cg * UNC + h * 8;
              *reinterpret_cast<uint4*>(out_hi + off) = make_uint4(0u, 0u, 0u, 0u);
              *reinterpret_cast<uint4*>(out_lo + off) = make_uint4(0u, 0u, 0u, 0u);
            }
          }
        }
        if constexpr (PROF) {
          tq[5] = clock64();
          prof_acc[0] += tq[1] - tq[0];
          prof_acc[1] += tq[2] - tq[1];
          prof_acc[2] += tq[3] - tq[2];
          prof_acc[3] += tq[6] - tq[3];
          prof_acc[4] += tq[7] - tq[6];
          prof_acc[5] += tq[4] - tq[7];
          prof_acc[6] += tq[5] - tq[4];
          prof_acc[7] += 1;
        }
        // slide the vertical window: rows 2y-1, 2y, 2y+1 become 2(y+1)-3 .. 2(y+1)-1
#pragma unroll
        for (int xi = 0; xi < 2; ++xi)
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            w0[xi][j] = w2[xi][j];
            w1[xi][j] = hf[0][xi][j];
            w2[xi][j] = hf[1][xi][j];
          }
      }
    }
    if (!NCHW && lane == 0) tma_store_wait_all();
    if constexpr (PROF) {
      if (lane == 0 && p.debug_prof != nullptr) {
        long long* dst = p.debug_prof + (static_cast<size_t>(blockIdx.x) * 8 + warp) * 16;
#pragma unroll
        for (int i = 0; i < 16; ++i) dst[i] = prof_acc[i];
      }
    }
  } else {
    // ------------------------------ TMA producer ------------------------------
    setmaxnreg_dec<kUProducerRegs>();
    if (warp != kUTmaWarp) return;
    // The A tile's rows are PERMUTED: inside every 32-pixel quarter, tile row 8 j + g holds pixel
    // 4 g + j (j < 4, g < 8), so that the wgmma accumulator rows of a warp pair hold, per thread,
    // four ADJACENT pixels.  The permutation is free: the tensor map lists the key planes' dimensions as
    // (channel, x / 4 % 8, x % 4, x / 32, row) — TMA fills shared memory in that order — so one
    // load still brings a whole image row (W >= 32; W < 32: (channel, x / 4, image, x % 4, y), one
    // load per quarter).  [Loading the eight rows of each (quarter, j) separately — 32 one-KB
    // boxes per plane and stage, strided or not — fed the MMAs at a third of their rate.]
    int stage = 0;
    uint32_t phase = 0;
    const bool wide = p.W >= 32;
    const int nop = wide ? G : 4;                  // loads per plane and stage
    const int plane = lane / nop, idx = lane % nop;
    const CUtensorMap* amap = plane ? &map_a_lo : &map_a_hi;
    const CUtensorMap* wmap = (lane & 1) ? &map_w_lo : &map_w_hi;
    const uint32_t a_off = plane * kUABytes + idx * (kUABytes / nop);
    for (int item = blockIdx.x; item < p.nitems; item += gridDim.x) {
      const UpItem it = decode_item(item, p);
      const int b0 = it.bg * G;
      const int wrow = it.cg * UN;
      for (int y = it.y_first; y < it.y_end; ++y) {
        for (int kb = 0; kb < kb_count; ++kb) {
          if (lane == 0) {
            mbar_wait_relaxed(&bars->empty[stage], phase ^ 1u);
            mbar_expect_tx(&bars->full[stage], kUStageBytes);
          }
          __syncwarp();
          uint8_t* st = smem + stage * kUStageBytes;
          if (lane < 2 * nop) {
            if (wide)
              tma_load_5d(st + a_off, amap, &bars->full[stage], kb * UBK, 0, 0, 0,
                          (b0 + idx) * (p.H + 1) + y);
            else
              tma_load_5d(st + a_off, amap, &bars->full[stage], kb * UBK, 0, b0 + idx * (32 / p.W), 0, y);
          } else if (lane >= 30) {
            tma_load_2d(st + 2 * kUABytes + (lane & 1) * kUBBytes, wmap, &bars->full[stage], kb * UBK,
                        wrow);
          }
          if (++stage == kUStages) { stage = 0; phase ^= 1u; }
        }
      }
    }
    return;
  }

}

}  // namespace

// weights: bf16 hi/lo planes [Cout/16][channel half][9 taps][8][Cin]  (rw_prep_weights, transpose_io = 2)
static int upconv_fused_launch(const UpFusedParams& pin, const void* a_hi, const void* a_lo,
                               const void* w_hi, const void* w_lo, cudaStream_t stream) {
  UpFusedParams p = pin;
  const int W = p.W, H = p.H;
  if (W < 4 || W > UM || (W & (W - 1)) != 0 || H < 1 || p.Cin % UBK != 0 || p.Cout % UNC != 0 ||
      p.B < 1) {
    set_last_error("upconv_fused: unsupported shape B=%d Cin=%d Cout=%d H=%d W=%d", p.B, p.Cin,
                   p.Cout, H, W);
    return RW_ERR_BAD_ARG;
  }
  const int G = UM / W;
  const int nbg = (p.B + G - 1) / G;
  p.ncg = p.Cout / UNC;
  const int sms = device_sm_count();
  // row bands: more items balance the static round-robin better, every band costs two warm-up
  // rows; pick the cheapest makespan
  int best = 1;
  long long best_cost = -1;
  for (int nb = 1; nb <= 32 && H / nb >= 4; nb *= 2) {
    const long long items = static_cast<long long>(nbg) * p.ncg * nb;
    const long long waves = (items + sms - 1) / sms;
    const long long cost = waves * ((H + nb - 1) / nb + 2);
    if (best_cost < 0 || cost < best_cost) {
      best_cost = cost;
      best = nb;
    }
  }
  p.nbands = best;
  p.nitems = nbg * p.ncg * p.nbands;

  CUtensorMap ma_hi, ma_lo, mw_hi, mw_lo, mo_hi, mo_lo;
  // key planes [B][H+1][W+1][Cin] with the dimensions listed so that shared memory receives the
  // rows of a 32-pixel quarter in the order 8 (x % 4) + x / 4 (see the producer)
  const uint32_t Wm = W < 32 ? W : 32;
  const uint64_t kpx = static_cast<uint64_t>(p.Cin) * 2;
  const uint64_t krow = static_cast<uint64_t>(W + 1) * kpx;
  int rc;
  if (W >= 32) {
    // (channel, x / 4 % 8, x % 4, x / 32, image * (H + 1) + y)
    const uint64_t dims[5] = {static_cast<uint64_t>(p.Cin), 8, 4, static_cast<uint64_t>(W / 32),
                              static_cast<uint64_t>(p.B) * (H + 1)};
    const uint64_t str[4] = {4 * kpx, kpx, 32 * kpx, krow};
    const uint32_t box[5] = {UBK, 8u, 4u, static_cast<uint32_t>(W / 32), 1u};
    if ((rc = make_tmap_nd_bf16(&ma_hi, a_hi, 5, dims, str, box, nullptr, 3))) return rc;
    if ((rc = make_tmap_nd_bf16(&ma_lo, a_lo, 5, dims, str, box, nullptr, 3))) return rc;
  } else {
    // (channel, x / 4, image, x % 4, y)
    const uint64_t dims[5] = {static_cast<uint64_t>(p.Cin), static_cast<uint64_t>(W / 4),
                              static_cast<uint64_t>(p.B), 4, static_cast<uint64_t>(H + 1)};
    const uint64_t str[4] = {4 * kpx, static_cast<uint64_t>(H + 1) * krow, kpx, krow};
    const uint32_t box[5] = {UBK, static_cast<uint32_t>(W / 4), 32u / Wm, 4u, 1u};
    if ((rc = make_tmap_nd_bf16(&ma_hi, a_hi, 5, dims, str, box, nullptr, 3))) return rc;
    if ((rc = make_tmap_nd_bf16(&ma_lo, a_lo, 5, dims, str, box, nullptr, 3))) return rc;
  }
  // output planes [B][Ho+1][Wo+1][Cout] seen as (channel, X / 8, X % 8, Y, image): one store = 16
  // channels of a quarter's 64 output pixels, staged as [image][X % 8][X / 8][16 ch] so that the
  // eight row addresses of a stmatrix fall into different banks (32-byte swizzle)
  if (p.y_out == nullptr) {
    const uint64_t Wo = 2 * static_cast<uint64_t>(W), Ho = 2 * static_cast<uint64_t>(H);
    const uint64_t px = static_cast<uint64_t>(p.Cout) * 2;
    const uint64_t od[5] = {static_cast<uint64_t>(p.Cout), Wo / 8, 8, Ho + 1, static_cast<uint64_t>(p.B)};
    const uint64_t os[4] = {8 * px, px, (Wo + 1) * px, (Ho + 1) * (Wo + 1) * px};
    const uint32_t ob[5] = {UNC, Wm / 4, 8u, 1u, 32u / Wm};
    if ((rc = make_tmap_nd_bf16(&mo_hi, p.next_hi, 5, od, os, ob, nullptr, 1))) return rc;
    if ((rc = make_tmap_nd_bf16(&mo_lo, p.next_lo, 5, od, os, ob, nullptr, 1))) return rc;
  } else {                                  // layer-level mode stores y directly: maps unused
    if ((reinterpret_cast<uintptr_t>(p.y_out) & 15u) != 0) {
      set_last_error("upconv_fused: y must be 16-byte aligned");
      return RW_ERR_BAD_ARG;
    }
    mo_hi = ma_hi;
    mo_lo = ma_lo;
  }
  const uint64_t wdims[2] = {static_cast<uint64_t>(p.Cin), static_cast<uint64_t>(p.ncg) * UN};
  const uint64_t wstr[1] = {static_cast<uint64_t>(p.Cin) * 2};
  const uint32_t wbox[2] = {UBK, UN};
  if ((rc = make_tmap_nd_bf16(&mw_hi, w_hi, 2, wdims, wstr, wbox, nullptr, 3))) return rc;
  if ((rc = make_tmap_nd_bf16(&mw_lo, w_lo, 2, wdims, wstr, wbox, nullptr, 3))) return rc;
  const int grid = p.nitems < sms ? p.nitems : sms;
  auto launch = [&](auto kernel, bool& attr_done) -> int {
    if (!attr_done) {
      int e = check_cuda(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                              kUSmemTotal),
                         "upconv_fused smem attr");
      if (e) return e;
      attr_done = true;
    }
    kernel<<<grid, kUThreads, kUSmemTotal, stream>>>(ma_hi, ma_lo, mw_hi, mw_lo, mo_hi, mo_lo, p);
    return check_cuda(cudaGetLastError(), "upconv_fused launch");
  };
  static bool attr_prof = false, attr_planes = false, attr_nchw = false;
  if (p.debug_prof != nullptr) return launch(upconv_fused_kernel<true, false>, attr_prof);
  if (p.y_out != nullptr) return launch(upconv_fused_kernel<false, true>, attr_nchw);
  return launch(upconv_fused_kernel<false, false>, attr_planes);
}

// the fused upsampling conv's parameters common to its entry points; next_* are null in
// layer-level mode (y_out)
static UpFusedParams up_fused_params(int B, int Cin, int Cout, int H, int W, const float* demod,
                                     const float* kernel4x4, const float* noise,
                                     long long noise_bstride, const float* noise_w,
                                     const float* bias, const float* next_scale, void* next_hi,
                                     void* next_lo) {
  UpFusedParams p;
  memset(&p, 0, sizeof(p));
  p.B = B; p.Cin = Cin; p.Cout = Cout; p.H = H; p.W = W;
  p.demod = demod; p.bias = bias; p.noise = noise; p.noise_bstride = noise_bstride;
  p.noise_w = noise_w; p.k4 = kernel4x4; p.next_scale = next_scale;
  p.next_hi = next_hi; p.next_lo = next_lo;
  return p;
}

}  // namespace rw

using namespace rw;

extern "C" {

int rw_modconv_up_fused(const void* kp_hi, const void* kp_lo, const void* wt_hi, const void* wt_lo,
                        const float* demod, const float* kernel4x4, const float* noise,
                        long long noise_bstride, const float* noise_w, const float* bias,
                        const float* next_scale, void* next_hi, void* next_lo, int B, int Cin,
                        int Cout, int H, int W, rw_stream_t stream) {
  if (!kp_hi || !kp_lo || !wt_hi || !wt_lo || !demod || !kernel4x4 || !noise || !noise_w || !bias ||
      !next_scale || !next_hi || !next_lo || (noise_bstride & 1)) {
    set_last_error("rw_modconv_up_fused: bad argument");
    return RW_ERR_BAD_ARG;
  }
  const UpFusedParams p = up_fused_params(B, Cin, Cout, H, W, demod, kernel4x4, noise,
                                          noise_bstride, noise_w, bias, next_scale, next_hi, next_lo);
  return upconv_fused_launch(p, kp_hi, kp_lo, wt_hi, wt_lo, stream);
}

int rw_modconv_up_fused_y(const void* kp_hi, const void* kp_lo, const void* wt_hi, const void* wt_lo,
                          const float* demod, const float* kernel4x4, const float* noise,
                          long long noise_bstride, const float* noise_w, const float* bias, int act,
                          float* y, int B, int Cin, int Cout, int H, int W, rw_stream_t stream) {
  if (!kp_hi || !kp_lo || !wt_hi || !wt_lo || !kernel4x4 || !y || (noise && (noise_bstride & 3)) ||
      ((noise != nullptr) != (noise_w != nullptr))) {
    set_last_error("rw_modconv_up_fused_y: bad argument");
    return RW_ERR_BAD_ARG;
  }
  UpFusedParams p = up_fused_params(B, Cin, Cout, H, W, demod, kernel4x4, noise, noise_bstride,
                                    noise_w, bias, nullptr, nullptr, nullptr);
  p.y_out = y;
  p.act = act;
  return upconv_fused_launch(p, kp_hi, kp_lo, wt_hi, wt_lo, stream);
}

int rw_debug_upconv_profile(const void* kp_hi, const void* kp_lo, const void* wt_hi,
                            const void* wt_lo, const float* demod, const float* kernel4x4,
                            const float* noise, long long noise_bstride, const float* noise_w,
                            const float* bias, const float* next_scale, void* next_hi, void* next_lo,
                            int B, int Cin, int Cout, int H, int W, long long* prof_out,
                            rw_stream_t stream) {
  UpFusedParams p = up_fused_params(B, Cin, Cout, H, W, demod, kernel4x4, noise, noise_bstride,
                                    noise_w, bias, next_scale, next_hi, next_lo);
  p.debug_prof = prof_out;
  return upconv_fused_launch(p, kp_hi, kp_lo, wt_hi, wt_lo, stream);
}

}  // extern "C"
