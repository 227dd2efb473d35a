// conv_tc.cu — wgmma implicit-GEMM over the padded-flat key layout ("row-GEMM").
//
//   acc[p, o] = sum_{tap} sum_{i} KP[p + shift(tap), i] * Wt[o, tap, i]
//
// KP is the style-modulated key  k = style (.) x  (reference: ApplyStyle,
// utils/stylegan2/models.py:616-620) stored channels-last as two bf16 planes
// (hi, lo) over a zero-padded flat pixel grid: one image = (H+1) x (W+1)
// positions, column W and row H are zero, so every 3x3 neighbour (and every
// conv_transpose phase neighbour) is a plain row shift of the same 2-D matrix
// and zero padding is implicit.  Wt is scale*W (models.py:315-319) as bf16
// hi/lo planes [Cout][tap][Cin].  Three MMAs per k-step (hi*hi + lo*hi + hi*lo)
// reproduce the fp32 conv of the reference to ~2^-17 relative (SURVEY.md §7:
// single-pass bf16/tf32 fails the 1e-3 pixel tolerance, 3xBF16 passes).
//
// Epilogue (fused, per accumulator element) follows DemodulatedConv2dF /
// NoiseInjectionF / FusedLeakyReLUF (models.py:320-328, 539-546;
// op/fused_bias_act_kernel.cu:27-47):
//   y = lrelu(acc * scale[b,o] + noise_w * noise[b, y*W+x] + bias[o], 0.2) * sqrt(2)
// each term optional, so the same kernel serves the un-fused `dconv` leaf of a
// nethook-split layer, the conv_transpose phases of an up layer and dgrad.
//
// Warp roles (384 threads): warpgroups 0 and 1 each issue wgmma for 64 of the tile's 128 rows and
// run the epilogue on their register accumulators, raised to 232 registers by setmaxnreg;
// warpgroup 2 is the producer, lowered to 40, whose warp 8 issues the TMA loads.  A 6-stage ring
// of 32 KB stages (BK = 32, 64-byte swizzle; BN = 64: 7 x 24 KB); the consumers keep one wgmma
// group in flight and release each stage one k-block behind.  The next layer's planes leave the
// epilogue through per-warp shared-memory slots and TMA stores.
// Persistent 2-CTA clusters: the two CTAs take adjacent m-tiles with the same (phase, n), so they
// read the same weight tile on every k-block; each loads one 64-row half of it and multicasts the
// half to both, cutting each CTA's L2 reads per k-block from 32 KB to 24 KB.
#include <cstdlib>
#include <cstring>

#include "../../include/rewriting_b200.h"
#include "rw_common.cuh"

namespace rw {

struct ConvTcParams {
  int rows;          // padded-flat rows = B * Hp * Wp  (GEMM M)
  int Cin;           // GEMM K per tap
  int Cout;          // GEMM N
  // Up to 4 "phases" share one launch (the 4 polyphase components of a stride-2
  // conv_transpose): tile index = (m, n, phase) with phase fastest, so the CTAs that
  // run concurrently read the same A tiles (L2 hits instead of 4 DRAM passes).
  int nphase;
  int ph_ntaps[4];
  int ph_shift[4][9];   // row shift applied to the A operand for this tap
  int ph_kofs[4][9];    // column offset of this tap inside the weight matrix
  int ph_acol[4][9];    // column offset of this tap inside the A planes (0 unless A holds
                        // several channel-concatenated tensors, e.g. the 4 gradient phases)
  int a_cols;           // total columns of the A planes (0 -> Cin)
  int ph_Hv[4], ph_Wv[4];       // valid output extent inside the padded grid
  long long ph_out_ofs[4];      // element offset of this phase's output origin
  int Hp, Wp;        // padded grid of one image
  int B;             // batch (only needed for the rgb partial layout)
  // epilogue
  const float* scale_bo;  // [B, Cout] per-sample per-channel scale (demod / style) or null
  const float* bias;      // [Cout] or null
  const float* noise;     // [B, noise_bstride] or null, indexed y*Wv + x
  long long noise_bstride;
  const float* noise_w;   // device scalar (read by the kernel: no host sync per layer)
  int act;                // 1 -> leaky_relu(0.2) * act_gain
  float act_gain;         // 0 -> sqrt(2) (FusedLeakyReLU); ProgGAN's nn.LeakyReLU uses 1
  float* out;             // may be null when only planes / rgb partials are wanted
  long long out_sb, out_sc, out_sy, out_sx;  // element strides: batch, channel, y, x
  // out_mode 0: strided (NCHW-like) store at valid positions only
  // out_mode 1: channels-last rows  out[(ph*rows + p)*Cout + o]  for every row p < rows
  int out_mode;
  // fused producer outputs (generation fast path): the NEXT layer's key planes
  //   next_{hi,lo}[p][o] = split_bf16(next_scale[b,o] * y)   (zero at pad positions), written by
  //   TMA stores: 16-byte aligned
  void* next_hi;
  void* next_lo;
  const float* next_scale;   // [B, Cout] style of the consuming layer
  // and this layer's ToRGB partial sums over the tile's 128 output channels
  //   rgb_part[nt][b][c][y*Wv+x] = sum_{o in tile} rgb_w[b][c][o] * y[b,o,y,x]
  float* rgb_part;
  const float* rgb_w;        // [B, 3, Cout] modulated 1x1 weights
  // non-null: launch the clock()-instrumented variant, which writes per-phase cycles of every
  // consumer warp to debug_prof[grid][8][8] (rw_debug_conv_profile)
  long long* debug_prof;
};

namespace {

constexpr int BM = 128;
// the tile's output channels, BN, is a template parameter: 128, or 64 where Cout % 128 != 0
// k-block of 32 channels = one 64-byte swizzle row: a 32 KB stage (BN = 128), so that six fit in
// shared memory next to the epilogue's plane slots
constexpr int BK = 32;
constexpr int MMA_K = 16;
constexpr int kNumThreads = 384;   // warps 0-7: wgmma + epilogue, warpgroup 2: producer
constexpr int kTmaWarp = 8;
// register split after setmaxnreg: 128 x 40 + 256 x 232 = 384 x 168, the launch allocation
constexpr uint32_t kProducerRegs = 40;
constexpr uint32_t kConsumerRegs = 232;
// CTAs per cluster: they share (multicast) the weight tile of a k-block
constexpr int kCluster = 2;
// The tensor core's fp32 accumulate truncates (round-toward-zero) on every MMA: a chain of n
// accumulations whose partial sums grow linearly shrinks by about n/2 * 2^-25 (measured: 1-1.3x
// that with chunks, up to 1.9x for one long chain).  So the wgmma accumulator only ever holds
// a CHUNK of kChunkKB k-blocks (K=512: 96 accumulations); the chunks are added in fp32 registers
// with round-to-nearest.  Measured on an H100 at K=4608 (DESIGN.md §4): 1.65e-6 with one-signed
// operands, 1.4e-6 with mean-zero ones (tests/test_gpu_tc_accumulation.py); with kChunkKB = 256
// (one chain) 2.2e-5..2.5e-5 and 1.2e-5..1.4e-5.
// (K=512 -> pixel error 5.2e-4, K=1024 -> 8.1e-4, K >= 2304 fails the 1e-3 bound)
constexpr int kChunkKB = 16;

// The next layer's hi / lo planes leave through shared memory: each consumer warp packs its 16
// rows of one 64-channel half into a slot per plane (16 rows x 128 bytes, 128-byte swizzle) with
// stmatrix, and one TMA store writes the slot to the [rows][Cout] plane.  (As 4-byte LSU stores,
// each touching 8 rows of the plane, they take half of the epilogue: DESIGN.md §6.)
constexpr int kSlotBytes = 16 * 64 * 2;
constexpr int kSlots = 2 * 8;          // hi and lo of each consumer warp: 32 KB

template <int BN>
struct ConvSmem {
  static constexpr int kABytes = BM * BK * 2;          // one plane: 8 KB
  static constexpr int kBBytes = BN * BK * 2;          // one plane: 8 KB (BN = 64: 4 KB)
  static constexpr int kStageBytes = 2 * kABytes + 2 * kBBytes;
  // BN = 128: six 32 KB stages leave room for the plane slots (seven measured no faster than
  // six, DESIGN.md §6); BN = 64: seven 24 KB stages
  static constexpr int kStages = BN == 128 ? 6 : 7;
  static constexpr int kSlotOfs = kStages * kStageBytes;
  static constexpr int kBarOfs = kSlotOfs + kSlots * kSlotBytes;
  static constexpr int kTotal = kBarOfs + 1024 /*align slack*/ + 256 /*barriers*/;
  // the slots are 1024-byte aligned, the period of the 128-byte swizzle
  static_assert(kSlotOfs % 1024 == 0, "conv_tc: plane slots off the swizzle period");
};
// 1024-byte alignment serves the swizzle atoms of the ring and the slots; the total must stay within
// the 227 KB a block may opt in to
static_assert(ConvSmem<128>::kTotal <= 232448, "conv_tc: shared memory over the per-block limit");
static_assert(ConvSmem<64>::kTotal <= 232448, "conv_tc: shared memory over the per-block limit");

template <int kStages>
struct Barriers {
  uint64_t full[kStages];
  uint64_t empty[kStages];
};

// work unit -> (phase, mn).  Phases have very different tap counts (4/2/2/1 for a stride-2
// conv_transpose); with a static round-robin every scheduler slot would keep drawing the same
// one or two phases, so the phase is rotated by the (m-pair, n) group index — a bijection inside
// every group of `nphase` consecutive units.
__device__ __forceinline__ void decode_tile(int tile, int nphase, int nsched, int& ph, int& mn) {
  mn = tile / nphase;
  ph = tile - mn * nphase;
  if (nphase > 1) ph = (ph + ((nsched % nphase) == 0 ? tile / nsched : mn)) % nphase;
}

// EPI = 0: full fused epilogue (demod, noise, bias, leaky-ReLU, NCHW / channels-last store, next
//          layer's planes, ToRGB partials — every feature a run-time switch).
// EPI = 1: lean epilogue — optional per-(b,o) scale and the store, nothing else.  The up-path
//          conv_transpose phases, dgrad and the plain row-GEMM use it.
// PROF = true: bring-up variant that accumulates, per consumer warp, the cycles of each phase of a
// tile (tools/prof_conv.py) into p.debug_prof; the product launches PROF = false.
// BN = 64 (Cout % 128 != 0, the 64-channel layers of the 512² generator): wgmma.m64n64k16 on a
// 64-row weight tile, still multicast as two 32-row halves across the CTA pair; the epilogue is
// the same code over 32 accumulators per thread instead of 64.
// map_n_hi / map_n_lo: the next layer's planes [p.rows][Cout], 64 x 16 boxes with 128-byte
// swizzle (read only when p.next_hi is set).
template <int BN, int EPI, bool PROF>
__global__ void __launch_bounds__(kNumThreads, 1)
conv_tc_kernel(const __grid_constant__ CUtensorMap map_a_hi,
               const __grid_constant__ CUtensorMap map_a_lo,
               const __grid_constant__ CUtensorMap map_w_hi,
               const __grid_constant__ CUtensorMap map_w_lo,
               const __grid_constant__ CUtensorMap map_n_hi,
               const __grid_constant__ CUtensorMap map_n_lo, const ConvTcParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                             ~static_cast<uintptr_t>(1023));
  using S = ConvSmem<BN>;
  constexpr int kStages = S::kStages;
  constexpr int NR = BN / 2;    // accumulator registers per thread
  constexpr int NJ = BN / 8;    // 8-column groups per thread row
  Barriers<kStages>* bars = reinterpret_cast<Barriers<kStages>*>(smem + S::kBarOfs);

  // broadcast from lane 0: the compiler then knows the role branches are warp-uniform, which it
  // needs to give the consumer code the registers setmaxnreg grants
  const int warp = __shfl_sync(0xffffffffu, static_cast<int>(threadIdx.x >> 5), 0);
  const int lane = threadIdx.x & 31;
  // a cluster of kCluster CTAs works on a unit of kCluster m-tiles with the same (phase, n): CTA
  // `rank` takes m-tile kCluster * mp + rank.  Beyond an odd last m-tile the second tile lies
  // wholly past p.rows: TMA zero-fills its rows and the epilogue's row guards store nothing.
  const int rank = static_cast<int>(cluster_ctarank());
  const int nsched = static_cast<int>(num_clusters_x());
  const int first_unit = static_cast<int>(cluster_id_x());

  const int m_tiles = (p.rows + BM - 1) / BM;
  const int n_tiles = p.Cout / BN;
  const int mn_units = (m_tiles + kCluster - 1) / kCluster * n_tiles;
  const int num_units = mn_units * p.nphase;
  const int kb_per_tap = p.Cin / BK;

  if (warp == kTmaWarp && lane == 0) {
    tma_prefetch_desc(&map_a_hi);
    tma_prefetch_desc(&map_a_lo);
    tma_prefetch_desc(&map_w_hi);
    tma_prefetch_desc(&map_w_lo);
    for (int s = 0; s < kStages; ++s) {
      mbar_init(&bars->full[s], 1);
      // one arrival per consumer warpgroup of every CTA: the stage's B tile is refilled in all
      // of them at once
      mbar_init(&bars->empty[s], 2 * kCluster);
    }
    fence_mbar_init();
  }
  // the barriers are initialised cluster-wide before any remote arrival or multicast
  cluster_sync();

  // the consumer branch comes first: with the producer first, ptxas keeps the consumer code at
  // the 168-register launch bound and spills
  if (warp < kTmaWarp) {
    // ------------------------- MMA + epilogue (consumers) ------------------------
    setmaxnreg_inc<kConsumerRegs>();
    const int wg = threadIdx.x >> 7;            // 64-row half of the tile
    const int c = lane & 3;
    const int img = p.Hp * p.Wp;
    // a stage is released in every CTA of the cluster (one arrival per consumer warpgroup)
    auto release = [&](int s) {
      if ((threadIdx.x & 127) == 0) {
#pragma unroll
        for (int r = 0; r < kCluster; ++r) mbar_arrive_cluster(mapa_shared(&bars->empty[s], r));
      }
    };
    // PROF: wait full, MMA issue, chunk drain + promotion, epilogue, tiles, total, and two parts
    // of the epilogue: ToRGB partials, next layer's planes (the rest of it is the per-element
    // terms: constant loads, scale, noise, bias, activation, fp32 stores)
    // (32-bit clock differences: a launch runs for far fewer than 2^32 cycles)
    auto clk = [] { return static_cast<uint32_t>(clock()); };
    uint32_t prof[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    uint32_t tp0 = 0, tp1 = 0;
    if constexpr (PROF) prof[5] = 0u - clk();
    int stage = 0;
    uint32_t phase = 0;
    for (int unit = first_unit; unit < num_units; unit += nsched) {
      int ph, mn;
      decode_tile(unit, p.nphase, nsched, ph, mn);
      const int num_kb = p.ph_ntaps[ph] * kb_per_tap;
      const int n_tile = mn % n_tiles;
      const int n0 = n_tile * BN;
      const int m0 = ((mn / n_tiles) * kCluster + rank) * BM;

      float acc[NR], d[NR];
#pragma unroll
      for (int j = 0; j < NR; ++j) acc[j] = 0.f;
      for (int kb0 = 0; kb0 < num_kb; kb0 += kChunkKB) {
        const int kb_end = (kb0 + kChunkKB < num_kb) ? kb0 + kChunkKB : num_kb;
        // one wgmma group stays in flight: a stage is released once the group after it has been
        // issued and the group that read it has completed
        int held = -1;
        for (int kb = kb0; kb < kb_end; ++kb) {
          if constexpr (PROF) tp0 = clk();
          mbar_wait(&bars->full[stage], phase);
          if constexpr (PROF) { tp1 = clk(); prof[0] += tp1 - tp0; }
          const uint32_t sa = smem_u32(smem + stage * S::kStageBytes);
          const uint64_t da_hi = make_smem_desc(sa + wg * (S::kABytes / 2), 16, 512, 2);
          const uint64_t da_lo = make_smem_desc(sa + S::kABytes + wg * (S::kABytes / 2), 16, 512, 2);
          const uint64_t db_hi = make_smem_desc(sa + 2 * S::kABytes, 16, 512, 2);
          const uint64_t db_lo = make_smem_desc(sa + 2 * S::kABytes + S::kBBytes, 16, 512, 2);
          wgmma_fence();
#pragma unroll
          for (int kk = 0; kk < BK / MMA_K; ++kk) {
            const uint64_t adv = static_cast<uint64_t>((kk * MMA_K * 2) >> 4);
            // smallest terms first, then the dominant hi*hi product
            wgmma_m64nN<0, 0>(d, da_lo + adv, db_hi + adv, ((kb - kb0) | kk) != 0);
            wgmma_m64nN<0, 0>(d, da_hi + adv, db_lo + adv, 1u);
            wgmma_m64nN<0, 0>(d, da_hi + adv, db_hi + adv, 1u);
          }
          wgmma_commit();
          wgmma_wait<1>();
          if (held >= 0) release(held);
          held = stage;
          if (++stage == kStages) { stage = 0; phase ^= 1u; }
          if constexpr (PROF) prof[1] += clk() - tp1;
        }
        if constexpr (PROF) tp0 = clk();
        // the chunk is complete before it is added; its last stage is released here, so the
        // producer refills the ring while the epilogue runs
        wgmma_wait<0>();
        release(held);
#pragma unroll
        for (int j = 0; j < NR; ++j) acc[j] += d[j];
        if constexpr (PROF) prof[2] += clk() - tp0;
      }
      if constexpr (PROF) tp0 = clk();

      // ---- fused epilogue: rows r = m0 + 64 wg + 16 (warp % 4) + g + 8 i, columns 8 j + 2 c + e ----
      // (the thread's row offset is formed here from a fresh %tid.x: hoisted above the main loop,
      // it is the one value ptxas spills in the full epilogue's variant)
      uint32_t tid;
      asm volatile("mov.u32 %0, %%tid.x;\n" : "=r"(tid));
      const int row0 = m0 + ((tid >> 7) << 6) + (((tid >> 5) & 3) << 4) + ((tid & 31) >> 2);
      // image and validity of the thread's two rows, for the next layer's planes after the row loop
      const int Hv = p.ph_Hv[ph], Wv = p.ph_Wv[ph];
      int rb[2];
      bool rvalid[2];
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        const int prow = row0 + 8 * i;
        const int b = prow / img;
        const int rem = prow - b * img;
        const int yy = rem / p.Wp;
        const int xx = rem - yy * p.Wp;
        const bool in_rows = prow < p.rows;
        const bool valid = in_rows && (yy < Hv) && (xx < Wv);
        rb[i] = b;
        rvalid[i] = valid;
        const float* scl = (p.scale_bo && in_rows) ? p.scale_bo + static_cast<size_t>(b) * p.Cout : nullptr;
        float* outp = (p.out != nullptr && p.out_mode == 0 && valid)
                          ? p.out + p.ph_out_ofs[ph] + static_cast<size_t>(b) * p.out_sb +
                                static_cast<size_t>(yy) * p.out_sy + static_cast<size_t>(xx) * p.out_sx
                          : nullptr;
        if (EPI == 1 || !valid) {
          // lean epilogue, and the pad rows of the full one: only the optional scale
          if (scl && (EPI == 1 || p.out_mode == 1)) {
#pragma unroll
            for (int j = 0; j < NJ; ++j) {
              const float2 sv = __ldg(reinterpret_cast<const float2*>(scl + n0 + 8 * j + 2 * c));
              acc[4 * j + 2 * i] *= sv.x;
              acc[4 * j + 2 * i + 1] *= sv.y;
            }
          }
          if (EPI == 1 && outp) {
#pragma unroll
            for (int j = 0; j < NJ; ++j)
#pragma unroll
              for (int e = 0; e < 2; ++e)
                outp[static_cast<size_t>(n0 + 8 * j + 2 * c + e) * p.out_sc] = acc[4 * j + 2 * i + e];
          }
        } else {
          float nz = 0.f;
          if (p.noise != nullptr)
            nz = __ldg(p.noise_w) * __ldg(p.noise + static_cast<size_t>(b) * p.noise_bstride +
                                          static_cast<size_t>(yy) * Wv + xx);
          const float act_gain = p.act_gain != 0.f ? p.act_gain : 1.4142135623730951f;
          // one pass over the row's 32 values per term, so that a term that is off costs no
          // instructions: in a single loop ptxas computes the strided store's addresses for every
          // element, although the generator's fast path stores no fp32 output.  Per-row base
          // pointers give the loads constant offsets.  Each element sees scale, noise, bias,
          // activation in that order.
          if (scl) {
            const float* sc = scl + n0 + 2 * c;
#pragma unroll
            for (int j = 0; j < NJ; ++j)
#pragma unroll
              for (int e = 0; e < 2; ++e) acc[4 * j + 2 * i + e] *= __ldg(sc + 8 * j + e);
          }
#pragma unroll
          for (int j = 0; j < NJ; ++j)
#pragma unroll
            for (int e = 0; e < 2; ++e) acc[4 * j + 2 * i + e] += nz;
          if (p.bias) {
            const float* bi = p.bias + n0 + 2 * c;
#pragma unroll
            for (int j = 0; j < NJ; ++j)
#pragma unroll
              for (int e = 0; e < 2; ++e) acc[4 * j + 2 * i + e] += __ldg(bi + 8 * j + e);
          }
          if (p.act) {
#pragma unroll
            for (int j = 0; j < 2 * NJ; ++j) {
              float& t = acc[4 * (j >> 1) + 2 * i + (j & 1)];
              t = (t > 0.f ? t : 0.2f * t) * act_gain;
            }
          }
          if (outp) {
#pragma unroll
            for (int j = 0; j < NJ; ++j)
#pragma unroll
              for (int e = 0; e < 2; ++e)
                outp[static_cast<size_t>(n0 + 8 * j + 2 * c + e) * p.out_sc] = acc[4 * j + 2 * i + e];
          }
        }
        // channels-last raw rows are written for every row (pad rows are never read back)
        if (p.out != nullptr && p.out_mode == 1 && in_rows) {
          float* orow = p.out + (static_cast<size_t>(ph) * p.rows + prow) * p.Cout + n0 + 2 * c;
#pragma unroll
          for (int j = 0; j < NJ; ++j)
            *reinterpret_cast<float2*>(orow + 8 * j) = make_float2(acc[4 * j + 2 * i], acc[4 * j + 2 * i + 1]);
        }
      }
      if (EPI == 0 && p.rgb_w != nullptr) {
        if constexpr (PROF) tp1 = clk();
        // one partial per 64-channel group: rgb_part[(n_tile*BN/64 + half)][b][c][y*Wv+x]; the
        // four lanes of a row hold 16 of the group's channels each.  Both rows of the thread in
        // one pass, which loads the weights once where the rows lie in the same image (all but
        // the rows at an image boundary).  Pad rows sum too (only their own lanes see the sums)
        // but store nothing.
        const int wb0 = rvalid[0] ? rb[0] : 0, wb1 = rvalid[1] ? rb[1] : 0;
        const float* wa = p.rgb_w + static_cast<size_t>(wb0) * 3 * p.Cout + n0 + 2 * c;
        const float* wb = p.rgb_w + static_cast<size_t>(wb1) * 3 * p.Cout + n0 + 2 * c;
#pragma unroll
        for (int half = 0; half < BN / 64; ++half) {
          float r[2][3] = {{0.f, 0.f, 0.f}, {0.f, 0.f, 0.f}};
          if (wb0 == wb1) {
#pragma unroll
            for (int j = 8 * half; j < 8 * half + 8; ++j)
#pragma unroll
              for (int e = 0; e < 2; ++e)
#pragma unroll
                for (int q = 0; q < 3; ++q) {
                  const float w = __ldg(wa + q * p.Cout + 8 * j + e);
                  r[0][q] = fmaf(w, acc[4 * j + e], r[0][q]);
                  r[1][q] = fmaf(w, acc[4 * j + 2 + e], r[1][q]);
                }
          } else {
#pragma unroll
            for (int j = 8 * half; j < 8 * half + 8; ++j)
#pragma unroll
              for (int e = 0; e < 2; ++e)
#pragma unroll
                for (int q = 0; q < 3; ++q) {
                  r[0][q] = fmaf(__ldg(wa + q * p.Cout + 8 * j + e), acc[4 * j + e], r[0][q]);
                  r[1][q] = fmaf(__ldg(wb + q * p.Cout + 8 * j + e), acc[4 * j + 2 + e], r[1][q]);
                }
          }
#pragma unroll
          for (int i = 0; i < 2; ++i) {
#pragma unroll
            for (int sh = 1; sh < 4; sh <<= 1)
#pragma unroll
              for (int q = 0; q < 3; ++q) r[i][q] += __shfl_xor_sync(0xffffffffu, r[i][q], sh);
            if (rvalid[i] && c == 0) {
              const int rem = row0 + 8 * i - rb[i] * img;
              const int yy = rem / p.Wp;
              const size_t hw = static_cast<size_t>(Hv) * Wv;
              float* rp = p.rgb_part +
                          ((static_cast<size_t>(n_tile * (BN / 64) + half) * p.B + rb[i]) * 3) * hw +
                          static_cast<size_t>(yy) * Wv + (rem - yy * p.Wp);
              rp[0] = r[i][0];
              rp[hw] = r[i][1];
              rp[2 * hw] = r[i][2];
            }
          }
        }
        if constexpr (PROF) prof[6] += clk() - tp1;
      }
      if (EPI == 0 && p.next_hi != nullptr) {
        if constexpr (PROF) tp1 = clk();
        // per 64-channel half: the bf16 hi / lo words of both rows (pad rows get zeros, the next
        // layer's implicit zero padding), stmatrix'd into the warp's two slots, 16 x 16 words per
        // stmatrix.x4 (matrices: rows 0-7 / 8-15 of column groups 2k, 2k + 1), then one TMA store
        // per plane; rows past p.rows are clipped by it.  Lane t addresses row r = 8 (t / 8 % 2) +
        // t % 8, 16-byte chunk 2k + t / 16 of its 128-byte slot row, swizzled by r % 8.
        const int wq = static_cast<int>(tid >> 5);
        const uint32_t slot_hi = smem_u32(smem + S::kSlotOfs + 2 * wq * kSlotBytes);
        const uint32_t slot_lo = slot_hi + kSlotBytes;
        const uint32_t r = ((tid >> 3) & 1) * 8 + (tid & 7);
        const uint32_t jx = (tid >> 4) & 1;
        const int srow = m0 + ((tid >> 7) << 6) + (((tid >> 5) & 3) << 4);
#pragma unroll
        for (int half = 0; half < BN / 64; ++half) {
          uint32_t nxh[2][8], nxl[2][8];
#pragma unroll
          for (int i = 0; i < 2; ++i) {
            const float* ns = p.next_scale + static_cast<size_t>(rvalid[i] ? rb[i] : 0) * p.Cout + n0 + 2 * c;
#pragma unroll
            for (int jj = 0; jj < 8; ++jj) {
              const int j = 8 * half + jj;
              float k0 = 0.f, k1 = 0.f;
              if (rvalid[i]) {
                const float2 sv = __ldg(reinterpret_cast<const float2*>(ns + 8 * j));
                k0 = sv.x * acc[4 * j + 2 * i];
                k1 = sv.y * acc[4 * j + 2 * i + 1];
              }
              const __nv_bfloat162 hh = __floats2bfloat162_rn(k0, k1);
              const float2 hf = __bfloat1622float2(hh);
              const __nv_bfloat162 ll = __floats2bfloat162_rn(k0 - hf.x, k1 - hf.y);
              nxh[i][jj] = *reinterpret_cast<const uint32_t*>(&hh);
              nxl[i][jj] = *reinterpret_cast<const uint32_t*>(&ll);
            }
          }
          // the slots are free once the warp's previous stores have read them
          if (lane == 0) tma_store_wait_read_n<0>();
          __syncwarp();
#pragma unroll
          for (int k = 0; k < 4; ++k) {
            const int j = 2 * k;
            const uint32_t a = r * 128 + (((2 * k + jx) ^ (r & 7)) << 4);
            const uint32_t wh[4] = {nxh[0][j], nxh[1][j], nxh[0][j + 1], nxh[1][j + 1]};
            const uint32_t wl[4] = {nxl[0][j], nxl[1][j], nxl[0][j + 1], nxl[1][j + 1]};
            stmatrix_x4(slot_hi + a, wh);
            stmatrix_x4(slot_lo + a, wl);
          }
          fence_proxy_async_smem();
          __syncwarp();
          if (lane == 0) {
            tma_store_2d(&map_n_hi, slot_hi, n0 + 64 * half, srow);
            tma_store_2d(&map_n_lo, slot_lo, n0 + 64 * half, srow);
          }
        }
        if constexpr (PROF) prof[7] += clk() - tp1;
      }
      if constexpr (PROF) { prof[3] += clk() - tp0; prof[4] += 1; }
    }
    if constexpr (PROF) {
      prof[5] += clk();
      if (lane == 0) {
        long long* dst = p.debug_prof + (static_cast<size_t>(blockIdx.x) * 8 + warp) * 8;
#pragma unroll
        for (int i = 0; i < 8; ++i) dst[i] = prof[i];
      }
    }
  } else {
    // ------------------------------ TMA producer ------------------------------
    // every CTA loads its own A tile and one BN / kCluster-row slice of the B tile, multicast to
    // the same stage offset in every CTA of the cluster; a full barrier thus receives a whole
    // stage, kStageBytes, and a stage is refilled only once all CTAs have released it
    setmaxnreg_dec<kProducerRegs>();
    if (warp == kTmaWarp && lane == 0) {
      constexpr uint16_t kMask = (1u << kCluster) - 1;
      constexpr int kBSlice = BN / kCluster;
      const uint32_t b_off = 2 * S::kABytes + rank * (S::kBBytes / kCluster);
      int stage = 0;
      uint32_t phase = 0;
      for (int unit = first_unit; unit < num_units; unit += nsched) {
        int ph, mn;
        decode_tile(unit, p.nphase, nsched, ph, mn);
        const int n0 = (mn % n_tiles) * BN + rank * kBSlice;
        const int m0 = ((mn / n_tiles) * kCluster + rank) * BM;
        for (int t = 0; t < p.ph_ntaps[ph]; ++t) {
          const int arow = m0 + p.ph_shift[ph][t];
          const int wcol = p.ph_kofs[ph][t];
          const int acol = p.ph_acol[ph][t];
          for (int kb = 0; kb < kb_per_tap; ++kb) {
            mbar_wait(&bars->empty[stage], phase ^ 1u);
            uint8_t* st = smem + stage * S::kStageBytes;
            mbar_expect_tx(&bars->full[stage], S::kStageBytes);
            tma_load_2d(st, &map_a_hi, &bars->full[stage], acol + kb * BK, arow);
            tma_load_2d(st + S::kABytes, &map_a_lo, &bars->full[stage], acol + kb * BK, arow);
            tma_load_2d_multicast(st + b_off, &map_w_hi, &bars->full[stage], wcol + kb * BK, n0,
                                  kMask);
            tma_load_2d_multicast(st + b_off + S::kBBytes, &map_w_lo, &bars->full[stage],
                                  wcol + kb * BK, n0, kMask);
            if (++stage == kStages) { stage = 0; phase ^= 1u; }
          }
        }
      }
    }
    __syncwarp();
  }
  // no CTA leaves while another CTA of its cluster can still multicast into its shared memory or
  // arrive on its barriers
  cluster_sync();
  // nor while its plane stores still read their slots.  (Waited for here rather than at the end
  // of the consumer branch, where ptxas then injects a warpgroup.wait into the main loop.)
  if (EPI == 0 && warp < kTmaWarp && lane == 0) tma_store_wait_all();
}

}  // namespace

template <int BN, int EPI, bool PROF>
static int conv_tc_launch_epi(const ConvTcParams& p, const void* a_hi, const void* a_lo,
                              const void* w_hi, const void* w_lo, int wk_total,
                              cudaStream_t stream) {
  CUtensorMap ma_hi, ma_lo, mw_hi, mw_lo, mn_hi, mn_lo;
  int rc;
  // 64-byte swizzle: a box row is one k-block of BK = 32 channels
  const uint64_t a_cols = p.a_cols > 0 ? p.a_cols : p.Cin;
  const uint64_t a_dims[2] = {a_cols, static_cast<uint64_t>(p.rows)}, a_str[1] = {a_cols * 2};
  const uint64_t w_dims[2] = {static_cast<uint64_t>(wk_total), static_cast<uint64_t>(p.Cout)};
  const uint64_t w_str[1] = {static_cast<uint64_t>(wk_total) * 2};
  const uint32_t a_box[2] = {BK, BM}, w_box[2] = {BK, BN / kCluster};
  if ((rc = make_tmap_nd_bf16(&ma_hi, a_hi, 2, a_dims, a_str, a_box, nullptr, 3))) return rc;
  if ((rc = make_tmap_nd_bf16(&ma_lo, a_lo, 2, a_dims, a_str, a_box, nullptr, 3))) return rc;
  if ((rc = make_tmap_nd_bf16(&mw_hi, w_hi, 2, w_dims, w_str, w_box, nullptr, 3))) return rc;
  if ((rc = make_tmap_nd_bf16(&mw_lo, w_lo, 2, w_dims, w_str, w_box, nullptr, 3))) return rc;
  // the next layer's planes: one warp's 16 rows x 64 channels per store, 128-byte swizzle
  std::memset(&mn_hi, 0, sizeof(mn_hi));
  std::memset(&mn_lo, 0, sizeof(mn_lo));
  if (EPI == 0 && p.next_hi != nullptr) {
    const uint64_t n_dims[2] = {static_cast<uint64_t>(p.Cout), static_cast<uint64_t>(p.rows)};
    const uint64_t n_str[1] = {static_cast<uint64_t>(p.Cout) * 2};
    const uint32_t n_box[2] = {64, 16};
    if ((rc = make_tmap_nd_bf16(&mn_hi, p.next_hi, 2, n_dims, n_str, n_box, nullptr, 2))) return rc;
    if ((rc = make_tmap_nd_bf16(&mn_lo, p.next_lo, 2, n_dims, n_str, n_box, nullptr, 2))) return rc;
  }

  cudaLaunchConfig_t cfg = {};
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = kCluster;
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = 1;
  cfg.blockDim = dim3(kNumThreads);
  cfg.dynamicSmemBytes = ConvSmem<BN>::kTotal;
  cfg.stream = stream;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  // persistent clusters: as many as can be resident at once (a GPC with an odd number of free
  // SMs cannot host a whole cluster, so this is fewer than SMs / kCluster)
  static int max_clusters = 0;
  if (max_clusters == 0) {
    rc = check_cuda(cudaFuncSetAttribute(conv_tc_kernel<BN, EPI, PROF>,
                                         cudaFuncAttributeMaxDynamicSharedMemorySize, ConvSmem<BN>::kTotal),
                    "conv_tc smem attr");
    if (rc) return rc;
    cfg.gridDim = dim3(kCluster * (device_sm_count() / kCluster));
    rc = check_cuda(cudaOccupancyMaxActiveClusters(&max_clusters, conv_tc_kernel<BN, EPI, PROF>, &cfg),
                    "conv_tc cluster occupancy");
    if (rc) return rc;
    if (max_clusters < 1) {
      set_last_error("conv_tc: no cluster of %d CTAs fits on the device", kCluster);
      return RW_ERR_UNSUPPORTED;
    }
  }
  const int m_tiles = (p.rows + BM - 1) / BM;
  const int n_tiles = p.Cout / BN;
  const int num_units = (m_tiles + kCluster - 1) / kCluster * n_tiles * p.nphase;
  const int clusters = max_clusters < num_units ? max_clusters : num_units;
  cfg.gridDim = dim3(kCluster * clusters);
  rc = check_cuda(cudaLaunchKernelEx(&cfg, conv_tc_kernel<BN, EPI, PROF>, ma_hi, ma_lo, mw_hi, mw_lo,
                                     mn_hi, mn_lo, p),
                  "conv_tc launch");
  if (rc) return rc;
  return check_cuda(cudaGetLastError(), "conv_tc launch");
}

template <int BN>
static int conv_tc_launch_bn(const ConvTcParams& p, const void* a_hi, const void* a_lo,
                             const void* w_hi, const void* w_lo, int wk_total, cudaStream_t stream) {
  // lean epilogue when only the optional scale and the store are asked for
  const bool lean = !p.noise && !p.bias && !p.act && !p.rgb_w && !p.rgb_part && !p.next_hi &&
                    p.out != nullptr && (reinterpret_cast<uintptr_t>(p.scale_bo) & 7u) == 0;
  if (p.debug_prof) return conv_tc_launch_epi<BN, 0, true>(p, a_hi, a_lo, w_hi, w_lo, wk_total, stream);
  if (lean) return conv_tc_launch_epi<BN, 1, false>(p, a_hi, a_lo, w_hi, w_lo, wk_total, stream);
  return conv_tc_launch_epi<BN, 0, false>(p, a_hi, a_lo, w_hi, w_lo, wk_total, stream);
}

// the one launch behind every entry point below: checks the shape and the epilogue's alignment,
// then picks the tile width and the epilogue variant
static int conv_tc_launch(const ConvTcParams& p, const void* a_hi, const void* a_lo,
                          const void* w_hi, const void* w_lo, int wk_total, cudaStream_t stream) {
  // the stated limit (DESIGN.md §1) stays Cin % 64, although the kernel only needs Cin % BK
  if (p.Cin % 64 != 0 || p.Cout % 64 != 0 || p.nphase < 1 || p.nphase > 4 || p.rows <= 0) {
    set_last_error("conv_tc: unsupported shape Cin=%d Cout=%d nphase=%d rows=%d", p.Cin, p.Cout,
                   p.nphase, p.rows);
    return RW_ERR_BAD_ARG;
  }
  for (int i = 0; i < p.nphase; ++i)
    if (p.ph_ntaps[i] < 1 || p.ph_ntaps[i] > 9) {
      set_last_error("conv_tc: phase %d has %d taps", i, p.ph_ntaps[i]);
      return RW_ERR_BAD_ARG;
    }
  // the epilogue's accesses, at offsets that keep each base pointer's alignment (Cout % 64 == 0,
  // even column): float2 loads of next_scale, and of scale_bo on the pad rows of a channels-last
  // store; float2 stores of channels-last out; bf16 pairs into next_hi / next_lo, which TMA stores
  // also need 16-byte aligned (checked below)
  const struct {
    const void* ptr;
    unsigned align;
    const char* name;
  } need[] = {
      {p.scale_bo, p.out_mode == 1 ? 8u : 4u, "scale_bo"},
      {p.out, p.out_mode == 1 ? 8u : 4u, "out"},
      {p.noise, 4u, "noise"},
      {p.noise_w, 4u, "noise_w"},
      {p.bias, 4u, "bias"},
      {p.next_scale, 8u, "next_scale"},
      {p.next_hi, 4u, "next_hi"},
      {p.next_lo, 4u, "next_lo"},
      {p.rgb_w, 4u, "rgb_w"},
      {p.rgb_part, 4u, "rgb_part"},
  };
  for (const auto& n : need)
    if (n.ptr != nullptr && (reinterpret_cast<uintptr_t>(n.ptr) & (n.align - 1)) != 0) {
      set_last_error("conv_tc: %s (%p) is not %u-byte aligned", n.name, n.ptr, n.align);
      return RW_ERR_BAD_ARG;
    }
  for (int i = 6; i < 8; ++i)      // next_hi, next_lo
    if (need[i].ptr != nullptr && (reinterpret_cast<uintptr_t>(need[i].ptr) & 15u) != 0) {
      set_last_error("conv_tc: %s (%p) is not 16-byte aligned (TMA store)", need[i].name, need[i].ptr);
      return RW_ERR_BAD_ARG;
    }
  // 128-channel tiles wherever Cout allows them; 64 only for the 64-channel layers
  if (p.Cout % 128 == 0) return conv_tc_launch_bn<128>(p, a_hi, a_lo, w_hi, w_lo, wk_total, stream);
  return conv_tc_launch_bn<64>(p, a_hi, a_lo, w_hi, w_lo, wk_total, stream);
}

// the 3x3 same-size conv over the padded-flat grid of B images H x W: one phase of 9 taps,
// NCHW output strides
static int fill_conv3x3(ConvTcParams& p, const char* who, int B, int Cin, int Cout, int H, int W) {
  memset(&p, 0, sizeof(p));
  p.Hp = H + 1;
  p.Wp = W + 1;
  p.B = B;
  p.nphase = 1;
  p.ph_Hv[0] = H;
  p.ph_Wv[0] = W;
  const long long rows = static_cast<long long>(B) * p.Hp * p.Wp;
  if (rows > 0x7fffffffLL) {
    set_last_error("%s: too many rows", who);
    return RW_ERR_BAD_ARG;
  }
  p.rows = static_cast<int>(rows);
  p.Cin = Cin;
  p.Cout = Cout;
  p.ph_ntaps[0] = 9;
  for (int u = 0; u < 3; ++u)
    for (int v = 0; v < 3; ++v) {
      p.ph_shift[0][u * 3 + v] = (u - 1) * p.Wp + (v - 1);
      p.ph_kofs[0][u * 3 + v] = (u * 3 + v) * Cin;
    }
  p.out_sb = static_cast<long long>(Cout) * H * W;
  p.out_sc = static_cast<long long>(H) * W;
  p.out_sy = W;
  p.out_sx = 1;
  return RW_OK;
}

static int modconv_up_impl(const void* kp_hi, const void* kp_lo, const void* wt_hi,
                           const void* wt_lo, const float* scale_bo, int B, int Cin, int Cout,
                           int H, int W, float* t_out, int channels_last, rw_stream_t stream) {
  if (!kp_hi || !kp_lo || !wt_hi || !wt_lo || !t_out || B < 1) {
    set_last_error("rw_modconv_up_fwd: bad argument");
    return RW_ERR_BAD_ARG;
  }
  // conv_transpose2d(stride 2, pad 0, k 3): out[2m+a, 2n+b] gathers
  //   a == 0: (u=0, in row m), (u=2, in row m-1);  a == 1: (u=1, in row m)   (same along x)
  // over the padded-flat grid every phase is a row-GEMM with <= 4 shifted taps.
  const int Hp = H + 1, Wp = W + 1;
  const int Ht = 2 * H + 1, Wt = 2 * W + 1;
  const long long rows = static_cast<long long>(B) * Hp * Wp;
  if (rows > 0x7fffffffLL) {
    set_last_error("rw_modconv_up_fwd: too many rows");
    return RW_ERR_BAD_ARG;
  }
  ConvTcParams p;
  memset(&p, 0, sizeof(p));
  p.Hp = Hp;
  p.Wp = Wp;
  p.B = B;
  p.rows = static_cast<int>(rows);
  p.Cin = Cin;
  p.Cout = Cout;
  p.nphase = 4;
  p.scale_bo = scale_bo;
  p.out = t_out;
  p.out_sb = static_cast<long long>(Cout) * Ht * Wt;
  p.out_sc = static_cast<long long>(Ht) * Wt;
  p.out_sy = 2LL * Wt;
  p.out_sx = 2;
  p.out_mode = channels_last ? 1 : 0;
  // heaviest phase first within every (m, n) group: (0,0) has 4 taps, (1,1) has 1
  for (int a = 0; a < 2; ++a) {
    for (int b = 0; b < 2; ++b) {
      const int ph = a * 2 + b;
      p.ph_Hv[ph] = Hp - a;
      p.ph_Wv[ph] = Wp - b;
      p.ph_out_ofs[ph] = static_cast<long long>(a) * Wt + b;
      int us[2], dys[2], nu;
      int vs[2], dxs[2], nv;
      if (a == 0) { nu = 2; us[0] = 0; dys[0] = 0; us[1] = 2; dys[1] = -1; }
      else        { nu = 1; us[0] = 1; dys[0] = 0; }
      if (b == 0) { nv = 2; vs[0] = 0; dxs[0] = 0; vs[1] = 2; dxs[1] = -1; }
      else        { nv = 1; vs[0] = 1; dxs[0] = 0; }
      int n = 0;
      for (int iu = 0; iu < nu; ++iu)
        for (int iv = 0; iv < nv; ++iv) {
          p.ph_shift[ph][n] = dys[iu] * Wp + dxs[iv];
          p.ph_kofs[ph][n] = (us[iu] * 3 + vs[iv]) * Cin;
          ++n;
        }
      p.ph_ntaps[ph] = n;
    }
  }
  return conv_tc_launch(p, kp_hi, kp_lo, wt_hi, wt_lo, 9 * Cin, stream);
}

static int modconv_fused_impl(const void* kp_hi, const void* kp_lo, const void* wt_hi,
                              const void* wt_lo, const float* scale_bo, const float* noise,
                              long long noise_bstride, const float* noise_w, const float* bias,
                              int act, int B, int Cin, int Cout, int H, int W, float* out,
                              const float* next_scale, void* next_hi, void* next_lo,
                              const float* rgb_w, float* rgb_part, long long* prof_out,
                              rw_stream_t stream) {
  if (!kp_hi || !kp_lo || !wt_hi || !wt_lo || B < 1 || (noise && !noise_w) ||
      ((next_hi != nullptr) != (next_lo != nullptr)) || (next_hi && !next_scale) ||
      ((rgb_w != nullptr) != (rgb_part != nullptr)) || (!out && !next_hi && !rgb_part)) {
    set_last_error("rw_modconv_fwd_fused: bad argument");
    return RW_ERR_BAD_ARG;
  }
  ConvTcParams p;
  int rc = fill_conv3x3(p, "rw_modconv_fwd_fused", B, Cin, Cout, H, W);
  if (rc) return rc;
  p.scale_bo = scale_bo;
  p.bias = bias;
  p.noise = noise;
  p.noise_bstride = noise_bstride;
  p.noise_w = noise_w;
  p.act = act;
  p.out = out;
  p.next_hi = next_hi;
  p.next_lo = next_lo;
  p.next_scale = next_scale;
  p.rgb_w = rgb_w;
  p.rgb_part = rgb_part;
  p.debug_prof = prof_out;
  return conv_tc_launch(p, kp_hi, kp_lo, wt_hi, wt_lo, 9 * Cin, stream);
}

}  // namespace rw

using namespace rw;

extern "C" {

int rw_modconv_fwd(const void* kp_hi, const void* kp_lo, const void* wt_hi, const void* wt_lo,
                   const float* scale_bo, const float* noise, long long noise_bstride,
                   const float* noise_w, const float* bias, int act, int B, int Cin, int Cout,
                   int H, int W, float* out, rw_stream_t stream) {
  if (!kp_hi || !kp_lo || !wt_hi || !wt_lo || !out || B < 1 || (noise && !noise_w)) {
    set_last_error("rw_modconv_fwd: bad argument");
    return RW_ERR_BAD_ARG;
  }
  ConvTcParams p;
  int rc = fill_conv3x3(p, "rw_modconv_fwd", B, Cin, Cout, H, W);
  if (rc) return rc;
  p.scale_bo = scale_bo;
  p.bias = bias;
  p.noise = noise;
  p.noise_bstride = noise_bstride;
  p.noise_w = noise_w;
  p.act = act;
  p.out = out;
  return conv_tc_launch(p, kp_hi, kp_lo, wt_hi, wt_lo, 9 * Cin, stream);
}

int rw_modconv_up_fwd(const void* kp_hi, const void* kp_lo, const void* wt_hi, const void* wt_lo,
                      const float* scale_bo, int B, int Cin, int Cout, int H, int W, float* t_out,
                      rw_stream_t stream) {
  return modconv_up_impl(kp_hi, kp_lo, wt_hi, wt_lo, scale_bo, B, Cin, Cout, H, W, t_out, 0, stream);
}

int rw_modconv_up_fwd_cl(const void* kp_hi, const void* kp_lo, const void* wt_hi,
                         const void* wt_lo, const float* scale_bo, int B, int Cin, int Cout, int H,
                         int W, float* t_cl, rw_stream_t stream) {
  return modconv_up_impl(kp_hi, kp_lo, wt_hi, wt_lo, scale_bo, B, Cin, Cout, H, W, t_cl, 1, stream);
}

int rw_conv3x3_bias_act(const void* kp_hi, const void* kp_lo, const void* wt_hi, const void* wt_lo,
                        const float* bias, int act, float act_gain, int B, int Cin, int Cout, int H,
                        int W, float* out, rw_stream_t stream) {
  if (!kp_hi || !kp_lo || !wt_hi || !wt_lo || !out || B < 1) {
    set_last_error("rw_conv3x3_bias_act: bad argument");
    return RW_ERR_BAD_ARG;
  }
  ConvTcParams p;
  int rc = fill_conv3x3(p, "rw_conv3x3_bias_act", B, Cin, Cout, H, W);
  if (rc) return rc;
  p.bias = bias;
  p.act = act;
  p.act_gain = act_gain;
  p.out = out;
  return conv_tc_launch(p, kp_hi, kp_lo, wt_hi, wt_lo, 9 * Cin, stream);
}

int rw_modconv_fwd_fused(const void* kp_hi, const void* kp_lo, const void* wt_hi,
                         const void* wt_lo, const float* scale_bo, const float* noise,
                         long long noise_bstride, const float* noise_w, const float* bias, int act,
                         int B, int Cin, int Cout, int H, int W, float* out,
                         const float* next_scale, void* next_hi, void* next_lo,
                         const float* rgb_w, float* rgb_part, rw_stream_t stream) {
  return modconv_fused_impl(kp_hi, kp_lo, wt_hi, wt_lo, scale_bo, noise, noise_bstride, noise_w,
                            bias, act, B, Cin, Cout, H, W, out, next_scale, next_hi, next_lo, rgb_w,
                            rgb_part, nullptr, stream);
}

int rw_debug_conv_profile(const void* kp_hi, const void* kp_lo, const void* wt_hi,
                          const void* wt_lo, const float* scale_bo, const float* noise,
                          long long noise_bstride, const float* noise_w, const float* bias, int act,
                          int B, int Cin, int Cout, int H, int W, float* out,
                          const float* next_scale, void* next_hi, void* next_lo,
                          const float* rgb_w, float* rgb_part, long long* prof_out,
                          rw_stream_t stream) {
  if (!prof_out) {
    set_last_error("rw_debug_conv_profile: prof_out is null");
    return RW_ERR_BAD_ARG;
  }
  return modconv_fused_impl(kp_hi, kp_lo, wt_hi, wt_lo, scale_bo, noise, noise_bstride, noise_w,
                            bias, act, B, Cin, Cout, H, W, out, next_scale, next_hi, next_lo, rgb_w,
                            rgb_part, prof_out, stream);
}

// tap (u,v) of the stride-2 conv_transpose reads gradient phase (u&1, v&1) at row shift
// (u>>1)*(W+1) + (v>>1) of the INPUT-resolution padded grid.
int rw_modconv_up_dgrad(const void* gph_hi, const void* gph_lo, const void* wt_hi,
                        const void* wt_lo, const float* scale_bi, int B, int Cin, int Cout, int H,
                        int W, float* dk, rw_stream_t stream) {
  if (!gph_hi || !gph_lo || !wt_hi || !wt_lo || !dk || B < 1) {
    set_last_error("rw_modconv_up_dgrad: bad argument");
    return RW_ERR_BAD_ARG;
  }
  // GEMM: M = input pixels, K = 9 taps x Cout (gradient channels), N = Cin
  ConvTcParams p;
  int rc = fill_conv3x3(p, "rw_modconv_up_dgrad", B, /*Cin(K)=*/Cout, /*Cout(N)=*/Cin, H, W);
  if (rc) return rc;
  p.a_cols = 4 * Cout;
  for (int u = 0; u < 3; ++u)
    for (int v = 0; v < 3; ++v) {
      const int t = u * 3 + v;
      p.ph_shift[0][t] = (u >> 1) * p.Wp + (v >> 1);
      p.ph_acol[0][t] = ((u & 1) * 2 + (v & 1)) * Cout;
      p.ph_kofs[0][t] = t * Cout;
    }
  p.scale_bo = scale_bi;
  p.out = dk;
  return conv_tc_launch(p, gph_hi, gph_lo, wt_hi, wt_lo, 9 * Cout, stream);
}

int rw_rowgemm(const void* a_hi, const void* a_lo, const void* w_hi, const void* w_lo, int rows, int K,
               int N, float* out, rw_stream_t stream) {
  if (!a_hi || !a_lo || !w_hi || !w_lo || !out || rows < 1 || K % 64 != 0 || N % 64 != 0) {
    set_last_error("rw_rowgemm: bad argument (rows=%d K=%d N=%d)", rows, K, N);
    return RW_ERR_BAD_ARG;
  }
  ConvTcParams p;
  memset(&p, 0, sizeof(p));
  p.rows = rows; p.Cin = K; p.Cout = N; p.nphase = 1; p.ph_ntaps[0] = 1;
  p.Hp = 1; p.Wp = rows; p.ph_Hv[0] = 1; p.ph_Wv[0] = rows;   // one "image" = all rows
  p.out = out; p.out_sb = 0; p.out_sc = 1; p.out_sy = 0; p.out_sx = N;  // row-major [rows][N]
  return conv_tc_launch(p, a_hi, a_lo, w_hi, w_lo, K, stream);
}

}  // extern "C"
