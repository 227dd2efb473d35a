// insert_wide.cu — the fused insert loop for key crops wider than insert_loop_kernel's register
// tile (w > 16) or larger than its shared-memory budget: whole-map goals (tight_paste=False) and
// wide selections.
//
// Same algorithm and per-element arithmetic as insert_loop_kernel (csrc/rewrite.cu): a CTA owns
// OC = 4 output channels, keeps their W rows in shared memory and runs every iteration in one
// launch with no grid-wide barrier, because every quantity of an iteration is local to one output
// channel.  What differs:
//   * t (raw conv output) and g*demod live in a caller-provided global scratch [Cout4][P] x 2
//     (Cout4 = Cout rounded up to OC) instead of shared memory.  Each CTA touches only its own
//     rows, so __syncthreads() orders the accesses; at 64x64 x 512 channels it is 16.8 MB and stays
//     in L2.
//   * the crop is tiled in column chunks of MW = 16, so the register tile is the one the small
//     kernel uses at w = 16, whatever the crop width.
//   * the weight gradient walks each column chunk down the rows with a sliding 3-row window of key
//     values in registers, so every key value is loaded once per (chunk, channel) instead of three
//     times.
// The demodulation, loss, demod-term, projection and Adam phases are insert_loop_kernel's code;
// they are repeated here rather than shared so that the small-crop kernel stays exactly as it is.
// kLinear selects the Λ mode (linear_insert), whose update phases both kernels share from
// csrc/insert_linear.cuh.
// kUp selects the upsampling target of the odd StyleGAN2 layers, dconv (conv_transpose, stride 2)
// -> blur (4x4 FIR, pad 1) -> noise -> activate, on a key crop [B,Cin,h,w] and a value crop
// [B,Cout,2h,2w].  The conv_transpose plane T is (2h+1)x(2w+1) and is computed in gather form,
// polyphase over the (h+1)x(w+1) grid of the zero-bordered key crop: output parity (p,q) reads
// padded key rows a and a+1 (taps u = 2, 0 for p = 0, u = 1 for p = 1) and columns likewise, so
// each key value feeds 9 taps as in the plain conv.  The blur and its adjoint run on the planes
// in the workspace: T, g (2h x 2w) and gT = demod * blur^T(g), from which the weight gradient is
// dW[o,i,u,v] = sc * sum gT[2y+u, 2x+v] k[i,y,x] - (the demod term, unchanged).
#include "../../include/rewriting_b200.h"
#include "rw_common.cuh"
#include "insert_linear.cuh"

namespace rw {

namespace {

constexpr int kMaxRank = 32;
constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;
constexpr int OC = 4;
constexpr int MW = 16;          // column chunk = register tile width
constexpr int kMinCin = 128;    // the sizes the tests hold to the oracle
constexpr int kMaxCin = 512;    // 2 * OC weight rows of Cin*9 floats in shared memory
constexpr int kMiscFloats = 64 + kWarps * OC * 5;       // demod, coef, loss and G tables
constexpr int kLamFloats = 3 * OC * kMaxRank * 9;       // Λ mode: Λ, exp_avg, exp_avg_sq
constexpr int MU = 4;           // up mode: key columns per forward register tile (x 4 phases)
constexpr int MWU = 8;          // up mode: key columns per weight-gradient chunk

// up mode only: the output-gradient plane and the layer's blur kernel, passed by value
struct UpArgs {
  float* gG;            // [Cout4][B*2h*2w] g = sign(y - v*) * gate / numel
  float blur[16];       // mconv.blur.kernel [4][4] as stored; applied flipped, as upfirdn2d does
};

template <bool kLinear, bool kUp>
__global__ void __launch_bounds__(kThreads, 1)
insert_wide_kernel(const InsertLoopParams p, const float* __restrict__ kpT, float* tG, float* gdG,
                   const UpArgs up) {
  extern __shared__ float sm[];
  const int Cin = p.Cin, h = p.h, w = p.w, B = p.B;
  const int P = B * h * w;
  // up mode: T and gT planes (2h+1)x(2w+1), g and value planes 2h x 2w
  const int Ht = 2 * h + 1, Wt = 2 * w + 1, Ho = 2 * h, Wo = 2 * w;
  const int PT = B * Ht * Wt, PO = B * Ho * Wo;
  const int wp = w + 2;
  const int nW = Cin * 9;
  const int nxc = (w + MW - 1) / MW;
  float* Ws = sm;                      // [OC][Cin*9]   current weight rows
  float* dWS = Ws + OC * nW;           // [OC][Cin*9]   gradient staging
  float* lam = dWS + OC * nW;          // [OC][kMaxRank*9]
  float* misc = lam + OC * kMaxRank * 9;
  float* demodS = misc;                // [OC][4]
  float* coefS = misc + 16;            // [OC][4]
  float* lossS = misc + 32;            // [kWarps][OC]
  float* GS = misc + 64;               // [kWarps][OC][4]
  float* lamS = misc + kMiscFloats;    // Λ mode: [OC][kMaxRank*9] Λ, then exp_avg, exp_avg_sq
  float* lamMS = lamS + OC * kMaxRank * 9;
  float* lamVS = lamMS + OC * kMaxRank * 9;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const bool plain = p.plain_conv != 0;  // nn.Conv2d target: no demodulation, no weight scale
  const float sc = plain ? 1.0f : rsqrtf(static_cast<float>(Cin * 9));
  const int nch = Cin / 32;            // channels per lane
  const float inv_numel = kUp
      ? 1.0f / static_cast<float>(static_cast<long long>(B) * p.Cout * Ho * Wo)
      : 1.0f / static_cast<float>(static_cast<long long>(B) * p.Cout * h * w);

  for (int o0 = blockIdx.x * OC; o0 < p.Cout; o0 += gridDim.x * OC) {
    const int noc = (p.Cout - o0 < OC) ? p.Cout - o0 : OC;
    float* tS = tG + static_cast<size_t>(o0) * (kUp ? PT : P);   // this CTA's rows of the scratch
    float* gdS = gdG + static_cast<size_t>(o0) * (kUp ? PT : P);
    float* gS = kUp ? up.gG + static_cast<size_t>(o0) * PO : nullptr;
    if constexpr (kLinear) {
      linear_mode::load_state<OC, kMaxRank * 9, kThreads>(p, o0, noc, lamS, lamMS, lamVS);
      __syncthreads();
      linear_mode::rebuild_weights<OC, kMaxRank * 9, kThreads>(p, o0, noc, lamS, Ws);
    } else {
      for (int i = threadIdx.x; i < OC * nW; i += kThreads) {
        const int oc = i / nW;
        Ws[i] = (oc < noc) ? p.W[static_cast<size_t>(o0) * nW + i] : 0.f;
      }
    }
    __syncthreads();

    for (int step = 0; step < p.nsteps; ++step) {
      const int it = p.it0 + step;
      // ---- demod[oc][b] = rsqrt(sum_i style^2 * sum_uv (sc W)^2 + 1e-8): warp <-> (oc, b)
      for (int ob = warp; ob < OC * B; ob += kWarps) {
        const int oc = ob / B, b = ob - oc * B;
        if (plain) {
          if (lane == 0) demodS[oc * 4 + b] = 1.0f;
          continue;
        }
        float acc = 0.f;
        for (int j = 0; j < nch; ++j) {
          const int i = lane + 32 * j;
          float ss = 0.f;
#pragma unroll
          for (int t = 0; t < 9; ++t) {
            const float v = sc * Ws[oc * nW + i * 9 + t];
            ss = fmaf(v, v, ss);
          }
          const float s = __ldg(p.style + b * Cin + i);
          acc = fmaf(s * s, ss, acc);
        }
#pragma unroll
        for (int off = 16; off; off >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, off);
        if (lane == 0) demodS[oc * 4 + b] = rsqrtf(acc + 1e-8f);
      }
      if constexpr (kUp) {
        // ---- forward conv_transpose: warp <-> (b, a, chunk of MU columns c), lane <-> input
        //      channel.  T[2a+p][2c+q] for the 4 parities from padded key rows a, a+1 and columns
        //      c, c+1 (key rows/columns a-1, a and c-1, c).
        const int nxu = (w + 1 + MU - 1) / MU;
        for (int u = warp; u < B * (h + 1) * nxu; u += kWarps) {
          const int row = u / nxu;                 // b * (h + 1) + a
          const int c0 = (u - row * nxu) * MU;
          const int b = row / (h + 1), a = row - b * (h + 1);
          float acc[OC][4][MU];
#pragma unroll
          for (int oc = 0; oc < OC; ++oc)
#pragma unroll
            for (int ph = 0; ph < 4; ++ph)
#pragma unroll
              for (int x = 0; x < MU; ++x) acc[oc][ph][x] = 0.f;
#pragma unroll 1
          for (int j = 0; j < nch; ++j) {
            const int i = lane + 32 * j;
            const float* k0 = kpT + ((static_cast<size_t>(b) * (h + 2) + a) * wp + c0) * Cin + i;
            const float* k1 = k0 + static_cast<size_t>(wp) * Cin;
            float kv0[MU + 1], kv1[MU + 1];
#pragma unroll
            for (int x = 0; x < MU + 1; ++x) {
              kv0[x] = (c0 + x < wp) ? __ldg(k0 + static_cast<size_t>(x) * Cin) : 0.f;
              kv1[x] = (c0 + x < wp) ? __ldg(k1 + static_cast<size_t>(x) * Cin) : 0.f;
            }
#pragma unroll
            for (int oc = 0; oc < OC; ++oc) {
              const float* wr = Ws + oc * nW + i * 9;
              const float w00 = wr[0], w01 = wr[1], w02 = wr[2];
              const float w10 = wr[3], w11 = wr[4], w12 = wr[5];
              const float w20 = wr[6], w21 = wr[7], w22 = wr[8];
#pragma unroll
              for (int x = 0; x < MU; ++x) {
                acc[oc][0][x] = fmaf(w00, kv1[x + 1], acc[oc][0][x]);
                acc[oc][0][x] = fmaf(w02, kv1[x], acc[oc][0][x]);
                acc[oc][0][x] = fmaf(w20, kv0[x + 1], acc[oc][0][x]);
                acc[oc][0][x] = fmaf(w22, kv0[x], acc[oc][0][x]);
                acc[oc][1][x] = fmaf(w01, kv1[x + 1], acc[oc][1][x]);
                acc[oc][1][x] = fmaf(w21, kv0[x + 1], acc[oc][1][x]);
                acc[oc][2][x] = fmaf(w10, kv1[x + 1], acc[oc][2][x]);
                acc[oc][2][x] = fmaf(w12, kv1[x], acc[oc][2][x]);
                acc[oc][3][x] = fmaf(w11, kv1[x + 1], acc[oc][3][x]);
              }
            }
          }
#pragma unroll
          for (int oc = 0; oc < OC; ++oc)
#pragma unroll
            for (int ph = 0; ph < 4; ++ph)
#pragma unroll
              for (int x = 0; x < MU; ++x) {
                float s = acc[oc][ph][x];
#pragma unroll
                for (int off = 16; off; off >>= 1) s += __shfl_xor_sync(0xffffffffu, s, off);
                const int ty = 2 * a + (ph >> 1), tx = 2 * (c0 + x) + (ph & 1);
                if (lane == ((ph * MU + x) & 31) && ty < Ht && tx < Wt)
                  tS[oc * PT + (b * Ht + ty) * Wt + tx] = sc * s;
              }
        }
      } else {
      // ---- forward conv: warp <-> (b, y, column chunk), lane <-> input channel;
      //      every key value loaded feeds the OC output channels
      for (int u = warp; u < B * h * nxc; u += kWarps) {
        const int row = u / nxc;                 // b * h + y
        const int x0 = (u - row * nxc) * MW;
        const int b = row / h, y = row - b * h;
        float acc[OC][MW];
#pragma unroll
        for (int oc = 0; oc < OC; ++oc)
#pragma unroll
          for (int x = 0; x < MW; ++x) acc[oc][x] = 0.f;
        for (int j = 0; j < nch; ++j) {
          const int i = lane + 32 * j;
#pragma unroll
          for (int r = 0; r < 3; ++r) {
            const float* krow = kpT + ((static_cast<size_t>(b) * (h + 2) + y + r) * wp + x0) * Cin + i;
            float kv[MW + 2];
#pragma unroll
            for (int x = 0; x < MW + 2; ++x)
              kv[x] = (x0 + x < wp) ? __ldg(krow + static_cast<size_t>(x) * Cin) : 0.f;
#pragma unroll
            for (int oc = 0; oc < OC; ++oc) {
              const float w0 = Ws[oc * nW + i * 9 + r * 3 + 0];
              const float w1 = Ws[oc * nW + i * 9 + r * 3 + 1];
              const float w2 = Ws[oc * nW + i * 9 + r * 3 + 2];
#pragma unroll
              for (int x = 0; x < MW; ++x) {
                acc[oc][x] = fmaf(w0, kv[x], acc[oc][x]);
                acc[oc][x] = fmaf(w1, kv[x + 1], acc[oc][x]);
                acc[oc][x] = fmaf(w2, kv[x + 2], acc[oc][x]);
              }
            }
          }
        }
#pragma unroll
        for (int oc = 0; oc < OC; ++oc)
#pragma unroll
          for (int x = 0; x < MW; ++x) {
            float a = acc[oc][x];
#pragma unroll
            for (int off = 16; off; off >>= 1) a += __shfl_xor_sync(0xffffffffu, a, off);
            if (lane == x && x0 + x < w) tS[oc * P + row * w + x0 + x] = sc * a;
          }
      }
      }
      __syncthreads();
      // ---- loss / output gradient: thread <-> (oc, pixel); block-reduce loss and G[oc][b]
      {
        float lsum[OC], gsum[OC][4];
#pragma unroll
        for (int oc = 0; oc < OC; ++oc) {
          lsum[oc] = 0.f;
#pragma unroll
          for (int bb = 0; bb < 4; ++bb) gsum[oc][bb] = 0.f;
        }
        if constexpr (kUp) {
          // z = demod * blur(T): upfirdn2d(pad 1) correlates with the flipped kernel,
          // z[Y][X] = sum_{r,c} T[Y+r-1][X+c-1] K[3-r][3-c]; G[oc][b] = sum g * blur(T)
          for (int q = threadIdx.x; q < PO; q += kThreads) {
            const int b = q / (Ho * Wo);
            const int pp = q - b * Ho * Wo;
            const int Y = pp / Wo, X = pp - Y * Wo;
            float nz = 0.f;
            if (p.has_noise_act && p.noise) nz = p.noise_w * __ldg(p.noise + b * Ho * Wo + pp);
#pragma unroll
            for (int oc = 0; oc < OC; ++oc) {
              if (oc >= noc) break;
              const int o = o0 + oc;
              const float* tp = tS + oc * PT + b * Ht * Wt;
              float t = 0.f;
#pragma unroll
              for (int r = 0; r < 4; ++r) {
                const int ty = Y + r - 1;
                if (ty < 0 || ty >= Ht) continue;
#pragma unroll
                for (int c = 0; c < 4; ++c) {
                  const int tx = X + c - 1;
                  if (tx >= 0 && tx < Wt) t = fmaf(up.blur[15 - (r * 4 + c)], tp[ty * Wt + tx], t);
                }
              }
              const float dm = demodS[oc * 4 + b];
              float yv = t * dm;
              float gate = 1.f;
              if (p.has_noise_act) {
                yv += nz;
                yv += __ldg(p.bias + o);
                gate = (yv > 0.f) ? 1.4142135623730951f : 0.2f * 1.4142135623730951f;
                yv = (yv > 0.f ? yv : 0.2f * yv) * 1.4142135623730951f;
              }
              const float tgt = __ldg(p.target + (static_cast<size_t>(b) * p.Cout + o) * Ho * Wo + pp);
              const float diff = yv - tgt;
              lsum[oc] += fabsf(diff);
              const float sgn = (diff > 0.f) ? 1.f : ((diff < 0.f) ? -1.f : 0.f);
              const float g = sgn * inv_numel * gate;
              gS[oc * PO + q] = g;
#pragma unroll
              for (int bb = 0; bb < 4; ++bb)
                if (bb == b) gsum[oc][bb] += g * t;
            }
          }
        } else {
        for (int q = threadIdx.x; q < P; q += kThreads) {
          const int b = q / (h * w);
          const int pp = q - b * h * w;
          float nz = 0.f;
          if (p.has_noise_act && p.noise) nz = p.noise_w * __ldg(p.noise + b * h * w + pp);
#pragma unroll
          for (int oc = 0; oc < OC; ++oc) {
            if (oc >= noc) break;
            const int o = o0 + oc;
            const float t = tS[oc * P + q];
            const float dm = demodS[oc * 4 + b];
            float yv = t * dm;
            float gate = 1.f;
            if (p.has_noise_act) {
              yv += nz;
              yv += __ldg(p.bias + o);
              gate = (yv > 0.f) ? 1.4142135623730951f : 0.2f * 1.4142135623730951f;
              yv = (yv > 0.f ? yv : 0.2f * yv) * 1.4142135623730951f;
            }
            const float tgt = __ldg(p.target + (static_cast<size_t>(b) * p.Cout + o) * h * w + pp);
            const float diff = yv - tgt;
            lsum[oc] += fabsf(diff);
            const float sgn = (diff > 0.f) ? 1.f : ((diff < 0.f) ? -1.f : 0.f);
            const float g = sgn * inv_numel * gate;
            gdS[oc * P + q] = g * dm;
#pragma unroll
            for (int bb = 0; bb < 4; ++bb)
              if (bb == b) gsum[oc][bb] += g * t;
          }
        }
        }
#pragma unroll
        for (int oc = 0; oc < OC; ++oc) {
#pragma unroll
          for (int off = 16; off; off >>= 1) {
            lsum[oc] += __shfl_xor_sync(0xffffffffu, lsum[oc], off);
#pragma unroll
            for (int bb = 0; bb < 4; ++bb)
              gsum[oc][bb] += __shfl_xor_sync(0xffffffffu, gsum[oc][bb], off);
          }
          if (lane == 0) {
            lossS[warp * OC + oc] = lsum[oc];
#pragma unroll
            for (int bb = 0; bb < 4; ++bb) GS[(warp * OC + oc) * 4 + bb] = gsum[oc][bb];
          }
        }
      }
      __syncthreads();
      if (threadIdx.x < noc) {
        float l = 0.f;
        for (int wv = 0; wv < kWarps; ++wv) l += lossS[wv * OC + threadIdx.x];
        p.loss_out[static_cast<size_t>(step) * p.Cout + o0 + threadIdx.x] = l;
      }
      if (threadIdx.x < OC * 4) {
        const int oc = threadIdx.x >> 2, bb = threadIdx.x & 3;
        float G = 0.f;
        for (int wv = 0; wv < kWarps; ++wv) G += GS[(wv * OC + oc) * 4 + bb];
        const float dm = demodS[oc * 4 + bb];
        coefS[oc * 4 + bb] = (bb < B && !plain) ? G * dm * dm * dm : 0.f;
      }
      __syncthreads();

      // Adam bias corrections as torch.optim.Adam computes them (python doubles)
      const double stepd = static_cast<double>(it + 1);
      const double bc1 = 1.0 - pow(p.beta1_exact, stepd);
      const double bc2 = 1.0 - pow(p.beta2_exact, stepd);
      const float step_size = static_cast<float>(static_cast<double>(p.lr) / bc1);
      const float bc2_sqrt = static_cast<float>(sqrt(bc2));
      const float one_m_b1 = p.one_minus_beta1;
      const float one_m_b2 = p.one_minus_beta2;

      if constexpr (kUp) {
        // ---- gT = demod * blur^T(g) on the (2h+1)x(2w+1) plane: thread <-> (oc, pixel)
        for (int q = threadIdx.x; q < PT; q += kThreads) {
          const int b = q / (Ht * Wt);
          const int pp = q - b * Ht * Wt;
          const int ty = pp / Wt, tx = pp - ty * Wt;
#pragma unroll
          for (int oc = 0; oc < OC; ++oc) {
            if (oc >= noc) break;
            const float* gp = gS + oc * PO + b * Ho * Wo;
            float s = 0.f;
#pragma unroll
            for (int r = 0; r < 4; ++r) {
              const int Y = ty + 1 - r;
              if (Y < 0 || Y >= Ho) continue;
#pragma unroll
              for (int c = 0; c < 4; ++c) {
                const int X = tx + 1 - c;
                if (X >= 0 && X < Wo) s = fmaf(up.blur[15 - (r * 4 + c)], gp[Y * Wo + X], s);
              }
            }
            gdS[oc * PT + q] = s * demodS[oc * 4 + b];
          }
        }
        __syncthreads();
        // ---- weight gradient: warp <-> channel group j, lane <-> input channel; OC x 9
        //      accumulators.  Key row y meets gT rows 2y, 2y+1, 2y+2 and, per column x, gT
        //      columns 2x, 2x+1, 2x+2 (broadcast loads, one gT row of a chunk at a time).
        for (int j = warp; j < nch; j += kWarps) {
          const int i = lane + 32 * j;
          float acc[OC][9];
#pragma unroll
          for (int oc = 0; oc < OC; ++oc)
#pragma unroll
            for (int t = 0; t < 9; ++t) acc[oc][t] = 0.f;
          for (int b = 0; b < B; ++b) {
            for (int x0 = 0; x0 < w; x0 += MWU) {
              for (int y = 0; y < h; ++y) {
                const float* krow =
                    kpT + ((static_cast<size_t>(b) * (h + 2) + y + 1) * wp + x0 + 1) * Cin + i;
                float kv[MWU];
#pragma unroll
                for (int x = 0; x < MWU; ++x)
                  kv[x] = (x0 + x < w) ? __ldg(krow + static_cast<size_t>(x) * Cin) : 0.f;
#pragma unroll
                for (int oc = 0; oc < OC; ++oc) {
                  if (oc >= noc) break;
                  const float* g0 = gdS + oc * PT + (b * Ht + 2 * y) * Wt + 2 * x0;
#pragma unroll
                  for (int r = 0; r < 3; ++r) {
                    float gv[2 * MWU + 1];
#pragma unroll
                    for (int c = 0; c < 2 * MWU + 1; ++c)
                      gv[c] = (2 * x0 + c < Wt) ? g0[r * Wt + c] : 0.f;
#pragma unroll
                    for (int x = 0; x < MWU; ++x) {
                      acc[oc][r * 3 + 0] = fmaf(gv[2 * x], kv[x], acc[oc][r * 3 + 0]);
                      acc[oc][r * 3 + 1] = fmaf(gv[2 * x + 1], kv[x], acc[oc][r * 3 + 1]);
                      acc[oc][r * 3 + 2] = fmaf(gv[2 * x + 2], kv[x], acc[oc][r * 3 + 2]);
                    }
                  }
                }
              }
            }
          }
          // demod term: - sc^2 * W * sum_b coef[b] * style[b,i]^2
#pragma unroll
          for (int oc = 0; oc < OC; ++oc) {
            float cs = 0.f;
            for (int b = 0; b < B; ++b) {
              const float s = __ldg(p.style + b * Cin + i);
              cs = fmaf(coefS[oc * 4 + b], s * s, cs);
            }
#pragma unroll
            for (int t = 0; t < 9; ++t) {
              const float wv = Ws[oc * nW + i * 9 + t];
              dWS[oc * nW + i * 9 + t] = sc * acc[oc][t] - (sc * sc) * wv * cs;
            }
          }
        }
      } else {
      // ---- weight gradient: warp <-> channel group j, lane <-> input channel; OC x 9
      //      accumulators.  Per column chunk the rows are walked top to bottom and the three key
      //      rows under the 3x3 window slide down one row per output row.
      for (int j = warp; j < nch; j += kWarps) {
        const int i = lane + 32 * j;
        float acc[OC][9];
#pragma unroll
        for (int oc = 0; oc < OC; ++oc)
#pragma unroll
          for (int t = 0; t < 9; ++t) acc[oc][t] = 0.f;
        for (int b = 0; b < B; ++b) {
          for (int x0 = 0; x0 < w; x0 += MW) {
            float kv[3][MW + 2];
            const float* kcol = kpT + (static_cast<size_t>(b) * (h + 2) * wp + x0) * Cin + i;
#pragma unroll
            for (int r = 0; r < 2; ++r)
#pragma unroll
              for (int x = 0; x < MW + 2; ++x)
                kv[r + 1][x] = (x0 + x < wp)
                                   ? __ldg(kcol + (static_cast<size_t>(r) * wp + x) * Cin) : 0.f;
            for (int y = 0; y < h; ++y) {
#pragma unroll
              for (int x = 0; x < MW + 2; ++x) {
                kv[0][x] = kv[1][x];
                kv[1][x] = kv[2][x];
                kv[2][x] = (x0 + x < wp)
                               ? __ldg(kcol + (static_cast<size_t>(y + 2) * wp + x) * Cin) : 0.f;
              }
              const float* grow = gdS + (b * h + y) * w + x0;
#pragma unroll
              for (int oc = 0; oc < OC; ++oc) {
#pragma unroll
                for (int x = 0; x < MW; ++x) {
                  const float gv = (oc < noc && x0 + x < w) ? grow[oc * P + x] : 0.f;
#pragma unroll
                  for (int r = 0; r < 3; ++r) {
                    acc[oc][r * 3 + 0] = fmaf(gv, kv[r][x], acc[oc][r * 3 + 0]);
                    acc[oc][r * 3 + 1] = fmaf(gv, kv[r][x + 1], acc[oc][r * 3 + 1]);
                    acc[oc][r * 3 + 2] = fmaf(gv, kv[r][x + 2], acc[oc][r * 3 + 2]);
                  }
                }
              }
            }
          }
        }
        // demod term: - sc^2 * W * sum_b coef[b] * style[b,i]^2
#pragma unroll
        for (int oc = 0; oc < OC; ++oc) {
          float cs = 0.f;
          if (!plain) {
            for (int b = 0; b < B; ++b) {
              const float s = __ldg(p.style + b * Cin + i);
              cs = fmaf(coefS[oc * 4 + b], s * s, cs);
            }
          }
#pragma unroll
          for (int t = 0; t < 9; ++t) {
            const float wv = Ws[oc * nW + i * 9 + t];
            dWS[oc * nW + i * 9 + t] = sc * acc[oc][t] - (sc * sc) * wv * cs;
          }
        }
      }
      }
      __syncthreads();
      if constexpr (kLinear) {
        // ---- Λ mode: dΛ = dW d^T, Adam on Λ, W = W0 + Λ d   (ganrewrite.py:219-240)
        linear_mode::adam_step<OC, kMaxRank * 9, kWarps>(p, noc, dWS, lamS, lamMS, lamVS,
                                                         step_size, bc2_sqrt, one_m_b1, one_m_b2);
        __syncthreads();
        linear_mode::rebuild_weights<OC, kMaxRank * 9, kThreads>(p, o0, noc, lamS, Ws);
        __syncthreads();
        continue;
      }
      // ---- optional gradient projection onto span(d)   (ganrewrite.py:285-286)
      if (p.project_gradient) {
        for (int ort = warp; ort < OC * p.rank * 9; ort += kWarps) {
          const int oc = ort / (p.rank * 9), rt = ort - oc * p.rank * 9;
          const int r = rt / 9, t = rt - r * 9;
          float a = 0.f;
          for (int i = lane; i < Cin; i += 32)
            a = fmaf(dWS[oc * nW + i * 9 + t], __ldg(p.d + r * Cin + i), a);
#pragma unroll
          for (int off = 16; off; off >>= 1) a += __shfl_xor_sync(0xffffffffu, a, off);
          if (lane == 0) lam[oc * kMaxRank * 9 + rt] = a;
        }
        __syncthreads();
        for (int e = threadIdx.x; e < OC * nW; e += kThreads) {
          const int oc = e / nW, ei = e - oc * nW;
          const int i = ei / 9, t = ei - i * 9;
          float pr = 0.f;
          for (int r = 0; r < p.rank; ++r)
            pr = fmaf(lam[oc * kMaxRank * 9 + r * 9 + t], __ldg(p.d + r * Cin + i), pr);
          dWS[e] = pr;
        }
        __syncthreads();
      }
      // ---- Adam (torch.optim.Adam, amsgrad=False, weight_decay=0)
      for (int e = threadIdx.x; e < noc * nW; e += kThreads) {
        const size_t ge = static_cast<size_t>(o0) * nW + e;
        const float g = dWS[e];
        float mm = p.m[ge], vv = p.v[ge];
        mm = mm + (g - mm) * one_m_b1;                 // exp_avg.lerp_(grad, 1-beta1)
        vv = vv * p.beta2 + one_m_b2 * g * g;          // mul_(beta2).addcmul_(g, g, 1-beta2)
        p.m[ge] = mm;
        p.v[ge] = vv;
        const float denom = sqrtf(vv) / bc2_sqrt + p.eps;
        Ws[e] = Ws[e] - step_size * (mm / denom);
      }
      __syncthreads();
      // ---- periodic projection  W <- W_ortho + P_d(W)   (ganrewrite.py:291-294)
      if (p.w_ortho != nullptr && (it % p.piter == 0 || it == p.niter_total - 1)) {
        for (int ort = warp; ort < OC * p.rank * 9; ort += kWarps) {
          const int oc = ort / (p.rank * 9), rt = ort - oc * p.rank * 9;
          const int r = rt / 9, t = rt - r * 9;
          float a = 0.f;
          for (int i = lane; i < Cin; i += 32)
            a = fmaf(Ws[oc * nW + i * 9 + t], __ldg(p.d + r * Cin + i), a);
#pragma unroll
          for (int off = 16; off; off >>= 1) a += __shfl_xor_sync(0xffffffffu, a, off);
          if (lane == 0) lam[oc * kMaxRank * 9 + rt] = a;
        }
        __syncthreads();
        for (int e = threadIdx.x; e < noc * nW; e += kThreads) {
          const int oc = e / nW, ei = e - oc * nW;
          const int i = ei / 9, t = ei - i * 9;
          float pr = 0.f;
          for (int r = 0; r < p.rank; ++r)
            pr = fmaf(lam[oc * kMaxRank * 9 + r * 9 + t], __ldg(p.d + r * Cin + i), pr);
          Ws[e] = __ldg(p.w_ortho + static_cast<size_t>(o0) * nW + e) + pr;
        }
        __syncthreads();
      }
    }
    for (int i = threadIdx.x; i < noc * nW; i += kThreads)
      p.W[static_cast<size_t>(o0) * nW + i] = Ws[i];
    if constexpr (kLinear)
      linear_mode::store_state<OC, kMaxRank * 9, kThreads>(p, o0, noc, lamS, lamMS, lamVS);
    __syncthreads();
  }
}

size_t wide_smem_bytes(int Cin, bool linear) {
  return (static_cast<size_t>(2 * OC) * Cin * 9 + OC * kMaxRank * 9 + kMiscFloats +
          (linear ? kLamFloats : 0)) * sizeof(float);
}

template <bool kLinear, bool kUp>
int wide_launch_mode(const InsertLoopParams& p, const float* blur, void* workspace,
                     size_t workspace_bytes, cudaStream_t stream) {
  const char* who = kUp ? "insert_loop_up" : "insert_loop_wide";
  // up mode: the T / gT planes are (2h+1)x(2w+1) per batch entry and channel
  const long long plane_px = kUp ? static_cast<long long>(p.B) * (2 * p.h + 1) * (2 * p.w + 1)
                                 : static_cast<long long>(p.B) * p.h * p.w;
  if (p.B < 1 || p.B > 4 || p.h < 1 || p.w < 1 || p.Cout < 1 || p.Cin < kMinCin || p.Cin % 32 != 0 ||
      p.Cin > kMaxCin || p.rank < 1 || p.rank > kMaxRank ||
      (p.Cout + OC) * plane_px > (1LL << 31) - 1) {
    set_last_error("%s: unsupported shape B=%d h=%d w=%d Cin=%d Cout=%d rank=%d "
                   "(B in [1,4], Cin %% 32 == 0 in [%d,%d], rank in [1,%d])",
                   who, p.B, p.h, p.w, p.Cin, p.Cout, p.rank, kMinCin, kMaxCin, kMaxRank);
    return RW_ERR_BAD_ARG;
  }
  if (kUp && (p.plain_conv != 0 || blur == nullptr)) {
    set_last_error("%s: %s", who, p.plain_conv ? "plain_conv has no upsampling target"
                                                : "NULL blur kernel");
    return RW_ERR_BAD_ARG;
  }
  const size_t need = kUp ? rw_insert_up_workspace_bytes(p.Cout, p.B, p.h, p.w)
                          : rw_insert_wide_workspace_bytes(p.Cout, p.B, p.h, p.w);
  if (workspace == nullptr || workspace_bytes < need) {
    set_last_error("%s: workspace %zu B < %zu B needed", who, workspace_bytes, need);
    return RW_ERR_BAD_ARG;
  }
  const size_t smem = wide_smem_bytes(p.Cin, kLinear);
  static size_t attr = 0;
  if (smem > attr) {
    int rc = check_cuda(cudaFuncSetAttribute(insert_wide_kernel<kLinear, kUp>,
                                             cudaFuncAttributeMaxDynamicSharedMemorySize,
                                             static_cast<int>(smem)),
                        "insert_loop_wide smem attr");
    if (rc) return rc;
    attr = smem;
  }
  const size_t cout4 = (static_cast<size_t>(p.Cout) + OC - 1) / OC * OC;
  const size_t plane = cout4 * static_cast<size_t>(plane_px);
  float* tG = static_cast<float*>(workspace);
  float* gdG = tG + plane;
  UpArgs up{};
  if (kUp) {
    up.gG = gdG + plane;                        // [Cout4][B*2h*2w]
    for (int t = 0; t < 16; ++t) up.blur[t] = blur[t];
  }
  int grid = (p.Cout + OC - 1) / OC;
  const int sms = device_sm_count();
  if (grid > sms) grid = sms;
  insert_wide_kernel<kLinear, kUp><<<grid, kThreads, smem, stream>>>(p, p.key, tG, gdG, up);
  return check_cuda(cudaGetLastError(), kUp ? "insert_loop_up launch" : "insert_loop_wide launch");
}

}  // namespace

}  // namespace rw

using namespace rw;

extern "C" {

size_t rw_insert_wide_workspace_bytes(int Cout, int B, int h, int w) {
  if (Cout < 1 || B < 1 || h < 1 || w < 1) return 0;
  const size_t cout4 = (static_cast<size_t>(Cout) + OC - 1) / OC * OC;
  return 2 * cout4 * static_cast<size_t>(B) * h * w * sizeof(float);
}

size_t rw_insert_up_workspace_bytes(int Cout, int B, int h, int w) {
  if (Cout < 1 || B < 1 || h < 1 || w < 1) return 0;
  const size_t cout4 = (static_cast<size_t>(Cout) + OC - 1) / OC * OC;
  const size_t t_px = static_cast<size_t>(2 * h + 1) * (2 * w + 1);   // T and gT
  const size_t g_px = static_cast<size_t>(2 * h) * (2 * w);           // g
  return cout4 * static_cast<size_t>(B) * (2 * t_px + g_px) * sizeof(float);
}

int rw_insert_loop_wide(const rw_insert_args* a, void* workspace, size_t workspace_bytes,
                        rw_stream_t stream) {
  InsertLoopParams p;
  int rc = insert_params(a, "rw_insert_loop_wide", p);
  if (rc) return rc;
  return wide_launch_mode<false, false>(p, nullptr, workspace, workspace_bytes, stream);
}

int rw_linear_insert_loop_wide(const rw_linear_insert_args* a, void* workspace,
                               size_t workspace_bytes, rw_stream_t stream) {
  InsertLoopParams p;
  int rc = linear_insert_params(a, "rw_linear_insert_loop_wide", p);
  if (rc) return rc;
  return wide_launch_mode<true, false>(p, nullptr, workspace, workspace_bytes, stream);
}

int rw_insert_loop_up(const rw_insert_args* a, const float blur[16], void* workspace,
                      size_t workspace_bytes, rw_stream_t stream) {
  InsertLoopParams p;
  int rc = insert_params(a, "rw_insert_loop_up", p);
  if (rc) return rc;
  return wide_launch_mode<false, true>(p, blur, workspace, workspace_bytes, stream);
}

int rw_linear_insert_loop_up(const rw_linear_insert_args* a, const float blur[16], void* workspace,
                             size_t workspace_bytes, rw_stream_t stream) {
  InsertLoopParams p;
  int rc = linear_insert_params(a, "rw_linear_insert_loop_up", p);
  if (rc) return rc;
  return wide_launch_mode<true, true>(p, blur, workspace, workspace_bytes, stream);
}

}  // extern "C"
