// rewrite.cu — the rank-r projected-gradient weight edit.
//
// Reference: ProgressiveGanRewriter.insert (rewrite/ganrewrite.py:254-298) and
// projected_conv (ganrewrite.py:806-813).  Per iteration the reference runs
//   loss = L1(v*, target_model(k*)) ; backward ; Adam.step ;
//   every `piter` its:  W <- W_ortho + P_d(W)
// as ~60 separate framework kernels over a 9.4 MB weight.
//
// Observation that shapes this kernel: with the key detached, *every* quantity
// of one iteration is local to one output channel o — t[o,:], demod[o], the L1
// gradient, dW[o,:,:,:], the Adam moments and the projection all touch only
// row o of W.  So the whole loop needs no grid-wide synchronisation: a CTA owns
// a few output channels, keeps W[o] (18 KB) in shared memory across iterations,
// streams m/v through L2 and writes one partial loss per (iteration, channel).
//
// Key crop layout: kpT [B][h+2][w+2][Cin] fp32 (zero border, channels-last) so
// that lanes <-> input channels gives coalesced 128-byte loads.
#include "../../include/rewriting_b200.h"
#include "rw_common.cuh"
#include "insert_linear.cuh"

namespace rw {

namespace {

constexpr int kMaxW = 16;      // crop width handled by the register tile
constexpr int kMaxRank = 32;
constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;


// out[o,i,t] = base[o,i,t] + sign * sum_r d[r,i] * (sum_j W[o,j,t] d[r,j])
// one CTA per output channel o; row o of W is contiguous (Cin*taps floats).
__global__ void __launch_bounds__(kThreads)
project_rank_kernel(const float* __restrict__ w, const float* __restrict__ base,
                    const float* __restrict__ d, int rank, int Cin, int taps, float sign,
                    float* __restrict__ out) {
  extern __shared__ float sm[];
  float* ws = sm;                      // [Cin*taps]
  float* lam = sm + Cin * taps;        // [rank*taps]
  const int o = blockIdx.x;
  const int n = Cin * taps;
  const float* wrow = w + static_cast<size_t>(o) * n;
  for (int i = threadIdx.x; i < n; i += blockDim.x) ws[i] = wrow[i];
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int rt = warp; rt < rank * taps; rt += kWarps) {
    const int r = rt / taps, t = rt - r * taps;
    float acc = 0.f;
    for (int j = lane; j < Cin; j += 32) acc = fmaf(ws[j * taps + t], __ldg(d + r * Cin + j), acc);
#pragma unroll
    for (int off = 16; off; off >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, off);
    if (lane == 0) lam[rt] = acc;
  }
  __syncthreads();
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    const int ci = i / taps, t = i - ci * taps;
    float p = 0.f;
    for (int r = 0; r < rank; ++r) p = fmaf(lam[r * taps + t], __ldg(d + r * Cin + ci), p);
    const float b = base ? base[static_cast<size_t>(o) * n + i] : 0.f;
    out[static_cast<size_t>(o) * n + i] = b + sign * p;
  }
}

// ---------------------------------------------------------------------------
// fused insert loop
//
// One CTA owns OC = 4 output channels and runs all iterations for them.  The key crop
// (kpT, ~225 KB for 512 channels x 10 x 11) does not fit next to the weights in shared memory,
// so it is streamed from L2 — the dominant cost.  Blocking four output channels per CTA makes
// every loaded key value feed four accumulators (4x less L2 traffic than one channel per CTA:
// measured 180 us -> see profiles), and the register tile is templated on the crop width.
//
// kLinear selects the Λ mode (linear_insert, csrc/insert_linear.cuh): the same forward, loss and
// weight gradient, then Adam on Λ and W = W0 + Λ d instead of Adam on W and the projections.
// ---------------------------------------------------------------------------
constexpr int OC = 4;
constexpr int kMiscFloats = 64 + kWarps * OC * 5 + 64;   // demod, coef, loss and G tables
constexpr int kLamFloats = 3 * OC * kMaxRank * 9;       // Λ mode: Λ, exp_avg, exp_avg_sq

template <int MW, bool kLinear>   // register tile width >= crop width w
__global__ void __launch_bounds__(kThreads, 1)
insert_loop_kernel(const InsertLoopParams p, const float* __restrict__ kpT) {
  extern __shared__ float sm[];
  const int Cin = p.Cin, h = p.h, w = p.w, B = p.B;
  const int P = B * h * w;
  const int wp = w + 2;
  const int nW = Cin * 9;
  float* Ws = sm;                      // [OC][Cin*9]   current weight rows
  float* dWS = Ws + OC * nW;           // [OC][Cin*9]   gradient staging
  float* tS = dWS + OC * nW;           // [OC][P]       raw conv output t
  float* gdS = tS + OC * P;            // [OC][P]       g * demod (wgrad coefficient)
  float* lam = gdS + OC * P;           // [OC][kMaxRank*9]
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
  const float inv_numel = 1.0f / static_cast<float>(static_cast<long long>(B) * p.Cout * h * w);

  for (int o0 = blockIdx.x * OC; o0 < p.Cout; o0 += gridDim.x * OC) {
    const int noc = (p.Cout - o0 < OC) ? p.Cout - o0 : OC;
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
      // ---- forward conv on the crop: warp <-> row unit (b, y), lane <-> input channel;
      //      every key value loaded feeds the OC output channels
      for (int u = warp; u < B * h; u += kWarps) {
        const int b = u / h, y = u - b * h;
        float acc[OC][MW];
#pragma unroll
        for (int oc = 0; oc < OC; ++oc)
#pragma unroll
          for (int x = 0; x < MW; ++x) acc[oc][x] = 0.f;
        for (int j = 0; j < nch; ++j) {
          const int i = lane + 32 * j;
#pragma unroll
          for (int r = 0; r < 3; ++r) {
            const float* krow = kpT + ((static_cast<size_t>(b) * (h + 2) + y + r) * wp) * Cin + i;
            float kv[MW + 2];
#pragma unroll
            for (int x = 0; x < MW + 2; ++x)
              kv[x] = (x < wp) ? __ldg(krow + static_cast<size_t>(x) * Cin) : 0.f;
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
            if (lane == x && x < w) tS[oc * P + u * w + x] = sc * a;
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

      // ---- weight gradient: warp <-> channel group j, lane <-> input channel; OC x 9 accumulators
      for (int j = warp; j < nch; j += kWarps) {
        const int i = lane + 32 * j;
        float acc[OC][9];
#pragma unroll
        for (int oc = 0; oc < OC; ++oc)
#pragma unroll
          for (int t = 0; t < 9; ++t) acc[oc][t] = 0.f;
        for (int b = 0; b < B; ++b) {
          for (int y = 0; y < h; ++y) {
            float kv[3][MW + 2];
#pragma unroll
            for (int r = 0; r < 3; ++r) {
              const float* krow = kpT + ((static_cast<size_t>(b) * (h + 2) + y + r) * wp) * Cin + i;
#pragma unroll
              for (int x = 0; x < MW + 2; ++x)
                kv[r][x] = (x < wp) ? __ldg(krow + static_cast<size_t>(x) * Cin) : 0.f;
            }
#pragma unroll
            for (int oc = 0; oc < OC; ++oc) {
#pragma unroll
              for (int x = 0; x < MW; ++x) {
                const float gv = (x < w) ? gdS[oc * P + (b * h + y) * w + x] : 0.f;
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

template <int MW, bool kLinear>
static int launch_insert(const InsertLoopParams& p, size_t smem, cudaStream_t stream) {
  static size_t attr = 0;
  if (smem > attr) {
    int rc = check_cuda(cudaFuncSetAttribute(insert_loop_kernel<MW, kLinear>,
                                             cudaFuncAttributeMaxDynamicSharedMemorySize,
                                             static_cast<int>(smem)),
                        "insert_loop smem attr");
    if (rc) return rc;
    attr = smem;
  }
  int grid = (p.Cout + OC - 1) / OC;
  const int sms = device_sm_count();
  if (grid > sms) grid = sms;
  insert_loop_kernel<MW, kLinear><<<grid, kThreads, smem, stream>>>(p, p.key);
  return check_cuda(cudaGetLastError(), "insert_loop launch");
}

}  // namespace

template <bool kLinear>
static int insert_loop_launch_mode(const InsertLoopParams& p, cudaStream_t stream) {
  if (p.w > kMaxW || p.B > 4 || p.B < 1 || p.Cin % 32 != 0 || p.rank > kMaxRank || p.rank < 1 ||
      static_cast<long long>(p.B) * p.h * p.w > 4096) {
    set_last_error("insert_loop: unsupported crop B=%d h=%d w=%d Cin=%d rank=%d", p.B, p.h, p.w,
                   p.Cin, p.rank);
    return RW_ERR_UNSUPPORTED;
  }
  const int P = p.B * p.h * p.w;
  const int nW = p.Cin * 9;
  const size_t smem = (static_cast<size_t>(2 * OC) * nW + static_cast<size_t>(2 * OC) * P +
                       OC * kMaxRank * 9 + kMiscFloats + (kLinear ? kLamFloats : 0)) *
                      sizeof(float);
  if (smem > 225 * 1024) {
    set_last_error("insert_loop: shared memory %zu B too large", smem);
    return RW_ERR_UNSUPPORTED;
  }
  if (p.w <= 8) return launch_insert<8, kLinear>(p, smem, stream);
  if (p.w <= 12) return launch_insert<12, kLinear>(p, smem, stream);
  return launch_insert<16, kLinear>(p, smem, stream);
}

}  // namespace rw

using namespace rw;

extern "C" {

int rw_project_rank(const float* w, const float* base, const float* d, int rank, int Cout,
                    int Cin, int taps, float sign, float* out, rw_stream_t stream) {
  if (!w || !d || !out) {
    set_last_error("rw_project_rank: bad argument");
    return RW_ERR_BAD_ARG;
  }
  if (rank < 1 || rank > 64) {
    set_last_error("project_rank: rank=%d out of range [1,64]", rank);
    return RW_ERR_BAD_ARG;
  }
  const size_t smem = (static_cast<size_t>(Cin) * taps + static_cast<size_t>(rank) * taps) * 4;
  if (smem > 200 * 1024) {
    set_last_error("project_rank: row too large for shared memory (%zu B)", smem);
    return RW_ERR_UNSUPPORTED;
  }
  static size_t attr = 0;
  if (smem > 48 * 1024 && smem > attr) {
    int rc = check_cuda(cudaFuncSetAttribute(project_rank_kernel,
                                             cudaFuncAttributeMaxDynamicSharedMemorySize,
                                             static_cast<int>(smem)),
                        "project_rank smem attr");
    if (rc) return rc;
    attr = smem;
  }
  project_rank_kernel<<<Cout, kThreads, smem, stream>>>(w, base, d, rank, Cin, taps, sign, out);
  return check_cuda(cudaGetLastError(), "project_rank launch");
}

int rw_insert_loop(const rw_insert_args* a, rw_stream_t stream) {
  InsertLoopParams p;
  int rc = insert_params(a, "rw_insert_loop", p);
  if (rc) return rc;
  return insert_loop_launch_mode<false>(p, stream);
}

int rw_linear_insert_loop(const rw_linear_insert_args* a, rw_stream_t stream) {
  InsertLoopParams p;
  int rc = linear_insert_params(a, "rw_linear_insert_loop", p);
  if (rc) return rc;
  return insert_loop_launch_mode<true>(p, stream);
}

}  // extern "C"
