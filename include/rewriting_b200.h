/* rewriting_b200.h — the C-ABI drop-in boundary of librw_b200.so.
 *
 * Every entry point takes plain device pointers, sizes and a cudaStream_t, returns
 * 0 on success or a negative rw_status (never throws, never allocates device
 * memory: scratch is a caller-provided workspace), and runs asynchronously on the
 * given stream.  Pointers are borrowed; the caller (PyTorch in the shipped host
 * code) owns all storage.  This is the surface the reference's two pybind11
 * extension modules plus its library-call "kernels" are replaced by:
 *
 *   reference interface (file:line, relative to davidbau/rewriting)      -> entry point here
 *   -------------------------------------------------------------------------------------------
 *   fused.fused_bias_act(input,bias,refer,act,grad,alpha,scale)
 *       utils/stylegan2/op/fused_bias_act.cpp:11-21                        -> rw_fused_bias_act
 *   upfirdn2d_op.upfirdn2d(input,kernel,up_x,up_y,down_x,down_y,pads)
 *       utils/stylegan2/op/upfirdn2d.cpp:4-22                              -> rw_upfirdn2d
 *   ApplyStyle  style[:,:,None,None]*fmap  utils/stylegan2/models.py:616-620 -> rw_prep_keys
 *   DemodulatedConv2dF.forward (F.conv2d / F.conv_transpose2d + demod)
 *       utils/stylegan2/models.py:313-329                                  -> rw_prep_weights,
 *                                                                              rw_demod,
 *                                                                              rw_modconv_fwd,
 *                                                                              rw_modconv_up_fwd
 *   BlurF -> NoiseInjectionF -> FusedLeakyReLUF of an upsampling StyledConv
 *       utils/stylegan2/models.py:275-281,535-546,622-626                  -> rw_blur_up_act
 *   NoiseInjectionF.forward  utils/stylegan2/models.py:539-546             -> rw_add_noise
 *   ToRGBF.forward           utils/stylegan2/models.py:639-655             -> rw_torgb
 *   autograd of the ToRGB modulated 1x1 conv (torch.einsum)                -> rw_torgb,
 *                                                                              rw_torgb_mod_bwd
 *   autograd of the conv (dgrad / wgrad)                                    -> rw_modconv_fwd on
 *                                                                              gradient planes,
 *                                                                              rw_conv_wgrad
 *   RunningSecondMoment.add -> mom2.addbmm_(a[:,:,None], a[:,None,:])
 *       utils/runningstats.py:1086-1097,1181-1190                          -> rw_split_rows,
 *                                                                              rw_second_moment_accum
 *   projected_conv(weight, direction)  rewrite/ganrewrite.py:806-813       -> rw_project_rank
 *   ProgressiveGanRewriter.insert hot loop rewrite/ganrewrite.py:279-294   -> rw_insert_loop,
 *                                                                              rw_insert_loop_wide
 *                                           (upsampling target)           -> rw_insert_loop_up
 *   ProgressiveGanRewriter.linear_insert   rewrite/ganrewrite.py:201-252   -> rw_linear_insert_loop,
 *                                                                              rw_linear_insert_loop_wide
 *                                           (upsampling target)           -> rw_linear_insert_loop_up
 *
 * Layout vocabulary
 *   key planes  : the style-modulated key k = style*x as two bf16 planes (hi, lo; k ~= hi+lo)
 *                 in "padded-flat" channels-last order: row index = (b*(H+1) + y)*(W+1) + x,
 *                 y in [0,H], x in [0,W]; row H and column W are zero.  rows = B*(H+1)*(W+1).
 *   weight planes: scale*W as bf16 hi/lo, [Cout][tap][Cin] (tap = u*3+v) — or [Cin][tap'][Cout]
 *                 with flipped taps for dgrad.
 */
#ifndef REWRITING_B200_H_
#define REWRITING_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct CUstream_st* rw_stream_t; /* == cudaStream_t */

enum rw_status {
  RW_STATUS_OK = 0,
  RW_STATUS_BAD_ARG = -1,
  RW_STATUS_CUDA = -2,
  RW_STATUS_NO_DRIVER_SYMBOL = -3,
  RW_STATUS_UNSUPPORTED = -4
};

/* ---- library ---- */
int rw_version(void);
const char* rw_last_error(void);
int rw_set_device(int device);
int rw_device_sm_count(void);

/* ---- operand preparation ---- */
int rw_prep_keys(const float* x, const float* style, int B, int C, int H, int W, void* kp_hi,
                 void* kp_lo, float* k_out, rw_stream_t stream);
int rw_split_rows(const float* a, long long n, void* hi, void* lo, rw_stream_t stream);
int rw_prep_weights(const float* w, int Cout, int Cin, float scale, int transpose_io,
                    int flip_taps, void* wt_hi, void* wt_lo, float* wsq, rw_stream_t stream);
int rw_demod(const float* style, const float* wsq, int B, int Cout, int Cin, float eps,
             float* demod, rw_stream_t stream);

/* ---- fused modulated 3x3 convolution (wgmma) ---- */
/* Alignment, for every entry point on the tensor-core row-GEMM (rw_modconv_fwd, _up_fwd,
 * _fwd_fused, _up_fwd_cl, _up_dgrad, rw_rowgemm, rw_conv3x3_bias_act): fp32 pointers are 4-byte
 * aligned; next_scale, and the channels-last t_cl and its scale_bo (rw_modconv_up_fwd_cl), are
 * 8-byte aligned; next_hi / next_lo are 4-byte aligned.  Otherwise the call returns
 * RW_STATUS_BAD_ARG before anything is launched, with the reason in rw_last_error().  A scale_bo
 * that is only 4-byte aligned is accepted elsewhere, on the slower full epilogue. */
/* out[b,o,y,x] = act( conv3x3(k, scale*W)[b,o,y,x] * scale_bo[b,o] + noise_w[0]*noise[b,y*W+x] + bias[o] )
 * scale_bo / noise / bias may be NULL; noise_w is a DEVICE scalar (the nn.Parameter's storage,
 * so no host sync per layer); act: 0 none, 1 leaky_relu(0.2)*sqrt(2). */
int rw_modconv_fwd(const void* kp_hi, const void* kp_lo, const void* wt_hi, const void* wt_lo,
                   const float* scale_bo, const float* noise, long long noise_bstride,
                   const float* noise_w, const float* bias, int act, int B, int Cin, int Cout,
                   int H, int W, float* out, rw_stream_t stream);
/* t[b,o,:,:] = conv_transpose2d(k, (scale*W)^T, stride 2, pad 0)[b,o] * scale_bo[b,o]; out is
 * [B,Cout,2H+1,2W+1].  One launch: the four polyphase components are tile-interleaved (exact
 * algorithmic FLOPs, A tiles shared through L2). */
int rw_modconv_up_fwd(const void* kp_hi, const void* kp_lo, const void* wt_hi, const void* wt_lo,
                      const float* scale_bo, int B, int Cin, int Cout, int H, int W, float* t_out,
                      rw_stream_t stream);
/* ---- generation fast path: producers write the consumer's operands directly ----
 * rw_modconv_fwd_fused = rw_modconv_fwd whose epilogue can additionally emit
 *   next_{hi,lo}[rows][Cout] : key planes of the NEXT layer, split_bf16(next_scale[b,o] * y)
 *   rgb_part[Cout/64][B][3][H*W] : this layer's ToRGB partial sums (one per 64-channel group)
 *                                   with rgb_w[B,3,Cout]
 * `out` (fp32 NCHW) becomes optional.  rw_modconv_up_fwd_cl writes the conv_transpose output
 * channels-last per phase, t_cl[4][rows][Cout]; rw_blur_up_fused turns it into the next layer's
 * planes, split_bf16(next_scale[b,c] * leaky_relu(blur(t) + noise_w[0]*noise + bias)*sqrt(2));
 * rw_rgb_combine = sum of partials + bias + 2x-upsampled skip.
 * rw_blur_up_fused requires every pointer, C % 64 == 0, bias and next_scale 16-byte aligned,
 * and fewer than 2^31 rows in t_cl and 8x16-output tiles x 64-channel blocks; otherwise it returns
 * RW_STATUS_BAD_ARG before anything is launched. */
int rw_modconv_fwd_fused(const void* kp_hi, const void* kp_lo, const void* wt_hi,
                         const void* wt_lo, const float* scale_bo, const float* noise,
                         long long noise_bstride, const float* noise_w, const float* bias, int act,
                         int B, int Cin, int Cout, int H, int W, float* out,
                         const float* next_scale, void* next_hi, void* next_lo,
                         const float* rgb_w, float* rgb_part, rw_stream_t stream);
int rw_modconv_up_fwd_cl(const void* kp_hi, const void* kp_lo, const void* wt_hi,
                         const void* wt_lo, const float* scale_bo, int B, int Cin, int Cout, int H,
                         int W, float* t_cl, rw_stream_t stream);
int rw_blur_up_fused(const float* t_cl, int B, int C, int Hin, int Win, const float* kernel4x4,
                     const float* noise, long long noise_bstride, const float* noise_w,
                     const float* bias, const float* next_scale, void* next_hi, void* next_lo,
                     rw_stream_t stream);
/* The whole upsampling StyledConv of the fast path in ONE kernel (csrc/upconv_tc.cu):
 * conv_transpose2d(stride 2) -> 4x4 blur (pad 1,1) -> * demod -> + noise_w*noise + bias ->
 * leaky-ReLU*sqrt(2) -> * next_scale -> the next layer's bf16 hi/lo planes (pad row/column zeroed).
 * Replaces the reference chain models.py:313-329 (DemodulatedConv2dF, upsample branch) -> :275-281
 * (BlurF / upfirdn2d_kernel.cu:52-137) -> :535-546 (NoiseInjectionF) -> fused_bias_act_kernel.cu
 * :27-47, without ever writing the (2H+1)x(2W+1) fp32 conv_transpose output.
 * wt_{hi,lo}: rw_prep_weights(transpose_io = 2) planes [Cout/16][2 channel halves][9 taps][8][Cin]
 * (opaque to the caller: produced and consumed by this library only).  W must be a power
 * of two in [4, 128], Cin % 64 == 0, Cout % 16 == 0, the 4x4 kernel rank one (separable). */
int rw_modconv_up_fused(const void* kp_hi, const void* kp_lo, const void* wt_hi, const void* wt_lo,
                        const float* demod, const float* kernel4x4, const float* noise,
                        long long noise_bstride, const float* noise_w, const float* bias,
                        const float* next_scale, void* next_hi, void* next_lo, int B, int Cin,
                        int Cout, int H, int W, rw_stream_t stream);

/* The same kernel as the LAYER-level op (the autograd forward of an upsampling StyledConv,
 * reference models.py:232-289 with upsample=True): writes this layer's activation y
 * [B, Cout, 2H, 2W] fp32 NCHW instead of the next layer's planes.  demod may be NULL (no
 * demodulation), noise / noise_w NULL together (no noise injection), act = 0 skips bias + leaky-ReLU
 * (bias may then be NULL). */
int rw_modconv_up_fused_y(const void* kp_hi, const void* kp_lo, const void* wt_hi, const void* wt_lo,
                          const float* demod, const float* kernel4x4, const float* noise,
                          long long noise_bstride, const float* noise_w, const float* bias, int act,
                          float* y, int B, int Cin, int Cout, int H, int W, rw_stream_t stream);
/* all modulation linears in one launch: out_l[b,c] = latent[b,lat_l,:] . (W_l[c,:]*scale) + bias_l[c]
 * (HOST arrays of n device pointers / ints; n <= 32) */
int rw_styles(const float* latent, int B, int n_latent, int K, float scale, int n,
              const float* const* w, const float* const* bias, float* const* out, const int* lat,
              const int* chans, rw_stream_t stream);
/* EqualLinear (utils/stylegan2/models.py:487-511): out[b,c] = sum_k x[b,k]*(w[c,k]*scale) +
 * bias[c]*bias_mul, then lrelu(0.2)*sqrt(2) when act != 0 (the mapping network's
 * fused_lrelu layers, lr_mul = 0.01).  One launch per layer instead of sgemm + bias_act + two
 * elementwise kernels. */
int rw_equal_linear(const float* x, int B, int K, const float* w, const float* bias, int Cout,
                    float scale, float bias_mul, int act, float* out, rw_stream_t stream);
/* PixelNormL (models.py:609-614): out = z * rsqrt(mean(z^2, dim 1) + 1e-8), z [B,K] */
int rw_pixel_norm(const float* z, int B, int K, float* out, rw_stream_t stream);
/* Everything that depends only on the styles, for all layers in one launch (n <= 32 jobs):
 * kind 0: out[b,o] = rsqrt(sum_i style[b,i]^2 * w[o,i] + eps)  (w = wsq of rw_prep_weights; the
 *         demodulation factor of models.py:325-327);
 * kind 1: out[b,c,i] = (wscale*w[c,i])*style[b,i]  (ToRGB's modulated 1x1 weights, cout = 3). */
int rw_demod_multi(int B, float eps, int n, const float* const* style, const float* const* w,
                   float* const* out, const int* cout, const int* cin, const int* kind,
                   const float* wscale, rw_stream_t stream);
int rw_rgb_combine(const float* part, int nparts, int B, int H, int W, const float* bias,
                   const float* prev, const float* kernel4x4, float* out, rw_stream_t stream);
/* same, and/or the image as NHWC bytes  clamp(x*127.5 + 127.5, 0, 255)  (uint8 truncation): the
 * output side of the sampling loops (metrics/sample.py:33-37, utils/get_samples.py:121-127 move
 * fp32 NCHW images to the host one by one); `out` may be NULL when only the bytes are wanted */
int rw_rgb_combine_u8(const float* part, int nparts, int B, int H, int W, const float* bias,
                      const float* prev, const float* kernel4x4, float* out,
                      unsigned char* out_u8_nhwc, rw_stream_t stream);
/* y = act( upfirdn2d(t, k4x4, pad=(1,1)) + noise_w*noise + bias ), t [B,C,2H+1,2W+1] -> y [B,C,2H,2W] */
int rw_blur_up_act(const float* t, int B, int C, int Hin, int Win, const float* kernel4x4,
                   const float* noise, long long noise_bstride, const float* noise_w,
                   const float* bias, int act, float* y, rw_stream_t stream);
int rw_add_noise(const float* x, const float* noise, long long noise_bstride,
                 const float* noise_w, int B, int C, int HW, float* y, rw_stream_t stream);
int rw_torgb(const float* x, const float* style, const float* w, const float* bias,
             const float* skip, int B, int C, int H, int W, float scale, float* out,
             rw_stream_t stream);
/* Backward of rw_torgb with no bias and no skip (the modulated 1x1 conv to 3 channels,
 * y[b,o,p] = sum_i scale w[o,i] style[b,i] x[b,i,p]; x [B,C,H,W], w [3,C], gy [B,3,H,W]):
 *   gx[b,i,p] = scale style[b,i] sum_o w[o,i] gy[b,o,p]     R[b,o,i] = sum_p gy[b,o,p] x[b,i,p]
 *   gw[o,i]   = scale sum_b style[b,i] R[b,o,i]             gs[b,i]  = scale sum_o w[o,i] R[b,o,i]
 * Three launches: one pass over x / gy writing gx and per-chunk partial sums of R into
 * `workspace` (at least rw_torgb_mod_bwd_workspace_bytes bytes; 0 means the shape is refused),
 * then fixed-order sums.  Any of gx / gs / gw may be NULL, not all three. */
size_t rw_torgb_mod_bwd_workspace_bytes(int B, int C, int H, int W);
int rw_torgb_mod_bwd(const float* x, const float* style, const float* w, const float* gy, int B,
                     int C, int H, int W, float scale, float* gx, float* gs, float* gw,
                     void* workspace, size_t workspace_bytes, rw_stream_t stream);

/* ---- operator-level ops of the reference ---- */
int rw_fused_bias_act(const float* x, const float* bias, const float* ref, int act, int grad,
                      float alpha, float scale, long long n, int step_b, int size_b, float* y,
                      rw_stream_t stream);
int rw_upfirdn2d(const float* in, const float* kernel, int major, int in_h, int in_w, int kh,
                 int kw, int up_x, int up_y, int down_x, int down_y, int pad_x0, int pad_x1,
                 int pad_y0, int pad_y1, float* out, int out_h, int out_w, rw_stream_t stream);

/* ---- key second moment / weight gradient (wgmma col-GEMM) ---- */
size_t rw_gram_workspace_bytes(int Cm, int Cn, long long rows, int ntaps);
/* mom2[C,C] += sum_r a_r a_r^T over `rows` rows of the hi/lo planes [rows][C]; C % 64 == 0 (the
 * col-GEMM takes channel counts in multiples of 64, tiles of 128 where the count allows) */
int rw_second_moment_accum(const void* hi, const void* lo, long long rows, int C, float* mom2,
                           void* workspace, size_t workspace_bytes, rw_stream_t stream);
/* dW[o][tap][i] = sum_p G[p,o] * K[p + shift(tap), i]  for a 3x3 conv over the padded-flat grid
 * (up=0) or the conv_transpose phases (up=1: G planes are given per phase, see host code). */
int rw_conv_wgrad(const void* g_hi, const void* g_lo, const void* kp_hi, const void* kp_lo,
                  long long rows, int Cout, int Cin, int Wp, float* dw_toi, void* workspace,
                  size_t workspace_bytes, rw_stream_t stream);

/* backward of the upsampling layer: gradient phase planes [rows][4*Cout] (rw_prep_phase_keys from the
 * gradient wrt the conv_transpose output [B,Cout,2H+1,2W+1], times demod), then
 *   dk[b,i,y,x] = sum_{o,u,v} g[b,o,2y+u,2x+v] * scale*W[o,i,u,v]      (rw_modconv_up_dgrad, weights
 *                 as [Cin][tap][Cout] planes, taps NOT flipped)
 *   dW[o][tap][i] = sum_p G_phase(tap)[p + shift(tap), o] * K[p, i]     (rw_conv_up_wgrad) */
int rw_prep_phase_keys(const float* g, const float* scale_bc, int B, int C, int H, int W,
                       void* hi, void* lo, rw_stream_t stream);
int rw_modconv_up_dgrad(const void* gph_hi, const void* gph_lo, const void* wt_hi,
                        const void* wt_lo, const float* scale_bi, int B, int Cin, int Cout, int H,
                        int W, float* dk, rw_stream_t stream);
int rw_conv_up_wgrad(const void* gph_hi, const void* gph_lo, const void* kp_hi, const void* kp_lo,
                     long long rows, int Cout, int Cin, int Wp, float* dw_toi, void* workspace,
                     size_t workspace_bytes, rw_stream_t stream);

/* ---- StyledConv backward: the HBM-bound passes between the tensor-core kernels ----
 * (autograd of FusedLeakyReLUF / NoiseInjectionF / BlurF / ApplyStyle / the demodulation:
 *  utils/stylegan2/op/fused_act.py:19-86, utils/stylegan2/models.py:275-281,320-328,535-546,616-620)
 *
 * rw_act_grad_reduce: one pass over (gy, y) of a [B,C,HW] layer output y = act(t + nw*noise + bias):
 *   g_pre = dL/d(pre-activation) (written unless g_pre == NULL; equal to gy when act == 0),
 *   s_sum[b,c] = sum_p g_pre, s_dot[b,c] = sum_p g_pre*t (t recovered from y), s_noise[b,c] =
 *   sum_p g_pre*noise[b,p].  noise / bias may be NULL.
 * rw_blur_adj_phase_keys: gradient phase planes [rows][4*C] (the layout of rw_prep_phase_keys) of
 *   scale[b,c] * blur^T(g_pre), g_pre [B,C,2H,2W]; the [B,C,2H+1,2W+1] tensor is never stored.
 * rw_dgrad_finish: gs_raw[b,i] = sum_p dk*x; dk <- dk*style[b,i] in place ([B,C,HW] planes).
 * rw_wgrad_finish: gw[o,i,tap] = scale*dw_toi[o,tap,i] - scale^2*w[o,i,tap]*sum_b s_dot[b,o]*
 *   demod[b,o]^2*style[b,i]^2 (s_dot == NULL: no demodulation term).
 * rw_style_grad_finish: g_style[b,i] = gs_raw[b,i] - style[b,i]*sum_o s_dot[b,o]*demod[b,o]^2*
 *   wsq[o,i] (gs_raw == NULL: 0). */
int rw_act_grad_reduce(const float* gy, const float* y, const float* noise,
                       long long noise_bstride, const float* noise_w, const float* bias, int act,
                       int B, int C, int HW, float* g_pre, float* s_sum, float* s_dot,
                       float* s_noise, rw_stream_t stream);
int rw_blur_adj_phase_keys(const float* g_pre, const float* scale_bc, const float* kernel4x4, int B,
                           int C, int H, int W, void* hi, void* lo, rw_stream_t stream);
int rw_dgrad_finish(float* dk, const float* x, const float* style, int B, int C, int HW,
                    float* gs_raw, rw_stream_t stream);
int rw_wgrad_finish(const float* dw_toi, const float* w, const float* s_dot, const float* demod,
                    const float* style, int B, int Cout, int Cin, float scale, float* gw,
                    rw_stream_t stream);
int rw_style_grad_finish(const float* gs_raw, const float* style, const float* s_dot,
                         const float* demod, const float* wsq, int B, int Cout, int Cin,
                         float* g_style, rw_stream_t stream);

/* ---- rank-r edit ---- */
/* out = base + sign * P_d(w);  P_d(w)[o,:,t] = sum_r (w[o,:,t] . d_r) d_r;  base may be NULL */
int rw_project_rank(const float* w, const float* base, const float* d, int rank, int Cout,
                    int Cin, int taps, float sign, float* out, rw_stream_t stream);

typedef struct rw_insert_args {
  float* W;               /* [Cout,Cin,3,3], updated in place */
  float* m;               /* Adam exp_avg     */
  float* v;               /* Adam exp_avg_sq  */
  const float* w_ortho;   /* W0 - P_d(W0) or NULL (low_rank_insert off) */
  const float* d;         /* [rank,Cin] orthonormal rows */
  const float* key_cl;    /* key crop, zero-bordered channels-last [B][h+2][w+2][Cin] */
  const float* style;     /* [B,Cin] */
  const float* target;    /* goal activations v* [B,Cout,h,w] */
  const float* noise;     /* [B,h*w] or NULL */
  const float* bias;      /* [Cout] or NULL */
  float* loss_out;        /* [nsteps,Cout] per-channel sums of |v*-y| */
  float noise_w, lr, beta1, beta2, eps;
  int rank, B, Cin, Cout, h, w;
  int has_noise_act;      /* 1: target = dconv->noise->activate, 0: dconv only */
  int it0, nsteps, niter_total, piter, project_gradient;
  /* appended in round 2 (zero = the StyleGAN2 behaviour of round 1): */
  int plain_conv;          /* 1: y = conv(k, W) with no style demodulation and no 1/sqrt(9 Cin)
                              weight scale — the `layerN.conv` target of ProgressiveGanRewriter
                              (ganrewrite.py:25-96; `style` is then ignored and may be NULL) */
  float one_minus_beta1;   /* torch.optim.Adam forms 1-beta in double and rounds once to float */
  float one_minus_beta2;   /* (0 -> computed in the kernel as 1.0f - beta) */
  double beta1_exact;      /* the betas as the Python doubles torch forms its bias corrections */
  double beta2_exact;      /* 1 - beta**step from (0 -> the float fields above, widened) */
} rw_insert_args;
int rw_insert_loop(const rw_insert_args* args, rw_stream_t stream);
/* The same loop for key crops beyond rw_insert_loop's limits (w > 16, B*h*w > 4096 or a shared-
 * memory overflow): whole-map goals and wide selections, all iterations in one launch, same
 * fp32 arithmetic.  t and g*demod go to `workspace`, at least rw_insert_wide_workspace_bytes(Cout,
 * B, h, w) bytes (2 fp32 planes [Cout rounded up to 4][B*h*w]; 16.8 MB at 512 x 64 x 64), which the
 * call owns until it completes on `stream`.  Needs 1 <= B <= 4, Cin % 32 == 0, 128 <= Cin <= 512,
 * 1 <= rank <= 32; an unsupported shape or a short workspace returns RW_STATUS_BAD_ARG before
 * anything is launched. */
size_t rw_insert_wide_workspace_bytes(int Cout, int B, int h, int w);
int rw_insert_loop_wide(const rw_insert_args* args, void* workspace, size_t workspace_bytes,
                        rw_stream_t stream);

/* linear_insert (reference rewrite/ganrewrite.py:201-252): the same loop with Adam on Λ in
 * W = W0 + Λ d instead of on W.  Per iteration: forward, L1 gradient and dW exactly as above, then
 * dΛ[o,r,t] = Σ_i dW[o,i,t] d[r,i], one Adam step on Λ, and W = W0 + Λ d with the product and the
 * sum rounded separately (a rank-1 rebuild equals the reference's `W0 + einsum(...)` bit for bit).
 * There is no projection: base->w_ortho must be NULL and base->project_gradient and
 * base->plain_conv 0; base->m, base->v and base->piter are unused.  base->W is not read; at the end
 * of the call it holds W0 + Λ d, and lam / lam_m / lam_v hold the state to continue from
 * (it0 = the next iteration).  W0 must not alias base->W.  Shape limits are those of
 * rw_insert_loop / rw_insert_loop_wide (rw_insert_loop needs 13.5 KB more shared memory for the
 * Λ state).  A wrong struct_size, a NULL W0 / lam / moment buffer or a set w_ortho,
 * project_gradient or plain_conv returns RW_STATUS_BAD_ARG before anything is launched. */
typedef struct rw_linear_insert_args {
  size_t struct_size;            /* sizeof(rw_linear_insert_args), checked */
  const rw_insert_args* base;    /* shapes, key_cl, style, target, noise/bias, Adam constants,
                                    it0/nsteps/niter_total, loss_out; base->W receives W0 + Λd */
  const float* W0;               /* [Cout,Cin,3,3] original weight, read only */
  float* lam;                    /* [Cout,rank,3,3] Λ (zero before it0 = 0), updated in place */
  float* lam_m; float* lam_v;    /* Adam state of Λ, same shape */
} rw_linear_insert_args;
int rw_linear_insert_loop(const rw_linear_insert_args* args, rw_stream_t stream);
int rw_linear_insert_loop_wide(const rw_linear_insert_args* args, void* workspace,
                               size_t workspace_bytes, rw_stream_t stream);

/* The two loops above for the upsampling target of an odd StyleGAN2 layer: dconv (conv_transpose,
 * stride 2, no padding) -> blur (upfirdn2d with `blur`, pad (1,1)) -> noise -> activate.  h and w
 * are the key crop's size (key_cl as above); target is [B,Cout,2h,2w] and noise [B,4*h*w] or NULL.
 * `blur` is the layer's 4x4 blur kernel exactly as stored (mconv.blur.kernel, row-major), applied
 * flipped as upfirdn2d applies it; it is a host array, copied into the launch.  The conv_transpose
 * plane T, the output gradient g and gT = demod * blur^T(g) go to `workspace`, at least
 * rw_insert_up_workspace_bytes(Cout, B, h, w) bytes (fp32 planes [Cout rounded up to 4][B][...]:
 * two of (2h+1)x(2w+1) and one of 2h x 2w), which the call owns until it completes on `stream`.
 * Everything after dW (projections, low_rank_gradient, Adam, the Λ mode) is as in
 * rw_insert_loop_wide / rw_linear_insert_loop_wide.  Needs 1 <= B <= 4, Cin % 32 == 0,
 * 128 <= Cin <= 512, 1 <= rank <= 32 and plain_conv 0 (ProgGAN has no upsampling target); any other
 * shape, a NULL blur or a NULL or short workspace returns RW_STATUS_BAD_ARG before anything is
 * launched, with the reason in rw_last_error(). */
size_t rw_insert_up_workspace_bytes(int Cout, int B, int h, int w);
int rw_insert_loop_up(const rw_insert_args* args, const float blur[16], void* workspace,
                      size_t workspace_bytes, rw_stream_t stream);
int rw_linear_insert_loop_up(const rw_linear_insert_args* args, const float blur[16],
                             void* workspace, size_t workspace_bytes, rw_stream_t stream);

/* out[rows][N] = A[rows][K] . W[N][K]^T on the tensor-core row-GEMM (3-term split bf16 planes from
 * rw_split_rows; K % 64 == 0, N % 64 == 0): the key algebra between key capture and the
 * direction d — ZCA . k and ZCA . v of ganrewrite.py:107-110, 339-374 — without a cuBLAS call */
int rw_rowgemm(const void* a_hi, const void* a_lo, const void* w_hi, const void* w_lo, int rows, int K,
               int N, float* out, rw_stream_t stream);

/* ---- ProgGAN generator leaves (reference utils/proggan.py:128-181): the target of
 * ProgressiveGanRewriter is a plain `layerN.conv` (ganrewrite.py:25-96) ----
 * rw_pixel_norm_nchw: PixelNormLayer, x / sqrt(mean_c x^2 + 1e-8), optionally fused with the
 *   following DoubleResolutionLayer (nearest 2x, up2 = 1: out is [B,C,2H,2W]);
 * rw_nearest_up2: DoubleResolutionLayer alone on [planes,H,W];
 * rw_conv3x3_bias_act: 3x3 conv (pad 1) over key planes on the tensor-core row-GEMM with
 *   + bias[o] and leaky-ReLU(0.2) * act_gain in the epilogue — NormConvBlock's conv -> WScaleLayer
 *   -> LeakyReLU when the WScale factor is folded into the weight planes (rw_prep_weights scale). */
int rw_pixel_norm_nchw(const float* x, int B, int C, int H, int W, int up2, float* out,
                       rw_stream_t stream);
int rw_nearest_up2(const float* x, long long planes, int H, int W, float* out, rw_stream_t stream);
/* Backwards of the two leaves (gradients of a training loss through PixelNormLayer and
 * DoubleResolutionLayer).  rw_pixel_norm_nchw_bwd: gx [B,C,H,W] from the forward's input x
 * [B,C,H,W] and gy ([B,C,2H,2W] when up2 = 1, 8-byte aligned); rw_nearest_up2_bwd: gx
 * [planes,H,W] = 2 x 2 sums of gy [planes,2H,2W] (8-byte aligned).  Null pointers and sizes < 1
 * return RW_STATUS_BAD_ARG before any launch; neither call allocates or synchronises. */
int rw_pixel_norm_nchw_bwd(const float* x, const float* gy, int B, int C, int H, int W, int up2,
                           float* gx, rw_stream_t stream);
int rw_nearest_up2_bwd(const float* gy, long long planes, int H, int W, float* gx,
                       rw_stream_t stream);
int rw_conv3x3_bias_act(const void* kp_hi, const void* kp_lo, const void* wt_hi, const void* wt_lo,
                        const float* bias, int act, float act_gain, int B, int Cin, int Cout, int H,
                        int W, float* out, rw_stream_t stream);

/* ---- ProgGAN layers off the tensor-core path: fp32 on CUDA cores, fp32 NCHW in and out ----
 * Every call sums in a fixed order (two calls on the same input give the same bits), neither
 * allocates nor synchronises, and returns RW_STATUS_BAD_ARG before any launch for a null pointer,
 * a size < 1, a misaligned pointer where one is required or a short workspace.
 *
 * rw_proggan_input_fwd: the 4x4 "dense" first layer, Conv2d(Z, C, 4, padding 3) on z [B,Z]
 *   (the 1x1 input): out[b,o,y,x] = sum_i z[b,i] w[o,i,3-y,3-x], w [C,Z,4,4], out [B,C,4,4].
 *   bias == NULL: the bare conv (wscale unused); otherwise the block's epilogue
 *   leaky_relu(out * wscale + bias[o], 0.2).
 * rw_proggan_input_bwd: gz [B,Z] = W^T gy and gw [C,Z,4,4] = sum over the batch, in order, of
 *   gy (x) z; either output may be NULL.  w, gy and gw must be 16-byte aligned.
 * rw_narrow_conv3x3: 3x3 conv (pad 1, no bias) for any Cin, Cout >= 1 (tuned for <= 64
 *   channels), x [B,Cin,H,W], w [Cout,Cin,3,3]; bias / wscale as for the input layer.
 * rw_narrow_conv3x3_dgrad: gx [B,Cin,H,W] from gy [B,Cout,H,W] (the same kernel, weights read
 *   transposed and flipped).
 * rw_narrow_conv3x3_wgrad: gw [Cout,Cin,3,3] from x and gy: partial sums over pixel tiles into
 *   `workspace` (at least rw_narrow_conv3x3_wgrad_workspace_bytes bytes; 0 means the shape is
 *   refused), then a fixed-order sum.
 * rw_torgb1x1 / _dgrad / _wgrad: the 1x1 conv of the ToRGB block, Cin -> Cout (1 <= Cout <= 4),
 *   w [Cout,Cin,1,1]; the wgrad as above with its own workspace query.
 * rw_proggan_output_block: OutputConvBlock in one kernel: pixel norm -> 1x1 conv -> * wscale +
 *   bias -> Hardtanh (clamp != 0) or identity; the same bits as the four leaves. */
int rw_proggan_input_fwd(const float* z, const float* w, const float* bias, float wscale, int B,
                         int Z, int C, float* out, rw_stream_t stream);
int rw_proggan_input_bwd(const float* z, const float* w, const float* gy, int B, int Z, int C,
                         float* gz, float* gw, rw_stream_t stream);
int rw_narrow_conv3x3(const float* x, const float* w, const float* bias, float wscale, int B,
                      int Cin, int Cout, int H, int W, float* out, rw_stream_t stream);
int rw_narrow_conv3x3_dgrad(const float* gy, const float* w, int B, int Cin, int Cout, int H, int W,
                            float* gx, rw_stream_t stream);
size_t rw_narrow_conv3x3_wgrad_workspace_bytes(int B, int Cin, int Cout, int H, int W);
int rw_narrow_conv3x3_wgrad(const float* x, const float* gy, int B, int Cin, int Cout, int H, int W,
                            float* gw, void* workspace, size_t workspace_bytes, rw_stream_t stream);
int rw_torgb1x1(const float* x, const float* w, int B, int Cin, int Cout, int H, int W, float* out,
                rw_stream_t stream);
int rw_torgb1x1_dgrad(const float* gy, const float* w, int B, int Cin, int Cout, int H, int W,
                      float* gx, rw_stream_t stream);
size_t rw_torgb1x1_wgrad_workspace_bytes(int B, int Cin, int Cout, int H, int W);
int rw_torgb1x1_wgrad(const float* x, const float* gy, int B, int Cin, int Cout, int H, int W,
                      float* gw, void* workspace, size_t workspace_bytes, rw_stream_t stream);
int rw_proggan_output_block(const float* x, const float* w, const float* bias, float wscale,
                            int clamp, int B, int Cin, int Cout, int H, int W, float* out,
                            rw_stream_t stream);

/* ---- VGG feature stack: the passes between its convolutions (HBM-bound, fp32 on CUDA cores) ----
 * rw_relu_pool: one read of a conv output a [B,C,H,W] fp32 NCHW: v = relu(a + bias[c]) (bias may be
 *   NULL), then, when pool != 0, the 2x2 / stride-2 max pool with floor semantics (an odd last row
 *   or column is dropped; H, W >= 2), giving [B,C,Ho,Wo].  Writes the next conv's bf16 planes
 *   out_hi / out_lo [B*(Ho+1)*(Wo+1)][C] (the layout and split of rw_prep_keys with no style:
 *   hi = bf16_rn(v), lo = bf16_rn(v - hi), zero pad row / column; C % 64 == 0, 16-byte aligned),
 *   fp32 NCHW out, or both.  relu keeps a NaN; the pool scans its window in row-major order and
 *   takes a strictly greater value or a NaN (torch's max_pool2d).
 * rw_relu_pool_bwd: the gradient with respect to a, from the same a / bias / pool and gy
 *   [B,C,Ho,Wo] fp32 NCHW: every ReLU gate and pool argmax is re-derived with the forward's
 *   arithmetic; the argmax element gets 0 + gy, every other element and a dropped row / column get
 *   0, and an element whose relu output is <= 0 gets 0 (torch's threshold_backward).  Writes
 *   planes g_hi / g_lo [B*(H+1)*(W+1)][C] (for the conv_tc dgrad), fp32 NCHW g [B,C,H,W], or both.
 * Outputs must not overlap a or gy.  A null input, a size < 1, a pool on H or W < 2, neither or
 * only one plane, planes with C % 64 != 0 or a plane pointer that is not 16-byte aligned return
 * RW_STATUS_BAD_ARG before any launch.  Neither call allocates or synchronises; two calls give the
 * same bits. */
int rw_relu_pool(const float* a, const float* bias, int B, int C, int H, int W, int pool,
                 void* out_hi, void* out_lo, float* out, rw_stream_t stream);
int rw_relu_pool_bwd(const float* a, const float* bias, const float* gy, int B, int C, int H, int W,
                     int pool, void* g_hi, void* g_lo, float* g, rw_stream_t stream);

/* ---- edit distances: spatial LPIPS v0.1 (VGG-16, "net-lin") and the masked L1 (HBM-bound) ----
 * rw_lpips_input: im0, im1 as fp32 NCHW [B,3,H,W] in [-1, 1] (u8 == 0) or uint8 NHWC [B,H,W,3]
 *   (u8 == 1, decoded as (u / 255 - 0.5) / 0.5, each step one IEEE fp32 operation) through the
 *   scaling layer (x - shift[c]) / scale[c], shift = (-.030, -.088, -.188), scale = (.458, .448,
 *   .450): out [2B,3,H,W] fp32, images 0..B-1 from im0, B..2B-1 from im1.  The same bits as torch's
 *   elementwise ops.
 * rw_lpips_head: one tap.  a [2B,C,h,w] fp32 is the tap conv's output for both halves of the batch
 *   (bias [C] added here when the conv left it out, else NULL); f = relu(a + bias) and
 *   d[b,y,x] = sum_c lin_w[c] (f0 / (|f0| + 1e-10) - f1 / (|f1| + 1e-10))^2 over the channel vector
 *   at (y, x), f0 from image b and f1 from image b + B; d [B,h,w] fp32, formed in float64.
 * rw_lpips_combine: D[b,0,y,x] = sum over the nmaps (1..8) maps, in order, of maps[l] [B,h_l,w_l]
 *   bilinearly resized to H x W (torch's align_corners=False with the output size given), in
 *   float64; map_hw is a host array {h_0, w_0, h_1, w_1, ...} and maps a host array of device
 *   pointers.  D [B,1,H,W] is written when not NULL.  With num / den (float64 [B]):
 *   num[b] = sum D * mask, den[b] = sum mask, mask [mask_b,1,H,W] fp32 with mask_b 1 or B, or NULL
 *   for a mask of ones; partial sums over 1024-pixel tiles go to `workspace` (8-byte aligned, at
 *   least rw_lpips_combine_workspace_bytes bytes; 0 means the shape is refused) and a fixed-order
 *   finish adds them per image.
 * rw_masked_l1: the same reduction of sum_c |im1 - im0| per pixel (images as for rw_lpips_input, in
 *   [-1, 1] units), channels added in order in fp32; num and den are required.
 * A null required pointer, a size < 1, B > 65535, an unknown format, a mask batch other than 1 or
 * B, only one of num / den, or a short workspace return RW_STATUS_BAD_ARG before any launch.  No
 * call allocates or synchronises, and none uses atomics: two calls give the same bits, and image
 * b's results do not depend on the other images of the batch. */
int rw_lpips_input(const void* im0, const void* im1, int u8, int B, int H, int W, float* out,
                   rw_stream_t stream);
int rw_lpips_head(const float* a, const float* bias, const float* lin_w, int B, int C, int h, int w,
                  float* d, rw_stream_t stream);
size_t rw_lpips_combine_workspace_bytes(int B, int H, int W);
int rw_lpips_combine(int nmaps, const float* const* maps, const int* map_hw, int B, int H, int W,
                     const float* mask, int mask_b, float* D, double* num, double* den,
                     void* workspace, size_t workspace_bytes, rw_stream_t stream);
int rw_masked_l1(const void* im0, const void* im1, int u8, int B, int H, int W, const float* mask,
                 int mask_b, double* num, double* den, void* workspace, size_t workspace_bytes,
                 rw_stream_t stream);

/* ---- unified-parsing segmenter (ResNet-50 deep stem + UPerNet): the passes between its convs ----
 * The convolutions run on rw_conv3x3_bias_act (3x3), rw_rowgemm (1x1 on the planes, giving
 * channels-last padded rows [B*(H+1)*(W+1)][N]) and rw_narrow_conv3x3 (the 3-channel stem).
 * rw_seg_input: images as for rw_lpips_input (fp32 NCHW in [-1, 1] or uint8 NHWC) to the
 *   network's input out [B,3,S,S] fp32: (x + 1) / 2 * 255, channels reversed (RGB -> BGR), minus
 *   the mean (102.9801, 115.9465, 122.7717); when S < H, W the mean over each (H/S) x (W/S) block
 *   (AdaptiveAvgPool2d with an integer factor; S must divide H and W).
 * rw_seg_map: v[b,c,y,x] = a sampled at output (y, x) + bias[c] + res[b,c,y,x], then relu when
 *   relu = 1.  a is fp32 NCHW [B,C,Hin,Win] (a_cl = 0) or channels-last padded rows
 *   [B*(Hin+1)*(Win+1)][C] (a_cl = 1, the rw_rowgemm output).  mode 0: a at (y, x) (Ho = Hin,
 *   Wo = Win); mode 1: a at (2y, 2x) (Ho = ceil(Hin/2), Wo = ceil(Win/2): a stride-2 conv computed
 *   at stride 1); mode 2: bilinear resize to Ho x Wo (torch's align_corners=False, weights in
 *   float64).  bias, res may be NULL.  Writes fp32 NCHW out [B,C,Ho,Wo] and / or bf16 hi/lo planes
 *   [B*(Ho+1)*(Wo+1)][ldc] in channels coff..coff+C-1 (zero pad row / column; ldc, coff multiples
 *   of 64; 16-byte aligned), so a concatenation's planes are written slice by slice.  C % 64 == 0.
 * rw_seg_maxpool: MaxPool2d(3, stride 2, padding 1): out [B,C,(H-1)/2+1,(W-1)/2+1]; -inf padding,
 *   the window scanned in row-major order, a strictly greater value or a NaN wins.
 * rw_seg_prroi: PrRoI pooling of the whole map (ROI [0, 0, W, H], spatial scale 1) into s x s bins:
 *   out[b,c,i,j] = the integral of the bilinear surface of x (zero outside the map) over bin
 *   [jW/s, (j+1)W/s] x [iH/s, (i+1)H/s], divided by the bin's area; float64, fixed order.
 * rw_seg_classes: the class maps at Ho x Wo from the heads' logits.  logits is a host array of
 *   3 * nsizes device pointers, per segmentation size (object, part, material head), each the
 *   head's 1x1 output as padded rows [B*(h_s+1)*(w_s+1)][ld[head]] without its bias; map_hw the
 *   host array {h_0, w_0, ...}; bias a host array of the three heads' device bias vectors.  groups
 *   is a host array of ngroups (1..128) records {head, first channel, count, owner}: per group,
 *   at each size, the logits + bias bilinearly up-sampled to Ho x Wo and a softmax over the
 *   group's channels; the probabilities summed over the sizes.  probs [B,sum of counts,Ho,Wo]
 *   (groups in order) is written when not NULL.  labels [B,3,Ho,Wo] int64, when not NULL:
 *   channel 0 the argmax of group 0 (objects), channel 1 the argmax m of group 1 (materials),
 *   written as m + mat_offset or 0 for m = 0, channel 2 trans[first channel + argmax] of the
 *   part group g >= 2 whose owner is the pixel's object, else 0 (trans: device int64, indexed by
 *   part-head channel).  The argmax is the first maximum.
 * A null required pointer, a size < 1 or a shape outside these rules returns RW_STATUS_BAD_ARG
 * before any launch.  No call allocates or synchronises, none uses atomics: two calls give the
 * same bits, and image b's results do not depend on the other images of the batch. */
int rw_seg_input(const void* im, int u8, int B, int H, int W, int S, float* out, rw_stream_t stream);
int rw_seg_map(const float* a, int a_cl, int B, int C, int Hin, int Win, int mode, int Ho, int Wo,
               const float* bias, const float* res, int relu, void* out_hi, void* out_lo, int ldc,
               int coff, float* out, rw_stream_t stream);
int rw_seg_maxpool(const float* x, int B, int C, int H, int W, float* out, rw_stream_t stream);
int rw_seg_prroi(const float* x, int B, int C, int H, int W, int s, float* out, rw_stream_t stream);
int rw_seg_classes(int nsizes, const float* const* logits, const int* map_hw, const float* const* bias,
                   const int* ld, int ngroups, const int* groups, const long long* trans,
                   long long mat_offset, int B, int Ho, int Wo, float* probs, long long* labels,
                   rw_stream_t stream);

/* ---- dissection: unit / label intersection counts (GAN dissection, utils/quickdissect) ----
 * Both calls up-sample a layer's activations act [B,U,h,w] fp32 to H x W as torch's grid_sample
 * with align_corners=True and padding_mode='zeros' does over an axis-affine grid: output (y, x)
 * reads the source at (y * sy + oy, x * sx + ox) in pixel units (0 the first pixel's centre);
 * the two taps per axis are weighted linearly and taps outside the map read 0, so the border
 * fades toward 0.  The value is computed in float64 and rounded once to float.
 * rw_upsample_bilinear: rows [B*H*W][U] fp32, row (b*H + y)*W + x.
 * rw_dissect_counts: with the same up-sampled values v (the same bits as the rows above), the
 *   per-unit levels level [U] fp32 and the label maps labels [B,K,H,W] int64 (0 = no label,
 *   values in 0..C-1), ADDS to the caller's int64 counters: isect [C,U] the pixels that carry
 *   label c in at least one of their K channels and have v[u] > level[u]; unit_total [U] the
 *   pixels with v[u] > level[u]; label_total [C] the pixels carrying label c; count [1] B*H*W.
 *   Label 0 is never counted; labels outside 1..C-1 are skipped (callers check the range: the
 *   call cannot report it).  Integer atomics: the counts are exact and independent of launch
 *   order and of how a sample set is split into batches.
 * Sizes 1..1024, U <= 65535, K 1..8, C 2..32768, the grid's source coordinates within 2^20;
 * a null pointer or a shape outside these returns RW_STATUS_BAD_ARG before any launch.  No call
 * allocates or synchronises. */
int rw_upsample_bilinear(const float* act, int B, int U, int h, int w, int H, int W, double sy,
                         double oy, double sx, double ox, float* rows, rw_stream_t stream);
int rw_dissect_counts(const float* act, const float* level, const long long* labels, int B, int U,
                      int h, int w, int H, int W, int K, int C, double sy, double oy, double sx,
                      double ox, long long* isect, long long* unit_total, long long* label_total,
                      long long* count, rw_stream_t stream);

/* ---- per-phase profiles (tools/prof_upconv.py, tools/prof_conv.py) ---- */
/* rw_modconv_up_fused instrumented with clock64(): prof_out[grid][8 epilogue warps][16] = cycles in
 * {wait for the MMAs, accumulator exchange, combine + mailbox + barrier, shuffles, edge-lane fix-ups,
 * horizontal FIR, vertical FIR + activation + stores}, the step count, and the last phase split into
 * {FIR + activation + bf16 split, wait for the staging slots, stmatrix + fence + pair barrier, TMA store issue} and
 * the third of those into {stmatrix, fence.proxy.async, pair barrier} */
int rw_debug_upconv_profile(const void* kp_hi, const void* kp_lo, const void* wt_hi,
                            const void* wt_lo, const float* demod, const float* kernel4x4,
                            const float* noise, long long noise_bstride, const float* noise_w,
                            const float* bias, const float* next_scale, void* next_hi, void* next_lo,
                            int B, int Cin, int Cout, int H, int W, long long* prof_out,
                            rw_stream_t stream);
/* rw_modconv_fwd_fused on conv_tc's clock()-instrumented variant: prof_out[grid][8 consumer
 * warps][8] = cycles in {waiting on full barriers, issuing the main loop's MMAs (up to the wgmma
 * wait that lets a stage go), chunk drains + promotion, epilogue}, the tile count, the cycles from
 * the first tile to the end, and two zeros; grid <= the SM count */
int rw_debug_conv_profile(const void* kp_hi, const void* kp_lo, const void* wt_hi,
                          const void* wt_lo, const float* scale_bo, const float* noise,
                          long long noise_bstride, const float* noise_w, const float* bias, int act,
                          int B, int Cin, int Cout, int H, int W, float* out,
                          const float* next_scale, void* next_hi, void* next_lo,
                          const float* rgb_w, float* rgb_part, long long* prof_out,
                          rw_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* REWRITING_B200_H_ */
