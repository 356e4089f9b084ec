/* hb200.h -- C ABI of libhb200.so: the H100 (sm_90a) DD-PPO learner hot path that
 * sits below habitat-baselines' Python registry classes.
 *
 * The reference (facebookresearch/habitat-lab) has NO native boundary: every hot-path
 * op is a PyTorch library call made from Python.  This header is the boundary a
 * maintainer would bind with ctypes from the reference's own classes; each entry point
 * cites the reference Python code it replaces (paths relative to the habitat-lab tree,
 * HB = habitat-baselines/habitat_baselines).
 *
 * Conventions
 *  - plain pointers + sizes only; all pointers are DEVICE pointers unless named h_*.
 *  - every function takes the cudaStream_t (as void*) to launch on and returns an int
 *    status: 0 ok, <0 error (message via hb200_last_error()).
 *  - the library never allocates or frees caller memory; scratch is passed in and sized
 *    by the *_workspace_bytes twin.
 *  - activations are NHWC.  16-bit tensors are raw uint16 storage typed by ROLE (both typedefs are uint16_t, the
 *    element format is fixed per argument): FORWARD values -- the pooled network input, conv outputs `y`, normalised
 *    activations, the packed forward weight images -- are IEEE fp16 (11-bit significand: what the reference's TF32
 *    cuDNN convolutions keep of their operands); GRADIENTS (g / dy / dx / gz / addend), the transposed (dgrad)
 *    weight images and the `*_bf16` twin outputs read by the weight-gradient kernels are bfloat16.  The
 *    tensor core (wgmma) needs both MMA operands in ONE format, so the forward kernels can write a second, bf16-rounded copy
 *    of an activation (`out_bf16`, optional): the weight gradient dW = sum x * dy then multiplies bf16 x with bf16 dy.
 *    Rounding x there is harmless (a linear perturbation); rounding it in the FORWARD pass is not (it flips ReLU /
 *    max-pool decisions), which is why the forward copy is fp16.
 */
#ifndef HB200_H_
#define HB200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define HB200_OK 0
#define HB200_ERR_INVALID_ARG (-1)
#define HB200_ERR_CUDA (-2)
#define HB200_ERR_UNSUPPORTED (-3)

typedef void* hb200_stream_t; /* cudaStream_t */
typedef uint16_t hb200_bf16; /* bfloat16 bits: gradients, dgrad weight images, bf16 activation twins */
typedef uint16_t hb200_f16;  /* IEEE fp16 bits: forward values */

/* ---- library ---------------------------------------------------------------- */
const char* hb200_last_error(void);
int hb200_version(void);
/* number of kernel launches issued through this library since load (bench's gpu_launches) */
long long hb200_launch_count(void);

/* ---- GAE return scan + advantages ---------------------------------------------
 * replaces RolloutStorage.compute_returns (HB/common/rollout_storage.py:174-205)
 * fused with PPO.get_advantages / _compute_var_mean (HB/rl/ppo/ppo.py:139-157).
 *
 * rewards, value_preds, returns, advantages: f32 [t_alloc, n_envs] (row pitch = n_envs)
 * masks: u8/bool [t_alloc, n_envs]; next_value: f32 [n_envs] written to value_preds[t_cur]
 * (use_gae) or returns[t_cur] (!use_gae) exactly like the reference.
 * t_cur = current_rollout_step_idx; t_alloc = numsteps+1 (advantages cover ALL t_alloc rows,
 * including the bootstrap row and stale rows -- reference quirk, ppo.py:140-149).
 * advantages may be NULL (returns only).  stats (f64[4], may be NULL): sum, sum of squares,
 * count over FINITE advantages, spare -- the raw material of the (distributed) var/mean.
 * variant: 0 auto, 1 thread-per-env serial scan (reference summation order), 2 warp-per-env
 * shuffle scan (affine-map composition; differs from the serial order by fp32 rounding only).
 */
int hb200_gae_adv(const float* rewards, float* value_preds, const uint8_t* masks,
                  const float* next_value, float* returns, float* advantages, double* stats,
                  int t_cur, int t_alloc, int n_envs, float gamma, float tau, int use_gae,
                  int variant, hb200_stream_t stream);

/* advantages <- (advantages - mean) * rsqrt(var + 1e-5) in place (ppo.py:151-153).
 * mode 0: single process, unbiased torch.var_mean over finite entries computed from stats
 * (ppo.py:155-157).  mode 1: mean/var given in mean_var[2] on device (distributed path,
 * HB/rl/ddppo/algo/ddppo.py:59-84, after the caller's all-reduce). */
int hb200_adv_normalize(float* advantages, long long n, const double* stats,
                        const float* mean_var, int mode, hb200_stream_t stream);

/* ---- action/value heads + PPO loss, forward and backward in one pass -------------
 * replaces CategoricalNet + CriticHead (HB/utils/common.py:64-96, HB/rl/ppo/policy.py:416-424)
 * and the loss section of PPO._update_from_batch (HB/rl/ppo/ppo.py:195-250, 260-275).
 *
 * features f32 [B,H]; w_act f32 [A,H], b_act [A]; w_val f32 [1,H], b_val [1]; actions i64 [B];
 * old_log_probs, advantages, old_values, returns f32 [B]; is_coeffs f32 [B] or NULL (VER).
 * Outputs: values, log_probs, entropy f32 [B] (any may be NULL); d_features f32 [B,H];
 * d_w_act [A,H], d_b_act [A], d_w_val [H], d_b_val [1] (OVERWRITTEN, not accumulated);
 * metrics f32 [HB200_LOSS_NMETRICS].  compute_grads=0 -> forward/metrics only.
 * workspace: hb200_ppo_loss_workspace_bytes(B,H,A).  1 <= A <= 8, H in {32, 64, 128, 256, 512}; anything else is
 * refused with an argument error.
 * NaN: min / max / clamp propagate NaN as torch.min / torch.max / torch.clamp do.  A NaN input reaches exactly the
 * outputs it reaches in the reference's autograd (a NaN old_value or value takes the value-clipped branch, whose value
 * gradient is 0); an action outside [0, A) has log-probability NaN, which poisons that frame's loss, ratio metrics,
 * d_features row and the action-head gradients.
 */
#define HB200_LOSS_NMETRICS 12
enum {
  HB200_M_VALUE_LOSS = 0, HB200_M_ACTION_LOSS = 1, HB200_M_DIST_ENTROPY = 2,
  HB200_M_VALUE_MIN = 3, HB200_M_VALUE_MEAN = 4, HB200_M_VALUE_MAX = 5,
  HB200_M_RATIO_MIN = 6, HB200_M_RATIO_MEAN = 7, HB200_M_RATIO_MAX = 8,
  HB200_M_FRAC_CLIPPED = 9, HB200_M_TOTAL_LOSS = 10, HB200_M_SPARE = 11
};
size_t hb200_ppo_loss_workspace_bytes(int batch, int hidden, int n_actions);
int hb200_ppo_loss(const float* features, const float* w_act, const float* b_act,
                   const float* w_val, const float* b_val, const int64_t* actions,
                   const float* old_log_probs, const float* advantages, const float* old_values,
                   const float* returns, const float* is_coeffs, int batch, int hidden,
                   int n_actions, float clip_param, float value_loss_coef, float entropy_coef,
                   int use_clipped_value_loss, int compute_grads, float* values, float* log_probs,
                   float* entropy, float* d_features, float* d_w_act, float* d_b_act,
                   float* d_w_val, float* d_b_val, float* metrics, void* workspace,
                   hb200_stream_t stream);

/* ---- clip_grad_norm_ + Adam on flat buffers ---------------------------------------
 * replaces nn.utils.clip_grad_norm_ + torch.optim.Adam(foreach=True).step()
 * (HB/rl/ppo/ppo.py:112-137, 257, 347-371).
 * params/grads/exp_avg/exp_avg_sq: f32 [n].  grad_norm_out: f32[1] device (the pre-clip total
 * L2 norm, what clip_grad_norm_ returns).  hyper: f32[8] DEVICE or NULL -> if non-NULL, lr is
 * read from hyper[0] (LambdaLR mutates lr every update; keeps the launch graph-capturable).
 * step = 1-based Adam step count for bias correction.  max_grad_norm <= 0 disables clipping.
 * grad_scale multiplies grads first (1/world_size when the all-reduce was a SUM).
 * workspace: hb200_clip_adam_workspace_bytes(n).  A NaN gradient norm makes every parameter and moment NaN when
 * max_grad_norm > 0, as clip_grad_norm_'s clamp does.
 */
size_t hb200_clip_adam_workspace_bytes(long long n);
int hb200_grad_sqnorm(const float* grads, long long n, float grad_scale, float* sqnorm_out,
                      void* workspace, hb200_stream_t stream);
int hb200_clip_adam(float* params, const float* grads, float* exp_avg, float* exp_avg_sq,
                    long long n, float lr, float beta1, float beta2, float eps, float weight_decay,
                    float max_grad_norm, float grad_scale, long long step, const float* hyper,
                    float* grad_norm_out, void* workspace, hb200_stream_t stream);

/* ---- visual input prep ----------------------------------------------------------------
 * replaces ResNetEncoder.forward's permute/float/scale/cat/avg_pool2d
 * (HB/rl/ddppo/policy/resnet_policy.py:255-271) and RunningMeanAndVar
 * (HB/rl/ddppo/policy/running_mean_and_var.py:24-78).
 *
 * Sources are the rollout buffers in place (no minibatch gather copy,
 * HB/common/rollout_storage.py:236-246): rgb u8 [rows,H,W,c_rgb] (may be NULL, c_rgb=0),
 * depth f32 [rows,H,W,c_depth] (may be NULL).  frame_rows i32 [B]: buffer row of each frame.
 * Channel order = rgb then depth (observation-space order).  C = c_rgb + c_depth <= 8.
 * stats_acc f64 [17]: [0,8) per-channel sum, [8,16) sum of squares of the 2x2-pooled input,
 * [16] number of frames (the reference's new_count = x.size(0)); with >1 ranks the caller
 * all-reduces (SUM) these 17 doubles -- one packed collective instead of the reference's three.
 */
int hb200_prep_stats(const uint8_t* rgb, const float* depth, const int32_t* frame_rows, int batch,
                     int height, int width, int c_rgb, int c_depth, float rgb_scale,
                     double* stats_acc, hb200_stream_t stream);
/* Welford merge of the batch stats into (_mean,_var,_count) f32 buffers [C],[C],[1]
 * (running_mean_and_var.py:50-68) and scale/shift f32 [2*8] for the normalise pass (:70-78).
 * world_size > 1: stats_acc must already hold the all-reduced SUM over ranks. update=0 skips
 * the merge (eval mode) and only refreshes scale_shift. */
int hb200_prep_finalize(const double* stats_acc, float* run_mean, float* run_var, float* run_count,
                        float* scale_shift, int channels, long long pixels_per_frame, int update,
                        hb200_stream_t stream);
/* pooled + normalised NHWC bf16 [B,H/2,W/2,8] (channels >= C zero padded), or with s2d != 0 the
 * space-to-depth form [B,H/4,W/4,16] (channel = (dy*2+dx)*4 + c) that turns the 7x7 stride-2 stem into
 * a 4x4 stride-1 convolution.  scale_shift NULL -> no normalisation (normalize_visual_inputs=False). */
int hb200_prep_apply(const uint8_t* rgb, const float* depth, const int32_t* frame_rows, int batch,
                     int height, int width, int c_rgb, int c_depth, float rgb_scale,
                     const float* scale_shift, hb200_f16* out, hb200_bf16* out_bf16, int s2d,
                     hb200_stream_t stream);

/* SimpleCNN input (HB/rl/models/simple_cnn.py:139-157): rgb/255 and raw depth concatenated, fp16 NHWC
 * [B,H,W,8] (forward values, act_t; channels past c_rgb + c_depth are zero), no pooling; rows gathered through
 * frame_rows.  The fp16 pack saturates: |depth| > 65504 and +-inf become +-65504, NaN stays NaN.  `out` holds fp16
 * bits despite its pointer type */
int hb200_prep_plain(const uint8_t* rgb, const float* depth, const int32_t* frame_rows, int batch, int height,
                     int width, int c_rgb, int c_depth, hb200_bf16* out, hb200_stream_t stream);
/* backward of conv+bias -> ReLU: dy = g * (out > 0) (out = post-ReLU activation; NULL -> no mask),
 * dbias[C] += per-channel sums of dy (caller zeroes); dy may be NULL (bias gradient only) */
int hb200_relu_bias_bwd(const hb200_bf16* g, const hb200_bf16* out, hb200_bf16* dy, float* dbias, long long npix,
                        int channels, hb200_stream_t stream);
/* fp16 NHWC [B,hw,C] (a forward activation, act_t; `x` holds fp16 bits despite its pointer type) -> f32 [B, C*hw]
 * in (c,h,w) order (nn.Flatten of the NCHW map) */
int hb200_bf16_hwc_to_f32_chw(const hb200_bf16* x, float* out, int batch, int hw, int channels,
                              hb200_stream_t stream);

/* ---- implicit-GEMM convolution on the tensor cores (wgmma) --------------------------------
 * replaces nn.Conv2d forward / backward-data / backward-weight as dispatched by
 * HB/rl/ddppo/policy/resnet.py:15-34,207-219 and resnet_policy.py:224-234 (cuDNN today).
 *
 * x bf16 NHWC [B,Hi,Wi,Ci]; w_packed bf16 [Co][kh*kw*Ci padded to 64] (hb200_pack_conv_weight);
 * y bf16 NHWC [B,Ho,Wo,Co].  Ci % 8 == 0, Co % 16 == 0, Co <= 256 or Co % 256 == 0.
 * gn_stats f64 [B, gn_groups, 2] or NULL (double accumulators: the atomics become order-independent
 * after rounding, so the forward pass is run-to-run reproducible): per-(frame,group) sum / sum-of-squares of the fp32
 * accumulators are atomically added (GroupNorm statistics fused into the conv epilogue).
 * addend (dgrad only) bf16 [B,Hi,Wi,Ci] or NULL: dx = conv_dgrad + addend (residual grad).
 */
typedef struct {
  int batch, hi, wi, ci, ho, wo, co, kh, kw, stride, pad;
} hb200_conv_shape;

int hb200_conv_fwd(const hb200_bf16* x, const hb200_bf16* w_packed, hb200_bf16* y,
                   double* gn_stats, int gn_groups, const hb200_conv_shape* s,
                   hb200_stream_t stream);
/* forward with per-channel bias (+ReLU) fused in the epilogue: SimpleCNN's biased convs
 * (HB/rl/models/simple_cnn.py:68-93) */
int hb200_conv_bias_act_fwd(const hb200_bf16* x, const hb200_bf16* w_packed, const float* bias, hb200_bf16* y,
                            int relu, const hb200_conv_shape* s, hb200_stream_t stream);
/* dy [B,Ho,Wo,Co] -> dx [B,Hi,Wi,Ci]; w_packed_t bf16 [Ci][kh*kw*Co padded] (transposed pack) */
int hb200_conv_dgrad(const hb200_bf16* dy, const hb200_bf16* w_packed_t, const hb200_bf16* addend,
                     hb200_bf16* dx, const hb200_conv_shape* s, hb200_stream_t stream);
/* dw_acc f32 [kh*kw*Ci][Co], ACCUMULATED (+=; caller zeroes): per-split partials summed in a fixed order */
int hb200_conv_wgrad(const hb200_bf16* x, const hb200_bf16* dy, float* dw_acc,
                     const hb200_conv_shape* s, hb200_stream_t stream);
/* f32 OIHW [Co,Ci_real,kh,kw] -> bf16 [Co][(r,s,ci) padded] (ci_pad >= ci_real, zero filled),
 * and the transposed pack [Ci_pad][(r,s,co) padded] used by dgrad.  Both are stored as
 * ready-to-copy shared-memory tile images (see hb200_set_umma_layout). */
int hb200_pack_conv_weight(const float* w_oihw, hb200_bf16* w_packed, hb200_bf16* w_packed_t,
                           int co, int ci_real, int ci_pad, int kh, int kw, hb200_stream_t stream);
/* dw_acc f32 [(r,s,ci_pad)][Co] -> f32 OIHW grad [Co,Ci_real,kh,kw] (overwrite) */
int hb200_unpack_conv_wgrad(const float* dw_acc, float* dw_oihw, int co, int ci_real, int ci_pad,
                            int kh, int kw, hb200_stream_t stream);

/* number of bf16 elements of a packed weight image with n_rows GEMM rows and
 * kh*kw*k_channels reduction length (padded to the 64-element K chunk) */
size_t hb200_packed_weight_elems(int n_rows, int k_channels, int kh, int kw);
/* shared-memory operand layout used by the conv kernels AND the weight images
 * (0 = no-swizzle interleaved core matrices, 1 = 128-byte swizzle); set before packing. */
int hb200_set_umma_layout(int layout);
int hb200_get_umma_layout(void);

/* ---- "halo" convolutions: stride-1 k x k layers (k=3 pad 1; k=4 = the space-to-depth stem) ----------
 * Each CTA loads the input halo of a 16x8 output tile once and addresses every filter tap with a
 * shifted wgmma shared-memory descriptor (no im2col re-reads); persistent CTAs keep the weights
 * (forward/dgrad) or the accumulators (wgrad) resident.  Same reference ops as hb200_conv_* above.
 * wimg: hb200_pack_halo_weight image [taps][C/8][N][8] (mode 0 forward, 1 dgrad, 2 stem).
 * mode 0 forward (gn_stats optional) / 1 data gradient (addend optional). */
int hb200_conv_halo_supported(int c, int n, int k, int h, int w);
int hb200_pack_halo_weight(const float* w_oihw, hb200_bf16* img, int co, int ci_real, int c, int n, int k,
                           int mode, hb200_stream_t stream);
int hb200_conv_halo(const hb200_bf16* x, const hb200_bf16* wimg, hb200_bf16* y, const hb200_bf16* addend,
                    double* gn_stats, int gn_groups, int batch, int h, int w, int c, int n, int k, int mode,
                    hb200_stream_t stream);
/* Halo loader of the forward / dgrad halo kernels: 0 = zero-filling cp.async gather (also HB200_NO_HALO_TMA=1 in the
 * environment), 1 = the measured best TMA variant per layer (default), 2 = TMA copies of whole pixel rows into the
 * swizzled K-major layout, 3 = warp-specialised pipeline over 16-byte channel slabs, 4 = warp-specialised + swizzled
 * rows, 5 = plain TMA slabs.  All are kept parity-tested (tests/test_gpu_kernels.py::test_conv_halo_3x3). */
int hb200_set_halo_tma(int mode);
int hb200_get_halo_tma(void);
/* x halo of the halo weight-gradient kernels: 0 = register staging / cp.async, 1 = one 5-D TMA box per tile (default;
 * HB200_WGRAD_XTMA=0 in the environment selects 0 at load time) */
int hb200_set_wgrad_xtma(int on);
int hb200_get_wgrad_xtma(void);

/* 1 if hb200_conv_halo_wgrad serves this 3x3 / stem shape: the hb200_conv_halo_supported shapes plus the small-image
 * layers (8x8 and 4x4 inputs, c % 32 == 0, n % 128 == 0: layer3 / layer4 / compression of
 * HB/rl/ddppo/policy/resnet.py:196-281, resnet_policy.py:200-240), whose tiles span several images. */
int hb200_conv_halo_wgrad_supported(int c, int n, int k, int h, int w);

/* ---- stride-2 block entry: 3x3 stride-2 pad-1 conv + 1x1 stride-2 downsample conv of the same input -------------------
 * (BasicBlock with a downsample branch, HB/rl/ddppo/policy/resnet.py:26-77, 143-160), one TMA-fed halo kernel per
 * direction over the 2x2 space-to-depth VIEW of x (5-D tensor map on the NHWC tensor, no copy): see csrc/conv_s2.cu.
 *   forward: x f16 [B,H,W,C] -> ya f16 [B,H/2,W/2,NA] (3x3 branch), yb f16 [B,H/2,W/2,NB] (1x1 branch), each with
 *            optional fused GroupNorm sums (stats f64 [B,G,2], pre-zeroed).
 *            wimg = hb200_pack_halo_weight(mode 0, c = C, n = NA + NB, k = 3) of the concatenated filter
 *            [NA + NB, C, 3, 3] whose last NB rows hold the 1x1 filter in the centre tap, zeros elsewhere.
 *   dgrad:   dx bf16 [B,H,W,C] = conv3x3^T(dya) + conv1x1^T(dyb) (+ addend); wimg_t = the same concatenated filter
 *            packed with mode 1 (c = NA + NB, n = C).
 * Supported: C = 32, NA = NB = 64, H % 32 == 0, W % 16 == 0 (layer2.0 of the resnet18 encoder at 256x256 input). */
int hb200_conv_s2_supported(int c, int na, int nb, int h, int w);
/* forward / dgrad variant: 1 (default) = warp-specialised pipeline over swizzled 128-byte pixel-row copies, 0 = one-thread
 * pipeline over 16-byte channel slabs (HB200_NO_CONV_S2_WS=1 in the environment selects 0 at load time) */
int hb200_set_conv_s2_ws(int on);
int hb200_get_conv_s2_ws(void);
/* weight gradient of the 3x3 stride-2 branch over the same space-to-depth view (x halo = one 5-D TMA box per tile):
 * x bf16 [B,H,W,C] (twin of the forward input), dy bf16 [B,H/2,W/2,N]; dw_acc f32 [16*C][N], pre-zeroed, rows
 * ((ky*2+kx)*4 + dy*2+dx)*C + c; hb200_unpack_s2_wgrad writes the 9 real taps as OIHW.  C = 32, N = 64. */
int hb200_conv_s2_wgrad_supported(int c, int n, int h, int w);
int hb200_conv_s2_wgrad(const hb200_bf16* x, const hb200_bf16* dy, float* dw_acc, int batch, int h, int w, int c, int n,
                        hb200_stream_t stream);
int hb200_unpack_s2_wgrad(const float* dw_acc, float* dw_oihw, int co, int ci, hb200_stream_t stream);
int hb200_conv_s2_fwd(const hb200_f16* x, const hb200_f16* wimg, hb200_f16* ya, hb200_f16* yb, double* stats_a,
                      int groups_a, double* stats_b, int groups_b, int batch, int h, int w, int c, int na, int nb,
                      hb200_stream_t stream);
int hb200_conv_s2_dgrad(const hb200_bf16* dya, const hb200_bf16* dyb, const hb200_bf16* wimg_t,
                        const hb200_bf16* addend, hb200_bf16* dx, int batch, int h, int w, int c, int na, int nb,
                        hb200_stream_t stream);

/* dw_acc f32 [(r*k+s)*C + ci][N] accumulated (+=; caller zeroes) in a fixed order, like hb200_conv_wgrad */
int hb200_conv_halo_wgrad(const hb200_bf16* x, const hb200_bf16* dy, float* dw_acc, int batch, int h, int w,
                          int c, int n, int k, hb200_stream_t stream);
/* stem accumulator [(a*4+b)*16 + (dy,dx,c)][Co] -> f32 OIHW [Co,Ci_real,7,7] */
int hb200_unpack_stem_wgrad(const float* dw_acc, float* dw_oihw, int co, int ci_real, hb200_stream_t stream);

/* raw wgmma GEMM probe: D[M,N] f32 = A[M,K] * B[N,K]^T (bf16, or fp16 with flags 16 | 32: both operands share one
 * format), M%128==0, N in {16, 32, 64, 128}, K%64==0.  layout: 0 = K-major no-swizzle interleaved core matrices,
 * 1 = K-major 128B swizzle, 2 = MN-major no-swizzle (then A is given as [K,M], B as [K,N]).
 * Used by the tests to pin the smem/instruction descriptor encodings on hardware. */
int hb200_umma_gemm_probe(const hb200_bf16* a, const hb200_bf16* b, float* d, int m, int n, int k,
                          int layout, hb200_stream_t stream);

/* ---- GroupNorm / ReLU / pooling / residual elementwise passes (bf16 NHWC) ---------------
 * replace nn.GroupNorm, nn.ReLU, nn.MaxPool2d and the residual add of BasicBlock
 * (HB/rl/ddppo/policy/resnet.py:37-69, 207-219, 272-281).
 * stats f64 [B,G,2] = (sum, sumsq) over the (C/G)*H*W elements of each group (conv epilogue).
 */
/* out = act(gamma * (y - mu) * rstd + beta);  relu: 0/1;  out_f32: 0 -> bf16 NHWC, 1 -> f32 NHWC,
 * 2 -> f32 [B, C*hw] flattened in (c,h,w) order (what nn.Flatten of the NCHW map feeds visual_fc) */
int hb200_gn_apply(const hb200_f16* y, const double* stats, const float* gamma, const float* beta,
                   void* out, hb200_bf16* out_bf16, int out_f32, int batch, int hw, int channels, int groups,
                   float eps, int relu, hb200_stream_t stream);
/* out = relu(GN(y) + res)  with res either an activation tensor (res_stats NULL) or a second
 * pre-norm tensor normalised with (res_stats, res_gamma, res_beta) (downsample branch). */
int hb200_gn_residual_relu(const hb200_f16* y, const double* stats, const float* gamma,
                           const float* beta, const hb200_f16* res, const double* res_stats,
                           const float* res_gamma, const float* res_beta, hb200_f16* out,
                           hb200_bf16* out_bf16, int batch, int hw, int channels, int groups, float eps,
                           hb200_stream_t stream);
/* out[B,H/2,W/2,C] = maxpool3x3s2p1(relu(GN(y[B,H,W,C]))); argmax u8 (0..8) saved for bwd */
int hb200_gn_relu_maxpool(const hb200_f16* y, const double* stats, const float* gamma,
                          const float* beta, hb200_f16* out, hb200_bf16* out_bf16, uint8_t* argmax, int batch,
                          int h, int w, int channels, int groups, float eps, hb200_stream_t stream);
/* dz[B,H,W,C] (grad wrt the GN output BEFORE relu masking is applied by the GN backward)
 * scattered from dout[B,H/2,W/2,C] through argmax */
int hb200_maxpool_bwd(const hb200_bf16* dout, const uint8_t* argmax, hb200_bf16* dz, int batch,
                      int h, int w, int channels, hb200_stream_t stream);
/* GroupNorm backward, two passes.  g = upstream grad wrt the activation that follows GN.
 * mask_mode 0: no ReLU (g is grad wrt z);  1: ReLU directly after GN (mask = z > 0, z recomputed);
 * 2: mask from `act` tensor (mask = act > 0; block output relu(GN(y)+res)).
 * pass 1 accumulates sums f32 [B,G,2] = (sum gamma*gz, sum gamma*gz*xhat) and dgamma/dbeta f32 [C]
 * (atomics, caller zeroes); pass 2 writes dy (grad wrt the conv output y) and, if gz_out != NULL,
 * the masked upstream grad gz (the residual-branch gradient). */
int hb200_gn_bwd_reduce(const hb200_bf16* g, const hb200_bf16* act, const hb200_bf16* y,
                        const double* stats, const float* gamma, const float* beta, float* sums,
                        float* dgamma, float* dbeta, int batch, int hw, int channels, int groups,
                        float eps, int mask_mode, hb200_stream_t stream);
/* both passes in one launch: a thread-block cluster owns a frame, stages it in shared memory (cp.async), reduces
 * through distributed shared memory and writes dy / gz_out from the staged copy, so every operand crosses HBM once.
 * dgamma/dbeta are accumulated (caller zeroes). */
int hb200_gn_bwd(const hb200_bf16* g, const hb200_bf16* act, const hb200_bf16* y, const double* stats,
                 const float* gamma, const float* beta, float* dgamma, float* dbeta, hb200_bf16* dy,
                 hb200_bf16* gz_out, int batch, int hw, int channels, int groups, float eps, int mask_mode,
                 hb200_stream_t stream);

/* Squeeze-excite block output (SEBottleneck, resnet.py:92-110, 155-180), one launch:
 *   z = GN(y);  p = mean_hw(z) [B,C];  h = relu(w1 p + b1) [B,reduced];  s = sigmoid(w2 h + b2) [B,C];
 *   out = relu(s * z + res)
 * w1 f32 [reduced, C], b1 [reduced], w2 [C, reduced], b2 [C] (nn.Linear layout); p, h, s f32 are written for the
 * backward.  res takes both forms of hb200_gn_residual_relu.  reduced = C / 16 in the reference; it must be a multiple
 * of 4 that divides 256. */
int hb200_gn_se_residual_relu(const hb200_f16* y, const double* stats, const float* gamma, const float* beta,
                              const hb200_f16* res, const double* res_stats, const float* res_gamma,
                              const float* res_beta, const float* w1, const float* b1, const float* w2,
                              const float* b2, float* p, float* h, float* s, hb200_f16* out, hb200_bf16* out_bf16,
                              int batch, int hw, int channels, int groups, int reduced, float eps,
                              hb200_stream_t stream);
/* Backward of hb200_gn_se_residual_relu's main branch: g = grad wrt out, act = out (ReLU mask).  Writes dy (grad wrt y),
 * gz_out = g * [out > 0] (the residual branch's gradient, may be NULL), adds the GroupNorm affine gradients to
 * dgamma / dbeta (caller zeroes), and writes a = (sum_hw gz * z) * s * (1 - s) [B,C] and dh = (w2^T a) * [h > 0]
 * [B,reduced]: the excitation weight gradients are dw2 = a^T h, db2 = sum_B a, dw1 = dh^T p, db1 = sum_B dh. */
int hb200_gn_se_bwd(const hb200_bf16* g, const hb200_bf16* act, const hb200_bf16* y, const double* stats,
                    const float* gamma, const float* beta, const float* s, const float* h, const float* w1,
                    const float* w2, float* dgamma, float* dbeta, hb200_bf16* dy, hb200_bf16* gz_out, float* a,
                    float* dh, int batch, int hw, int channels, int groups, int reduced, float eps,
                    hb200_stream_t stream);

/* Stem backward in one pass: MaxPool2d(3,2,1) backward (argmax codes from hb200_gn_relu_maxpool) + ReLU backward +
 * GroupNorm backward (resnet.py:244-252).  dpool bf16 [B,H/2,W/2,C] is the gradient of the pooled activation, y / dy
 * bf16 [B,H,W,C] the stem conv output and its gradient; the full-resolution pooled gradient is never written.
 * _supported() tells whether a (h, w, channels) shape can be tiled (else: hb200_maxpool_bwd + hb200_gn_bwd). */
int hb200_gn_relu_maxpool_bwd_supported(int h, int w, int channels, int groups);
int hb200_gn_relu_maxpool_bwd(const hb200_bf16* dpool, const uint8_t* argmax, const hb200_bf16* y,
                              const double* stats, const float* gamma, const float* beta, float* dgamma,
                              float* dbeta, hb200_bf16* dy, int batch, int h, int w, int channels, int groups,
                              float eps, hb200_stream_t stream);
int hb200_gn_bwd_apply(const hb200_bf16* g, const hb200_bf16* act, const hb200_bf16* y,
                       const double* stats, const float* gamma, const float* beta,
                       const float* sums, hb200_bf16* dy, hb200_bf16* gz_out, int batch, int hw,
                       int channels, int groups, float eps, int mask_mode, hb200_stream_t stream);

/* ---- fp32 SIMT GEMM (linears, LSTM projections) ---------------------------------------------
 * C[M,N] = alpha * op(A)[M,K] * op(B)[K,N] (+ bias[N]) (+ C if accumulate), optional ReLU.
 * A(m,k) = a[m*a_ms + k*a_ks], B(k,n) = b[k*b_ks + n*b_ns], C row pitch ldc.
 * replaces nn.Linear forward/backward (cuBLAS sgemm): visual_fc (resnet_policy.py:587-594),
 * LSTM/GRU input projections and weight gradients (rnn_state_encoder.py:380-422).
 */
int hb200_sgemm(const float* a, long long a_ms, long long a_ks, const float* b, long long b_ks,
                long long b_ns, float* c, long long ldc, const float* bias, int m, int n, int k,
                float alpha, int accumulate, int relu, hb200_stream_t stream);
/* Same contract on the tensor cores: wgmma .tf32 (operands stay fp32 in memory, read as TF32 --
 * the precision of the reference's cuDNN RNN path on CUDA -- fp32 accumulation).  Both operands must be
 * K-major (a_ks == 1 and b_ks == 1; transposed operands go through hb200_transpose_f32) with 16-byte
 * aligned rows (leading dimensions multiples of 4 floats).  Weight gradients
 * (accumulate != 0, long K) are split over K; the splits are summed in split order. */
int hb200_tgemm(const float* a, long long a_ms, long long a_ks, const float* b, long long b_ks, long long b_ns,
                float* c, long long ldc, const float* bias, int m, int n, int k, int accumulate, int relu,
                hb200_stream_t stream);
/* operand feed of hb200_tgemm: 1 (default) = TMA box loads, 0 = the 16-byte cp.async gather (kept for A/B tests;
 * environment HB200_NO_TGEMM_TMA=1 selects it at load time) */
int hb200_set_tgemm_tma(int on);
int hb200_get_tgemm_tma(void);
/* dst[c,r] = src[r,c] (fp32): feeds hb200_tgemm K-major operands for the data / weight gradient GEMMs */
int hb200_transpose_f32(const float* src, long long ld_src, float* dst, long long ld_dst, int rows, int cols,
                        hb200_stream_t stream);
/* out_bf16[i] = bf16(x_f16[i]) (n % 8 == 0): the bf16 twin of a forward activation produced by a conv epilogue
 * (SimpleCNN, HB/rl/models/simple_cnn.py:68-93), read by the weight-gradient kernels */
int hb200_f16_to_bf16(const hb200_f16* x, hb200_bf16* out, long long n, hb200_stream_t stream);
/* out[i] = f32(x_bf16[i]) and out_bf16[i] = bf16(x_f32[i]) (round to nearest even), n a positive multiple of 8 */
int hb200_bf16_to_f32(const hb200_bf16* x, float* out, long long n, hb200_stream_t stream);
int hb200_f32_to_bf16(const float* x, hb200_bf16* out, long long n, hb200_stream_t stream);

/* ---- recurrent state encoder ------------------------------------------------------------------
 * replaces RNNStateEncoder.seq_forward/single_forward with nn.LSTM / nn.GRU and the whole
 * packed-sequence machinery build_pack_info_from_dones/build_rnn_inputs/build_rnn_out_from_seq
 * (HB/rl/models/rnn_state_encoder.py:35-277, 301-371): the masked recurrence
 *   h_in = h_{t-1} * m_t ; (h_t, c_t) = cell(x_t, h_in, c_in)
 * is exactly what that machinery computes (pinned by test/test_rnn_state_encoder.py:72-94).
 *
 * One call = one time step of one layer (frames of step t are rows [t*n, (t+1)*n)).
 * xproj f32 [n, 4H] = x_t W_ih^T + b_ih precomputed for all frames by hb200_sgemm; b_hh f32 [4H]
 * (may be NULL) is added in the step kernel.
 * w_hh f32 [G*H, H] (PyTorch gate order i,f,g,o / r,z,n).  masks u8 [n] (1 = not done).
 * h_prev/c_prev f32 [n,H] (row pitch H); outputs h,c [n,H]; gates_out f32 [n,G*H] saved
 * activations for backward (i,f,g,o post-nonlinearity).  GRU (config #3) is a "next" row.
 */
int hb200_lstm_step_fwd(const float* xproj, const float* w_hh, const float* b_hh, const uint8_t* masks,
                        const float* h_prev, long long h_prev_stride, const float* c_prev,
                        long long c_prev_stride, float* h, float* c, float* gates_out, int n,
                        int hidden, hb200_stream_t stream);
/* backward of one step: dh_out f32 [n,H] = grad wrt h_t from above (layer output, may be NULL);
 * dh_rec/dc_rec f32 [n,H] = recurrent grads from step t+1 (already masked; NULL at the last
 * step).  Writes dgates f32 [n,4H] (pre-activation grads = d xproj), dh_prev, dc_prev [n,H]
 * (masked by m_t, i.e. grads wrt h_{t-1}, c_{t-1}). */
int hb200_lstm_step_bwd(const float* dh_out, const float* dh_rec, const float* dc_rec,
                        const float* gates, const float* c, const float* c_prev,
                        long long c_prev_stride, const float* w_hh, const uint8_t* masks,
                        float* dgates, float* dh_prev, float* dc_prev, int n, int hidden,
                        hb200_stream_t stream);
/* Whole-sequence persistent versions (ONE cooperative launch per layer; W_hh slices stay in shared
 * memory for all T steps, CTAs exchange h_t / dgates_t through L2 with one grid barrier per step).
 * xproj [T*n,4H], masks u8 [T*n], hs/cs [T,n,H], gates [T,n,4H] (NULL in inference), h0/c0 [n,H]
 * with row strides.  workspace: >= 64 bytes of device memory (barrier counter). */
int hb200_lstm_seq_fwd(const float* xproj, const float* w_hh, const float* b_hh, const uint8_t* masks,
                       const float* h0, long long h0_stride, const float* c0, long long c0_stride,
                       float* hs, float* cs, float* gates_out, int t_steps, int n, int hidden,
                       void* workspace, hb200_stream_t stream);
/* dh_out [T,n,H] = gradient wrt the layer output; writes dgates [T,n,4H] (= d xproj), which must be 16-byte aligned
 * (it is read back with 16-byte loads; a misaligned pointer is an argument error). */
int hb200_lstm_seq_bwd(const float* dh_out, const float* gates, const float* cs, const float* c0,
                       long long c0_stride, const float* w_hh, const uint8_t* masks, float* dgates,
                       int t_steps, int n, int hidden, void* workspace, hb200_stream_t stream);
/* The same launch over a time chunk of a longer sequence (chunks are processed last-to-first): carry f32 [2][n][H]
 * holds (dh, dc) flowing into the step before the chunk's first one -- read when carry_in, written when carry_out.
 * c0 must then be the cell state of the step before the chunk (cs row of step t0 - 1, stride H).  hidden == 512 only.
 * With hb200_lstm_seq_fwd called per chunk (h0 / c0 = the previous chunk's last hs / cs rows) two stacked layers run
 * as a wavefront on two streams; every launch needs its own workspace. */
int hb200_lstm_seq_bwd_chunk(const float* dh_out, const float* gates, const float* cs, const float* c0,
                             long long c0_stride, const float* w_hh, const uint8_t* masks, float* dgates,
                             int t_steps, int n, int hidden, void* workspace, float* carry, int carry_in,
                             int carry_out, hb200_stream_t stream);
/* GRU (gate order r,z,n), same persistent cooperative structure.  xproj [T*n,3H] = x W_ih^T + b_ih;
 * saved [T,n,4H] = (r, z, n, W_hn h + b_hn) for backward (NULL in inference).  Backward writes
 * dgx [T,n,3H] = d xproj (-> dW_ih, db_ih, dx) and dgh [T,n,3H] = d(h-side pre-activations) (-> dW_hh, db_hh); dgh must
 * be 16-byte aligned (it is read back with 16-byte loads; a misaligned pointer is an argument error). */
int hb200_gru_seq_fwd(const float* xproj, const float* w_hh, const float* b_hh, const uint8_t* masks,
                      const float* h0, long long h0_stride, float* hs, float* saved, int t_steps, int n, int hidden,
                      void* workspace, hb200_stream_t stream);
int hb200_gru_seq_bwd(const float* dh_out, const float* saved, const float* hs, const float* h0, long long h0_stride,
                      const float* w_hh, const uint8_t* masks, float* dgx, float* dgh, int t_steps, int n, int hidden,
                      void* workspace, hb200_stream_t stream);
/* h_in[t] = (t == 0 ? h0 : h_seq[t-1]) * m_t for the whole sequence (input of dW_hh = dG^T h_in) */
int hb200_rnn_shift_mask(const float* h_seq, const float* h0, long long h0_row_stride,
                         const uint8_t* masks, float* h_in, int t_steps, int n, int hidden,
                         hb200_stream_t stream);
/* out[N] (+)= column sums of x[M,N] (bias gradients) */
int hb200_colsum(const float* x, long long ld, float* out, long long m, int n, int accumulate,
                 hb200_stream_t stream);
/* d[r,c] = 0 where y[r,c] <= 0, c < cols (ReLU backward on a column block; row pitches ld_*) */
int hb200_relu_bwd(float* d, const float* y, long long ld_d, long long ld_y, long long rows, int cols,
                   hb200_stream_t stream);
/* out[f, :] = src[frame_rows[f], :] for f < batch (f32 rows of row_elems, a multiple of 4; 16-byte aligned buffers):
 * the minibatch's cached visual features of a frozen encoder, read from the rollout storage for the visual_fc GEMM */
int hb200_gather_rows(const float* src, const int32_t* frame_rows, float* out, int batch, long long row_elems,
                      hb200_stream_t stream);
/* f32 [B, C*hw] flattened in (c,h,w) order (nn.Flatten of NCHW, resnet_policy.py:587-594)
 * -> bf16 NHWC [B,hw,C]: the gradient of visual_fc's input re-enters the NHWC conv stack */
int hb200_f32_chw_to_bf16_hwc(const float* x, hb200_bf16* out, int batch, int hw, int channels,
                              hb200_stream_t stream);
/* actor path: logits f32 [B,A] and values f32 [B] only (HB/rl/ppo/policy.py:300-359) */
int hb200_heads_fwd(const float* features, const float* w_act, const float* b_act, const float* w_val,
                    const float* b_val, int batch, int hidden, int n_actions, float* logits,
                    float* values, hb200_stream_t stream);
/* the whole tail of Policy.act (HB/rl/ppo/policy.py:300-359: action_distribution(features), critic(features),
 * distribution.sample() / .mode(), distribution.log_probs(action)) in one launch.  log_probs f32 [B,A] = normalised
 * logits (what CustomFixedCategorical holds); actions i64 [B]; action_log_probs f32 [B].  uniform f32 [B] in [0,1): the
 * draw is the inverse CDF at uniform[b] (same distribution as torch.multinomial, different random stream);
 * uniform == NULL takes the mode (deterministic=True). */
int hb200_heads_act(const float* features, const float* w_act, const float* b_act, const float* w_val,
                    const float* b_val, const float* uniform, int batch, int hidden, int n_actions,
                    float* log_probs, float* values, long long* actions, float* action_log_probs,
                    hb200_stream_t stream);

/* ---- goal / previous-action embeddings --------------------------------------------------------
 * replaces tgt_embeding + prev_action_embedding + torch.cat of PointNavResNetNet.forward
 * (HB/rl/ddppo/policy/resnet_policy.py:658-692, 747-763).
 * goal f32 [rows,2] gathered through frame_rows; prev_actions i64 [B]; masks u8 [B] (per frame).
 * Writes columns [col0, col0+32) (goal) and [col0+32, col0+64) (prev action) of out f32 [B,ld].
 */
int hb200_embed_fwd(const float* goal, const int64_t* prev_actions, const uint8_t* masks,
                    const int32_t* frame_rows, const float* w_tgt, const float* b_tgt,
                    const float* emb_table, float* out, int ld, int col0, int batch,
                    hb200_stream_t stream);
/* d_out f32 [B,ld]; d_w_tgt [32,3], d_b_tgt [32], d_emb [A+1,32] accumulated (+=) in a fixed frame order */
int hb200_embed_bwd(const float* goal, const int64_t* prev_actions, const uint8_t* masks,
                    const int32_t* frame_rows, const float* d_out, int ld, int col0, int batch,
                    int n_emb, float* d_w_tgt, float* d_b_tgt, float* d_emb,
                    hb200_stream_t stream);

/* ---- generic 1-D sensors of PointNavResNetNet.forward (HB/rl/ddppo/policy/resnet_policy.py:658-763) ------------
 * x f32 [rows, in_dim] is a rollout observation buffer addressed through frame_rows (int32 [batch]).
 * transform: 0 identity (gps :730-733, pointgoal :695-697, proximity :699-701, 1-D fuse keys :649-656),
 *            1 2-D polar pointgoal (r, cos(-t), sin(-t)) (:662-673), 2 3-D polar (:674-691),
 *            3 angle -> (cos, sin) (compass :718-728, heading :703-712).
 * out[f, col0 + j] = b[j] + sum_k w[j, k] feat_k  (w f32 [out_dim, n_feat], nn.Linear layout; out_dim <= 64);
 * w == NULL copies the features themselves (fuse keys).  _bwd adds to d_w / d_b; frames are summed in a fixed order
 * (per-chunk partials, then reduce_partials), so the result is the same every run. */
int hb200_sensor_linear_fwd(const float* x, int in_dim, const int32_t* frame_rows, int batch, int transform,
                            const float* w, const float* b, float* out, int ld, int col0, int out_dim,
                            hb200_stream_t stream);
int hb200_sensor_linear_bwd(const float* x, int in_dim, const int32_t* frame_rows, int batch, int transform,
                            const float* d_out, int ld, int col0, int out_dim, float* d_w, float* d_b,
                            hb200_stream_t stream);
/* nn.Embedding lookups: out[f, col0 + j] = table[k_f, j] with k_f = idx[frame_rows[f]] (objectgoal, :714-716;
 * frame_rows NULL -> idx[f]) or, when masks (u8 [batch]) is given, masks[f] ? idx[f] + 1 : 0 (previous action with
 * its start token, :747-757).  An index outside the table poisons the row with NaN.  _bwd: d_table[k_f] += d_out row. */
int hb200_index_embed_fwd(const int64_t* idx, const int32_t* frame_rows, const uint8_t* masks, int batch,
                          int table_rows, const float* table, int width, float* out, int ld, int col0,
                          hb200_stream_t stream);
int hb200_index_embed_bwd(const int64_t* idx, const int32_t* frame_rows, const uint8_t* masks, int batch,
                          int table_rows, int width, const float* d_out, int ld, int col0, float* d_table,
                          hb200_stream_t stream);
/* Generic visual input prep (ResNetEncoder.forward, HB/rl/ddppo/policy/resnet_policy.py:255-271) for ANY sensor mix
 * and size: up to 4 HWC sources (h_* are HOST arrays of n_srcs entries: device pointers, dtype 0 u8 / 1 f32 / 2 i32,
 * channels, pre-pool scale = 1/high for u8 keys), <= 8 channels in total, concatenated in order, avg_pool2d(2) (odd
 * last row / column dropped).  stats_acc != NULL: statistics pass (17 doubles like hb200_prep_stats); otherwise the
 * apply pass writes out f16 [batch, H/2, W/2, 8] (+ optional bf16 twin) normalised with scale_shift (NULL: raw). */
int hb200_prep_generic(const void* const* h_srcs, const int* h_dtypes, const int* h_channels, const float* h_scales,
                       int n_srcs, const int32_t* frame_rows, int batch, int height, int width,
                       const float* scale_shift, hb200_f16* out, hb200_bf16* out_bf16, double* stats_acc,
                       hb200_stream_t stream);

/* Observation transforms (HB/common/obs_transformers.py ResizeShortestEdge + CenterCropper, HB/utils/common.py
 * image_resize_shortest_edge / center_crop) for NHWC batches, every key in ONE launch.  src[i]: [batch, H, W, C],
 * dst[i]: a contiguous [batch, h, w, C] region (normally one time slot of the rollout storage).  desc: HOST array of
 * n_keys (<= 8) x 11 ints: dtype (0 u8, 1 f32, 2 i32), mode, H, W, C, Hr, Wr, y0, x0, h, w.  Only the window
 * (y0, x0, h, w) of the image resampled to Hr x Wr is computed.  Modes, each bit-identical to torch on the CPU running
 * F.interpolate(img.float(), (Hr, Wr), mode).to(dtype): 0 area (adaptive average pooling), 1 nearest; 2 copy
 * (Hr = H, Wr = W: the window's bits).  Pointers must be aligned to their element size; src and dst must not overlap. */
int hb200_obs_resample(const void* const* src, void* const* dst, const int32_t* desc, int n_keys, int batch,
                       hb200_stream_t stream);

/* Not on the product path yet: mechanism probe (verified on hardware) for the TMA halo load of the halo convolutions
 * (NOTES_NEXT.md): loads the halo_h x halo_w halo of the tile whose first output pixel is (oh0, ow0) of frame b from the
 * NHWC bf16 tensor x [batch, h, w, channels] with channels/8 `cp.async.bulk.tensor.4d` box copies (out-of-bounds rows /
 * columns zero-filled = conv padding `pad`) and writes the staged slabs to out [channels/8][halo_h][halo_w][8]. */
int hb200_tma_halo_probe(const hb200_bf16* x, hb200_bf16* out, int batch, int h, int w, int channels, int b, int oh0,
                         int ow0, int halo_h, int halo_w, int pad, hb200_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* HB200_H_ */
