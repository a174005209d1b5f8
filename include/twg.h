/* twg.h -- C ABI of libtwg.so, the sm_90a (H100) kernel library behind twingan_b200.
 *
 * Drop-in boundary (SURVEY.md 8b).  The reference (jerryli27/TwinGAN) has NO FFI: every FLOP of its
 * hot path runs inside TensorFlow-1.8 library kernels reached through the Python plug-in points
 * nets/pggan.py:93-123,338-349,403-418 (network fns) and nets/pggan_utils.py:86-98 (arg-scope
 * normalizer/activation hooks).  Each entry point below cites the reference op(s) it replaces.
 *
 * Conventions
 *  - every pointer is a CUDA device pointer owned by the caller (twg_sum_scalars takes a HOST array of device
 *    pointers); the library never allocates or frees device memory at run time.  Mutable global state: the thread-local
 *    last-error string, the launch counter, one-time kernel attribute set-up, and one 32 MB device buffer per device
 *    (allocated when the library loads) for the partial sums of cross-block reductions (plus 64 KB of fp64 partial sums
 *    for the twg_swd_* evaluation entries);
 *  - results are bit-identical from run to run: reductions add their partial sums in a fixed order, never with fp32
 *    atomics;
 *  - every call takes a cudaStream_t (passed as void*), is asynchronous and graph-capturable.  Calls for one device must
 *    be ordered on one stream (the partial-sum buffer is shared); calls from several host threads are safe when they are;
 *  - returns 0 on success, <0 on invalid argument / unsupported shape / CUDA error (see twg_last_error);
 *  - activations are NHWC fp32, conv weights HWIO fp32 ([kh][kw][Cin][Cout]), like the reference
 *    (libs/batch_norm.py:409; tf.contrib.layers.conv2d);
 *  - "rows" = N*H*W pixels, "C" = channels.
 *  - sm_90a only.  There is no CPU path.
 */
#ifndef TWG_H_
#define TWG_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef void* twg_stream_t; /* cudaStream_t */

#define TWG_OK 0
#define TWG_ERR_INVALID (-1)
#define TWG_ERR_UNSUPPORTED (-2)
#define TWG_ERR_CUDA (-3)

/* norm_act flags */
#define TWG_FLAG_LRELU 1     /* util_misc.py:68-86, alpha 0.2 */
#define TWG_FLAG_PIXNORM 2   /* nets/pggan_utils.py:330-331, eps 1e-6 */

/* normaliser kinds (nets/pggan_utils.py:35-41) */
#define TWG_NORM_NONE 0
#define TWG_NORM_INSTANCE 1  /* libs/instance_norm.py:31-138, stats per (n,c) */
#define TWG_NORM_BATCH 2     /* libs/batch_norm.py:396-470, stats per c */
#define TWG_NORM_RENORM 3    /* libs/batch_norm.py:329-393 */

int twg_version(void);
const char* twg_last_error(void);
/* number of kernels launched by this library in the calling process since load (for bench gpu_launches) */
int64_t twg_launch_count(void);

/* ---- convolution: replaces tf.contrib.layers.conv2d (nets/pggan_utils.py:316-320) and its
 *      tf.gradients-generated Conv2DBackpropInput / Conv2DBackpropFilter -------------------------------
 * Stride 1.  x:[N,H,W,Cin]  w:[k,k,Cin,Cout]  y:[N,Ho,Wo,Cout], Ho = H + 2*pad - k + 1.
 * SAME for k=3 is pad=1, k=1 pad=0; VALID is pad=0.
 * Two kernel families: exact fp32 on fp32 operands (any shape), and wgmma tensor cores on split-bf16 planes (3 MMAs per
 * product, ~fp32 accuracy) for the shapes twg_conv_path reports as TWG_CONV_TC.                                       */
#define TWG_CONV_SIMT 0  /* exact fp32, CUDA cores */
#define TWG_CONV_PW 1    /* exact fp32, the thin 1x1 layers (fromRGB / toRGB): twg_conv_fwd/dgrad/wgrad use it in any case */
#define TWG_CONV_TC 2    /* tensor cores: 3x3 SAME / 1x1 with 16, 32, 64 or a multiple of 128 channels */
/* which family covers this stride-1 conv shape (one of TWG_CONV_*) */
int twg_conv_path(int N, int H, int W, int Cin, int Cout, int k, int pad);
/* exact fp32: y = conv(x, w) */
int twg_conv_fwd(const float* x, const float* w, float* y, int N, int H, int W, int Cin, int Cout, int k, int pad,
                 twg_stream_t stream);
/* gx:[N,H,W,Cin] = d/dx of sum(gy*y) */
int twg_conv_dgrad(const float* gy, const float* w, float* gx, int N, int H, int W, int Cin, int Cout, int k, int pad,
                   twg_stream_t stream);
/* gw:[k,k,Cin,Cout] (+)= d/dw; accumulate!=0 adds into gw */
int twg_conv_wgrad(const float* x, const float* gy, float* gw, int N, int H, int W, int Cin, int Cout, int k, int pad,
                   int accumulate, twg_stream_t stream);

/* ---- tensor-core convolution on pre-split operands ("split-bf16 planes": hi plane then lo plane, bf16, same
 *      NHWC element order as the fp32 tensor; x = hi + lo).  Lets the caller split an activation once and reuse
 *      it for forward + wgrad, a gradient once for dgrad + wgrad, and a weight once per optimiser step.        */
/* planes: 2*n bf16 */
int twg_split_act(const float* x, void* planes, int64_t n, twg_stream_t stream);
/* planes: 2*k*k*Cin*Cout bf16; dgrad=0: [tap][Cout][Cin] (forward operand), dgrad=1: [flip(tap)][Cin][Cout] */
int twg_split_weights(const float* w, void* planes, int k, int Cin, int Cout, int dgrad, twg_stream_t stream);
/* Fused epilogue of the forward conv (sign mask, statistics, evaluation-mode affine): the number of statistics records
 * per image it writes for this shape, 0 when the shape has no fused epilogue (the small-channel high-resolution layers
 * have one: a pixel's Cout channels sit in one CTA). */
int twg_conv_epilogue_slots(int N, int H, int W, int Cin, int Cout, int k, int pad);
/* y = lrelu?(conv(x, w) + bias): bias (nullable) and act = 1 (leaky-ReLU, needs bias) give the discriminator layer in one
 * kernel (nets/pggan_utils.py:116-127), so the pre-activation never touches HBM.  Optional outputs (each nullable):
 *  - z_planes: y also as split planes, for the next conv;
 *  - act_mask (act = 1): the SIGN MASK of y, act_mask[i] one byte per 4 consecutive channels, bit j = y[4i+j] > 0, which
 *    is all the first-order backward of tf.maximum(0.2x, x) needs (util_misc.py:86) -- the backward then reads 0.25 B
 *    instead of 4 B per element (twg_lrelu_bwd_colsum);
 *  - stats (no bias, no z_planes): the statistics tf.nn.moments would take over y (libs/instance_norm.py:131-135 after
 *    nets/pggan.py:78-81), from the conv epilogue: stats[n][slot][c] = {count, pivot, sum (y - pivot), sum (y - pivot)^2}
 *    (float4) over the pixels one epilogue warp drained, slot < twg_conv_epilogue_slots(...) per image -- no second pass
 *    over y, no atomics.  N * slots * Cout float4, fully written by the call.
 * act_mask and stats need twg_conv_epilogue_slots(...) > 0. */
int twg_conv_fwd_planes(const void* x_planes, const void* w_planes, const float* bias, int act, float* y, void* z_planes,
                        void* act_mask, float* stats, int N, int H, int W, int Cin, int Cout, int k, int pad,
                        twg_stream_t stream);
/* Inference-mode generator / encoder layer in ONE kernel (nets/pggan.py:78-81 with is_training=False:
 * libs/batch_norm.py:266-278 turns the normaliser into the per-channel affine a = gamma / sqrt(moving_var + eps),
 * b = beta - moving_mean * a, twg_norm_eval_affine):  z = pixel_norm?(lrelu?(a[c] * conv(x, w) + b[c])), flags =
 * TWG_FLAG_LRELU | TWG_FLAG_PIXNORM, written as fp32 z and / or split planes (either may be NULL, not both).  Covered
 * shapes: twg_conv_epilogue_slots(...) > 0. */
int twg_conv_affine_act_fwd_planes(const void* x_planes, const void* w_planes, const float* a, const float* b, int flags,
                                   float* z, void* z_planes, int N, int H, int W, int Cin, int Cout, int k, int pad,
                                   twg_stream_t stream);
int twg_conv_dgrad_planes(const void* gy_planes, const void* w_planes, float* gx, int N, int H, int W, int Cin,
                          int Cout, int k, int pad, twg_stream_t stream);
int twg_conv_wgrad_planes(const void* x_planes, const void* gy_planes, float* gw, int N, int H, int W, int Cin,
                          int Cout, int k, int pad, int accumulate, twg_stream_t stream);

/* host utility (no GPU): CRC-32C (Castagnoli) of `n` bytes continuing from `crc` (0 to start) -- the checksum of
 * TensorFlow's checkpoint format (twingan_b200/tf_checkpoint.py) */
int64_t twg_crc32c(const void* data, int64_t n, int64_t crc);

/* ---- normaliser + activation + pixel-norm: replaces tf.nn.moments/tf.nn.batch_normalization
 *      (libs/batch_norm.py:430,470; libs/instance_norm.py:131-135), tf.maximum(0.2x,x) (util_misc.py:86)
 *      and _pixel_norm (nets/pggan_utils.py:330-331) and their gradients --------------------------------- */
/* Shifted sums (tf.nn.moments is two-pass; raw single-pass sums cancel once |mean| >> std):
 * sums[n][c] = {sum_hw (y - p), sum_hw (y - p)^2}, p = y[first sample of n's pivot group][pixel 0][c]
 * (pivot_group = 1 for instance norm, = the statistics group size for the batch kinds).  2*N*C floats, fully written
 * by the call. */
int twg_moments(const float* y, float* sums, int N, int HW, int C, int pivot_group, twg_stream_t stream);
/* Turn the sums into the per-(n,c) affine z = a*y + b of the chosen normaliser (training mode) plus
 * mean/rstd for the backward.  The batch is N/group_size groups of group_size samples -- one group per original
 * network pass when passes that share conv weights run as one batch (twingan.py:196-284); bit g of dom_mask picks the
 * group's domain: gamma0/beta0/renorm0 ('_s' say) or gamma1/beta1/renorm1 (the reference's per-domain
 * conditional_layer_var_scope_postfix variables, nets/pggan_utils.py:141-166).  Batch kinds take their statistics over
 * the group.  `y` is read for the pivots only.  For RENORM `renormX` points at {renorm_mean[C], renorm_stddev[C],
 * renorm_mean_weight, renorm_stddev_weight} (2C+2 floats, pre-update values), r,d are clipped to `clip` =
 * {rmin, rmax, dmax} in DEVICE memory (twg_step_schedule; null: 1,1,0); rd_out:[groups][2][C] receives r,d.
 * batch_stats:[groups][2][C] (optional) receives the batch mean and (variance | stddev for RENORM).          */
int twg_norm_finalize(const float* sums, const float* y, const float* gamma0, const float* beta0, const float* gamma1,
                      const float* beta1, int dom_mask, int group_size, const float* renorm0, const float* renorm1,
                      int kind, float eps, const float* clip, float* a, float* b, float* mean, float* rstd, float* rd_out,
                      float* batch_stats, int N, int HW, int C, twg_stream_t stream);
/* Instance-norm variant of twg_norm_finalize that merges the epilogue statistics records of twg_conv_fwd_planes (records
 * re-based to one pivot drawn from the data: the accuracy of tf.nn.moments' two-pass form, libs/instance_norm.py:131-135) */
int twg_norm_finalize_partials(const float* stats, int slots, const float* gamma0, const float* beta0, const float* gamma1,
                               const float* beta1, int dom_mask, int group_size, float eps, float* a, float* b, float* mean,
                               float* rstd, int N, int C, twg_stream_t stream);
/* Evaluation-mode affine from moving statistics (libs/batch_norm.py:266-278): a,b:[N][C] broadcast */
int twg_norm_eval_affine(const float* gamma, const float* beta, const float* moving_mean, const float* moving_var,
                         float eps, float* a, float* b, int N, int C, twg_stream_t stream);
/* z = pixnorm?( lrelu?( a[n,c]*y + b[n,c] ) ) as fp32 z and / or split-bf16 planes for the next tensor-core conv
 * (either may be NULL, not both) */
int twg_norm_act_fwd(const float* y, const float* a, const float* b, float* z, void* planes, int N, int HW, int C,
                     int flags, twg_stream_t stream);
/* first backward pass: gu = d/du of the activation/pixel-norm part, red[n][c] = {sum gu, sum gu*yhat}.  For a layer
 * whose output also feeds a 2x2 average pool (nets/pggan.py:436,468), `gpool` [N,H/2,W/2,C] is the gradient w.r.t. the
 * pooled tensor; its contribution 0.25*gpool[h/2][w/2] is added on the fly (the full-resolution pool gradient and
 * autograd's accumulation with a UNet-skip gradient `gz` are never materialised).  gz or gpool may be NULL, not both.
 * W = row length of the full-resolution tensor (read only with gpool). */
int twg_norm_act_bwd_reduce(const float* y, const float* a, const float* b, const float* mean, const float* rstd,
                            const float* gz, const float* gpool, int W, float* gu, float* red, int N, int HW, int C,
                            int flags, twg_stream_t stream);
/* second pass: gy = a*(gu - S1/M - yhat*S2/M) with the reduction domain of `kind` (fp32 and/or split-bf16 planes, the
 * operand dgrad and wgrad consume); ggammaX[C], gbetaX[C] = parameter gradients of domain X over its groups (groups /
 * dom_mask as in twg_norm_finalize; += when accumulate, e.g. straight into the flat gradient buffer); rd:[groups][2][C]
 * (r,d; null => r=1,d=0) */
int twg_norm_act_bwd_apply(const float* y, const float* a, const float* mean, const float* rstd, const float* gu,
                           const float* red, const float* rd, float* gy, void* gy_planes, float* ggamma0, float* gbeta0,
                           float* ggamma1, float* gbeta1, int accumulate, int dom_mask, int group_size, int kind, int N,
                           int HW, int C, twg_stream_t stream);
/* EMA pushes (libs/batch_norm.py:295-319, 359-393); decay 0.99 for batch_renorm (nets/pggan_utils.py:165), 0.999 for
 * plain batch_norm (libs/batch_norm.py:44 default): state layout per (layer,domain):
 * moving_mean[C], moving_var[C], renorm_mean[C], renorm_stddev[C], renorm_mean_weight, renorm_stddev_weight */
int twg_norm_update_stats(float* state, const float* batch_stats, int kind, float decay, float eps, int C,
                          twg_stream_t stream);

/* ---- discriminator-style bias + leaky-ReLU (nets/pggan_utils.py:116-127) -------------------------- */
/* z = lrelu?(y + bias); z additionally as split-bf16 planes (for the tensor-core conv that consumes it) and / or as its
 * sign mask (one byte per 4 channels, bit j = z[4i+j] > 0, for twg_lrelu_bwd_colsum); either may be NULL, and needs
 * C % 4 == 0 */
int twg_bias_lrelu_fwd(const float* y, const float* bias, float* z, void* planes, void* mask, int64_t rows, int C,
                       int lrelu_on, twg_stream_t stream);
/* out = g * (ref>0 ? 1 : 0.2)   (gradient of tf.maximum(0.2x,x); ref may be the activation output) */
int twg_lrelu_bwd(const float* g, const float* ref, float* out, int64_t n, twg_stream_t stream);
/* fused: out = lrelu_on ? g*slope(ref) : g (not written when lrelu_on=0) and colsum[c] (+)= sum_rows out[row][c].
 * `out` fp32 and / or (`planes`) split planes; the activation's sign from `mask` (twg_conv_fwd_planes, twg_bias_lrelu_fwd)
 * instead of `ref` when mask != NULL; `g` optionally given as the gradient w.r.t. avg_pool2(z) ([N,poolH/2,poolW/2,C];
 * poolW = 0: plain form). */
int twg_lrelu_bwd_colsum(const float* g, const float* ref, const void* mask, float* out, void* planes, float* colsum,
                         int64_t rows, int C, int lrelu_on, int poolH, int poolW, int accumulate, twg_stream_t stream);
/* out[c] (+)= sum_rows g[row][c] */
int twg_colsum(const float* g, float* out, int64_t rows, int C, int accumulate, twg_stream_t stream);

/* ---- resampling (nets/pggan_utils.py:349-350; tf.nn.avg_pool nets/pggan.py:274,306,436,468) -------- */
/* out[N,H/2,W/2,C] = scale * sum of the 2x2 block (scale .25 = avg-pool; 1 = gradient of nearest x2); `out` fp32 and / or
 * split planes */
int twg_pool2(const float* x, float* out, void* planes, int N, int H, int W, int C, float scale, twg_stream_t stream);
/* out[N,2H,2W,C] = scale * x[i/2,j/2] (scale 1 = nearest x2; .25 = gradient of avg-pool) */
int twg_upsample2(const float* x, float* out, int N, int H, int W, int C, float scale, twg_stream_t stream);
/* UNet join (nets/pggan_utils.py:281-298 + :349): out[N,2H,2W,Ca+Cb] = concat(nearest2(a[N,H,W,Ca]), b[n % Nb]) with
 * b:[Nb,2H,2W,Cb] -- Nb < N when several generator passes that share one encoder pass run as one batch.  `out` fp32
 * and/or split planes. */
int twg_upsample_concat(const float* a, const float* b, float* out, void* planes, int N, int H, int W, int Ca, int Cb,
                        int Nb, twg_stream_t stream);
/* its gradient: ga[N,H,W,Ca] = sum2x2(gout[..., :Ca]); gb[m] = sum_j gout[m + j*Nb][..., Ca:] */
int twg_upsample_concat_bwd(const float* gout, float* ga, float* gb, int N, int H, int W, int Ca, int Cb, int Nb,
                            twg_stream_t stream);
/* out = alpha*x + beta*y (y may be null); fade-in lerp (nets/pggan.py:205,314,475) */
int twg_axpby(const float* x, const float* y, float* out, float alpha, float beta, int64_t n, twg_stream_t stream);
/* out = x * (*dev_scalar) * alpha   (scale by a device-resident scalar, e.g. an upstream loss gradient) */
int twg_scale_by_dev(const float* x, const float* dev_scalar, float* out, float alpha, int64_t n, twg_stream_t stream);
/* channel concat / split for row-major [rows][C] tensors (minibatch-stddev plumbing) */
int twg_copy_cols(const float* src, float* dst, int64_t rows, int Csrc, int src_off, int Cdst, int dst_off, int ncols,
                  twg_stream_t stream);

/* ---- minibatch stddev (nets/pggan_utils.py:353-366) -------------------------------------------------
 * x:[N][F] (F=4*4*C).  s = mean_f sqrt(var_n(x)+1e-8).  out:[N][4*4][Ct] = [x | s | zeros], Ct >= C+1: Ct = C+1 is
 * the reference tensor; a larger Ct pads the following conv's input channels to a tensor-core channel count (its
 * weights are padded with zero rows the same way, see twg_copy_cols).
 * `groups`: the N samples are `groups` independent minibatches of N/groups (one per original discriminator pass). */
int twg_mbstd_fwd(const float* x, float* out, float* s_out, int N, int P, int C, int Ct, int groups,
                  twg_stream_t stream);
/* gx[N][P][C] = gout[..., :C] + G * ds/dx with G = sum of gout[..., C]; gout:[N][P][Ct] */
int twg_mbstd_bwd(const float* x, const float* gout, float* gx, int N, int P, int C, int Ct, int groups,
                  twg_stream_t stream);
/* double backward of the s-branch: given ggx (cotangent of gx) returns
 * dG_out[N][P][Ct]: cotangent for gout (identity on the first C channels, sum_nf ggx*c in channel C, 0 above) and
 * dx[N][P][C] = G * sum ggx * dc/dx                                                                  */
int twg_mbstd_bwd2(const float* x, const float* gout, const float* ggx, float* dgout, float* dx, int N, int P, int C,
                   int Ct, int groups, twg_stream_t stream);

/* ---- losses (image_generation.py:341,392,397; twingan.py:464,502; image_generation.py:441-476) ------ */
/* loss_out[0] (+)= weight*mean(sigmoid_ce(label, logits)); grad[i] = weight/n * (sigmoid(x)-label) */
int twg_sigmoid_ce(const float* logits, float label, float weight, float* loss_out, float* grad, int64_t n,
                   int accumulate, twg_stream_t stream);
/* WGAN / hinge terms (image_generation.py:330-389, optional --loss_architecture values): loss_out[0] = weight *
 * mean_i f(sign*x_i + margin), f = identity (kind 0), relu (1), square (2); _bwd: gx[i] = gl[0]*weight/n*sign*f'(.) */
int twg_logit_mean(const float* x, float* loss_out, int64_t n, float sign, float margin, int kind, float weight,
                   twg_stream_t stream);
int twg_logit_mean_bwd(const float* x, const float* gl, float* gx, int64_t n, float sign, float margin, int kind,
                       float weight, twg_stream_t stream);
/* loss_out[0] (+)= weight*mean|a-b|; grad_a = weight/n*sign(a-b) */
int twg_l1(const float* a, const float* b, float weight, float* loss_out, float* grad_a, int64_t n, int accumulate,
           twg_stream_t stream);
/* DRAGAN perturbation: xhat = x + alpha[n]*(0.5*var(x)*noise), var over ALL elements (image_generation.py:445) */
int twg_dragan_xhat(const float* x, const float* alpha, const float* noise, float* xhat, float* scratch2, int N,
                    int64_t per_sample, twg_stream_t stream);
/* penalty: loss (+)= lambda*mean_n (||g_n||-1)^2 ; coef[n] = lambda*2*(s_n-1)/(N*s_n)  (so dL/dg = coef[n]*g) */
int twg_grad_penalty(const float* g, float lambda, float* loss_out, float* coef, int N, int64_t per_sample,
                     int accumulate, twg_stream_t stream);
/* out[n][i] = x[n][i] * coef[n] * (*dev_scalar) */
int twg_scale_rows(const float* x, const float* coef, const float* dev_scalar, float* out, int N, int64_t per_sample,
                   twg_stream_t stream);

/* ---- TwinGAN wiring for batched passes (twingan.py:196-284, 370-381, 451-505).  The four generator passes run as one
 *      batch gout = [s_cycle | t_cycle | t_prime | s_prime] (B samples of per_sample floats each), x = [sources | targets].
 * One pass over gout writes the discriminator batches ds = [sources | s_cycle | s_prime], dt = [targets | t_cycle |
 * t_prime], the second encoder batch e2 = [t_prime | s_prime], loss2 = {l_cyc_s, l_cyc_t} = weight*mean|x - cycle|
 * (tf.losses.absolute_difference, twingan.py:464) and their gradient seeds sign_grad [2B] (weight/n * sign).   */
int twg_fanout_fwd(const float* gout, const float* x, float* ds, float* dt, float* e2, float* sign_grad, float* loss2,
                   float weight, int B, int64_t per_sample, twg_stream_t stream);
/* ggout = sum of the gradients coming back through ds, dt, e2 (each nullable) and gl_s/gl_t * sign_grad (device scalars,
 * nullable) */
int twg_fanout_bwd(const float* gds, const float* gdt, const float* ge2, const float* sign_grad, const float* gl_s,
                   const float* gl_t, float* ggout, int B, int64_t per_sample, twg_stream_t stream);
/* loss[g] = weight*mean|a_g - b_g| over `groups` equal blocks (l_content_{s,t}, twingan.py:485-505); grad_a = w/n*sign */
int twg_l1_groups(const float* a, const float* b, float weight, float* loss, float* grad_a, int groups, int64_t per_group,
                  twg_stream_t stream);
/* out block g (g = 0,1) = grad block g * sign * (*gl_g)   (gl_g device scalars; null => zeros) */
int twg_scale_groups2(const float* grad, const float* gl0, const float* gl1, float sign, float* out, int64_t per_group,
                      twg_stream_t stream);
/* GAN losses of one discriminator batch logits = [real | cycle | prime] (B each), image_generation.py:341-344, 392-401
 * via tf.losses.sigmoid_cross_entropy: loss6 = {generator_fool_cycle, generator_fool_prime, discriminator_fake_cycle,
 * discriminator_real (cycle term), discriminator_fake_prime, discriminator_real (prime term)}; sig = sigmoid(logits). */
int twg_gan_losses(const float* logits, float weight, float* loss6, float* sig, int B, twg_stream_t stream);
/* grad = d(sum_k g_k*loss_k)/d logits; g_k device scalars (nullable = 0) */
int twg_gan_losses_bwd(const float* sig, float weight, const float* g0, const float* g1, const float* g2, const float* g3,
                       const float* g4, const float* g5, float* grad, int B, twg_stream_t stream);
/* out[0] = scale * sum_i *ptrs[i]: `device_ptrs_host_array` is a HOST array of n <= 16 device pointers to fp32 scalars
 * (total loss = sum of the named losses / num_clones, deployment/model_deploy.py:265-267) */
int twg_sum_scalars(const void* device_ptrs_host_array, int n, float scale, float* out, twg_stream_t stream);

/* ---- step counters on the device: counters = int32 {adam_t, global_step}.  twg_step_schedule writes the bias-corrected
 *      Adam step sizes of the step's two applies, lr_out2[i] = lr*sqrt(1-b2^(t+1+i))/(1-b1^(t+1+i)) (model/
 *      model_inheritor.py:537-542; one optimizer => shared beta powers), and the batch-renorm clipping
 *      {rmin, rmax, dmax} of global_step (nets/pggan_utils.py:44-47), so a captured CUDA graph of the step stays correct
 *      while time advances; twg_step_advance adds to the counters. */
int twg_step_schedule(const void* counters, float lr, float beta1, float beta2, float* lr_out2, float* clip_out3,
                      twg_stream_t stream);
int twg_step_advance(void* counters, int d_adam_t, int d_global_step, twg_stream_t stream);
/* every conv weight of the model -> split-bf16 planes in ONE launch (after the Adam apply): table = rows of
 * {int64 src offset in `flat` (floats), int64 dst offset in `planes` (bf16 elements), int32 taps, Cin, Cout, dgrad};
 * the hi plane of a row sits at dst, its lo plane at dst + taps*Cin*Cout; layouts as twg_split_weights */
int twg_split_weights_table(const float* flat, void* planes, const void* table, int rows, int64_t max_elems,
                            twg_stream_t stream);

/* ---- optimizer: tf.train.AdamOptimizer (model/model_inheritor.py:537-542), one launch over a flat buffer */
int twg_adam(float* p, const float* g, float* m, float* v, int64_t n, float lr_t, float beta1, float beta2, float eps,
             twg_stream_t stream);
/* same, with the bias-corrected step size lr_t read from device memory (so a captured CUDA graph of the step
 * can be replayed while the Adam time step advances) */
int twg_adam_dev_lr(float* p, const float* g, float* m, float* v, int64_t n, const float* lr_t_dev, float beta1,
                    float beta2, float eps, twg_stream_t stream);

/* ---- sliced Wasserstein distance, an evaluation outside the step: --calc_swd (image_generation.py:147-156, 868-927),
 *      whose library the reference does not ship (:926-927).  The metric is PGGAN's (Karras et al., ICLR 2018, section 5
 *      and appendix D; metrics/sliced_wasserstein.py of its release): Laplacian pyramid, 7x7 neighbourhood descriptors,
 *      per-channel normalisation (finalize_descriptors), sliced W1 over random unit directions (sliced_wasserstein).
 *      Images are NHWC fp32 RGB.  Finite inputs are a precondition: NaN or infinity gives undefined results. */
/* Laplacian pyramid (pyr_down / pyr_up with g = [1,4,6,4,1]^T[1,4,6,4,1]/256, mirror borders as
 * scipy.ndimage.convolve(mode='mirror'); the last level stays Gaussian) of x:[N,R,R,3] into pyr: level l = 0..levels-1 is
 * [N, R>>l, R>>l, 3] at float offset N*3*sum_{k<l} (R>>k)^2.  R a power of two, R >> (levels-1) >= 4. */
int twg_swd_pyramid(const float* x, float* pyr, int N, int R, int levels, twg_stream_t stream);
/* desc[(n*nhoods + k)][c*s*s + dy*s + dx] = level[n][cy - s/2 + dy][cx - s/2 + dx][c] (PGGAN's NCHW component order),
 * s = nhood_size (odd), centres: int32 {cy, cx} per [n][k], clamped into [s/2, Rl - 1 - s/2] */
int twg_swd_gather(const float* level, const void* centres, float* desc, int N, int Rl, int nhoods, int nhood_size,
                   twg_stream_t stream);
/* stats = {mean[3], rstd[3]} of desc:[rows][3*s*s] per channel over all rows and s*s positions, population std (ddof 0),
 * summed in fp64; rstd = 1/std, 0 for a channel whose std is 0 */
int twg_swd_stats(const float* desc, float* stats, int64_t rows, int nhood_size, twg_stream_t stream);
/* proj[j][i] (column-major, [ndirs][rows]) = sum_k (desc[i][k] - mean[c(k)]) * rstd[c(k)] * dirs[k][j], exact fp32 FMA;
 * dirs:[3*s*s][ndirs], ndirs a multiple of 128 */
int twg_swd_project(const float* desc, const float* stats, const float* dirs, float* proj, int64_t rows, int nhood_size,
                    int ndirs, twg_stream_t stream);
/* bytes of device workspace twg_swd_sort needs (<0: invalid sizes) */
int64_t twg_swd_sort_workspace(int segments, int64_t seg_len);
/* sorts each of `segments` consecutive columns of seg_len (< 2^31) fp32 keys ascending, in place (stable LSD radix sort
 * over order-preserving uint32 keys; -0 sorts before +0) */
int twg_swd_sort(float* keys, void* workspace, int segments, int64_t seg_len, twg_stream_t stream);
/* out_f64[0] = sum_i |a[i] - b[i]| accumulated in fp64 (one double in device memory) */
int twg_swd_sorted_l1(const float* a, const float* b, void* out_f64, int64_t n, twg_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* TWG_H_ */
