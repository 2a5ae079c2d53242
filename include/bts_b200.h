/* bts_b200 -- C ABI of the GPU-native BTS hot path (libbts_b200.so, built for the H100: sm_90a).
 *
 * This is the native boundary underneath the Python module surface `bts` (BtsModel / encoder / bts /
 * local_planar_guidance / reduction_1x1 / silog_loss, reference pytorch/bts.py).  The reference's only
 * native interface is the TensorFlow custom op (tensorflow/custom_layer/local_planar_guidance.h:22-49:
 * LocalPlanarGuidanceKernel / LocalPlanarGuidanceGradKernel functors taking raw float pointers + sizes);
 * bts_lpg_fwd / bts_lpg_bwd replace exactly those two functors (layout=BTS_LAYOUT_NHWC, tf_compat=1
 * reproduces the op bit-for-formula); every other entry point replaces an ATen/cuDNN call sequence of
 * pytorch/bts.py cited per function.
 *
 * Conventions (all entry points):
 *   - plain pointers are DEVICE pointers (fp32 unless noted); no torch / TF types.
 *   - asynchronous on the caller-supplied CUDA stream (void* == cudaStream_t); never allocates,
 *     never synchronises (the reference op calls d.synchronize() after each launch, .cu:91,170 -- we do not).
 *   - returns 0 on success, a negative BTS_E* on bad arguments, a positive cudaError_t on launch failure.
 *   - `*_h` variants take HOST pointers, do the H2D/D2H copies themselves and synchronise; they are the
 *     reference-facing plugin form used for end-to-end (e2e) measurements and by non-torch callers.
 */
#ifndef BTS_B200_H_
#define BTS_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define BTS_LAYOUT_NCHW 0 /* plane (B,4,h,w)  -- pytorch/bts.py:135-138 */
#define BTS_LAYOUT_NHWC 1 /* plane (B,h,w,4)  -- custom_layer/local_planar_guidance.cc:102-107 */

#define BTS_EINVAL (-1)   /* bad argument (null pointer, non-positive size, unsupported upratio) */
#define BTS_EALIGN (-2)   /* pointer not 16-byte aligned where the kernel needs it */

/* library / build identification: returns the target architecture (90 for sm_90a); writes a short version string */
int bts_version(char *buf, int buflen);

/* ---- Local planar guidance --------------------------------------------------------------------
 * Forward  (pytorch/bts.py:132-146; custom_layer/local_planar_guidance.cu:33-72, .cc:74-115):
 *     depth[b,y,x] = n4 / ((n1*u(x) + n2*v(y)) + n3),  plane of patch (y/r, x/r),
 *     u(x) = ((x mod r) - (r-1)/2)/r  (bit-exact dyadic grid), v(y) likewise.
 * `focal` is unused by the reference in both implementations (SURVEY Q1) and is not a parameter.
 * upratio r must be 1 or even. */
int bts_lpg_fwd(const float *plane, float *depth, int B, int h, int w, int r, int layout, void *stream);

/* Backward (autograd of pytorch/bts.py:146; custom_layer/local_planar_guidance.cu:95-150, .cc:241-298):
 *     dplane[b,:,i,j] = sum over the r x r tile of (-dY*n4*u/den^2, -dY*n4*v/den^2, -dY*n4/den^2, dY/den)
 * tf_compat=1 drops n4 from the first three (the reference TF kernel's formula, SURVEY Q5). */
int bts_lpg_bwd(const float *dy, const float *plane, float *dplane, int B, int h, int w, int r,
                int layout, int tf_compat, void *stream);

/* Host-pointer plugin form of the TF op pair (input (B,h,w,4) NHWC, output (B,h*r,w*r)); copies in/out
 * and synchronises.  Mirrors LocalPlanarGuidanceOp::Compute / LocalPlanarGuidanceGradOp::Compute
 * (custom_layer/local_planar_guidance.cc:190-229, 364-416). */
int bts_lpg_fwd_h(const float *plane_host, float *depth_host, int B, int h, int w, int r, int layout);
int bts_lpg_bwd_h(const float *dy_host, const float *plane_host, float *dplane_host, int B, int h, int w,
                  int r, int layout, int tf_compat);

/* ---- silog loss (pytorch/bts.py:41-48) ---------------------------------------------------------
 * mask: uint8/bool, n elements.  ws: >= 4 doubles of device workspace, zeroed by the call.
 * fwd:  d_i = ln est_i - ln gt_i over mask; loss = 10*sqrt(mean(d^2) - lambda*mean(d)^2)  -> loss[0]
 *       ws keeps (sum d, sum d^2, N) for the backward.
 * bwd:  dest_i = gout[0] * mask_i * (10/sqrt(S)) * (d_i - lambda*m1) / (N*est_i)   (SURVEY Appendix B) */
int bts_silog_fwd(const float *est, const float *gt, const uint8_t *mask, long long n, float lambda,
                  double *ws, float *loss, void *stream);
int bts_silog_bwd(const float *est, const float *gt, const uint8_t *mask, long long n, float lambda,
                  const double *ws, const float *gout, float *dest, void *stream);

/* ---- plane-coefficient head tail (pytorch/bts.py:112-120 + 223-229 per scale) -------------------
 * c3: (B,3,h,w) output of reduc.plane_params.  Computes theta=sig(c0)*pi/3, phi=sig(c1)*2pi,
 * dist=sig(c2)*max_depth, n=(sin th cos ph, sin th sin ph, cos th), n^=n/max(|n|,1e-12), plane=(n^,dist),
 * then LPG(r) -> scaled=(depth/max_depth) (B,H,W) and ds (optional, nearest down-sample by ds_stride).
 * plane_out (B,4,h,w) optional (saved for backward / inspection). */
int bts_plane_head_fwd(const float *c3, float *plane_out, float *scaled, float *ds, float max_depth,
                       int ds_stride, int B, int h, int w, int r, void *stream);
/* backward of the above: inputs d_scaled (B,H,W), d_ds (optional), c3; output dc3 (B,3,h,w) */
int bts_plane_head_bwd(const float *d_scaled, const float *d_ds, const float *c3, float *dc3,
                       float max_depth, int ds_stride, int B, int h, int w, int r, void *stream);

/* ---- wgmma implicit-GEMM convolution (pytorch/bts.py:51-80,153-194; torchvision dense/bottleneck layers) ----
 * NHWC activations, fp32 in / fp32 out, parity-grade 3xTF32 on the Hopper tensor cores (precision=0) or
 * single-pass TF32 (precision=1, opt-in, not parity).  precision=1 launches the dedicated single-pass kernels
 * (conv_tf32_kernel, wgrad_tf32_kernel, wgrad2_tf32_kernel): one product per k8 step, and shared-memory stages that hold
 * only the hi half of the weight / dY operand.  The packed weights are the same for both values.
 *   out[p,co] = act( sum_{tap,ci} pre(x[p (+) tap, ci]) * w[co,ci,tap] )
 *   pre : x*pre_scale[ci]+pre_shift[ci] (folded BatchNorm; both NULL to skip), then ReLU if pre_relu;
 *         zero padding is applied after pre.
 *   act : 0 none, 1 ELU, 2 sigmoid.
 * x: source (B,Hs,Ws,*) with x_pixel_stride floats between pixels (a channel slice of a wider slab is fine);
 * out likewise with out_pixel_stride.  Weights must first be packed (split hi/lo, K-major, 128B-swizzled tiles):
 *   bts_conv_packed_floats(n_rows, k_channels, KH, KW) -> number of floats of the packed buffer
 *   bts_conv_pack_weights(w, strides of (co,ci,kh,kw) in floats, ..., transpose_flip, wpack)
 *       transpose_flip=0: forward operator (rows = Cout);  1: dgrad operator (rows = Cin, taps flipped) so that
 *       dX = bts_conv_fwd(dY, wpack_T, Cin<->Cout swapped, pad' = dil*(K-1) - pad).
 *   bts_conv_n_tile(Cout) -> the N tile the engine uses for that many output channels. */
int bts_conv_n_tile(int Cout);
long long bts_conv_packed_floats(int n_rows, int k_channels, int KH, int KW);
int bts_conv_pack_weights(const float *w, long long s_co, long long s_ci, long long s_kh, long long s_kw,
                          int Cout, int Cin, int KH, int KW, int transpose_flip, float *wpack, void *stream);
/* bts_conv_fwd: the forward / dgrad launch above, with
 *   source_mode 0 plain | 1 nearest x2 up-sample of the source folded in | 2 ZERO-STUFFED x2 source with an explicit
 *       out_h x out_w output (out_h / out_w are ignored otherwise): with the transposed, tap-flipped packed operator,
 *       stride = 1 and pad' = dil*(K-1) - pad this is the input gradient of a STRIDE-2 convolution whose input was
 *       out_h x out_w (x = dY of that layer; replaces cuDNN's strided dgrad behind the ResNet / ResNeXt encoders, reference
 *       pytorch/bts.py:282-296 via torchvision.models.resnet);
 *   kwin > 0 block-diagonal ("grouped") operator packed by bts_conv_pack_weights_grouped: output channels
 *       [nt*kwin, (nt+1)*kwin) read input channels [nt*kwin, (nt+1)*kwin) only; Cin == Cout == the layer width; 0 = dense;
 *   stat_sum / stat_sumsq (both or neither): the BatchNorm batch statistics of the output, stat_sum[co] += sum_p out[p,co],
 *       stat_sumsq[co] += sum_p out[p,co]^2 (fp64, accumulated with atomics -> zero them first; any Cout, act must be 0).
 *       Replaces a separate bts_bn_stats pass over the tensor just written (torchvision _DenseLayer: conv1 -> norm2,
 *       conv2 -> every later norm1);
 *   x_bn / bn_st (both or neither; needs the statistics pointers and act 0): BatchNorm(+ReLU)-backward epilogue of the
 *       layer in front of a dgrad.  The tile written is g = dL/d[relu](bn(x_bn)); the statistics pointers receive
 *       S1[c] += sum_p g*mask and S2[c] += sum_p g*mask*xhat instead (zero them first), mask = [bn(x_bn)>0] when relu
 *       else 1, xhat = (x_bn-mean)*invstd.  x_bn: the BatchNorm INPUT at the output's pixels and channels, pixel stride
 *       x_bn_stride; bn_st = [4][Cout] scale|shift|mean|invstd (the bts_bn_finalize layout).  Replaces the
 *       bts_bn_bwd_reduce pass over (x, g); follow with bts_bn_bwd_coef + bts_bn_bwd_apply;
 *   workspace != NULL: split-K, for launches whose tiles (128-pixel x n-tile output blocks) leave SMs idle (batch-1
 *       inference): each tile's K range is cut into `splits` ranges run by separate CTAs, which write raw fp32 partial
 *       tile sums into `workspace` ([splits][M][Cout rounded up to 4], 16-byte aligned); a second kernel adds them in a
 *       fixed order (the result is reproducible run to run) and applies `act` into out.  The split kernel has no
 *       statistics or BatchNorm-backward epilogue: both are refused with a workspace.  workspace == NULL does not split;
 *       splits must then be 1.
 * Refused argument combinations return BTS_EINVAL (a misaligned workspace BTS_EALIGN) before any CUDA runtime call.
 *   bts_conv_fwd_splitk_plan(B, Hout, Wout, kwin, Cin, KH, KW, Cout, &splits, &workspace_floats): with *splits = 0 on
 *   entry, the engine's choice (1 = do not split: the launch already fills more than half the SMs, or K is too short);
 *   with *splits = n > 0, n reduced so that no split is empty.  *workspace_floats: the workspace that count needs. */
int bts_conv_fwd(const float *x, long long x_pixel_stride, int B, int Hs, int Ws, int source_mode, int out_h, int out_w,
                 int kwin, int Cin, int KH, int KW, int stride, int pad, int dil, const float *wpack, int Cout,
                 const float *pre_scale, const float *pre_shift, int pre_relu, float *out, long long out_pixel_stride,
                 int act, int precision, double *stat_sum, double *stat_sumsq, const float *x_bn, long long x_bn_stride,
                 const float *bn_st, int relu, int splits, float *workspace, void *stream);
int bts_conv_fwd_splitk_plan(int B, int Hout, int Wout, int kwin, int Cin, int KH, int KW, int Cout, int *splits,
                             long long *workspace_floats);
/* Tuning / bring-up switches of the narrow-output wgrad (csrc/wgrad2_tc.cu).  set_tma(0): the producers load the operands
 * from global memory (round-1 path) instead of the TMA landing ring; set_min_pixels(n): smallest map (input pixels) routed to
 * this kernel (default 12000, n < 0 restores it; tests pass 0 to reach it with small shapes). */
int bts_wgrad2_set_tma(int on);
int bts_wgrad2_set_min_pixels(long long n);
int bts_wgrad2_set_min_kblocks(int n);
int bts_wgrad2_set_pointwise(int on);        /* 1 (default): 1x1 layers with 64 < Cout <= 256 use this kernel too */

/* (k0, k1) of bts_bn_bwd_apply from sums reduced elsewhere (the BatchNorm-backward epilogue of bts_conv_fwd) */
int bts_bn_bwd_coef(const double *S1, const double *S2, long long M, int C, const float *scale, const float *mean,
                    const float *invstd, float *coef, void *stream);
/* grouped 3x3 (ResNeXt: 32 groups of cpg channels): w is (width, cpg, KH, KW).  bts_conv_group_window -> the diagonal block
 * width kwin the packed operator uses (128 when width % 128 == 0 and 128 % cpg == 0; 0 = not supported). */
int bts_conv_group_window(int width, int cpg);
/* n-tile width of the grouped operator of window kwin (the widest multiple of 16 <= 64 dividing kwin; 0 if kwin is invalid) */
int bts_conv_group_n_tile(int kwin);
long long bts_conv_packed_floats_grouped(int width, int cpg, int KH, int KW);
int bts_conv_pack_weights_grouped(const float *w, long long s_co, long long s_ci, long long s_kh, long long s_kw, int width,
                                  int cpg, int KH, int KW, int transpose_flip, float *wpack, void *stream);
int bts_conv_wgrad_grouped_plan(int B, int Hout, int Wout, int width, int cpg, int KH, int KW, int *splitK_out,
                                long long *workspace_floats);
int bts_conv_wgrad_grouped(const float *x, long long x_pixel_stride, int B, int Hs, int Ws, int width, int cpg, int KH, int KW,
                           int stride, int pad, int dil, const float *dy, long long dy_pixel_stride, float *workspace,
                           int splitK, float *dw, long long s_co, long long s_ci, long long s_kh, long long s_kw,
                           int precision, void *stream);

/* wgrad on the same engine: dW[co,ci,tap] = sum_p dY[p,co] * pre(x[p (+) tap, ci]), both operands transposed
 * to K-major in shared memory,
 * split-K partials in `workspace` reduced deterministically into dw (strides in floats).
 *   bts_conv_wgrad_plan(...) -> splitK and the workspace size (floats) the call needs. */
int bts_conv_wgrad_plan(int B, int Hout, int Wout, int Cin, int Cout, int KH, int KW, int stride, int *splitK_out,
                        long long *workspace_floats);
int bts_conv_wgrad(const float *x, long long x_pixel_stride, int B, int Hs, int Ws, int upsample2, int Cin,
                   int KH, int KW, int stride, int pad, int dil, const float *pre_scale, const float *pre_shift,
                   int pre_relu, const float *dy, long long dy_pixel_stride, int Cout, float *workspace, int splitK,
                   float *dw, long long s_co, long long s_ci, long long s_kh, long long s_kw, int precision,
                   void *stream);

/* ---- single-output-channel convolutions (get_depth 3x3 32->1 + sigmoid, bts.py:193-194; reduc1x1 final 1x1 8->1 +
 * sigmoid, bts.py:94-96) as HBM-bound CUDA-core kernels.  x NHWC, C in {8,16,32,64,128}, K in {1,3}, stride 1,
 * pad K/2.  w: the (1,C,K,K) parameter addressed by its (ci,kh,kw) strides.  act: 0 none, 2 sigmoid.
 * Backward entry points take dy and, when the forward applied the sigmoid, the saved output `sig` (else NULL):
 * the effective gradient is dy*sig*(1-sig).  wgrad needs bts_conv_c1_workspace_floats(C,K) floats of workspace. */
int bts_conv_c1_workspace_floats(int C, int K);
int bts_conv_c1_fwd(const float *x, long long x_pixel_stride, int B, int H, int W, int C, int K, const float *w,
                    long long s_ci, long long s_kh, long long s_kw, int act, float *y, void *stream);
int bts_conv_c1_dgrad(const float *dy, const float *sig, int B, int H, int W, int C, int K, const float *w,
                      long long s_ci, long long s_kh, long long s_kw, float *dx, long long dx_pixel_stride,
                      void *stream);
int bts_conv_c1_wgrad(const float *x, long long x_pixel_stride, const float *dy, const float *sig, int B, int H,
                      int W, int C, int K, float *workspace, float *dw, long long s_ci, long long s_kh,
                      long long s_kw, void *stream);

/* ---- train-mode BatchNorm pieces for fused BN -> ReLU -> conv chains (torchvision _DenseLayer norm1/relu1/conv1/
 * norm2/relu2/conv2; decoder BNs bts.py:154-182).  The normalisation is applied inside the consumer conv
 * (bts_conv_fwd pre_scale/pre_shift/pre_relu); these entry points provide the per-channel reductions and the
 * backward pass over NHWC tensors (explicit pixel strides -> channel slices of slabs work in place).
 *   bts_bn_stats            : sum / sum of squares per channel (fp64 accumulators, zeroed by the call)
 *   bts_bn_finalize         : -> scale = gamma*invstd, shift = beta - mean*scale, mean, invstd (+ running-stat update,
 *                             momentum m, unbiased variance; running_* may be NULL; num_batches_tracked += 1 unless NULL)
 *   bts_bn_fold             : the same four vectors from frozen running statistics (eval mode)
 *   bts_bn_bwd_reduce       : S1 = sum g*mask, S2 = sum g*mask*xhat (y = x*scale+shift, mask = the backward mask of `act`
 *                             at y) and the fp32 backward coefficients coef[0:C] = k0, coef[C:2C] = k1
 *                             (dx = mask*scale*g + k1*x + k0)
 *   bts_bn_bwd_apply        : out (=|+=) mask*scale*g + k1*x + k0   (coef == NULL: frozen statistics, k0 = k1 = 0)
 * `act` is the activation after the normalisation: 0 none (plain BatchNorm, as the decoder's bn5/bn4/bn4_2/bn3/bn2 which
 * feed a concat, bts.py:200-246), 1 ReLU (mask [y>0]), 2 ReLU6 (torchvision mobilenet_v2's Conv2dNormActivation /
 * InvertedResidual, bts.py:297-300; its backward mask is 0 < y < 6, strictly, as hardtanh_backward). */
int bts_bn_stats(const float *x, long long x_pixel_stride, long long M, int C, double *sum, double *sumsq, void *stream);
int bts_bn_finalize(const double *sum, const double *sumsq, long long N, int C, const float *gamma, const float *beta,
                    float eps, float momentum, float *running_mean, float *running_var, long long *num_batches_tracked,
                    float *scale, float *shift, float *mean, float *invstd, void *stream);
int bts_bn_fold(int C, const float *gamma, const float *beta, float eps, const float *running_mean,
                const float *running_var, float *scale, float *shift, float *mean, float *invstd, void *stream);
int bts_bn_bwd_reduce(const float *x, long long x_pixel_stride, const float *g, long long g_pixel_stride, long long M,
                      int C, const float *scale, const float *shift, const float *mean, const float *invstd, int act,
                      double *S1, double *S2, float *coef, void *stream);
int bts_bn_bwd_apply(const float *x, long long x_pixel_stride, const float *g, long long g_pixel_stride, long long M,
                     int C, const float *scale, const float *shift, const float *coef, int act, float *out,
                     long long out_pixel_stride, int accumulate, void *stream);

/* One-pass BatchNorm+ReLU backward into a concat gradient slab (the dense-block fan-out, torchvision densenet.py
 * _DenseLayer / _DenseBlock backward): out += [y>0]*scale*g in the same pass that reduces S1, S2; the per-channel affine
 * remainder k1*x + k0 is added into K0/K1 (fp64, K0 == K1 == NULL for frozen statistics) and applied later, once per
 * channel slice, by bts_bn_bwd_correct (out += K1*x + K0) -- before that slice's gradient is consumed. */
int bts_bn_relu_bwd_fused(const float *x, long long x_pixel_stride, const float *g, long long g_pixel_stride, long long M,
                          int C, const float *scale, const float *shift, const float *mean, const float *invstd,
                          double *S1, double *S2, float *out, long long out_pixel_stride, double *K0, double *K1,
                          void *stream);
int bts_bn_bwd_correct(const float *x, long long x_pixel_stride, long long M, int C, const double *K0, const double *K1,
                       float *out, long long out_pixel_stride, void *stream);

/* ---- streaming NHWC glue kernels of the decoder / encoder transitions (csrc/elem.cu) ---------------------------
 * All take explicit pixel strides (floats) so channel slices of wider slabs are read / written in place.
 *   bts_bn_apply       out = act(x*scale + shift)       -- BatchNorm2d forward given (scale, shift) from bts_bn_finalize /
 *                      bts_bn_fold (decoder BNs bts.py:154-182; torchvision norm0 / norm5); `act` is the activation code
 *                      0 none, 1 ReLU, 2 ReLU6 (min(max(y, 0), 6): mobilenet_v2's BN + ReLU6 pairs)
 *   bts_elu_bwd        out = gy * (y > 0 ? 1 : y + 1)   -- backward of nn.ELU() through its saved OUTPUT y (bts.py:72,79,...)
 *   bts_upsample2_sum  out[b,y,x,:] = sum of g[b,2y..2y+1,2x..2x+1,:]  -- backward of F.interpolate(scale_factor=2,
 *                      mode='nearest') (bts.py:77); relu_src != NULL additionally gates by relu_src > 0 (torch.nn.ReLU in
 *                      front of upconv5, bts.py:198)
 *   bts_copy_channels  dst (=|+=) src over M pixels x C channels -- torch.cat along channels / its backward (bts.py:201-260)
 *   bts_zero_channels  dst[:, c0:c1] = 0                -- alignment padding channels of concat3 (225) / concat2 (161)
 *   bts_avgpool2_fwd/bwd  2x2 stride-2 average pooling of the DenseNet transitions (torchvision densenet.py `pool`) */
int bts_bn_apply(const float *x, long long x_pixel_stride, long long M, int C, const float *scale, const float *shift,
                 int act, float *out, long long out_pixel_stride, void *stream);
int bts_elu_bwd(const float *gy, long long gy_pixel_stride, const float *y, long long y_pixel_stride, long long M, int C,
                float *out, long long out_pixel_stride, void *stream);
int bts_upsample2_sum(const float *g, long long g_pixel_stride, int B, int H, int W, int C, const float *relu_src,
                      long long relu_pixel_stride, float *out, long long out_pixel_stride, void *stream);
int bts_copy_channels(const float *src, long long src_pixel_stride, long long M, int C, float *dst,
                      long long dst_pixel_stride, int accumulate, void *stream);
int bts_zero_channels(float *dst, long long dst_pixel_stride, long long M, int c0, int c1, void *stream);
int bts_avgpool2_fwd(const float *x, long long x_pixel_stride, int B, int Hout, int Wout, int C, float *out,
                     long long out_pixel_stride, void *stream);
int bts_avgpool2_bwd(const float *g, long long g_pixel_stride, int B, int Hout, int Wout, int C, float *gx,
                     long long gx_pixel_stride, void *stream);

/* ---- weight gradient of the narrow 1x1 convolutions of the reduction heads (bts.py:83-108) on CUDA cores (csrc/pointwise.cu):
 * dW[co,ci] = sum_p dY[p,co]*x[p,ci] for Cin in {8,16,32,64}, Cout <= 32 -- HBM-bound, deterministic two-pass reduction.
 * workspace: bts_conv_pw_wgrad_workspace_floats(Cin, Cout) floats; dw addressed by its (co, ci) strides in floats. */
/* Forward / dgrad of the same narrow 1x1 layers on CUDA cores (HBM-bound): out[p, co] = act(sum_ci x[p, ci] * W[co, ci]),
 * Cin in {8,16,32,64}, Cout <= 64; (s_out, s_in) are the element strides of W[out, in] -- for dgrad pass the conv weight's
 * (s_ci, s_co) and dY as x.  act: 0 none, 1 ELU, 2 sigmoid.  Replaces the tensor engine for reduc1x1/2x2/4x4 (bts.py:83-108). */
int bts_conv_pw_fwd_eligible(int Cin, int Cout);
int bts_conv_pw_fwd(const float *x, long long x_pixel_stride, long long M, int Cin, const float *w, long long s_out,
                    long long s_in, int Cout, int act, float *out, long long out_pixel_stride, void *stream);
int bts_conv_pw_wgrad_eligible(int Cin, int Cout);
long long bts_conv_pw_wgrad_workspace_floats(int Cin, int Cout);
int bts_conv_pw_wgrad(const float *x, long long x_pixel_stride, const float *dy, long long dy_pixel_stride, long long M,
                      int Cin, int Cout, float *workspace, float *dw, long long s_co, long long s_ci, void *stream);

/* ResNet / ResNeXt encoder glue (torchvision.models.resnet behind reference pytorch/bts.py:282-296):
 *   bts_bn_add_relu   out = max(x*scale + shift + res, 0)            Bottleneck tail  relu(bn3(conv3(.)) + identity)
 *   bts_bn_add        out = x*scale + shift + res                    MobileNetV2 inverted-residual tail x + bn3(conv3(.))
 *                                                                    (torchvision InvertedResidual, use_res_connect)
 *   bts_relu_bwd      out = gy * (y > 0)                             its backward (through the saved output y)
 *   bts_maxpool3s2_*  3x3 / stride 2 / pad 1 max-pool (the encoder stems' pool0 / maxpool), NHWC; forward records the
 *                     winning window position (uint8 per OUTPUT element, dense [B,Ho,Wo,C]) -> deterministic gather backward */
int bts_bn_add_relu(const float *x, long long x_pixel_stride, long long M, int C, const float *scale, const float *shift,
                    const float *res, long long res_pixel_stride, float *out, long long out_pixel_stride, void *stream);
int bts_bn_add(const float *x, long long x_pixel_stride, long long M, int C, const float *scale, const float *shift,
               const float *res, long long res_pixel_stride, float *out, long long out_pixel_stride, void *stream);
int bts_relu_bwd(const float *gy, long long gy_pixel_stride, const float *y, long long y_pixel_stride, long long M, int C,
                 float *out, long long out_pixel_stride, void *stream);
int bts_maxpool3s2_fwd(const float *x, long long x_pixel_stride, int B, int H, int W, int C, float *out,
                       long long out_pixel_stride, unsigned char *argmax, void *stream);
int bts_maxpool3s2_bwd(const float *g, long long g_pixel_stride, const unsigned char *argmax, int B, int H, int W, int C,
                       float *gx, long long gx_pixel_stride, void *stream);

/* ---- depthwise 3x3 convolution of the MobileNetV2 inverted-residual blocks (csrc/dwconv.cu; torchvision mobilenet_v2
 * features[1..17] `conv.*` groups == C layer behind reference pytorch/bts.py:297-300, replacing cuDNN's depthwise
 * forward / backward-data / backward-filter).  NHWC fp32, pad 1, stride 1 or 2, no bias, C % 4 == 0, H x W the INPUT size,
 * output (H-1)/stride+1 x (W-1)/stride+1.  x, y, dy, dx: 16-byte aligned with pixel strides that are multiples of 4 (channel
 * slices of wider slabs work).  w: the (C,1,3,3) parameter read in place through its (c, kh, kw) strides.  Anything else
 * returns BTS_EINVAL before any launch.
 *   bts_dw3x3_fwd    y = dw(pre(x)) [-> relu6(y*post_scale + post_shift)]
 *                    pre: relu6(x*pre_scale + pre_shift) per channel (both NULL to skip), applied once per staged element;
 *                    the zero padding is applied after it.  post: the eval-mode epilogue relu6(bn2(y)) from folded running
 *                    statistics (both NULL to skip).  stat_sum / stat_sumsq (both or neither; not with post): fp64 per-channel
 *                    sum and sum of squares of y, WRITTEN (no zeroing needed), reduced deterministically through
 *                    `workspace` = bts_dw3x3_fwd_workspace_floats(...) floats (8-byte aligned).
 *   bts_dw3x3_dgrad  dx from dy (dy is (B, Ho, Wo, C)); stride 1 is the forward over flipped taps, stride 2 gathers only the
 *                    taps that land.
 *   bts_dw3x3_wgrad  dw[c,kh,kw] = sum_p dy[p,c] * pre(x)[p*stride + (kh,kw) - 1, c], the same optional prologue recomputed
 *                    from the raw x; per-CTA fp64 partials in `workspace` = bts_dw3x3_wgrad_workspace_floats(...) floats,
 *                    summed in a fixed order by a second kernel (bit-reproducible).  dw written through its strides.
 * The *_workspace_floats queries return BTS_EINVAL for shapes the kernels do not take. */
long long bts_dw3x3_fwd_workspace_floats(int B, int H, int W, int C, int stride);
int bts_dw3x3_fwd(const float *x, long long x_pixel_stride, int B, int H, int W, int C, int stride, const float *w, long long s_c,
                  long long s_kh, long long s_kw, const float *pre_scale, const float *pre_shift, const float *post_scale,
                  const float *post_shift, float *y, long long y_pixel_stride, double *stat_sum, double *stat_sumsq,
                  float *workspace, void *stream);
int bts_dw3x3_dgrad(const float *dy, long long dy_pixel_stride, int B, int H, int W, int C, int stride, const float *w,
                    long long s_c, long long s_kh, long long s_kw, float *dx, long long dx_pixel_stride, void *stream);
long long bts_dw3x3_wgrad_workspace_floats(int B, int H, int W, int C, int stride);
int bts_dw3x3_wgrad(const float *x, long long x_pixel_stride, const float *dy, long long dy_pixel_stride, int B, int H, int W,
                    int C, int stride, const float *pre_scale, const float *pre_shift, float *workspace, float *dw,
                    long long s_c, long long s_kh, long long s_kw, void *stream);

/* ---- optimizer step of the training loop (reference pytorch/bts_main.py:371-373 torch.optim.AdamW, two groups, eps 1e-3;
 * :456-460 poly LR) as ONE multi-tensor kernel, csrc/optim.cu.  ptrs: device int64 [4n] = param | grad | exp_avg | exp_avg_sq
 * addresses; numel: device int64 [n]; group: device int32 [n] -> index into the n_groups (<= 8) scalar sets;
 * chunk_tensor / chunk_off: device tables cutting every tensor into bts_adamw_chunk()-element pieces;
 * scalars: HOST float [7*n_groups], seven blocks of n_groups: 1-lr*wd | 1-beta1 | beta2 | 1-beta2 | sqrt(1-beta2^t) | eps |
 * -lr/(1-beta1^t).  Element arithmetic follows torch's _multi_tensor_adam operation by operation. */
int bts_adamw_chunk(void);
int bts_adamw_multi(const long long *ptrs, const long long *numel, const int *group, int n, const int *chunk_tensor,
                    const long long *chunk_off, int n_chunks, const float *scalars, int n_groups, void *stream);
/* every packed conv operator of a model in one launch: descs = device array of n 96-byte descriptors
 * {w, wpack, s_co, s_ci, s_kh, s_kw, start (int64 each), Cout, Cin, KH, KW, transpose_flip, n_tile, n_tiles, kwin, cpg, pad
 * (int32 each)}, start = prefix sum of packed_floats/2; total = their sum. */
int bts_conv_pack_weights_multi(const void *descs, int n, long long total, void *stream);

/* ---- data formats either side of the hot path (SURVEY 8f ranks 2-3), csrc/io.cu
 * bts_input_prep: the reference loader's per-sample transform after decoding (pytorch/bts_dataloader.py:128-140,202-235,
 *   244-249), fused: uint8 HWC frames [B,Hs,Ws,3] (+ optional uint16 depth [B,Hs,Ws]) -> crop -> flip -> gamma/brightness/
 *   colour augmentation + clip -> ImageNet normalisation -> fp32 NHWC image [B,H,W,(stride)] and depth/depth_div [B,H,W].
 *   params: device float [B][9] = y0, x0, flip, augment, gamma, brightness, colour r,g,b (the random draws stay on the host).
 * bts_input_prep_rotated: bts_input_prep after the random rotation of the whole frame (pytorch/bts_dataloader.py:122-125,
 *   187-189): the crop window is cut from the frame as PIL's Image.rotate leaves it, bilinear for the image and nearest for
 *   the depth, 0 outside the frame, bit-exact with Pillow.  affine: device double [B][6] = a..f of each sample's inverse
 *   map, source point (a*(x+.5) + b*(y+.5) + c, d*(x+.5) + e*(y+.5) + f) of rotated-frame pixel (x, y), the matrix
 *   Image.rotate passes to Image.transform (bts_b200.data.rotate_affine).  affine == NULL gives bts_input_prep's output.
 * bts_eval_errors: online-eval clamps + masks + the nine metrics of one image (pytorch/bts_main.py:144-165,275-296):
 *   metrics_out[10] = silog, abs_rel, log10, rms, sq_rel, log_rms, d1, d2, d3, n_valid; crop rows [y0,y1) cols [x0,x1);
 *   workspace = 10 doubles.
 * bts_depth_to_u16: the 16-bit PNG wire format of pytorch/bts_test.py:179-185, uint16(depth * scale). */
int bts_input_prep(const unsigned char *img_u8, int Hs, int Ws, const unsigned short *depth_u16, float depth_div,
                   const float *params, int B, int H, int W, float *image_out, long long out_pixel_stride, float *depth_out,
                   void *stream);
int bts_input_prep_rotated(const unsigned char *img_u8, int Hs, int Ws, const unsigned short *depth_u16, float depth_div,
                           const float *params, const double *affine, int B, int H, int W, float *image_out,
                           long long out_pixel_stride, float *depth_out, void *stream);
int bts_eval_errors(const float *pred, const float *gt, int H, int W, float min_depth, float max_depth, int crop_y0,
                    int crop_y1, int crop_x0, int crop_x1, double *workspace, float *metrics_out, void *stream);
int bts_depth_to_u16(const float *depth, float scale, long long n, unsigned short *out, void *stream);

/* zero n floats on the stream (grad_focal output of the TF-op surface, integration/tf_op/bts_lpg_tf_op.cc) */
int bts_fill_zero_f32(float *p, long long n, void *stream);

#ifdef __cplusplus
}
#endif
#endif /* BTS_B200_H_ */
