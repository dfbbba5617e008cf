/*
 * b200seg.h — C ABI of libb200seg.so: the H100 (sm_90a) kernels behind the
 * 3D-segmentation training hot path of yhygao/CBIM-Medical-Image-Segmentation.
 *
 * The reference has NO native interface (it is 100% Python, SURVEY.md §2): every
 * entry point below replaces a *library call site* in the reference, cited as
 * reference file:line.  All pointers are DEVICE pointers owned by the caller
 * (PyTorch's caching allocator in the drop-in); kernels never allocate, free,
 * or keep a pointer past return.  Every call takes the CUDA stream to launch on
 * (as a void* holding a cudaStream_t) and returns 0 on success or a negative
 * B200SEG_E* code; b200seg_strerror() maps codes to text.  No entry point
 * synchronises the host.
 *
 * Layout conventions
 *   activations : NDHWC ("channels-last-3d"), element (b,d,h,w,c) of a tensor
 *                 with leading dimension `ld` (channels physically stored per
 *                 voxel) and channel offset `coff` lives at
 *                 base[(((b*D+d)*H+h)*W+w)*ld + coff + c]            (c < C)
 *   dtype       : B200SEG_F32 (0) or B200SEG_F16 (1) storage; accumulation is
 *                 always fp32 (wgmma / mma.sync or FFMA).
 *   stats       : per-(batch,channel) InstanceNorm sums, double[B][C][2] =
 *                 {sum, sum of squares} over D*H*W.  Producers ACCUMULATE into
 *                 them (caller zeroes first); consumers derive mean / rstd.
 *   weights     : "packed" conv weights, [taps][Cout][Cin] in the activation
 *                 dtype, tap = (kd_i*kh + kh_i)*kw + kw_i; produced from the
 *                 reference's [Cout][Cin][kd][kh][kw] fp32 parameter by
 *                 b200seg_pack_weight (optionally flipped+transposed for dgrad).
 */
#ifndef B200SEG_H
#define B200SEG_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B200SEG_VERSION 100

enum { B200SEG_F32 = 0, B200SEG_F16 = 1 };

enum {
  B200SEG_OK = 0,
  B200SEG_EINVAL = -1,      /* bad argument (null pointer, non-positive dim, bad dtype)      */
  B200SEG_EUNSUPPORTED = -2,/* shape not supported by the requested algorithm (hard error)   */
  B200SEG_ECUDA = -3,       /* a CUDA runtime call failed (see b200seg_last_cuda_error)      */
  B200SEG_ENODEVICE = -4    /* device is not sm_90 (this library has no fallback)            */
};

/* conv algorithms.  conv3d_fwd takes TC, TC_TF32 or DIRECT (whatever b200seg_conv3d_algo /
 * b200seg_conv3d_algo_tf32 returned when the weights were packed); wgrad also accepts AUTO since it
 * consumes no packed weights.  TC runs fp16 operands; TC_TF32 runs fp32 tensors on the same
 * tensor-core kernel with TF32 operands (dtype = B200SEG_F32 only) and is never chosen unless the
 * caller asks for it. */
enum { B200SEG_ALGO_AUTO = 0, B200SEG_ALGO_DIRECT = 1, B200SEG_ALGO_TC = 2, B200SEG_ALGO_TC_TF32 = 3 };

/* activation applied to the (optionally normalised) conv input in the loader */
enum { B200SEG_ACT_NONE = 0, B200SEG_ACT_RELU = 1,
       B200SEG_ACT_LRELU = 2 /* LeakyReLU(negative_slope = 0.01): monai UnetResBlock, swin_unetr.py:129-226 */ };

int         b200seg_version(void);
const char* b200seg_strerror(int code);
const char* b200seg_last_cuda_error(void);
/* 0 if the current device can run this library (compute capability 10.x). */
int         b200seg_check_device(void);

/* ---------------------------------------------------------------------------
 * Fused softmax + adaptive-Tversky Dice + weighted cross-entropy.
 * Replaces training/losses.py:18-58 (DiceLoss.forward), nn.CrossEntropyLoss at
 * train_ddp.py:93,189-191 and the sum at train_ddp.py:186-191.
 *
 * logits element (b,v,c) is at logits[b*stride_b + v*stride_v + c*stride_c]
 * (NCDHW: stride_c=V, stride_v=1; NDHWC: stride_c=1, stride_v=C).
 * labels: int64 (label_bytes=8) or uint8 (label_bytes=1), [B][V].
 * ce_weight: float[C] or NULL (=ones).  partial: double[3*C+2] scratch, zeroed
 * by the call itself.  out: float[4+4*C]:
 *   out[0]=ce_scale*CE + dice_scale*Dice, out[1]=CE, out[2]=Dice, out[3]=sum_w,
 *   out[4+c]      = dDice/dTP_c (total derivative, alpha kept differentiable)
 *   out[4+C+c]    = dDice/dSP_c
 *   out[4+2C+c]   = alpha_c,  out[4+3C+c] = dice_c
 * ------------------------------------------------------------------------- */
int b200seg_dice_ce_fwd(const void* logits, int dtype,
                        int64_t stride_b, int64_t stride_v, int64_t stride_c,
                        const void* labels, int label_bytes,
                        const float* ce_weight,
                        int B, int64_t V, int C,
                        float ce_scale, float dice_scale,
                        double* partial, float* out, void* stream);

/* dlogits gets the same strides as logits.  grad_out: device float scalar
 * (upstream gradient, e.g. GradScaler's scale) or NULL (=1). */
int b200seg_dice_ce_bwd(const void* logits, int dtype,
                        int64_t stride_b, int64_t stride_v, int64_t stride_c,
                        const void* labels, int label_bytes,
                        const float* ce_weight,
                        int B, int64_t V, int C,
                        float ce_scale, float dice_scale,
                        const float* fwd_out, const float* grad_out,
                        void* dlogits, void* stream);

/* ---------------------------------------------------------------------------
 * InstanceNorm statistics (nn.InstanceNorm3d, conv_layers.py:40,42 — the
 * reduction half).  Accumulates {sum, sumsq} of x[..., coff:coff+C] into
 * stats[B][C][2].
 * ------------------------------------------------------------------------- */
int b200seg_instnorm_stats(const void* x, int dtype, int ld, int coff,
                           int B, int64_t V, int C, double* stats, void* stream);

/* y = act((x - mean) * rstd), materialised (used where the normalise cannot be
 * folded into a consumer's loader: SingleConv post-activation, conv_layers.py:46-53). */
int b200seg_instnorm_apply(const void* x, int dtype, int x_ld, int x_coff,
                           const double* stats, float eps, int act,
                           void* y, int y_ld, int y_coff,
                           int B, int64_t V, int C, void* stream);

/* Backward of y = act(IN(x)), stage 1: g = dy * act'(xhat); accumulates
 * bstats[B][C][2] += {sum g, sum g*xhat}; writes g.  */
int b200seg_instnorm_bwd_reduce(const void* dy, int dy_ld, int dy_coff,
                                const void* x, int x_ld, int x_coff, int dtype,
                                const double* stats, float eps, int act,
                                void* g, int g_ld, int g_coff,
                                double* bstats, int B, int64_t V, int C, void* stream);

/* Stage 2: dx = rstd * (g - S1/n - xhat*S2/n) (+ add).  `add` (nullable, may
 * alias dx) carries a gradient arriving over another branch, e.g. the identity
 * residual of a BasicBlock (conv_layers.py:92). */
int b200seg_instnorm_bwd_apply(const void* g, int g_ld, int g_coff,
                               const void* x, int x_ld, int x_coff, int dtype,
                               const double* stats, const double* bstats, float eps,
                               const void* add, int add_ld, int add_coff,
                               void* dx, int dx_ld, int dx_coff,
                               int B, int64_t V, int C, void* stream);

/* ---------------------------------------------------------------------------
 * Conv3d family (nn.Conv3d call sites conv_layers.py:29-38, unet_utils.py:14,
 * unet.py:47; autograd of same at train_ddp.py:193/208).  Stride 1, padding
 * k/2, odd k, dilation 1, groups 1.
 * ------------------------------------------------------------------------- */

/* w_packed[tap][Cout][Cin] <- w[Cout][Cin][kd][kh][kw] (fp32 parameter).
 * transpose_flip!=0 builds the dgrad operand instead:
 *   w_packed[T-1-tap][Cin][Cout] (roles of Cin/Cout swapped, taps mirrored).
 * co_off / co_total place this weight's output channels inside a wider fused
 * weight (conv1+shortcut of a BasicBlock share one GEMM, conv_layers.py:79,84).
 * layout is B200SEG_ALGO_DIRECT, _TC (dtype F16) or _TC_TF32 (dtype F32). */
int b200seg_pack_weight(const float* w, int Cout, int Cin, int taps,
                        void* w_packed, int dtype, int transpose_flip,
                        int co_off, int co_total, int layout, void* stream);

/* Multi-tensor form of b200seg_pack_weight: one launch re-packs every weight of a
 * model (called once per forward, so an in-place `.data` update of a parameter —
 * the reference's EMA, training/utils.py:99-102 — can never leave a stale image).
 *   jobs_dev  : int64 [njobs][10] = {w ptr, out ptr, Cout, Cin, taps, dtype,
 *               transpose_flip, co_off, co_total, layout code}; layout code 0 = DIRECT,
 *               1 = TC, 2 = TC_TF32
 *   chunks_dev: int64 [nchunks][2] = {job index, code}, one thread block each:
 *               code >= 0: ELEMENT chunk, b200seg_pack_chunk_elems() consecutive elements of w
 *                          starting at `code`;
 *               code <  0: TILE chunk (Cout and Cin multiples of 8), -(code+1) = co0*65536 + ci0:
 *                          output channels [co0, co0+8) x input channels [ci0, ci0 +
 *                          b200seg_pack_tile_ci(taps)) x all taps, staged through shared memory
 *                          and written as 16-byte runs of the packed image. */
int b200seg_pack_chunk_elems(void);
/* input channels per TILE chunk of b200seg_pack_weights_multi for a `taps`-tap kernel (0 = element chunks only) */
int b200seg_pack_tile_ci(int taps);
int b200seg_pack_weights_multi(const int64_t* jobs_dev, const int64_t* chunks_dev,
                               int nchunks, void* stream);

/* Which algorithm (B200SEG_ALGO_TC or _DIRECT) serves a conv of this shape.  The
 * packed-weight layout is per algorithm (`layout` above = this value):
 *   DIRECT : [tap][Cout][Cin];
 *   TC     : the shared-memory image the tensor-core kernel streams with bulk TMA,
 *            [ntile][tap][kchunk][KC/8][NT][8] fp16  (NT / KC: csrc/conv_args.h);
 *   TC_TF32: the same image in 16-byte planes of 4 fp32 channels, rounded to TF32,
 *            [ntile][tap][kchunk][KC/4][NT][4]  (KC: tc_pick_kc_tf32).
 * fp32 convolutions are always DIRECT here: TF32 is an opt-in (b200seg_conv3d_algo_tf32). */
int b200seg_conv3d_algo(int Cin, int Cout, int kd, int kh, int kw, int dtype, int B);
/* TC_TF32 when an fp32 conv of this shape can run on TF32 tensor cores (same kernel-size and
 * batch limits as the fp16 rule; Cin a multiple of 8, Cout of 16), else DIRECT. */
int b200seg_conv3d_algo_tf32(int Cin, int Cout, int kd, int kh, int kw, int B);

/* y[.., y_coff:y_coff+Cout] = conv(act(IN(x))) (+bias) (+residual); optionally
 * accumulates InstanceNorm sums of the STORED y into y_stats.
 *   x_stats==NULL  -> no normalisation of the input (raw conv, e.g. the stem)
 *   residual==NULL -> no residual add (conv_layers.py:92 `out += shortcut`)
 * When dgrad_x != NULL the call is the data-gradient of a pre-activation conv:
 * the accumulator `da` is multiplied by act'(xhat(dgrad_x)) before the store
 * and y_stats receives {sum g, sum g*xhat} instead (stage 1 of IN backward),
 * with dgrad_stats the forward statistics of dgrad_x. */
int b200seg_conv3d_fwd(const void* x, int x_ld, int x_coff,
                       const double* x_stats, float eps, int act,
                       const void* w_packed, const float* bias,
                       const void* residual, int r_ld, int r_coff,
                       void* y, int y_ld, int y_coff, double* y_stats,
                       const void* dgrad_x, int dx_ld, int dx_coff,
                       const double* dgrad_stats, float dgrad_eps, int dgrad_act,
                       int B, int D, int H, int W, int Cin, int Cout,
                       int kd, int kh, int kw, int dtype, int algo, void* stream);

/* dw[Cout][Cin][kd][kh][kw] (fp32, the reference parameter layout, what DDP
 * all-reduces) += sum_vox dy[vox][co] * act(IN(x))[vox+tap][ci].
 * dw must be zeroed by the caller unless accumulating.  dbias (float[Cout] or
 * NULL) += sum_vox dy.  b200seg_conv3d_wgrad_workspace() reports the scratch
 * bytes a call needs: per-block partial slices (tensor-core split-K, Cin-1 stem,
 * 1x1x1 head, bias-gradient pass), summed in a fixed order so that dw / dbias
 * are the same on every run; 0 for the CUDA-core path.  A smaller or NULL
 * workspace where one is needed is B200SEG_EINVAL. */
size_t b200seg_conv3d_wgrad_workspace(int x_ld, int x_coff, int normalised,
                                      int dy_ld, int dy_coff, int want_bias,
                                      int B, int D, int H, int W, int Cin, int Cout,
                                      int kd, int kh, int kw, int dtype, int algo);
int b200seg_conv3d_wgrad(const void* x, int x_ld, int x_coff,
                         const double* x_stats, float eps, int act,
                         const void* dy, int dy_ld, int dy_coff,
                         float* dw, float* dbias,
                         int B, int D, int H, int W, int Cin, int Cout,
                         int kd, int kh, int kw, int dtype, int algo,
                         void* workspace, size_t ws_bytes, void* stream);

/* ---- per-channel (BatchNorm) mode of the convolutions -------------------------
 * The input enters as act(x[vox][c] * s[c] + t[c]) from x_affine, a float
 * [Cin][2] {s, t} table (b200seg_batchnorm_fwd_fold), or as act(x) when
 * x_affine is NULL.  The table is one row for the whole batch, so the algorithm
 * and packed-weight layout of these launches are b200seg_conv3d_algo(..., B=1)
 * at any B.  There is no data-gradient mask: the data gradient of a BatchNorm
 * layer is a raw b200seg_conv3d_fwd_pc launch followed by
 * b200seg_batchnorm_bwd_reduce / _fold / _apply.  Everything else (bias,
 * residual, y_stats, workspace, accumulation into dw) is as in
 * b200seg_conv3d_fwd / b200seg_conv3d_wgrad. */
int b200seg_conv3d_fwd_pc(const void* x, int x_ld, int x_coff, const float* x_affine, int act,
                          const void* w_packed, const float* bias,
                          const void* residual, int r_ld, int r_coff,
                          void* y, int y_ld, int y_coff, double* y_stats,
                          int B, int D, int H, int W, int Cin, int Cout,
                          int kd, int kh, int kw, int dtype, int algo, void* stream);
size_t b200seg_conv3d_wgrad_pc_workspace(int x_ld, int x_coff, int transformed,
                                         int dy_ld, int dy_coff, int want_bias,
                                         int B, int D, int H, int W, int Cin, int Cout,
                                         int kd, int kh, int kw, int dtype, int algo);
int b200seg_conv3d_wgrad_pc(const void* x, int x_ld, int x_coff, const float* x_affine, int act,
                            const void* dy, int dy_ld, int dy_coff,
                            float* dw, float* dbias,
                            int B, int D, int H, int W, int Cin, int Cout,
                            int kd, int kh, int kw, int dtype, int algo,
                            void* workspace, size_t ws_bytes, void* stream);

/* ---- BatchNorm (nn.BatchNorm2d, training and eval) ------------------------------
 * sums: fp64 [nb][C][2] {sum x, sum x^2} (nb = B for the per-(sample, channel) sums
 * a convolution epilogue writes, 1 for sums already added over the batch or the
 * ranks), count = values per channel.  Training: batch mean and biased variance;
 * running_mean / running_var updated with `momentum` (running_var with the
 * unbiased variance) and *num_batches_tracked += 1 (may be NULL); count <= 1 is
 * B200SEG_EINVAL.  Eval: the running statistics.  Writes table [C][2] {s, t} =
 * {gamma*rstd, beta - mean*gamma*rstd} and mean_rstd [C][2]. */
int b200seg_batchnorm_fwd_fold(const double* sums, int nb, int C, double count,
                               const float* gamma, const float* beta,
                               float* running_mean, float* running_var, int64_t* num_batches_tracked,
                               float momentum, float eps, int training,
                               float* table, float* mean_rstd, void* stream);
/* y = act(x*s + t) (post-activation blocks); C, ld and offsets multiples of 8. */
int b200seg_batchnorm_apply(const void* x, int dtype, int x_ld, int x_coff, const float* table, int act,
                            void* y, int y_ld, int y_coff, int64_t nvox, int C, void* stream);
/* sums [C][2] (fp64, zeroed by the caller) += {sum dz, sum dz*xhat}, where
 * dz = g * act'(x*s + t) (g itself when table is NULL or act is NONE) and
 * xhat = (x - mean) * rstd.  C <= 2048. */
int b200seg_batchnorm_bwd_reduce(const void* g, int g_ld, int g_coff, const void* x, int x_ld, int x_coff,
                                 int dtype, const float* table, int act, const float* mean_rstd,
                                 int64_t nvox, int C, double* sums, void* stream);
/* dgamma = sum dz*xhat, dbeta = sum dz (fp32, written), and coef [C][4]
 * {a, b, mean, k} with dx = a*dz + b*(x - mean) + k (training: batch-statistic
 * terms included; eval: b = k = 0). */
int b200seg_batchnorm_bwd_fold(const double* sums, double count, const float* gamma, const float* mean_rstd,
                               int training, int C, float* dgamma, float* dbeta, float* coef, void* stream);
/* out = a*dz + b*(x - mean) + k (+ add); dz as in b200seg_batchnorm_bwd_reduce.
 * out may be add (accumulation in place). */
int b200seg_batchnorm_bwd_apply(const void* g, int g_ld, int g_coff, const void* x, int x_ld, int x_coff,
                                int dtype, const float* table, int act, const float* coef,
                                const void* add, int add_ld, int add_coff,
                                void* out, int out_ld, int out_coff, int64_t nvox, int C, void* stream);

/* ---------------------------------------------------------------------------
 * MaxPool3d, kernel == stride (unet_utils.py:36), floor mode, + IN sums of the
 * pooled tensor.  idx: uint8[B][Do][Ho][Wo][C] argmax offset inside the window.
 * ------------------------------------------------------------------------- */
int b200seg_maxpool3d_fwd(const void* x, int x_ld, int x_coff,
                          void* y, int y_ld, int y_coff, uint8_t* idx, double* y_stats,
                          int B, int D, int H, int W, int C, int sd, int sh, int sw,
                          int dtype, void* stream);
int b200seg_maxpool3d_bwd(const void* dy, int dy_ld, int dy_coff, const uint8_t* idx,
                          void* dx, int dx_ld, int dx_coff,
                          int B, int D, int H, int W, int C, int sd, int sh, int sw,
                          int dtype, void* stream);

/* ---------------------------------------------------------------------------
 * Trilinear upsample (align_corners=True) fused with the channel concat
 * (unet_utils.py:69-71): y[.., y_coff:y_coff+C] = upsample(x) to (Do,Ho,Wo),
 * + IN sums of the written channels.  bwd is a deterministic gather (no atomics):
 * dx (+)= sum of the output-voxel gradients whose stencil touches each input voxel.
 * ------------------------------------------------------------------------- */
int b200seg_upsample_trilinear_fwd(const void* x, int x_ld, int x_coff,
                                   void* y, int y_ld, int y_coff, double* y_stats,
                                   int B, int Di, int Hi, int Wi, int Do, int Ho, int Wo,
                                   int C, int dtype, void* stream);
int b200seg_upsample_trilinear_bwd(const void* dy, int dy_ld, int dy_coff,
                                   void* dx, int dx_ld, int dx_coff, int accumulate,
                                   int B, int Di, int Hi, int Wi,
                                   int Do, int Ho, int Wo, int C, int dtype, void* stream);

/* Strided channel-slice copy / cast / add:  y[..,y_coff+c] (+)= x[..,x_coff+c].
 * x_dtype and y_dtype may differ (cast).  Used for concat of the skip tensor,
 * NCDHW<->NDHWC boundary casts and gradient accumulation. */
int b200seg_copy_channels(const void* x, int x_dtype, int x_ld, int x_coff,
                          void* y, int y_dtype, int y_ld, int y_coff, int accumulate,
                          int64_t nvox, int C, void* stream);

/* ---------------------------------------------------------------------------
 * MedFormer bidirectional attention core (B-MHA), medformer_utils.py:63-97
 * (BidirectionAttention.forward between the q/v projections and the output
 * projections).  N = D*H*W feature voxels, M <= 64 semantic-map tokens,
 * dim_head must be 32 (every BASELINE MedFormer level).  All tensors are
 * channels-last with channel index  c = d*heads + h  inside the `inner` block
 * (rearrange1, :43-51):
 *   fq, fv : [B][N][*_ld] (+coff)      feature query / value
 *   mq, mv : [B][M][m_ld] (+coff)      map query / value
 *   fo     : [B][N][fo_ld]             softmax_j(S) @ map_v          (:80,84)
 *   mo     : [B][M][mo_ld]             softmax_i(S)^T @ feat_v       (:82,89)
 *   colstat: float[B][heads][M][2]     {max_i, sum_i exp} of the column softmax,
 *                                      kept for the backward
 *   workspace: b200seg_biattn_workspace() bytes (per-block partials)
 * One pass over the voxels per direction; S/A1/A2 are never materialised.
 * ------------------------------------------------------------------------- */
size_t b200seg_biattn_workspace(int B, int64_t N, int M, int heads);
int b200seg_biattn_fwd(const void* fq, int fq_ld, int fq_coff, const void* fv, int fv_ld, int fv_coff,
                       const void* mq, int mq_coff, const void* mv, int mv_coff, int m_ld,
                       void* fo, int fo_ld, int fo_coff, void* mo, int mo_ld, int mo_coff,
                       float* colstat, float* workspace, int B, int64_t N, int M, int heads, int dim_head,
                       float scale, int dtype, void* stream);
int b200seg_biattn_bwd(const void* fq, int fq_ld, int fq_coff, const void* fv, int fv_ld, int fv_coff,
                       const void* mq, int mq_coff, const void* mv, int mv_coff, int m_ld,
                       const void* mo, int mo_ld, int mo_coff, const float* colstat,
                       const void* dfo, int dfo_ld, int dfo_coff, const void* dmo, int dmo_ld, int dmo_coff,
                       void* dfq, int dfq_ld, int dfq_coff, void* dfv, int dfv_ld, int dfv_coff,
                       void* dmq, int dmq_coff, void* dmv, int dmv_coff, int dm_ld,
                       float* workspace, int B, int64_t N, int M, int heads, int dim_head, float scale,
                       int dtype, void* stream);

/* Wide B-MHA: the same operands and conventions as b200seg_biattn_fwd / _bwd for the
 * shapes those refuse: dim_head 32 with 65..80 map tokens, dim_head 64 or 80 with
 * 1..80 map tokens (ACDC's 2x6x6 maps at dim_head 32 / 64 / 80).  Every other shape,
 * dim_head 32 with M <= 64 included, returns B200SEG_EUNSUPPORTED, so each shape has
 * exactly one path.  workspace: b200seg_biattn_wide_workspace() bytes; it takes
 * dim_head because the per-block partials are 2*dim_head floats per map token. */
size_t b200seg_biattn_wide_workspace(int B, int64_t N, int M, int heads, int dim_head);
int b200seg_biattn_wide_fwd(const void* fq, int fq_ld, int fq_coff, const void* fv, int fv_ld, int fv_coff,
                            const void* mq, int mq_coff, const void* mv, int mv_coff, int m_ld,
                            void* fo, int fo_ld, int fo_coff, void* mo, int mo_ld, int mo_coff,
                            float* colstat, float* workspace, int B, int64_t N, int M, int heads, int dim_head,
                            float scale, int dtype, void* stream);
int b200seg_biattn_wide_bwd(const void* fq, int fq_ld, int fq_coff, const void* fv, int fv_ld, int fv_coff,
                            const void* mq, int mq_coff, const void* mv, int mv_coff, int m_ld,
                            const void* mo, int mo_ld, int mo_coff, const float* colstat,
                            const void* dfo, int dfo_ld, int dfo_coff, const void* dmo, int dmo_ld, int dmo_coff,
                            void* dfq, int dfq_ld, int dfq_coff, void* dfv, int dfv_ld, int dfv_coff,
                            void* dmq, int dmq_coff, void* dmv, int dmv_coff, int dm_ld,
                            float* workspace, int B, int64_t N, int M, int heads, int dim_head, float scale,
                            int dtype, void* stream);

/* ---------------------------------------------------------------------------
 * Depthwise 3-D convolution (groups == C), stride 1, "same" padding, no bias:
 * DepthwiseSeparableConv.depthwise conv_layers.py:135-143 (MedFormer attention
 * projections medformer_utils.py:30-31, MBConv).  Channels-last, C % 8 == 0,
 * kernel extents 1 or 3.  flip is a bit set: bit 0 reads the taps reversed (= the
 * data-gradient of the same layer); bit 1 says w is float[C][kd*kh*kw] — the
 * module's own [C,1,kd,kh,kw] parameter, consumed in place — instead of the
 * tap-major float[kd*kh*kw][C].  Optional fused prologue a = act(IN(x)) from
 * x_stats (NULL: raw x), optional IN sums of y (y_stats).
 * wgrad: dw += sum dy * a (float, caller zeroes / accumulates), laid out
 * [tap][c] (dw_layout 0) or [c][tap] = the parameter's layout (dw_layout 1).
 * ------------------------------------------------------------------------- */
int b200seg_dwconv3d_fwd(const void* x, int x_ld, int x_coff, const double* x_stats, float eps, int act,
                         const float* w, int flip, void* y, int y_ld, int y_coff, double* y_stats,
                         int B, int D, int H, int W, int C, int kd, int kh, int kw, int dtype, void* stream);
int b200seg_dwconv3d_wgrad(const void* x, int x_ld, int x_coff, const double* x_stats, float eps, int act,
                           const void* dy, int dy_ld, int dy_coff, float* dw, int dw_layout,
                           int B, int D, int H, int W, int C, int kd, int kh, int kw, int dtype, void* stream);

/* ---------------------------------------------------------------------------
 * MedFormer operators that are not convolutions (all channels-last).
 *
 * space_to_depth: PatchMerging gather medformer_utils.py:165-171,
 *   y[b,d,h,w,q*C+c] = x[b,d*sd+i,h*sh+j,w*sw+k,c], q=(i*sh+j)*sw+k; reverse!=0
 *   scatters y back into x (the gradient).  Do/Ho/Wo are the OUTPUT extents.
 * mapgen: SemanticMapGeneration medformer_utils.py:221-226,
 *   map[b,k,c] = sum_j softmax_j(wl[b,j,k]) * f[b,j,c]   (K <= 80 map codes),
 *   colstat float[B][K][2]; bwd writes df and dwl (dw_pad >= K logits channels,
 *   the padding gets zeros) into the gradient of the fused projection output.
 * se_gate: SEBlock conv_layers.py:159-174 on the channel means taken from IN
 *   sums: gate = sigmoid(W2 relu(W1 mean + b1) + b2); w1 [R][C], w2 [C][R].
 *   bwd accumulates (+=) dw1/db1/dw2/db2 and returns dmean.
 * channel_scale: y = x*gate[b][c]; bwd_reduce: dgate += sum_vox dy*x, added in a
 *   fixed order through a float workspace of channel_scale_bwd_workspace bytes;
 *   bwd_apply: dx = dy*gate + dmean/V (dmean may be NULL).
 * layernorm: nn.LayerNorm(C, eps) trans_layers.py:36-41 over rows [R][C];
 *   mean_rstd float[R][2]; bwd accumulates (+=) dgamma/dbeta.
 * gelu: exact erf GELU trans_layers.py:22; dy==NULL -> forward, else out=dy*gelu'(x).
 * mhsa: Attention core trans_layers.py:84-93 for dim_head 32 with L<=192 tokens
 *   and dim_head 64 with L<=216 tokens;
 *   qkv [B][L][3*inner] ('(heads dim_head)' order), out [B][L][inner];
 *   forward when dout==NULL, otherwise writes dqkv.
 * ------------------------------------------------------------------------- */
int b200seg_space_to_depth(void* x, void* y, int B, int Do, int Ho, int Wo, int C, int sd, int sh, int sw,
                           int reverse, int dtype, void* stream);
size_t b200seg_mapgen_workspace(int B, int64_t N, int K, int C);
int b200seg_mapgen_fwd(const void* f, int f_ld, int f_coff, const void* wl, int w_ld, int w_coff,
                       void* map, float* colstat, float* workspace, int B, int64_t N, int K, int C,
                       int dtype, void* stream);
int b200seg_mapgen_bwd(const void* f, int f_ld, int f_coff, const void* wl, int w_ld, int w_coff,
                       const void* map, const float* colstat, const void* dmap,
                       void* df, int df_ld, int df_coff, void* dwl, int dw_ld, int dw_coff, int dw_pad,
                       int B, int64_t N, int K, int C, int dtype, void* stream);
int b200seg_se_gate_fwd(const double* stats, int64_t nvox, const float* w1, const float* b1, const float* w2,
                        const float* b2, float* gate, float* hidden, float* mean, int B, int C, int R, void* stream);
int b200seg_se_gate_bwd(const float* dgate, const float* gate, const float* hidden, const float* mean,
                        const float* w1, const float* w2, float* dw1, float* db1, float* dw2, float* db2,
                        float* dmean, int B, int C, int R, void* stream);
int b200seg_channel_scale_fwd(const void* x, const float* gate, void* y, int B, int64_t V, int C, int dtype, void* stream);
size_t b200seg_channel_scale_bwd_workspace(int B, int64_t V, int C);
int b200seg_channel_scale_bwd_reduce(const void* dy, const void* x, float* dgate, float* workspace, int B, int64_t V, int C, int dtype, void* stream);
int b200seg_channel_scale_bwd_apply(const void* dy, const float* gate, const float* dmean, void* dx, int B, int64_t V, int C, int dtype, void* stream);
int b200seg_layernorm_fwd(const void* x, const float* gamma, const float* beta, void* y, float* mean_rstd,
                          int R, int C, float eps, int dtype, void* stream);
int b200seg_layernorm_bwd(const void* dy, const void* x, const float* gamma, const float* mean_rstd, void* dx,
                          float* dgamma, float* dbeta, int R, int C, int dtype, void* stream);
int b200seg_gelu(const void* x, const void* dy, void* out, int64_t n, int dtype, void* stream);
int b200seg_mhsa(const void* qkv, const void* dout, void* out, void* dqkv, int B, int L, int heads, int dim_head,
                 float scale, int dtype, void* stream);

/* ---------------------------------------------------------------------------
 * SwinUNETR operators (model/dim3/swin_unetr.py; monai 1.1.0 blocks at its call
 * sites :129-228).  Channels-last tensors.
 *
 * resblock_out: output stage of monai's UnetResBlock,
 *   y = act( IN(r2) + res ),  res = IN(r3) when stats3 != NULL (the block's 1x1
 *   projection branch) else r3 itself; act = B200SEG_ACT_LRELU.
 *   bwd_reduce: g = dy * act'(y) (dense [V][C]) and sums[b][c][3] =
 *   {sum g, sum g*xhat2, sum g*xhat3} for the two InstanceNorm backward passes.
 * window_attn: WindowAttention.forward :467-490 between the qkv and proj Linears,
 *   fused with forward_part1's pad / roll / window_partition / window_reverse
 *   (:554-606), compute_mask (:737-773) and the relative-position-bias gather
 *   (:417-459,473-476).  qkv [B,D,H,W,3*heads*dh] ({q,k,v} x heads x dh), out
 *   [B,D,H,W,heads*dh]; window/shift are the module's nominal int[3] (clamping to
 *   short axes, get_window_size :358-381, happens inside).  qkv_bias (nullable)
 *   stands in for the q/k/v of padding tokens (the reference pads before the qkv
 *   Linear); bwd adds those tokens' gradients to dbias_pad [3*heads*dh] and the
 *   bias-table gradient to dtable [(2w0-1)(2w1-1)(2w2-1)][heads] (both +=).
 *   lse / delta: fp32 buffers of b200seg_window_attn_workspace() bytes.
 * swin_merge: PatchMerging gather, v2 == 0: the v0.9 slice list of :717-727 WITH its
 *   duplicated slices (x5 == x2, x6 == x3), v2 != 0: PatchMergingV2's product order
 *   (:693-695); x [B,D,H,W,C] -> y [B,ceil(D/2),ceil(H/2),ceil(W/2),8C] (odd
 *   extents zero-padded, :714-716); reverse != 0: x is dy, y receives dx.
 * ------------------------------------------------------------------------- */
int b200seg_resblock_out_fwd(const void* r2, int r2_ld, const double* stats2,
                             const void* r3, int r3_ld, int r3_coff, const double* stats3,
                             float eps, int act, void* y, int y_ld,
                             int B, int64_t V, int C, int dtype, void* stream);
int b200seg_resblock_out_bwd_reduce(const void* dy, int dy_ld, const void* y, int y_ld,
                                    const void* r2, int r2_ld, const double* stats2,
                                    const void* r3, int r3_ld, int r3_coff, const double* stats3,
                                    float eps, int act, void* g, double* sums,
                                    int B, int64_t V, int C, int dtype, void* stream);
size_t b200seg_window_attn_workspace(int B, int D, int H, int W, int heads, const int* window);
int b200seg_window_attn_fwd(const void* qkv, const float* qkv_bias, const float* bias_table,
                            void* out, float* lse, int B, int D, int H, int W, int heads, int dh,
                            const int* window, const int* shift, int dtype, void* stream);
int b200seg_window_attn_bwd(const void* qkv, const float* qkv_bias, const float* bias_table,
                            const void* out, const void* dout, const float* lse, float* delta,
                            void* dqkv, float* dtable, float* dbias_pad,
                            int B, int D, int H, int W, int heads, int dh,
                            const int* window, const int* shift, int dtype, void* stream);
int b200seg_swin_merge(const void* x, void* y, int B, int D, int H, int W, int C,
                       int reverse, int v2, int dtype, void* stream);

/* ---------------------------------------------------------------------------
 * UNETR operators (model/dim3/unetr.py; its ViT encoder is monai 1.1.0's).
 *
 * attention: the core of monai's SABlock between its qkv and out_proj Linears,
 *   out = softmax(q k^T * dim_head^-0.5) v per (batch, head) over all L tokens.
 *   qkv [B][L][3*heads*dim_head], channel which*inner + h*dim_head + d (q, k, v);
 *   out [B][L][heads*dim_head], channel h*dim_head + d.  lse: fp32 [B][heads][L]
 *   row log-sum-exp written by fwd and read by bwd; delta: fp32 [B][heads][L]
 *   scratch of bwd.  bwd writes every element of dqkv (same layout as qkv) and is
 *   deterministic.  dim_head must be 64 (else B200SEG_EUNSUPPORTED), any L >= 1;
 *   qkv / out / dout / dqkv 16-byte aligned.
 * ------------------------------------------------------------------------- */
int b200seg_attention_fwd(const void* qkv, void* out, float* lse, int B, int L, int heads, int dim_head,
                          int dtype, void* stream);
int b200seg_attention_bwd(const void* qkv, const void* out, const void* dout, const float* lse, float* delta,
                          void* dqkv, int B, int L, int heads, int dim_head, int dtype, void* stream);

/* ---------------------------------------------------------------------------
 * Optimiser tail (SURVEY.md 8f.1): GradScaler non-finite check + unscale, AdamW
 * (training/utils.py:8-14, eps 1e-5) and the EMA update (training/utils.py:98-105,
 * ema_alpha = this iteration's min(1 - 1/(iter+1), cap), computed by the caller) as
 * multi-tensor kernels over a device table.
 *   table_dev : int64 [ntensors][6] = {grad, param, exp_avg, exp_avg_sq, ema param
 *               (0 = none), numel}; all fp32, contiguous
 *   chunks_dev: int64 [nchunks][2] = {tensor index, first element}; a chunk covers
 *               b200seg_optim_chunk_elems() elements
 * grads_nonfinite raises *found_inf (device float, zeroed by the caller) when any
 * gradient element is inf / nan.  adamw_ema_step applies one AdamW step unless
 * *found_inf != 0 (the EMA update runs either way, as in the reference loop);
 * gradients are divided by *scale (nullable); *step_dev counts the APPLIED steps
 * (bias corrections) and is advanced on device.
 * ------------------------------------------------------------------------- */
int b200seg_optim_chunk_elems(void);
int b200seg_grads_nonfinite(const int64_t* table_dev, const int64_t* chunks_dev, int nchunks,
                            float* found_inf, void* stream);
int b200seg_adamw_ema_step(const int64_t* table_dev, const int64_t* chunks_dev, int nchunks,
                           float lr, float beta1, float beta2, float eps, float weight_decay,
                           float ema_alpha, float* step_dev, const float* scale,
                           const float* found_inf, void* stream);

/* ---------------------------------------------------------------------------
 * Evaluation consumers of net(x) (SURVEY.md 8f.2).
 * softmax_accumulate: sliding-window inference, inference/inference3d.py:77-89:
 *   prob[b][c][d0+d][h0+h][w0+w] += softmax_c(logits[b*sb + v*sv + c*sc]),
 *   counter[b][..] += 1 for the window's wd x wh x ww voxels; prob fp32
 *   [B][C][D][H][W], counter fp32 [B][D][H][W].
 * normalize_argmax: prob /= counter (:91); label (nullable, uint8 [B][V]) = argmax_c.
 * dice_metric: metric/utils.py:62-82, out uint64 [C][2] += {|pred==c & target==c|,
 *   |pred==c| + |target==c|}; label maps uint8 (bytes = 1) or int64 (bytes = 8).
 * ------------------------------------------------------------------------- */
int b200seg_softmax_accumulate(const void* logits, int dtype, int64_t sb, int64_t sv, int64_t sc,
                               float* prob, float* counter, int B, int C, int wd, int wh, int ww,
                               int D, int H, int W, int d0, int h0, int w0, void* stream);
int b200seg_normalize_argmax(float* prob, const float* counter, uint8_t* label, int B, int C,
                             int64_t V, void* stream);
int b200seg_dice_metric(const void* pred, int pred_bytes, const void* target, int target_bytes,
                        int64_t N, int C, unsigned long long* out, void* stream);

/* ---------------------------------------------------------------------------
 * Validation surface distances: metric/utils.py:8-28 (calculate_distance) with the semantics of
 * metric/metrics.py:265-720.  For every class c in 1..C-1 of the label maps gt / pred (uint8 or int64,
 * bytes = 1 / 8, [D][H][W]): asd[c-1] = the mean of the two directed area-weighted average surface distances,
 * hd[c-1] = the larger of the two directed `percent` percentile distances (fp64, device pointers).  A class
 * absent from one or both maps gives nan / inf, as the reference.  table: device fp64 [256] surfel area per
 * neighbour code at spacing (s0, s1, s2) (b200seg.surface.surface_area_table).  Results are bit-identical
 * from run to run.  The call waits for one small device-to-host copy (the per-class bounding boxes).
 * workspace: b200seg_surface_distance_workspace() bytes (0: unsupported size, C > 256).
 * ------------------------------------------------------------------------- */
size_t b200seg_surface_distance_workspace(int D, int H, int W, int C);
int b200seg_surface_distance(const void* pred, int pred_bytes, const void* gt, int gt_bytes, int D, int H, int W,
                             int C, double s0, double s1, double s2, double percent, const double* table,
                             double* asd, double* hd, void* workspace, size_t workspace_bytes, void* stream);

/* ---------------------------------------------------------------------------
 * GPU augmentation (SURVEY.md 8f.3; `aug_device: gpu`, training/augmentation.py, driven per sample by
 * training/dataset/dim3/dataset_kits.py:116-153).  Images are fp32 [C][D][H][W] (the reference's
 * [1,C,D,H,W]); label maps uint8 (bytes = 1) or int64 (bytes = 8).  The small geometry / parameter
 * arrays (`*_dims`, `*_origin`, `theta`, `a`, `b`, `weights`) are HOST pointers read during the call.
 *
 * `stats`: one 32-byte row per statistics row of the reference's `view(tmp_C, -1)` (rows = 1, or C for
 * per_channel): {uint64 min key, uint64 max key, double sum, double sum of squares}; the caller initialises
 * a row to {0xffffffff, 0, 0.0, 0.0}; kernels ACCUMULATE (atomics).  key(f) = bits(f) ^ (sign ? ~0 : 1<<31).
 *
 * aug_resample: crop_3d(random) -> random_scale_rotate_translate_3d -> crop_3d(center) -> mirror x3
 *   (augmentation.py:226-291,320-343,176-197) as one gather.  The affine grid is defined on the sub-volume
 *   [sub_origin, sub_origin + sub_dims) of the source (F.affine_grid / F.grid_sample, align_corners=True,
 *   zeros padding OUTSIDE THE SUB-VOLUME, trilinear image / nearest label); only the patch
 *   [out_origin, out_origin + out_dims) of that grid is produced; flip_mask bit a mirrors output axis a.
 *   theta = the 3x4 matrix handed to F.affine_grid (12 floats, row-major), or NULL for the exact-copy branch.
 *   lab / out_lab may both be NULL; img / out_img may both be NULL with C = 0 (label map only).
 *   stats (nullable) receives the statistics of out_img.
 * aug_pointwise: op 0 brightness_multiply y = x*a[r] (:88-101); 1 brightness_additive y = x + a[r] (:66-85);
 *   2 gamma pow pass y = ((x-min)/rng)^a[r]*rng + min (:123-127, needs stats_in); 3 gamma retain_stats pass
 *   y = (x - mean_in)/std_in*std_in2 + mean_in2 (:129-131; stats_in = after the pow, stats_in2 = before);
 *   4 contrast y = (x-mean)*a[r] + mean, clamped to [min,max] when b[r] != 0 (:136-168);
 *   5 gaussian_noise y = x + N(0,1)*a[r] + b[r] (:14-16; Philox4x32-10 keyed by seed, counter = element / 4);
 *   6 statistics only (y may be NULL).  rows <= 8, n = elements per row; stats_out (nullable) receives the
 *   statistics of y, so a chain of ops never needs a separate reduction pass.
 * aug_gaussian_blur: gaussian_blur (:18-64) with the 1-D weights of the separable kernel (ksize 1..7, odd),
 *   zero padding like F.conv3d(padding = k//2); x != y.
 * ------------------------------------------------------------------------- */
int b200seg_aug_resample(const float* img, const void* lab, int lab_bytes, int C, const int* src_dims,
                         const int* sub_origin, const int* sub_dims, const float* theta,
                         const int* out_origin, const int* out_dims, int flip_mask, float* out_img,
                         void* out_lab, int out_lab_bytes, void* stats, int stats_rows, void* stream);
int b200seg_aug_pointwise(const float* x, float* y, int rows, int64_t n, int op, const float* a,
                          const float* b, const void* stats_in, const void* stats_in2, void* stats_out,
                          uint64_t seed, void* stream);
int b200seg_aug_gaussian_blur(const float* x, float* y, int C, int D, int H, int W, const float* weights,
                              int ksize, void* stats_out, int stats_rows, void* stream);
/* aug_gaussian_blur2d: gaussian_blur on a [1,C,H,W] image (F.conv2d with the normalised k x k kernel, which is
 *   the outer product of the normalised 1-D weights), zero padding k//2; otherwise as aug_gaussian_blur. */
int b200seg_aug_gaussian_blur2d(const float* x, float* y, int C, int H, int W, const float* weights, int ksize,
                                void* stats_out, int stats_rows, void* stream);

/* ---------------------------------------------------------------------------
 * Batched 2-D training branch (training/dataset/dim2/dataset_acdc.py:128-142) for B ragged slices:
 *   y1 = x + noise_std*N(0,1) + beta        gaussian_noise (Philox keyed by noise_key, counter = element / 4,
 *                                           the stream aug_pointwise op 5 draws) and brightness_additive
 *   y2 = ((y1 - min1)/rng1)^gamma*rng1 + min1,  y3 = (y2 - mean2)/std2*std1 + mean1
 *                                           gamma(retain_stats=True); statistics of the whole slice, std unbiased
 *   random_scale_rotate_translate_2d with the 2x3 theta (F.affine_grid / F.grid_sample over the whole H x W slice,
 *   align_corners=True, bilinear image / nearest label, zeros padding), of which only the h x w crop at
 *   (crop_y, crop_x) is produced (crop_2d).
 * rows: DEVICE array of B b200seg_aug2d_row (88 bytes each).  img fp32 [H][W]; lab uint8 (lab_bytes = 1) or
 * int64 (8) [H][W]; y1 (nullable) receives y1, [H][W] fp32.  max_elems >= every H*W.  out_img fp32 [B][h][w],
 * out_lab int64 [B][h][w].  Three launches whatever B; statistics stay on the device, reduced in a fixed order
 * without atomics, so a given table always gives the same bits.
 * workspace: b200seg_aug2d_workspace(B, max_elems) bytes of device memory.
 * ------------------------------------------------------------------------- */
typedef struct {
  const float* img;
  const void* lab;
  float* y1;
  int H, W;
  uint64_t noise_key;
  float noise_std, beta, gamma;
  float theta[6];          /* row-major 2x3, as handed to F.affine_grid */
  int crop_y, crop_x;
  int reserved;
} b200seg_aug2d_row;
size_t b200seg_aug2d_workspace(int B, int64_t max_elems);
int b200seg_aug2d_train(const void* rows, int B, int64_t max_elems, int lab_bytes, int h, int w, float* out_img,
                        int64_t* out_lab, void* workspace, size_t workspace_bytes, void* stream);

/* ---------------------------------------------------------------------------
 * Attention-UNet gate (SURVEY.md 8f.4), model/dim3/attention_unet_utils.py:7-37.  With
 * t = relu(IN(W_g g) + IN(W_x x)) already formed (conv3d_fwd x2 + resblock_out_fwd, act = RELU):
 * attn_gate_fwd:  p[b][v] = sum_c w[c] t[b][v][c]          (`psi` Conv3d(int_ch, 1, 1, bias=False), :20)
 *                 pstats[b] += {sum p, sum p^2}              (InstanceNorm3d(1), :21, eps = 1e-5)
 *                 out[b][v][o_coff + c] = x[b][v][x_coff + c] * sigmoid(IN(p)[b][v])     (:22,37)
 *                 ostats[b][c] += {sum, sumsq} of out (nullable; the next conv's loader normalises with them)
 *   t [B][V][Ct] (leading dimension t_ld), w fp32 [Ct], p fp32 [B][V]; Ct, Cx multiples of 8.
 * attn_gate_bwd:  dx = dout * psi (dense [B][V][Cx]); dt = dp * w (dense [B][V][Ct], before t's ReLU mask, which
 *   resblock_out_bwd_reduce applies); dw[c] += sum dp * t; dz fp32 [B][V] and bsums double [B][2] are scratch
 *   (bsums zeroed by the caller, like pstats / ostats / dw).
 * ------------------------------------------------------------------------- */
int b200seg_attn_gate_fwd(const void* t, int t_ld, const float* w, const void* x, int x_ld, int x_coff,
                          float eps, float* p, double* pstats, void* out, int o_ld, int o_coff,
                          double* ostats, int B, int64_t V, int Ct, int Cx, int dtype, void* stream);
int b200seg_attn_gate_bwd(const void* dout, int d_ld, int d_coff, const void* x, int x_ld, int x_coff,
                          const void* t, int t_ld, const float* w, const float* p, const double* pstats,
                          float eps, void* dx, void* dt, float* dw, float* dz, double* bsums, int B,
                          int64_t V, int Ct, int Cx, int dtype, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* B200SEG_H */
