/*
 * b200gan.h -- C ABI of libb200gan.so: the sm_90a implementation of the
 * Generator/Discriminator hot path of eriklindernoren/PyTorch-GAN.
 *
 * The reference has no FFI of its own: its operator boundary is the torch.nn.Module
 * protocol (SURVEY.md section 8b).  Each entry point below replaces the arithmetic that one
 * reference call site hands to third-party torch; the reference file:line is cited per
 * function.  All signatures are plain C: raw device pointers, sizes, a cudaStream_t passed
 * as void*.  No torch types cross this boundary.
 *
 * Conventions
 *   - Activations are fp32, NHWC ("channels_last"), dense: x[n][h][w][c].
 *   - Weight parameters stay in PyTorch's external layout (Conv2d: OIHW, ConvTranspose2d:
 *     IOHW) so state_dict keys/shapes are unchanged (pix2pix.py:71-72, cyclegan.py:75-78);
 *     packed copies are derived caches produced by b200gan_pack_weights().
 *   - Every launch is asynchronous on the given stream; nothing allocates or frees device
 *     memory; nothing synchronises the host.  All buffers are caller-owned.
 *   - Return value: 0 = OK, negative = B200GAN_E_*; b200gan_last_error() gives the text
 *     (thread-local).  There is no CPU fallback anywhere in this library.
 */
#ifndef B200GAN_H
#define B200GAN_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B200GAN_VERSION 100

enum {
  B200GAN_OK = 0,
  B200GAN_E_UNSUPPORTED = -1, /* geometry not supported by the requested algorithm */
  B200GAN_E_BAD_ARG = -2,     /* null pointer, misalignment, inconsistent sizes */
  B200GAN_E_CUDA = -3,        /* a CUDA runtime/driver call failed */
  B200GAN_E_ARCH = -4         /* device is not sm_90 */
};

/* activation fused into an epilogue / applied by a norm kernel */
enum { B200GAN_ACT_NONE = 0, B200GAN_ACT_LRELU = 1, B200GAN_ACT_RELU = 2, B200GAN_ACT_TANH = 3,
       B200GAN_ACT_SIGMOID = 4 };

/* algorithm selector for the convolution entry points */
enum { B200GAN_ALGO_AUTO = 0, /* wgmma TF32 when the geometry qualifies, else SIMT */
       B200GAN_ALGO_SIMT = 1, /* fp32 FFMA implicit GEMM (any geometry) */
       B200GAN_ALGO_TC = 2 }; /* wgmma TF32 implicit GEMM (error if unsupported) */

/* padding mode of the (virtual) padded input */
enum { B200GAN_PAD_ZERO = 0, B200GAN_PAD_REFLECT = 1 };

/* packed-weight layouts produced by b200gan_pack_weights() */
enum {
  B200GAN_PACK_SIMT_FPROP = 0, /* [R][S][Cin][Cout]   : fprop (Conv2d and ConvTranspose2d), SIMT */
  B200GAN_PACK_SIMT_DGRAD = 1, /* [R][S][Cout][Cin]   : dgrad (Conv2d and ConvTranspose2d), SIMT */
  B200GAN_PACK_TC_FPROP = 2,   /* [R*S][Cout][Cin]    tf32-rounded, K-major, wgmma fprop      */
  B200GAN_PACK_TC_DGRAD = 3,   /* [R*S][Cin][Cout]    tf32-rounded, taps in filter order (the
                                  scatter form's tap offsets do the flip), dgrad               */
  B200GAN_PACK_TC_FPROP_UP2 = 4, /* [4 phases][4 taps][Cout][Cin]: 3x3 s1 p1 conv folded with a
                                    preceding nearest x2 upsample into four 2x2 phase filters  */
  B200GAN_PACK_TC_DGRAD_UP2 = 5  /* [4 phases][4 taps][Cin][Cout]: its data gradient           */
};

/*
 * Geometry of one convolution call site.  Replaces the constructor arguments of
 *   nn.Conv2d           dcgan.py:55,59,62,78  pix2pix/models.py:23,79,115,127
 *                       cyclegan/models.py:28,32,50,60,75,82,106,118
 *   nn.ConvTranspose2d  pix2pix/models.py:39
 * optionally composed with the shape-only modules the reference places directly in front:
 *   nn.Upsample(scale_factor=2)   dcgan.py:54,58  cyclegan/models.py:74  pix2pix/models.py:77
 *   nn.ZeroPad2d((1,0,1,0))       pix2pix/models.py:78,126   cyclegan/models.py:117
 *   nn.ReflectionPad2d(k)         cyclegan/models.py:27,31,49,81
 * The "virtual input" is  pad(upsample(x)): size (H*up + pad_t + pad_b) x (W*up + pad_l + pad_r).
 */
typedef struct b200gan_conv_geom {
  int32_t N, H, W, C;  /* stored input tensor (before upsample / padding), NHWC          */
  int32_t K;           /* output channels                                                  */
  int32_t R, S;        /* filter height, width                                             */
  int32_t stride;      /* same in h and w                                                  */
  int32_t pad_t, pad_l, pad_b, pad_r; /* total padding of the virtual input (conv padding +
                                         any folded ZeroPad2d / ReflectionPad2d)           */
  int32_t pad_mode;    /* B200GAN_PAD_*                                                    */
  int32_t up;          /* 1, or 2 = nearest-neighbour x2 upsample folded in front          */
  int32_t transposed;  /* 0 = Conv2d, 1 = ConvTranspose2d (pad_* = its `padding`, up == 1) */
  int32_t P, Q;        /* output height, width (checked against the other fields)          */
} b200gan_conv_geom;

/* Epilogue fused into fprop:  y = chan_scale[n,k] * act(conv + bias[k])  (each part optional).
 * stats (optional) receives, atomically accumulated in fp64, the per-group sums of y and y*y
 * that the following BatchNorm2d / InstanceNorm2d needs: stats[0..G) = sum, stats[G..2G) =
 * sum of squares, G = K (stats_per_sample == 0) or N*K (== 1).  Caller zeroes it.  Both kinds
 * are produced for every algorithm and tiling: where the kernel cannot fuse them (e.g. a wgmma
 * tile that spans two images) the library adds one b200gan_norm_stats pass on the same stream. */
typedef struct b200gan_epilogue {
  const float *bias;       /* [K] or NULL                                                  */
  int32_t act;             /* B200GAN_ACT_*                                                */
  float slope;             /* LeakyReLU negative slope                                     */
  const float *chan_scale; /* [N][K] Dropout2d keep-mask / (1-p)  (dcgan.py:77) or NULL    */
  double *stats;           /* [2][G] or NULL                                               */
  int32_t stats_per_sample;
  int32_t round_tf32;      /* store y rounded to TF32 (RN) so that a following wgmma conv
                              consumes exactly-representable operands                      */
} b200gan_epilogue;

int b200gan_version(void);
const char *b200gan_last_error(void);
/* 0 if the current device is sm_90 and the wgmma/TMA paths can run, else B200GAN_E_ARCH */
int b200gan_check_device(void);

/* ---- weights ------------------------------------------------------------------------ */
size_t b200gan_packed_weight_floats(const b200gan_conv_geom *g, int pack);
/* w: the nn.Parameter storage (Conv2d [K][C][R][S]; ConvTranspose2d [C][K][R][S]). */
int b200gan_pack_weights(const b200gan_conv_geom *g, int pack, const float *w, float *packed,
                         void *stream);

/* Every packed copy of an optimizer's weights in ONE launch (the job table travels as a kernel argument): called by
 * b200gan.optim.Adam right after the parameter update, so a training step carries 2 pack launches instead of ~20. */
typedef struct b200gan_pack_job {
  const float *w;
  float *packed;
  b200gan_conv_geom geom;
  int32_t pack; /* B200GAN_PACK_* */
} b200gan_pack_job;
int b200gan_pack_weights_multi(const b200gan_pack_job *jobs, int32_t count, void *stream);

/* ---- convolution: forward, data gradient, weight gradient ---------------------------- */
/* 1 if algo (B200GAN_ALGO_TC) supports this geometry for the given pass (0 fprop,1 dgrad,2 wgrad) */
int b200gan_conv2d_supported(const b200gan_conv_geom *g, int pass, int algo);

/* y[N][P][Q][K] = epilogue(conv(x, w)).  `packed` must be the layout the algorithm wants:
 * SIMT: PACK_SIMT_FPROP (Conv2d and ConvTranspose2d alike);
 * TC  : PACK_TC_FPROP, or PACK_TC_FPROP_UP2 when g->up == 2.
 * Replaces cudnnConvolutionForward behind nn.Conv2d.forward (dcgan.py:69,95). */
int b200gan_conv2d_fprop(const b200gan_conv_geom *g, const b200gan_epilogue *ep, const float *x,
                         const float *packed, float *y, int algo, void *stream);

/* dx[N][H][W][C] = d(loss)/dx given dy[N][P][Q][K] (gradient w.r.t. the pre-epilogue conv
 * output, i.e. after the caller applied act'/mask).  For up == 2 or reflect padding the SIMT
 * path needs `workspace` of b200gan_conv2d_dgrad_workspace_floats() floats.
 * Replaces cudnnConvolutionBackwardData behind autograd of nn.Conv2d (dcgan.py:168,182). */
size_t b200gan_conv2d_dgrad_workspace_floats(const b200gan_conv_geom *g, int algo);
int b200gan_conv2d_dgrad(const b200gan_conv_geom *g, const float *dy, const float *packed,
                         float *dx, float *workspace, int algo, void *stream);

/* dw (parameter layout: Conv2d [K][C][R][S], ConvTranspose2d [C][K][R][S]) and db[K] (or NULL).
 * dw/db are OVERWRITTEN.  workspace: b200gan_conv2d_wgrad_workspace_floats() floats.
 * Replaces cudnnConvolutionBackwardFilter (dcgan.py:168,182). */
size_t b200gan_conv2d_wgrad_workspace_floats(const b200gan_conv_geom *g, int algo);
int b200gan_conv2d_wgrad(const b200gan_conv_geom *g, const float *x, const float *dy, float *dw,
                         float *db, float *workspace, int algo, void *stream);
/* The same, except that on the tensor-core route of a Conv2d db is summed by the weight-gradient kernel from the dy
 * values it already holds, instead of by a separate pass over dy (the other routes and ConvTranspose2d: as above). */
int b200gan_conv2d_wgrad_fused_bias(const b200gan_conv_geom *g, const float *x, const float *dy, float *dw,
                                    float *db, float *workspace, int algo, void *stream);

/* dz = dy * act'(y) * chan_scale  -- backward of the fused fprop epilogue, from the saved
 * output y (LeakyReLU/ReLU sign and Tanh/Sigmoid derivative are functions of y).
 * n = N*P*Q*K elements, K channels, PQ pixels per sample (for chan_scale indexing). */
int b200gan_epilogue_bwd(const float *dy, const float *y, const float *chan_scale, int32_t act,
                         float slope, int64_t n, int32_t K, int64_t PQ, int32_t round_tf32,
                         float *dz, void *stream);

/* db[k] = sum over (n,p,q) of dy * act'(y) * chan_scale -- the bias gradient of a fused conv block computed from
 * UNROUNDED values (when dz is TF32-rounded for the tensor-core dgrad/wgrad, summing the rounded values loses the
 * cancellation a bias gradient lives on).  db is overwritten. */
int b200gan_bias_grad(const float *dy, const float *y, const float *chan_scale, int32_t act, float slope,
                      int64_t rows, int32_t K, int64_t PQ, float *db, void *stream);

/* ---- BatchNorm2d (training) / InstanceNorm2d ------------------------------------------ */
/* Normalisation over groups: G = C (per_sample == 0: BatchNorm2d, dcgan.py:53,56,60,80) or
 * N*C (per_sample == 1: InstanceNorm2d, pix2pix/models.py:25,40,117, cyclegan/models.py:29...). */
typedef struct b200gan_norm_desc {
  int32_t N, HW, C;
  int32_t per_sample;
  float eps;      /* dcgan.py:56 passes 0.8 here (second positional arg of BatchNorm2d)         */
  float momentum; /* running-stat momentum (BatchNorm2d only)                                  */
  int32_t act;    /* activation fused after the affine transform                               */
  float slope;
  int32_t round_tf32;
} b200gan_norm_desc;

/* stats[2][G] (fp64, zeroed by the caller) += (sum x, sum x^2).  Skip when the producing conv
 * already accumulated them in its epilogue. */
int b200gan_norm_stats(const b200gan_norm_desc *d, const float *x, double *stats, void *stream);
/* From stats: mean_rstd[2][G]; scale_shift[2][G] (= gamma*rstd, beta-mean*gamma*rstd; gamma,
 * beta may be NULL = 1,0); running_mean/var (may be NULL) updated with the UNBIASED variance,
 * num_batches_tracked (int64, may be NULL) += 1 -- torch.nn.BatchNorm2d semantics.
 * `stats` is CONSUMED: it is zeroed on return, so a persistent accumulator never needs a memset. */
int b200gan_norm_finalize(const b200gan_norm_desc *d, double *stats, const float *gamma,
                          const float *beta, float *mean_rstd, float *scale_shift,
                          float *running_mean, float *running_var, int64_t *num_batches_tracked,
                          void *stream);
/* y = act(x * scale + shift); may run in place (y == x). */
int b200gan_norm_apply(const b200gan_norm_desc *d, const float *x, const float *scale_shift,
                       float *y, void *stream);
/* Backward.  Inputs: dy, saved input x, mean_rstd, gamma (or NULL), and scale_shift (or NULL).  With scale_shift
 * a LeakyReLU / ReLU mask is recomputed from x; the saved output y is required only for Tanh / Sigmoid, or for
 * LeakyReLU / ReLU when scale_shift is NULL (otherwise y may be NULL).
 * sums[2][G] fp64 workspace: zero on entry, handed back zeroed.
 * Outputs: dx; dgamma_dbeta[2][G] (only meaningful for per_sample == 0 with affine; may be NULL). */
int b200gan_norm_bwd(const b200gan_norm_desc *d, const float *dy, const float *x, const float *y,
                     const float *mean_rstd, const float *scale_shift, const float *gamma, double *sums, float *dx,
                     float *dgamma_dbeta, void *stream);

/* Double backward of b200gan_norm_bwd (gradient penalties through a training-mode norm): given u = dL/d(dx) and
 * ugamma_ubeta[2][C] = dL/d(dgamma), dL/d(dbeta) per channel (NULL = 0), writes gx = dL/dx, gdy = dL/d(dy) and
 * ggamma_per_group[G] = dL/dgamma per group (summed over samples by the caller for InstanceNorm); any of the three may
 * be NULL.  The mean and rstd are the batch statistics of x, so gx includes their dependence on x.  act NONE, or LRELU /
 * RELU with scale_shift (the mask is piecewise constant: no second-order term); TANH / SIGMOID give
 * B200GAN_E_UNSUPPORTED.  sums: fp64 [5][G] workspace, zero on entry, handed back zeroed.  No host synchronisation. */
int b200gan_norm_dbwd(const b200gan_norm_desc *d, const float *dy, const float *x, const float *mean_rstd,
                      const float *scale_shift, const float *gamma, const float *u, const float *ugamma_ubeta,
                      double *sums, float *gx, float *gdy, float *ggamma_per_group, void *stream);

/* ---- BatchNorm2d [-> LeakyReLU / ReLU] [-> Upsample x2] -> Conv2d backward (dcgan.py:53-55,56-59) ------------------ */
/* The conv's data gradient dx as b200gan_conv2d_dgrad (ALGO_TC, packed PACK_TC_DGRAD[_UP2]) writes it, bit for bit, and
 * in the same epilogue the sums the norm backward needs: sums[0..C) += sum dy', sums[C..2C) += sum dy' * xhat, with
 * dy' = dx * act'(x * scale + shift) and xhat = (x - mean) * rstd.  x: the norm input [N][H][W][C] (the conv's input
 * grid); d: the norm (per_sample 0, act NONE / LRELU / RELU); mean_rstd, scale_shift from b200gan_norm_finalize.  sums:
 * fp64 [2][C], zero on entry.  B200GAN_E_UNSUPPORTED unless b200gan_conv2d_dgrad_norm_supported(g): Conv2d, stride 1,
 * zero padding, up 1 or 2, a tensor-core data gradient whose contraction is not split over CTAs. */
int b200gan_conv2d_dgrad_norm_supported(const b200gan_conv_geom *g);
int b200gan_conv2d_dgrad_norm(const b200gan_conv_geom *g, const b200gan_norm_desc *d, const float *dy,
                              const float *packed, const float *x, const float *mean_rstd, const float *scale_shift,
                              double *sums, float *dx, void *stream);
/* The rest of b200gan_norm_bwd once `sums` holds what its reduction would have produced (b200gan_conv2d_dgrad_norm):
 * dx and dgamma_dbeta; act NONE, or LRELU / RELU with scale_shift.  sums is handed back zeroed. */
int b200gan_norm_bwd_from_sums(const b200gan_norm_desc *d, const float *dy, const float *x, const float *mean_rstd,
                               const float *scale_shift, const float *gamma, double *sums, float *dx,
                               float *dgamma_dbeta, void *stream);

/* ---- Generator tail: BatchNorm2d -> LeakyReLU/ReLU -> Conv2d(C, K<=3, 3, 1, 1) -> Tanh, fused -------------- */
/* Replaces the module run dcgan.py:60-63
 *     nn.BatchNorm2d(64, 0.8), nn.LeakyReLU(0.2, inplace=True), nn.Conv2d(64, opt.channels, 3, stride=1, padding=1), nn.Tanh()
 * acting on `a`, the raw output of the preceding convolution: the normalised/activated tensor, its gradient and the
 * conv's data gradient are never written to memory (csrc/tail.cu).  scale_shift / mean_rstd come from
 * b200gan_norm_finalize (batch statistics of `a`).  Supported: C in {32, 64, 128}, K in 1..3, W a power of two in
 * [16, 128], act_mid in {NONE, LRELU, RELU}. */
typedef struct b200gan_tail_desc {
  int32_t N, H, W, C; /* a: [N][H][W][C] */
  int32_t K;          /* conv output channels; the conv is 3x3, stride 1, zero padding 1 */
  int32_t act_mid;    /* activation between the norm and the conv */
  float slope;
  int32_t act_out;    /* activation after the conv (+bias) */
} b200gan_tail_desc;
int b200gan_tail_supported(const b200gan_tail_desc *d);
/* out[N][H][W][K] = act_out(conv3x3(act_mid(a * scale + shift), w) + bias); w: the Conv2d parameter [K][C][3][3].
 * The convolution runs on wgmma (TF32). */
int b200gan_tail_fprop(const b200gan_tail_desc *d, const float *a, const float *scale_shift, const float *w,
                       const float *bias, float *out, void *stream);
/* Backward of the same composite given g = d(loss)/d(conv output before act_out) [N][H][W][K]:
 *   da[N][H][W][C]  gradient w.r.t. `a` through conv, activation and the training-mode BatchNorm
 *   dgamma_dbeta[2][C] (may be NULL), dw[K][C][3][3], db[K] (may be NULL) -- all OVERWRITTEN.
 * workspace: b200gan_tail_bwd_workspace_bytes() bytes, 16-byte aligned (zeroed by the call). */
size_t b200gan_tail_bwd_workspace_bytes(const b200gan_tail_desc *d);
int b200gan_tail_bwd(const b200gan_tail_desc *d, const float *a, const float *mean_rstd, const float *scale_shift,
                     const float *w, const float *g, void *workspace, float *da, float *dgamma_dbeta, float *dw,
                     float *db, int32_t round_tf32, void *stream);

/* ---- shape / index ops (bit-exact) ---------------------------------------------------- */
/* NCHW <-> NHWC transposes of a dense fp32 tensor. */
int b200gan_nchw_to_nhwc(const float *x, float *y, int32_t N, int32_t C, int32_t HW, void *stream);
int b200gan_nhwc_to_nchw(const float *x, float *y, int32_t N, int32_t C, int32_t HW, void *stream);
/* Stand-alone versions of the modules that are normally folded into a conv:
 * nearest x2 upsample and its gradient (sum over the 2x2 replicas), NHWC. */
int b200gan_upsample2x_fwd(const float *x, float *y, int32_t N, int32_t H, int32_t W, int32_t C,
                           void *stream);
int b200gan_upsample2x_bwd(const float *dy, float *dx, int32_t N, int32_t H, int32_t W, int32_t C,
                           void *stream);
/* Constant-zero or reflection padding and its gradient (crop / fold), NHWC. */
/* round_tf32: store RN-rounded TF32 values (the padded copy feeds a wgmma conv) */
int b200gan_pad2d_fwd(const float *x, float *y, int32_t N, int32_t H, int32_t W, int32_t C,
                      int32_t pad_t, int32_t pad_l, int32_t pad_b, int32_t pad_r, int32_t mode,
                      int32_t round_tf32, void *stream);
int b200gan_pad2d_bwd(const float *dy, float *dx, int32_t N, int32_t H, int32_t W, int32_t C,
                      int32_t pad_t, int32_t pad_l, int32_t pad_b, int32_t pad_r, int32_t mode,
                      void *stream);
/* Element-wise activation (optionally times a per-element or per-(n,c) mask) and backward. */
int b200gan_act_fwd(const float *x, const float *mask, int32_t mask_per_channel, int32_t act,
                    float slope, int64_t n, int32_t C, int64_t HW, float *y, void *stream);

/* ---- MLP critic: forward, backward, double backward of the input gradient; WGAN-GP critic step */
/* The same critic D(x) = W3 lrelu(W2 lrelu(W1 x + b1) + b2) + b3, Din -> H1 -> H2 -> 1, one LeakyReLU
 * slope for both activations, as three generic passes with no penalty built in, so that a script's own
 * autograd.grad(create_graph=True) penalty (wgan_gp.py:125-137, wgan_div.py:143-163) runs every critic GEMM
 * here (csrc/mlp_critic.cu).  Each is ONE cooperative launch; any N, Din, H1, H2 >= 1; all outputs are
 * OVERWRITTEN, never accumulated.  Weights in torch layout: W1[H1][Din], W2[H2][H1], W3[H2], b3[1]. */
typedef struct b200gan_mlp_critic_desc {
  int32_t N, Din, H1, H2;
  float slope;
} b200gan_mlp_critic_desc;
/* Forward, x[N][Din]:
 *   h1 = x W1^T + b1,  m1 = (h1 > 0 ? 1 : slope),  a1 = h1 * m1          m1, a1: [N][H1]
 *   h2 = a1 W2^T + b2, m2 = (h2 > 0 ? 1 : slope),  a2 = h2 * m2          m2, a2: [N][H2]
 *   out[n] = a2[n] . W3 + b3
 * m1, a1, m2, a2 are kept for the two backward passes.  No workspace. */
int b200gan_mlp_critic_fwd(const b200gan_mlp_critic_desc *d, const float *x, const float *W1,
                           const float *b1, const float *W2, const float *b2, const float *W3,
                           const float *b3, float *out, float *m1, float *a1, float *m2, float *a2,
                           void *stream);
/* First-order backward for the output gradient dout[N]:
 *   U2 = dout W3 * m2  [N][H2],   U1 = (U2 W2) * m1  [N][H1],   dx = U1 W1  [N][Din]
 *   dW1 = U1^T x,  dW2 = U2^T a1,  dW3 = dout^T a2,  db1 = sum_n U1,  db2 = sum_n U2,  db3 = sum_n dout.
 * Every output (dx, dW1, db1, dW2, db2, dW3, db3) may be NULL and is then not computed; x, a1, a2 and W1
 * are read only for dW1, dW2, dW3 and dx respectively and may otherwise be NULL.  U1, U2: written when
 * non-NULL (the double backward needs them); when either is NULL `workspace` must hold
 * b200gan_mlp_critic_bwd_workspace_floats() floats. */
size_t b200gan_mlp_critic_bwd_workspace_floats(const b200gan_mlp_critic_desc *d);
int b200gan_mlp_critic_bwd(const b200gan_mlp_critic_desc *d, const float *dout, const float *x,
                           const float *W1, const float *W2, const float *W3, const float *m1,
                           const float *a1, const float *m2, const float *a2, float *dx, float *dW1,
                           float *db1, float *dW2, float *db2, float *dW3, float *db3, float *U1,
                           float *U2, float *workspace, void *stream);
/* Double backward of dx = U1 W1 for the gradient u[N][Din] arriving at dx.  The masks are piecewise
 * constant (LeakyReLU'' = 0 almost everywhere), so:
 *   dW1 = U1^T u;   t = (u W1^T) * m1;   dW2 = U2^T t;   s = (t W2^T) * m2;
 *   dW3 = sum_n dout_n s_n;   ddout[n] = s_n . W3   (the gradient w.r.t. dout).
 * The gradients w.r.t. x and the biases are exactly zero and not produced.  dW1, dW2, dW3, ddout may be
 * NULL (not computed).  workspace: b200gan_mlp_critic_dbwd_workspace_floats() floats. */
size_t b200gan_mlp_critic_dbwd_workspace_floats(const b200gan_mlp_critic_desc *d);
int b200gan_mlp_critic_dbwd(const b200gan_mlp_critic_desc *d, const float *u, const float *dout,
                            const float *U1, const float *U2, const float *m1, const float *m2,
                            const float *W1, const float *W2, const float *W3, float *dW1, float *dW2,
                            float *dW3, float *ddout, float *workspace, void *stream);
/* The whole WGAN-GP critic iteration of wgan_gp.py:164-173 for this critic in ONE cooperative kernel:
 *   losses[0] = -mean(D(real)) + mean(D(fake)) + lambda_gp * gp,   losses[1] = lambda_gp * gp,
 *   gp = mean_n (||dD/dx_n||_2 - 1)^2 at the interpolates x = alpha * real + (1 - alpha) * fake, formed inside
 * (alpha [N], wgan_gp.py:122-137), and the gradient of losses[0] w.r.t. every parameter of D (all OVERWRITTEN): the
 * first-order backward of the real / fake passes and the closed-form double backward of the penalty share their GEMMs.
 * real, fake: [N][Din].  workspace: b200gan_critic_step_workspace_floats() floats. */
size_t b200gan_critic_step_workspace_floats(const b200gan_mlp_critic_desc *d);
int b200gan_critic_step_mlp(const b200gan_mlp_critic_desc *d, float lambda_gp, const float *real, const float *fake,
                            const float *alpha, const float *W1, const float *b1, const float *W2, const float *b2,
                            const float *W3, const float *b3, float *losses, float *dW1, float *db1, float *dW2,
                            float *db2, float *dW3, float *db3, float *workspace, void *stream);
/* The vanilla GAN discriminator (gan.py:64-80, bgan.py:66-80, aae.py:90-104): the same critic followed by a Sigmoid,
 *   y[n] = 1 / (1 + exp(-(a2[n] . W3 + b3))),
 * on the same two kernels as b200gan_mlp_critic_fwd / _bwd (one cooperative launch each).  The forward writes y[N] in
 * place of out and keeps m1, a1, m2, a2 as the critic forward does.  The backward first forms the gradient at the
 * logits, g[n] = dout[n] y[n] (1 - y[n]) (torch's sigmoid backward), then runs the critic backward for g; its outputs
 * and their NULL rules are those of b200gan_mlp_critic_bwd.  workspace: b200gan_mlp_disc_bwd_workspace_floats()
 * floats (U1, U2 and g). */
int b200gan_mlp_disc_fwd(const b200gan_mlp_critic_desc *d, const float *x, const float *W1, const float *b1,
                         const float *W2, const float *b2, const float *W3, const float *b3, float *y, float *m1,
                         float *a1, float *m2, float *a2, void *stream);
size_t b200gan_mlp_disc_bwd_workspace_floats(const b200gan_mlp_critic_desc *d);
int b200gan_mlp_disc_bwd(const b200gan_mlp_critic_desc *d, const float *dout, const float *y, const float *x,
                         const float *W1, const float *W2, const float *W3, const float *m1, const float *a1,
                         const float *m2, const float *a2, float *dx, float *dW1, float *db1, float *dW2, float *db2,
                         float *dW3, float *db3, float *workspace, void *stream);

/* ---- MLP generator: forward and backward (csrc/mlp_generator/mlp_generator.cu) ------------------------------------ */
/* The MLP generator of wgan_gp.py:42-65 / gan.py:38-61 (Linear weights W[l][width[l+1]][width[l]], biases b[l]):
 *   a_{-1} = z [N][width[0]]
 *   h_l = a_{l-1} W_l^T + b_l;  y_l = BatchNorm1d_l(h_l) when has_norm[l], else h_l;  a_l = lrelu(y_l)     l < L - 1
 *   out = tanh(a_{L-2} W_{L-1}^T + b_{L-1})                                                  [N][width[L]]
 * BatchNorm1d in training mode: batch mean and biased variance, y = gamma (h - mean) / sqrt(var + eps) + beta; the
 * running statistics (when the three pointers are non-NULL) are updated on the device with torch's rule,
 *   running_mean = (1 - momentum) running_mean + momentum mean,
 *   running_var  = (1 - momentum) running_var  + momentum var N / (N - 1),   num_batches_tracked += 1,
 * so a call can be captured in a CUDA graph.  One LeakyReLU slope >= 0, one eps and one momentum for every layer.
 * Each call is ONE cooperative launch of 32 x 32 fp32 FFMA tiles; every output element and column sum is formed in a
 * fixed order, so results are bit-identical from call to call and do not depend on the grid size.
 * Limits: 1 <= L <= B200GAN_MLP_GEN_MAX_LAYERS; 1 <= width <= B200GAN_MLP_GEN_MAX_WIDTH; 1 <= N <=
 * B200GAN_MLP_GEN_MAX_N, and N >= 2 when a layer has a norm (torch refuses one value per channel in training).  The
 * column statistics run one thread per column over all N rows, which bounds N; the reference sizes are N 64 with
 * widths 100 -> 128 -> 256 -> 512 -> 1024 -> 1024 (wgan_gp.py, 32 x 32) or -> 784 (gan.py, 28 x 28). */
#define B200GAN_MLP_GEN_MAX_LAYERS 8
#define B200GAN_MLP_GEN_MAX_WIDTH 8192
#define B200GAN_MLP_GEN_MAX_N 8192
typedef struct b200gan_mlp_gen_desc {
  int32_t L, N;
  int32_t width[B200GAN_MLP_GEN_MAX_LAYERS + 1];
  int32_t has_norm[B200GAN_MLP_GEN_MAX_LAYERS];    /* only l < L - 1 may be set */
  float slope, eps, momentum;
  const float *W[B200GAN_MLP_GEN_MAX_LAYERS], *b[B200GAN_MLP_GEN_MAX_LAYERS];
  const float *gamma[B200GAN_MLP_GEN_MAX_LAYERS], *beta[B200GAN_MLP_GEN_MAX_LAYERS];  /* norm layers: non-NULL */
  float *running_mean[B200GAN_MLP_GEN_MAX_LAYERS], *running_var[B200GAN_MLP_GEN_MAX_LAYERS];
  int64_t *num_batches_tracked[B200GAN_MLP_GEN_MAX_LAYERS];
} b200gan_mlp_gen_desc;
/* Gradients of the backward, all OVERWRITTEN; each may be NULL and is then not computed (norm layers only for dgamma
 * and dbeta). */
typedef struct b200gan_mlp_gen_grads {
  float *dW[B200GAN_MLP_GEN_MAX_LAYERS], *db[B200GAN_MLP_GEN_MAX_LAYERS];
  float *dgamma[B200GAN_MLP_GEN_MAX_LAYERS], *dbeta[B200GAN_MLP_GEN_MAX_LAYERS];
} b200gan_mlp_gen_grads;
/* What the backward reads from the forward, in this order: a_l [N][width[l+1]] for l < L - 1, then for each norm layer
 * xhat_l = (h_l - mean) / sqrt(var + eps) [N][width[l+1]], then for each norm layer 1 / sqrt(var + eps) [width[l+1]]. */
size_t b200gan_mlp_gen_saved_floats(const b200gan_mlp_gen_desc *d);
/* Scratch of both passes: 3 N max(width[1..L]) floats. */
size_t b200gan_mlp_gen_workspace_floats(const b200gan_mlp_gen_desc *d);
/* out [N][width[L]].  saved: b200gan_mlp_gen_saved_floats() floats for a later backward, or NULL (a forward under
 * torch.no_grad(): only out and the running statistics are written). */
int b200gan_mlp_gen_fwd(const b200gan_mlp_gen_desc *d, const float *z, float *out, float *saved, float *workspace,
                        void *stream);
/* Backward for the output gradient dout [N][width[L]], from z, the forward's out and saved; dz [N][width[0]] may be
 * NULL. */
int b200gan_mlp_gen_bwd(const b200gan_mlp_gen_desc *d, const float *dout, const float *z, const float *out,
                        const float *saved, float *dz, const b200gan_mlp_gen_grads *grads, float *workspace,
                        void *stream);

/* ---- Discriminator conv blocks as a fused chain (csrc/narrow_block.cu) -------------------------------------------- */
/* Replaces, for the narrow strided layers of dcgan.py:77-88
 *     [nn.Conv2d(in, out, 3, 2, 1), nn.LeakyReLU(0.2, inplace=True), nn.Dropout2d(0.25), nn.BatchNorm2d(out, 0.8)] x 4
 * every kernel between two convolutions: a layer stores a_l = dropout(lrelu(conv_l(x_l) + b_l)) and the batch sums of
 * a_l; the normalised tensor x_{l+1} = BN_l(a_l) is applied while the consumer gathers its operands and is never
 * written.  A BatchNorm seen from these kernels is the raw batch statistics plus its parameters: */
typedef struct b200gan_nb_bn {
  const double *stats; /* [groups][2][C] sum, sum of squares of the normalised tensor over a group's N*H*W; NULL = no
                          BatchNorm */
  const float *gamma;  /* [C] or NULL (= 1) */
  const float *beta;   /* [C] or NULL (= 0) */
  float eps;
  double count;        /* (N / groups)*H*W */
  int32_t groups;      /* <= 1: the whole batch is one BatchNorm batch.  G > 1: the batch is G equal runs of images with
                          independent batch statistics and weight gradients summed over all of them -- G forward passes of
                          the reference (dcgan.py:178-179: discriminator(real_imgs), discriminator(gen_imgs.detach())) in
                          one launch per layer; running statistics are updated G times in batch order.  Every stats / sums
                          buffer of the chain entry points then has a leading [groups] dimension. */
  int32_t reserved;
} b200gan_nb_bn;
/* 1 if the geometry can run in the fused chain (Conv2d, zero padding, stride 1/2, 3x3 or 4x4, C <= 128 (1 or a
 * multiple of 4), K a power of two in [4, 128]) */
int b200gan_nb_supported(const b200gan_conv_geom *g);
/* ... and with the batch split into `groups` statistics groups (see b200gan_nb_bn) */
int b200gan_nb_groups_supported(const b200gan_conv_geom *g, int32_t groups);
/* y = chan_scale[n,k] * act(conv(BN_in(x)) + bias): x = a_{l-1} [N][H][W][C]; packed = B200GAN_PACK_SIMT_FPROP.
 * in_bn (may be NULL): the BatchNorm between the producer and this conv, finalised in the prologue; running_mean/var and
 * num_batches_tracked (may be NULL) are updated once per call (per group, in order) with torch semantics.  groups: see
 * b200gan_nb_bn (must equal in_bn->groups when in_bn is given).  out_stats [groups][2][K] (may be NULL):
 * OVERWRITTEN with the batch sums of y for the next BatchNorm. */
int b200gan_nb_fprop(const b200gan_conv_geom *g, const b200gan_nb_bn *in_bn, float *running_mean, float *running_var,
                     int64_t *num_batches_tracked, float momentum, const float *x, const float *packed,
                     const float *bias, int32_t act, float slope, const float *chan_scale, float *y,
                     double *out_stats, int32_t groups, void *stream);
/* dz = BN_out-backward(g) * chan_scale * act'(a) and db[K] = column sums of dz (may be NULL).  g: gradient w.r.t. the
 * (virtual) BatchNorm output, or w.r.t. a itself when out_bn is NULL; sums [2][K]: sum g, sum g * ahat (complete). */
int b200gan_nb_dz(int32_t N, int64_t PQ, int32_t K, const float *g, const float *a, const float *chan_scale,
                  int32_t act, float slope, const b200gan_nb_bn *out_bn, const double *sums, float *dz, float *db,
                  void *stream);
/* dw [K][C][R][S] (OVERWRITTEN) from dz [N][P][Q][K] and x = BN_in(a_{l-1}) recomputed on the fly.  workspace:
 * b200gan_nb_wgrad_workspace_floats() floats of per-block partial slabs (summed in a fixed order: deterministic); NULL or
 * a size of 0: fp32 atomics into dw. */
size_t b200gan_nb_wgrad_workspace_floats(const b200gan_conv_geom *g);
int b200gan_nb_wgrad(const b200gan_conv_geom *g, const b200gan_nb_bn *in_bn, const float *x, const float *dz, float *dw,
                     float *workspace, void *stream);
/* g_out [N][H][W][C] = gradient w.r.t. the conv's (virtual) input; packed = B200GAN_PACK_SIMT_DGRAD.  With in_bn, a_prev
 * (= the stored input a_{l-1}) and sums [2][C]: sums is OVERWRITTEN with sum g_out, sum g_out * ahat_prev, which is what
 * the backward of the BatchNorm in front of this conv needs (and its dbeta / dgamma). */
int b200gan_nb_dgrad(const b200gan_conv_geom *g, const float *dz, const float *packed, const b200gan_nb_bn *in_bn,
                     const float *a_prev, float *g_out, double *sums, void *stream);
/* End of a chain: out = BN(a) as a real tensor, [N][C][HW] (nchw != 0: what the script's .view expects, dcgan.py:96) or
 * [N][HW][C]; and its backward: g [N][HW][C] = dout re-laid-out, sums [2][C] OVERWRITTEN. */
int b200gan_nb_tail_fwd(int32_t N, int32_t HW, int32_t C, const b200gan_nb_bn *bn, float *running_mean,
                        float *running_var, int64_t *num_batches_tracked, float momentum, const float *a, float *out,
                        int32_t nchw, void *stream);
int b200gan_nb_tail_bwd(int32_t N, int32_t HW, int32_t C, const b200gan_nb_bn *bn, const float *a, const float *dout,
                        int32_t nchw, float *g, double *sums, void *stream);

/* ---- Discriminator head and adversarial loss (csrc/head.cu) --------------------------------------------------- */
/* y[n] = act(dot(x[n], w) + b): nn.Linear(K, 1) [+ nn.Sigmoid]  (dcgan.py:92).  x [N][K] row-major. */
int b200gan_linear1_fwd(const float *x, const float *w, const float *b, float *y, int32_t N, int32_t K, int32_t act,
                        void *stream);
/* Backward from the saved output y: dx [N][K] (may be NULL), dw [K], db [1] (may be NULL) are OVERWRITTEN. */
int b200gan_linear1_bwd(const float *x, const float *w, const float *y, const float *dy, float *dx, float *dw,
                        float *db, int32_t N, int32_t K, int32_t act, void *stream);
/* torch.nn.BCELoss(), reduction 'mean', log terms clamped at -100 (dcgan.py:103,166,178-179). */
int b200gan_bce_fwd(const float *v, const float *t, float *loss, int64_t n, void *stream);
int b200gan_bce_bwd(const float *v, const float *t, const float *gout, float *dv, int64_t n, void *stream);

/* ---- MSELoss / L1Loss, reduction 'mean' (csrc/pixel_loss/) --------------------------------------------------------- */
/* torch.nn.MSELoss() / torch.nn.L1Loss() of an input a and a target b of one logical shape [N][C][H][W] (fewer
 * dimensions padded with leading 1s): the adversarial loss of LSGAN, Pix2Pix and CycleGAN (lsgan.py:102, pix2pix.py:50,
 * cyclegan.py:50) and the pixel, cycle and identity losses of the image translators (pix2pix.py:51, cyclegan.py:51-52).
 * Each operand is dense in its own layout: NCHW-contiguous, or channels_last (NHWC, 4-D only).  0 < n < 2^31. */
enum { B200GAN_PIXEL_LOSS_MSE = 0, B200GAN_PIXEL_LOSS_L1 = 1 };
enum { B200GAN_LAYOUT_NCHW = 0, B200GAN_LAYOUT_NHWC = 1 };
typedef struct b200gan_pixel_loss_desc {
  int32_t mode;                 /* B200GAN_PIXEL_LOSS_*                          */
  int32_t layout_a, layout_b;   /* B200GAN_LAYOUT_* of the input and the target  */
  int32_t reserved;
  int64_t n;                    /* N * C * H * W                                 */
  int32_t N, C, H, W;           /* logical shape, padded to 4-D                  */
} b200gan_pixel_loss_desc;
/* Bytes of the forward's workspace (0 for an invalid desc).  It holds a completion ticket that must be zero before the
 * first call; every call leaves it zero again, so one buffer serves any number of calls (and CUDA-graph replays) issued
 * in order on one stream. */
size_t b200gan_pixel_loss_workspace_bytes(const b200gan_pixel_loss_desc *d);
/* loss[0] = mean over the elements of (a - b)^2 (MSE) or |a - b| (L1), summed in a fixed order (fp32 per thread, fp64
 * across threads and blocks): bit-identical from call to call on one device.  ONE launch.  workspace: 16-byte aligned. */
int b200gan_pixel_loss_fwd(const b200gan_pixel_loss_desc *d, const float *a, const float *b, float *loss,
                           void *workspace, void *stream);
/* Given gout[0] = dL/dloss (read on the device): da = 2 (a - b) gout / n (MSE) or sign(a - b) gout / n (L1, sign(0) =
 * 0) in a's layout, and db = -da in b's layout when db is not NULL.  ONE launch; da and db are OVERWRITTEN. */
int b200gan_pixel_loss_bwd(const b200gan_pixel_loss_desc *d, const float *a, const float *b, const float *gout,
                           float *da, float *db, void *stream);

/* ---- Adam (torch.optim.Adam semantics: dcgan.py:134-135) ---------------------------------------------------------- */
/* p -= lr * mhat / (sqrt(vhat) + eps), bias-corrected with the step count read from the device.  lr, betas and eps are
 * doubles like torch's Python-side hyper-parameters: torch forms 1 - beta, 1 - beta^t and lr / (1 - beta1^t) in double
 * and casts them to fp32 where they meet a tensor.  grad_scale multiplies g first (1/world_size after an all-reduce
 * sum).  Every parameter tensor of one optimizer in ONE launch per 48 tensors (the table travels as a kernel argument;
 * `g` is whatever tensor autograd left in param.grad; n > 0).  step: TWO floats on the device, zero-initialised by the
 * caller: step[0] = number of steps taken (advanced once per call, by the last block of the last launch -> CUDA-graph
 * capturable; count 0 only advances it), step[1] = internal ticket counter. */
typedef struct b200gan_adam_tensor {
  float *p;
  const float *g;
  float *m;
  float *v;
  int64_t n;
} b200gan_adam_tensor;
int b200gan_adam_multi(const b200gan_adam_tensor *tensors, int32_t count, double lr, double beta1, double beta2,
                       double eps, float grad_scale, float *step, void *stream);

#ifdef __cplusplus
}
#endif
#endif /* B200GAN_H */
