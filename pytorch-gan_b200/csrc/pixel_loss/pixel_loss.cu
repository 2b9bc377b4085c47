// pixel_loss.cu -- torch.nn.MSELoss() and torch.nn.L1Loss() (reduction 'mean'), forward and backward, one kernel each.
//
// Reference call sites:
//   criterion_GAN = torch.nn.MSELoss()                         pix2pix.py:50, cyclegan.py:50, lsgan.py:102 (adversarial)
//   criterion_pixelwise = torch.nn.L1Loss()                    pix2pix.py:51 (pixel), cyclegan.py:51-52 (cycle, identity)
//   loss_pixel = criterion_pixelwise(fake_B, real_B)           pix2pix.py:145, on [16, 3, 256, 256]
// Stock torch runs MSE as one element-wise kernel plus a mean reduction forward and two or three element-wise kernels
// backward; L1 is a composite (sub, abs, mean) with as many again.  Here: one launch per direction.
//
// Each operand is dense in one of two layouts of the same logical [N][C][H][W] (shapes of fewer dimensions are padded
// with leading 1s): NCHW-contiguous or channels_last (NHWC).  The operands may differ: a drop-in generator's output is
// channels_last while the data loader's target is NCHW.  Elements are visited in the input's (a's) memory order and b is
// read at the same logical index; with one layout on both sides that is the same offset, and float4 loads are used.
// The kernels are in pixel_loss_kernels.cuh; this file plans their grids, checks the arguments and launches them.
#include "pixel_loss_kernels.cuh"

namespace b200gan {

static int pl_fwd_grid(int64_t n) {
  int64_t blocks = ceil_div64(n, (int64_t)PL_THREADS * PL_PER_THREAD);
  const int64_t cap = (int64_t)2 * num_sms() < PL_MAX_BLOCKS ? (int64_t)2 * num_sms() : PL_MAX_BLOCKS;
  if (blocks > cap) blocks = cap;
  return (int)blocks;
}

static int pl_bwd_grid(int64_t n) {
  int64_t blocks = ceil_div64(n, (int64_t)PL_THREADS * 4);
  if (blocks > (int64_t)4 * num_sms()) blocks = (int64_t)4 * num_sms();
  return (int)blocks;
}

static int pl_check_desc(const b200gan_pixel_loss_desc *d) {
  B2_CHECK_ARG(d, "pixel_loss: desc is NULL");
  B2_CHECK_ARG(d->mode == B200GAN_PIXEL_LOSS_MSE || d->mode == B200GAN_PIXEL_LOSS_L1, "pixel_loss: unknown mode %d",
               d->mode);
  B2_CHECK_ARG(d->layout_a == B200GAN_LAYOUT_NCHW || d->layout_a == B200GAN_LAYOUT_NHWC,
               "pixel_loss: unknown layout %d of the input", d->layout_a);
  B2_CHECK_ARG(d->layout_b == B200GAN_LAYOUT_NCHW || d->layout_b == B200GAN_LAYOUT_NHWC,
               "pixel_loss: unknown layout %d of the target", d->layout_b);
  B2_CHECK_ARG(d->n > 0, "pixel_loss: n = %lld (an empty loss is not taken)", (long long)d->n);
  B2_CHECK_ARG(d->N > 0 && d->C > 0 && d->H > 0 && d->W > 0, "pixel_loss: shape [%d, %d, %d, %d]", d->N, d->C, d->H,
               d->W);
  B2_CHECK_ARG((int64_t)d->N * d->C * d->H * d->W == d->n, "pixel_loss: shape [%d, %d, %d, %d] does not hold n = %lld",
               d->N, d->C, d->H, d->W, (long long)d->n);
  if (d->n > INT32_MAX) B2_UNSUPPORTED("pixel_loss: n = %lld > 2^31 - 1", (long long)d->n);
  return B200GAN_OK;
}

static PixelLossArgs pl_args(const b200gan_pixel_loss_desc *d, const float *a, const float *b) {
  PixelLossArgs p;
  p.a = a;
  p.b = b;
  p.n = (int32_t)d->n;
  p.C = d->C;
  p.H = d->H;
  p.W = d->W;
  p.mode = d->mode;
  p.same = d->layout_a == d->layout_b;
  p.a_nhwc = d->layout_a == B200GAN_LAYOUT_NHWC;
  p.vec = p.same && (((uintptr_t)a | (uintptr_t)b) & 15) == 0;
  return p;
}

}  // namespace b200gan

using namespace b200gan;

extern "C" size_t b200gan_pixel_loss_workspace_bytes(const b200gan_pixel_loss_desc *d) {
  if (pl_check_desc(d) != B200GAN_OK) return 0;
  return (size_t)PL_TICKET_BYTES + sizeof(double) * (size_t)pl_fwd_grid(d->n);
}

extern "C" int b200gan_pixel_loss_fwd(const b200gan_pixel_loss_desc *d, const float *a, const float *b, float *loss,
                                      void *workspace, void *stream) {
  const int rc = pl_check_desc(d);
  if (rc != B200GAN_OK) return rc;
  B2_CHECK_ARG(a && b && loss && workspace, "pixel_loss_fwd: NULL pointer");
  B2_CHECK_ARG(((uintptr_t)workspace & 15) == 0, "pixel_loss_fwd: workspace is not 16-byte aligned");
  const PixelLossArgs p = pl_args(d, a, b);
  const int blocks = pl_fwd_grid(d->n);
  int32_t chunk = (int32_t)ceil_div64(d->n, blocks);
  chunk = (chunk + 3) & ~3;  // float4-aligned block slices
  pixel_loss_fwd_kernel<<<(unsigned)blocks, PL_THREADS, 0, as_stream(stream)>>>(p, chunk, workspace, loss);
  B2_LAUNCH_CHECK();
  return B200GAN_OK;
}

extern "C" int b200gan_pixel_loss_bwd(const b200gan_pixel_loss_desc *d, const float *a, const float *b,
                                      const float *gout, float *da, float *db, void *stream) {
  const int rc = pl_check_desc(d);
  if (rc != B200GAN_OK) return rc;
  B2_CHECK_ARG(a && b && gout && da, "pixel_loss_bwd: NULL pointer");
  PixelLossArgs p = pl_args(d, a, b);
  p.vec = p.vec && (((uintptr_t)da | (uintptr_t)db) & 15) == 0;
  pixel_loss_bwd_kernel<<<(unsigned)pl_bwd_grid(d->n), PL_THREADS, 0, as_stream(stream)>>>(p, gout, da, db);
  B2_LAUNCH_CHECK();
  return B200GAN_OK;
}
