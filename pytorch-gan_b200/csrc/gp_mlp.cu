// gp_mlp.cu -- WGAN-GP gradient penalty of the MLP critic as ONE kernel (cooperative launch).
//
// Reference: compute_gradient_penalty (wgan_gp.py:119-138) builds the penalty with
// autograd.grad(create_graph=True) and d_loss.backward() (wgan_gp.py:173) differentiates through that
// graph: ~40 tiny cuBLAS/ATen launches, all latency.  The critic (wgan_gp.py:72-78) is
//   D(x) = W3 lrelu(W2 lrelu(W1 x + b1) + b2) + b3,      Din -> H1 -> H2 -> 1.
// LeakyReLU'' = 0 almost everywhere, so the double backward has a closed form (SURVEY.md 8a row a7):
//   h1 = x W1^T + b1, m1 = lrelu'(h1);   a1 = h1 * m1
//   h2 = a1 W2^T + b2, m2 = lrelu'(h2);  g2 = W3 * m2            [N,H2]   (= dD/dh2)
//   g1 = (g2 W2) * m1  [N,H1];   gx = g1 W1  [N,Din]  (= dD/dx);   r = ||gx||_2
//   gp = lambda * mean((r-1)^2);          u = lambda * (2/N) (r-1)/r * gx
//   dW1 = g1^T u;  dg1 = u W1^T;  t = dg1 * m1;  dW2 = g2^T t;  dg2 = t W2^T;  dW3 = sum_n dg2 * m2
// (bias gradients are exactly zero).  Eight dependent phases of small fp32 GEMMs are separated by
// grid-wide barriers inside one persistent kernel; every phase spreads 32x32 output tiles over the
// grid.  fp32 FFMA throughout: the whole problem is ~0.6 GFLOP and purely latency bound.
#include "common.cuh"
#include "tile_gemm.cuh"
#include <cooperative_groups.h>

namespace cg = cooperative_groups;

namespace b200gan {

struct GpP {
  int N, Din, H1, H2;
  float slope, lambda_gp;
  const float *xi, *W1, *b1, *W2, *b2, *W3;
  float *gp, *dW1, *dW2, *dW3;
  float *m1, *a1, *g1, *g1s, *t;   // [N][H1]
  float *m2, *g2, *dg2m;           // [N][H2]
  float *gx;                       // [N][Din]
  float *coef;                     // [N]
};

__global__ void __launch_bounds__(256) gp_mlp_kernel(GpP p) {
  __shared__ float As[GT][GT + 1];
  __shared__ float Bs[GT][GT + 1];
  cg::grid_group grid = cg::this_grid();
  const int N = p.N, Din = p.Din, H1 = p.H1, H2 = p.H2;
  const int nb = gridDim.x, bid = blockIdx.x;

  if (bid == 0 && threadIdx.x == 0) *p.gp = 0.f;
  // P1: h1 = xi W1^T + b1
  for (int t = bid; t < ntiles(N, H1); t += nb)
    tile_gemm(p.xi, Din, 1, p.W1, 1, Din, N, H1, Din, t,
              [&](int n, int j, float acc) {
                float h = acc + p.b1[j];
                float m = h > 0.f ? 1.f : p.slope;
                p.m1[(size_t)n * H1 + j] = m;
                p.a1[(size_t)n * H1 + j] = h * m;
              }, As, Bs);
  grid.sync();
  // P2: h2 = a1 W2^T + b2 ; g2 = W3 * m2
  for (int t = bid; t < ntiles(N, H2); t += nb)
    tile_gemm(p.a1, H1, 1, p.W2, 1, H1, N, H2, H1, t,
              [&](int n, int j, float acc) {
                float h = acc + p.b2[j];
                float m = h > 0.f ? 1.f : p.slope;
                p.m2[(size_t)n * H2 + j] = m;
                p.g2[(size_t)n * H2 + j] = p.W3[j] * m;
              }, As, Bs);
  grid.sync();
  // P3: g1 = (g2 W2) * m1
  for (int t = bid; t < ntiles(N, H1); t += nb)
    tile_gemm(p.g2, H2, 1, p.W2, H1, 1, N, H1, H2, t,
              [&](int n, int i, float acc) { p.g1[(size_t)n * H1 + i] = acc * p.m1[(size_t)n * H1 + i]; }, As, Bs);
  grid.sync();
  // P4: gx = g1 W1
  for (int t = bid; t < ntiles(N, Din); t += nb)
    tile_gemm(p.g1, H1, 1, p.W1, Din, 1, N, Din, H1, t,
              [&](int n, int d, float acc) { p.gx[(size_t)n * Din + d] = acc; }, As, Bs);
  grid.sync();
  // P5: per-sample norm, penalty, coefficient; g1s = coef * g1
  {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (int n = bid * 8 + warp; n < N; n += nb * 8) {
      float s = 0.f;
      for (int d = lane; d < Din; d += 32) {
        float v = p.gx[(size_t)n * Din + d];
        s = fmaf(v, v, s);
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
      float r = sqrtf(s);
      float c = p.lambda_gp * (2.f / (float)N) * (r - 1.f) / r;
      if (lane == 0) {
        p.coef[n] = c;
        atomicAdd(p.gp, p.lambda_gp * (r - 1.f) * (r - 1.f) / (float)N);
      }
      for (int i = lane; i < H1; i += 32) p.g1s[(size_t)n * H1 + i] = p.g1[(size_t)n * H1 + i] * c;
    }
  }
  grid.sync();
  // P6: dW1 = g1s^T gx   and   t = (coef * (gx W1^T)) * m1
  {
    const int ta = ntiles(H1, Din), tb = ntiles(N, H1);
    for (int t = bid; t < ta + tb; t += nb) {
      if (t < ta)
        tile_gemm(p.g1s, 1, H1, p.gx, Din, 1, H1, Din, N, t,
                  [&](int i, int d, float acc) { p.dW1[(size_t)i * Din + d] = acc; }, As, Bs);
      else
        tile_gemm(p.gx, Din, 1, p.W1, 1, Din, N, H1, Din, t - ta,
                  [&](int n, int i, float acc) {
                    p.t[(size_t)n * H1 + i] = acc * p.coef[n] * p.m1[(size_t)n * H1 + i];
                  }, As, Bs);
    }
  }
  grid.sync();
  // P7: dW2 = g2^T t   and   dg2m = (t W2^T) * m2
  {
    const int ta = ntiles(H2, H1), tb = ntiles(N, H2);
    for (int t = bid; t < ta + tb; t += nb) {
      if (t < ta)
        tile_gemm(p.g2, 1, H2, p.t, H1, 1, H2, H1, N, t,
                  [&](int j, int i, float acc) { p.dW2[(size_t)j * H1 + i] = acc; }, As, Bs);
      else
        tile_gemm(p.t, H1, 1, p.W2, 1, H1, N, H2, H1, t - ta,
                  [&](int n, int j, float acc) { p.dg2m[(size_t)n * H2 + j] = acc * p.m2[(size_t)n * H2 + j]; }, As,
                  Bs);
    }
  }
  grid.sync();
  // P8: dW3 = sum_n dg2m
  for (int j = bid * blockDim.x + threadIdx.x; j < H2; j += nb * blockDim.x) {
    float s = 0.f;
    for (int n = 0; n < N; ++n) s += p.dg2m[(size_t)n * H2 + j];
    p.dW3[j] = s;
  }
}


// ---- the whole critic iteration of wgan_gp.py:164-173 in ONE kernel -----------------------------------------------------------
//   d_loss = -mean(D(real)) + mean(D(fake)) + lambda * gp(D, alpha * real + (1 - alpha) * fake)
// and its gradient w.r.t. every parameter of D.  The three batches (real, fake, interpolates) are stacked into one 3N-row
// problem; the first-order backward of the real/fake rows and the closed-form double backward of the penalty rows share
// their GEMMs: with dout = (-1/N, +1/N, 1) per row group,
//   U2 = dout * W3 * m2          rows < 2N: dL/dh2,        penalty rows: g2
//   U1 = (U2 W2) * m1            rows < 2N: dL/dh1,        penalty rows: g1 (then scaled by coef -> g1s)
//   X3 penalty rows <- gx = g1 W1 (the interpolates themselves are dead after layer 1)
//   dW1 = U1^T X3                = dh1^T x  +  g1s^T gx
//   A1 penalty rows <- t = coef * (gx W1^T) * m1;     dW2 = U2^T A1 = dh2^T a1 + g2^T t
//   A2 penalty rows <- (t W2^T) * m2;                 dW3 = sum_r dout_r * A2_r
// Bias gradients come from the real/fake rows only (the penalty does not depend on the biases).
struct CsP {
  int N, Din, H1, H2;
  float slope, lambda_gp;
  const float *real, *fake, *alpha, *W1, *b1, *W2, *b2, *W3, *b3;
  float *losses;  // [2]: d_loss, lambda * gp
  float *dW1, *db1, *dW2, *db2, *dW3, *db3;
  float *X3, *A1, *U1, *M1, *A2, *U2, *M2, *dout, *coef;
};

__global__ void __launch_bounds__(256) critic_step_kernel(CsP p) {
  __shared__ float As[GT][GT + 1];
  __shared__ float Bs[GT][GT + 1];
  cg::grid_group grid = cg::this_grid();
  const int N = p.N, Din = p.Din, H1 = p.H1, H2 = p.H2, R = 3 * p.N;
  const int nb = gridDim.x, bid = blockIdx.x;
  const int64_t gtid = (int64_t)bid * blockDim.x + threadIdx.x, gthreads = (int64_t)nb * blockDim.x;

  // P0: stack the three batches, per-row output gradients
  for (int64_t i = gtid; i < (int64_t)N * Din; i += gthreads) {
    const int n = (int)(i / Din);
    const float r = p.real[i], f = p.fake[i], a = p.alpha[n];
    p.X3[i] = r;
    p.X3[(int64_t)N * Din + i] = f;
    p.X3[(int64_t)2 * N * Din + i] = a * r + (1.f - a) * f;
  }
  for (int64_t i = gtid; i < R; i += gthreads) p.dout[i] = i < N ? -1.f / (float)N : (i < 2 * N ? 1.f / (float)N : 1.f);
  if (gtid < 2) p.losses[gtid] = 0.f;
  grid.sync();
  // P1: h1 = X3 W1^T + b1
  for (int t = bid; t < ntiles(R, H1); t += nb)
    tile_gemm(p.X3, Din, 1, p.W1, 1, Din, R, H1, Din, t,
              [&](int r, int j, float acc) {
                const float h = acc + p.b1[j];
                const float m = h > 0.f ? 1.f : p.slope;
                p.M1[(size_t)r * H1 + j] = m;
                p.A1[(size_t)r * H1 + j] = h * m;
              }, As, Bs);
  grid.sync();
  // P2: h2 = a1 W2^T + b2; U2 = dout * W3 * m2
  for (int t = bid; t < ntiles(R, H2); t += nb)
    tile_gemm(p.A1, H1, 1, p.W2, 1, H1, R, H2, H1, t,
              [&](int r, int j, float acc) {
                const float h = acc + p.b2[j];
                const float m = h > 0.f ? 1.f : p.slope;
                p.M2[(size_t)r * H2 + j] = m;
                p.A2[(size_t)r * H2 + j] = h * m;
                p.U2[(size_t)r * H2 + j] = p.dout[r] * p.W3[j] * m;
              }, As, Bs);
  grid.sync();
  // P3: critic outputs of the real / fake rows -> Wasserstein part of the loss;  U1 = (U2 W2) * m1
  {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (int r = bid * 8 + warp; r < 2 * N; r += nb * 8) {
      float s = 0.f;
      for (int j = lane; j < H2; j += 32) s = fmaf(p.A2[(size_t)r * H2 + j], p.W3[j], s);
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
      if (lane == 0) atomicAdd(p.losses, (s + p.b3[0]) * p.dout[r]);
    }
  }
  for (int t = bid; t < ntiles(R, H1); t += nb)
    tile_gemm(p.U2, H2, 1, p.W2, H1, 1, R, H1, H2, t,
              [&](int r, int i, float acc) { p.U1[(size_t)r * H1 + i] = acc * p.M1[(size_t)r * H1 + i]; }, As, Bs);
  grid.sync();
  // P4: gx = g1 W1 over the penalty rows, written over the (dead) interpolates
  for (int t = bid; t < ntiles(N, Din); t += nb)
    tile_gemm(p.U1 + (size_t)2 * N * H1, H1, 1, p.W1, Din, 1, N, Din, H1, t,
              [&](int n, int d, float acc) { p.X3[(size_t)(2 * N + n) * Din + d] = acc; }, As, Bs);
  grid.sync();
  // P5: per-sample gradient norm, penalty, coefficient; g1 -> g1s = coef * g1
  {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (int n = bid * 8 + warp; n < N; n += nb * 8) {
      const float *gx = p.X3 + (size_t)(2 * N + n) * Din;
      float s = 0.f;
      for (int d = lane; d < Din; d += 32) s = fmaf(gx[d], gx[d], s);
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
      const float r = sqrtf(s);
      const float c = p.lambda_gp * (2.f / (float)N) * (r - 1.f) / r;
      if (lane == 0) {
        p.coef[n] = c;
        const float term = p.lambda_gp * (r - 1.f) * (r - 1.f) / (float)N;
        atomicAdd(p.losses, term);
        atomicAdd(p.losses + 1, term);
      }
      float *g1 = p.U1 + (size_t)(2 * N + n) * H1;
      for (int i = lane; i < H1; i += 32) g1[i] *= c;
    }
  }
  grid.sync();
  // P6: dW1 = U1^T X3;  t = coef * (gx W1^T) * m1 over the (dead) a1 of the penalty rows;  db1
  {
    const int ta = ntiles(H1, Din), tb = ntiles(N, H1);
    for (int t = bid; t < ta + tb; t += nb) {
      if (t < ta)
        tile_gemm(p.U1, 1, H1, p.X3, Din, 1, H1, Din, R, t,
                  [&](int i, int d, float acc) { p.dW1[(size_t)i * Din + d] = acc; }, As, Bs);
      else
        tile_gemm(p.X3 + (size_t)2 * N * Din, Din, 1, p.W1, 1, Din, N, H1, Din, t - ta,
                  [&](int n, int i, float acc) {
                    p.A1[(size_t)(2 * N + n) * H1 + i] = acc * p.coef[n] * p.M1[(size_t)(2 * N + n) * H1 + i];
                  }, As, Bs);
    }
    for (int64_t i = gtid; i < H1; i += gthreads) {
      float s = 0.f;
      for (int r = 0; r < 2 * N; ++r) s += p.U1[(size_t)r * H1 + i];
      p.db1[i] = s;
    }
  }
  grid.sync();
  // P7: dW2 = U2^T A1;  A2 penalty rows <- (t W2^T) * m2;  db2
  {
    const int ta = ntiles(H2, H1), tb = ntiles(N, H2);
    for (int t = bid; t < ta + tb; t += nb) {
      if (t < ta)
        tile_gemm(p.U2, 1, H2, p.A1, H1, 1, H2, H1, R, t,
                  [&](int j, int i, float acc) { p.dW2[(size_t)j * H1 + i] = acc; }, As, Bs);
      else
        tile_gemm(p.A1 + (size_t)2 * N * H1, H1, 1, p.W2, 1, H1, N, H2, H1, t - ta,
                  [&](int n, int j, float acc) {
                    p.A2[(size_t)(2 * N + n) * H2 + j] = acc * p.M2[(size_t)(2 * N + n) * H2 + j];
                  }, As, Bs);
    }
    for (int64_t j = gtid; j < H2; j += gthreads) {
      float s = 0.f;
      for (int r = 0; r < 2 * N; ++r) s += p.U2[(size_t)r * H2 + j];
      p.db2[j] = s;
    }
  }
  grid.sync();
  // P8: dW3 = sum_r dout_r * A2_r;  db3 = sum over the real / fake rows of dout
  for (int64_t j = gtid; j < H2; j += gthreads) {
    float s = 0.f;
    for (int r = 0; r < R; ++r) s = fmaf(p.dout[r], p.A2[(size_t)r * H2 + j], s);
    p.dW3[j] = s;
  }
  if (gtid == 0) {
    float s = 0.f;
    for (int r = 0; r < 2 * N; ++r) s += p.dout[r];
    p.db3[0] = s;
  }
}

}  // namespace b200gan

using namespace b200gan;

extern "C" size_t b200gan_gp_mlp_workspace_floats(const b200gan_gp_mlp_desc *d) {
  if (!d) return 0;
  return (size_t)d->N * ((size_t)5 * d->H1 + (size_t)3 * d->H2 + d->Din + 1) + 64;
}

extern "C" int b200gan_gp_mlp_fwd_bwd(const b200gan_gp_mlp_desc *d, const float *xi, const float *W1,
                                      const float *b1, const float *W2, const float *b2, const float *W3, float *gp,
                                      float *dW1, float *dW2, float *dW3, float *workspace, void *stream) {
  B2_CHECK_ARG(d && xi && W1 && b1 && W2 && b2 && W3 && gp && dW1 && dW2 && dW3 && workspace,
               "gp_mlp_fwd_bwd: null pointer");
  B2_CHECK_ARG(d->N > 0 && d->Din > 0 && d->H1 > 0 && d->H2 > 0, "gp_mlp_fwd_bwd: bad dims");
  GpP p;
  p.N = d->N; p.Din = d->Din; p.H1 = d->H1; p.H2 = d->H2; p.slope = d->slope; p.lambda_gp = d->lambda_gp;
  p.xi = xi; p.W1 = W1; p.b1 = b1; p.W2 = W2; p.b2 = b2; p.W3 = W3;
  p.gp = gp; p.dW1 = dW1; p.dW2 = dW2; p.dW3 = dW3;
  float *w = workspace;
  const size_t nh1 = (size_t)d->N * d->H1, nh2 = (size_t)d->N * d->H2;
  p.m1 = w; w += nh1; p.a1 = w; w += nh1; p.g1 = w; w += nh1; p.g1s = w; w += nh1; p.t = w; w += nh1;
  p.m2 = w; w += nh2; p.g2 = w; w += nh2; p.dg2m = w; w += nh2;
  p.gx = w; w += (size_t)d->N * d->Din;
  p.coef = w;
  int dev = 0, sms = 0, per_sm = 0;
  B2_CUDA(cudaGetDevice(&dev));
  B2_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  B2_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, gp_mlp_kernel, 256, 0));
  B2_CHECK_ARG(per_sm >= 1, "gp_mlp_fwd_bwd: kernel cannot be made resident");
  int grid = sms * (per_sm > 2 ? 2 : per_sm);
  void *args[] = {&p};
  B2_CUDA(cudaLaunchCooperativeKernel((const void *)gp_mlp_kernel, dim3(grid), dim3(256), args, 0, as_stream(stream)));
  return B200GAN_OK;
}

extern "C" size_t b200gan_critic_step_workspace_floats(const b200gan_gp_mlp_desc *d) {
  if (!d) return 0;
  const size_t R = (size_t)3 * d->N;
  return R * ((size_t)d->Din + 3 * (size_t)d->H1 + 3 * (size_t)d->H2 + 1) + d->N + 64;
}

extern "C" int b200gan_critic_step_mlp(const b200gan_gp_mlp_desc *d, const float *real, const float *fake,
                                       const float *alpha, const float *W1, const float *b1, const float *W2,
                                       const float *b2, const float *W3, const float *b3, float *losses, float *dW1,
                                       float *db1, float *dW2, float *db2, float *dW3, float *db3, float *workspace,
                                       void *stream) {
  B2_CHECK_ARG(d && real && fake && alpha && W1 && b1 && W2 && b2 && W3 && b3 && losses && dW1 && db1 && dW2 && db2 &&
                   dW3 && db3 && workspace, "critic_step_mlp: null pointer");
  B2_CHECK_ARG(d->N > 0 && d->Din > 0 && d->H1 > 0 && d->H2 > 0, "critic_step_mlp: bad dims");
  CsP p;
  p.N = d->N; p.Din = d->Din; p.H1 = d->H1; p.H2 = d->H2; p.slope = d->slope; p.lambda_gp = d->lambda_gp;
  p.real = real; p.fake = fake; p.alpha = alpha; p.W1 = W1; p.b1 = b1; p.W2 = W2; p.b2 = b2; p.W3 = W3; p.b3 = b3;
  p.losses = losses; p.dW1 = dW1; p.db1 = db1; p.dW2 = dW2; p.db2 = db2; p.dW3 = dW3; p.db3 = db3;
  const size_t R = (size_t)3 * d->N;
  float *w = workspace;
  p.X3 = w; w += R * d->Din;
  p.A1 = w; w += R * d->H1; p.U1 = w; w += R * d->H1; p.M1 = w; w += R * d->H1;
  p.A2 = w; w += R * d->H2; p.U2 = w; w += R * d->H2; p.M2 = w; w += R * d->H2;
  p.dout = w; w += R;
  p.coef = w;
  int dev = 0, sms = 0, per_sm = 0;
  B2_CUDA(cudaGetDevice(&dev));
  B2_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  B2_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, critic_step_kernel, 256, 0));
  B2_CHECK_ARG(per_sm >= 1, "critic_step_mlp: kernel cannot be made resident");
  int grid = sms * (per_sm > 2 ? 2 : per_sm);
  void *args[] = {&p};
  B2_CUDA(cudaLaunchCooperativeKernel((const void *)critic_step_kernel, dim3(grid), dim3(256), args, 0, as_stream(stream)));
  return B200GAN_OK;
}
