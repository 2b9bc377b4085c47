// mlp_critic.cu -- the MLP critic (wgan_gp.py:72-78, wgan_div.py:72-78) as cooperative kernels:
//   D(x) = W3 lrelu(W2 lrelu(W1 x + b1) + b2) + b3,      Din -> H1 -> H2 -> 1, one LeakyReLU slope.
// Its autograd is three kernels with no penalty built in: the forward, the first-order backward for an arbitrary output
// gradient dout, and the double backward of the input gradient for an arbitrary upstream gradient u = dL/d(dD/dx) are
// separate entry points, so a script's own penalty arithmetic (||g|| - 1)^2, ||g||^p, ... stays in its autograd graph
// while every critic GEMM runs here.
//   forward        h1 = x W1^T + b1, m1 = lrelu'(h1), a1 = h1 m1;   h2 = a1 W2^T + b2, m2 = lrelu'(h2), a2 = h2 m2
//                  out = a2 W3^T + b3
//   backward       U2 = dout W3 * m2;  U1 = (U2 W2) * m1;  dx = U1 W1
//                  dW1 = U1^T x, dW2 = U2^T a1, dW3 = dout^T a2, db1 = sum_n U1, db2 = sum_n U2, db3 = sum_n dout
//   double bwd     (LeakyReLU'' = 0 almost everywhere: the masks are constants)
//                  dW1 = U1^T u;  t = (u W1^T) * m1;  dW2 = U2^T t;  s = (t W2^T) * m2;
//                  dW3 = sum_n dout_n s_n;  d(dout)_n = s_n . W3      (x and the biases get exactly zero)
// Each pass is ~0.1 GFLOP at the WGAN-GP size and latency bound, so each is ONE persistent cooperative launch whose
// dependent phases are separated by grid.sync(); every phase spreads 32x32 fp32 FFMA output tiles (tile_gemm.cuh)
// over the grid.  Column sums run one thread per column in a fixed order: the results are deterministic.
// critic_step_kernel (below) is the whole WGAN-GP critic iteration, penalty included, in one such launch.
// The vanilla GAN's discriminator (gan.py:64-80, bgan.py:66-80, aae.py:90-104) is the same critic followed by a Sigmoid:
// a run-time mode of the forward and backward kernels (b200gan_mlp_disc_*), off for the critic entry points.
//   forward        y = 1 / (1 + exp(-out))
//   backward       g = dout * y * (1 - y) (torch's sigmoid backward), then the critic backward above with dout := g
#include "common.cuh"
#include "tile_gemm.cuh"
#include <cooperative_groups.h>

namespace cg = cooperative_groups;

namespace b200gan {

struct McFwdP {
  int N, Din, H1, H2;
  float slope;
  int sigmoid;  // out = sigmoid(W3 a2 + b3)
  const float *x, *W1, *b1, *W2, *b2, *W3, *b3;
  float *out, *m1, *a1, *m2, *a2;
};

struct McBwdP {
  int N, Din, H1, H2;
  const float *dout, *x, *W1, *W2, *W3, *m1, *a1, *m2, *a2;
  float *dx, *dW1, *db1, *dW2, *db2, *dW3, *db3, *U1, *U2;
  const float *y;  // non-NULL: the Sigmoid mode; y is the forward's output, g [N] the gradient at the logits
  float *g;
};

struct McDbwdP {
  int N, Din, H1, H2;
  const float *u, *dout, *U1, *U2, *m1, *m2, *W1, *W2, *W3;
  float *dW1, *dW2, *dW3, *ddout, *t, *s;
};

// out[r] = sum_c A[r][c] * w[c] (+ bias), one warp per row; sigmoid of that when sig
__device__ __forceinline__ void row_dots(const float *A, const float *w, const float *bias, float *out, int R, int C,
                                         int sig = 0) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int r = blockIdx.x * 8 + warp; r < R; r += gridDim.x * 8) {
    float s = 0.f;
    for (int c = lane; c < C; c += 32) s = fmaf(A[(size_t)r * C + c], w[c], s);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (lane == 0) {
      const float v = bias ? s + bias[0] : s;
      out[r] = sig ? 1.f / (1.f + expf(-v)) : v;
    }
  }
}

// out[c] = sum_r (wr ? wr[r] : 1) * A[r][c], one thread per column
__device__ __forceinline__ void col_sums(const float *A, const float *wr, float *out, int R, int C) {
  for (int c = blockIdx.x * blockDim.x + threadIdx.x; c < C; c += gridDim.x * blockDim.x) {
    float s = 0.f;
    if (wr)
      for (int r = 0; r < R; ++r) s = fmaf(wr[r], A[(size_t)r * C + c], s);
    else
      for (int r = 0; r < R; ++r) s += A[(size_t)r * C + c];
    out[c] = s;
  }
}

// one LeakyReLU layer over R rows: h = A W^T + b with A [R][K], W [J][K];  m = lrelu'(h), a = h m, both [R][J]
__device__ __forceinline__ void lrelu_layer(const float *A, const float *W, const float *b, float slope, float *m,
                                            float *a, int R, int K, int J, float (*As)[GT + 1], float (*Bs)[GT + 1]) {
  for (int t = blockIdx.x; t < ntiles(R, J); t += gridDim.x)
    tile_gemm(A, K, 1, W, 1, K, R, J, K, t,
              [&](int r, int j, float acc) {
                const float h = acc + b[j];
                const float mk = h > 0.f ? 1.f : slope;
                m[(size_t)r * J + j] = mk;
                a[(size_t)r * J + j] = h * mk;
              }, As, Bs);
}

__global__ void __launch_bounds__(256) mlp_critic_fwd_kernel(McFwdP p) {
  __shared__ float As[GT][GT + 1];
  __shared__ float Bs[GT][GT + 1];
  cg::grid_group grid = cg::this_grid();
  // P1: h1 = x W1^T + b1
  lrelu_layer(p.x, p.W1, p.b1, p.slope, p.m1, p.a1, p.N, p.Din, p.H1, As, Bs);
  grid.sync();
  // P2: h2 = a1 W2^T + b2
  lrelu_layer(p.a1, p.W2, p.b2, p.slope, p.m2, p.a2, p.N, p.H1, p.H2, As, Bs);
  grid.sync();
  // P3: out = a2 W3^T + b3 (or its sigmoid)
  row_dots(p.a2, p.W3, p.b3, p.out, p.N, p.H2, p.sigmoid);
}

__global__ void __launch_bounds__(256) mlp_critic_bwd_kernel(McBwdP p) {
  __shared__ float As[GT][GT + 1];
  __shared__ float Bs[GT][GT + 1];
  cg::grid_group grid = cg::this_grid();
  const int N = p.N, Din = p.Din, H1 = p.H1, H2 = p.H2;
  const int nb = gridDim.x, bid = blockIdx.x;
  const int64_t gtid = (int64_t)bid * blockDim.x + threadIdx.x, gthreads = (int64_t)nb * blockDim.x;
  // P0 (Sigmoid mode): g = dout * y * (1 - y), the gradient at the logits, which P1-P3 read in place of dout
  if (p.y) {
    for (int64_t i = gtid; i < N; i += gthreads) p.g[i] = p.dout[i] * p.y[i] * (1.f - p.y[i]);
    grid.sync();
  }
  const float *dout = p.y ? p.g : p.dout;
  // P1: U2 = dout W3 * m2;  dW3 = dout^T a2;  db3 = sum dout
  for (int64_t i = gtid; i < (int64_t)N * H2; i += gthreads) {
    const int n = (int)(i / H2), j = (int)(i % H2);
    p.U2[i] = dout[n] * p.W3[j] * p.m2[i];
  }
  if (p.dW3) col_sums(p.a2, dout, p.dW3, N, H2);
  if (p.db3 && gtid == 0) {
    float s = 0.f;
    for (int n = 0; n < N; ++n) s += dout[n];
    p.db3[0] = s;
  }
  grid.sync();
  // P2: dW2 = U2^T a1;  U1 = (U2 W2) * m1;  db2 = sum_n U2
  {
    const int ta = p.dW2 ? ntiles(H2, H1) : 0, tb = ntiles(N, H1);
    for (int t = bid; t < ta + tb; t += nb) {
      if (t < ta)
        tile_gemm(p.U2, 1, H2, p.a1, H1, 1, H2, H1, N, t,
                  [&](int j, int i, float acc) { p.dW2[(size_t)j * H1 + i] = acc; }, As, Bs);
      else
        tile_gemm(p.U2, H2, 1, p.W2, H1, 1, N, H1, H2, t - ta,
                  [&](int n, int i, float acc) { p.U1[(size_t)n * H1 + i] = acc * p.m1[(size_t)n * H1 + i]; }, As,
                  Bs);
    }
    if (p.db2) col_sums(p.U2, nullptr, p.db2, N, H2);
  }
  grid.sync();
  // P3: dW1 = U1^T x;  dx = U1 W1;  db1 = sum_n U1
  {
    const int ta = p.dW1 ? ntiles(H1, Din) : 0, tb = p.dx ? ntiles(N, Din) : 0;
    for (int t = bid; t < ta + tb; t += nb) {
      if (t < ta)
        tile_gemm(p.U1, 1, H1, p.x, Din, 1, H1, Din, N, t,
                  [&](int i, int d, float acc) { p.dW1[(size_t)i * Din + d] = acc; }, As, Bs);
      else
        tile_gemm(p.U1, H1, 1, p.W1, Din, 1, N, Din, H1, t - ta,
                  [&](int n, int d, float acc) { p.dx[(size_t)n * Din + d] = acc; }, As, Bs);
    }
    if (p.db1) col_sums(p.U1, nullptr, p.db1, N, H1);
  }
}

__global__ void __launch_bounds__(256) mlp_critic_dbwd_kernel(McDbwdP p) {
  __shared__ float As[GT][GT + 1];
  __shared__ float Bs[GT][GT + 1];
  cg::grid_group grid = cg::this_grid();
  const int N = p.N, Din = p.Din, H1 = p.H1, H2 = p.H2;
  const int nb = gridDim.x, bid = blockIdx.x;
  const bool want_s = p.dW3 || p.ddout, want_t = want_s || p.dW2;
  // P1: dW1 = U1^T u;  t = (u W1^T) * m1
  {
    const int ta = p.dW1 ? ntiles(H1, Din) : 0, tb = want_t ? ntiles(N, H1) : 0;
    for (int t = bid; t < ta + tb; t += nb) {
      if (t < ta)
        tile_gemm(p.U1, 1, H1, p.u, Din, 1, H1, Din, N, t,
                  [&](int i, int d, float acc) { p.dW1[(size_t)i * Din + d] = acc; }, As, Bs);
      else
        tile_gemm(p.u, Din, 1, p.W1, 1, Din, N, H1, Din, t - ta,
                  [&](int n, int i, float acc) { p.t[(size_t)n * H1 + i] = acc * p.m1[(size_t)n * H1 + i]; }, As,
                  Bs);
    }
  }
  grid.sync();
  // P2: dW2 = U2^T t;  s = (t W2^T) * m2
  {
    const int ta = p.dW2 ? ntiles(H2, H1) : 0, tb = want_s ? ntiles(N, H2) : 0;
    for (int t = bid; t < ta + tb; t += nb) {
      if (t < ta)
        tile_gemm(p.U2, 1, H2, p.t, H1, 1, H2, H1, N, t,
                  [&](int j, int i, float acc) { p.dW2[(size_t)j * H1 + i] = acc; }, As, Bs);
      else
        tile_gemm(p.t, H1, 1, p.W2, 1, H1, N, H2, H1, t - ta,
                  [&](int n, int j, float acc) { p.s[(size_t)n * H2 + j] = acc * p.m2[(size_t)n * H2 + j]; }, As,
                  Bs);
    }
  }
  grid.sync();
  // P3: dW3 = sum_n dout_n s_n;  d(dout)_n = s_n . W3
  if (p.dW3) col_sums(p.s, p.dout, p.dW3, N, H2);
  if (p.ddout) row_dots(p.s, p.W3, nullptr, p.ddout, N, H2);
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
// with gx = dD/dx, r_n = ||gx_n||_2, the penalty term lambda * mean((r - 1)^2) and coef_n = lambda * (2/N) (r_n - 1) / r_n
// (the term's derivative w.r.t. r_n, over r_n), and coef_n = 0 where r_n = 0.
// Bias gradients come from the real/fake rows only (the penalty does not depend on the biases).
struct CsP {
  int N, Din, H1, H2;
  float slope, lambda_gp;
  const float *real, *fake, *alpha, *W1, *b1, *W2, *b2, *W3, *b3;
  float *losses;  // [2]: d_loss, lambda * gp
  float *dW1, *db1, *dW2, *db2, *dW3, *db3;
  float *X3, *A1, *U1, *M1, *A2, *U2, *M2, *dout, *coef;
};

// The bound only caps ptxas at 64 registers; launch_coop still runs two blocks per SM.  Without it ptxas spills values
// live across the division subroutine calls; under a two-block bound (128 registers) the kernel runs ~3% slower than
// at 64 (206.5 vs 200.6 us per launch, N = 64, 1024 -> 512 -> 256, H100 80GB HBM3 at 700 W).
__global__ void __launch_bounds__(256, 4) critic_step_kernel(CsP p) {
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
  lrelu_layer(p.X3, p.W1, p.b1, p.slope, p.M1, p.A1, R, Din, H1, As, Bs);
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
      // r = 0 (a zero input gradient): torch's norm backward passes 0 there, and 0 * (-inf) would be NaN
      const float c = r == 0.f ? 0.f : p.lambda_gp * (2.f / (float)N) * (r - 1.f) / r;
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
    col_sums(p.U1, nullptr, p.db1, 2 * N, H1);
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
    col_sums(p.U2, nullptr, p.db2, 2 * N, H2);
  }
  grid.sync();
  // P8: dW3 = sum_r dout_r * A2_r;  db3 = sum over the real / fake rows of dout
  col_sums(p.A2, p.dout, p.dW3, R, H2);
  if (gtid == 0) {
    float s = 0.f;
    for (int r = 0; r < 2 * N; ++r) s += p.dout[r];
    p.db3[0] = s;
  }
}

// one persistent cooperative launch, grid sized to the device's SMs (at most two blocks per SM)
template <class P>
static int launch_coop(void (*kernel)(P), P &p, void *stream, const char *what) {
  int per_sm = 0;
  B2_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, 256, 0));
  B2_CHECK_ARG(per_sm >= 1, "%s: kernel cannot be made resident", what);
  const int grid = num_sms() * (per_sm > 2 ? 2 : per_sm);
  void *args[] = {&p};
  B2_CUDA(cudaLaunchCooperativeKernel((const void *)kernel, dim3(grid), dim3(256), args, 0, as_stream(stream)));
  return B200GAN_OK;
}

static bool dims_ok(const b200gan_mlp_critic_desc *d) {
  return d->N > 0 && d->Din > 0 && d->H1 > 0 && d->H2 > 0;
}

static int critic_fwd(const b200gan_mlp_critic_desc *d, const float *x, const float *W1, const float *b1,
                      const float *W2, const float *b2, const float *W3, const float *b3, float *out, float *m1,
                      float *a1, float *m2, float *a2, int sigmoid, void *stream, const char *what) {
  B2_CHECK_ARG(d && x && W1 && b1 && W2 && b2 && W3 && b3 && out && m1 && a1 && m2 && a2, "%s: null pointer", what);
  B2_CHECK_ARG(dims_ok(d), "%s: bad dims", what);
  McFwdP p;
  p.N = d->N; p.Din = d->Din; p.H1 = d->H1; p.H2 = d->H2; p.slope = d->slope; p.sigmoid = sigmoid;
  p.x = x; p.W1 = W1; p.b1 = b1; p.W2 = W2; p.b2 = b2; p.W3 = W3; p.b3 = b3;
  p.out = out; p.m1 = m1; p.a1 = a1; p.m2 = m2; p.a2 = a2;
  return launch_coop(mlp_critic_fwd_kernel, p, stream, what);
}

// y == NULL: the critic backward for dout; else the Sigmoid mode, g in the workspace after U1 and U2
static int critic_bwd(const b200gan_mlp_critic_desc *d, const float *dout, const float *y, const float *x,
                      const float *W1, const float *W2, const float *W3, const float *m1, const float *a1,
                      const float *m2, const float *a2, float *dx, float *dW1, float *db1, float *dW2, float *db2,
                      float *dW3, float *db3, float *U1, float *U2, float *workspace, void *stream, const char *what) {
  B2_CHECK_ARG(d && dout && W2 && W3 && m1 && m2, "%s: null pointer", what);
  B2_CHECK_ARG(dims_ok(d), "%s: bad dims", what);
  B2_CHECK_ARG(!dx || W1, "%s: dx needs W1", what);
  B2_CHECK_ARG(!dW1 || x, "%s: dW1 needs x", what);
  B2_CHECK_ARG(!dW2 || a1, "%s: dW2 needs a1", what);
  B2_CHECK_ARG(!dW3 || a2, "%s: dW3 needs a2", what);
  B2_CHECK_ARG((U1 && U2) || workspace, "%s: U1/U2 need a workspace when not requested", what);
  McBwdP p;
  p.N = d->N; p.Din = d->Din; p.H1 = d->H1; p.H2 = d->H2;
  p.dout = dout; p.x = x; p.W1 = W1; p.W2 = W2; p.W3 = W3; p.m1 = m1; p.a1 = a1; p.m2 = m2; p.a2 = a2;
  p.dx = dx; p.dW1 = dW1; p.db1 = db1; p.dW2 = dW2; p.db2 = db2; p.dW3 = dW3; p.db3 = db3;
  p.U1 = U1 ? U1 : workspace;
  p.U2 = U2 ? U2 : workspace + (size_t)d->N * d->H1;
  p.y = y;
  p.g = y ? workspace + (size_t)d->N * ((size_t)d->H1 + d->H2) : nullptr;
  return launch_coop(mlp_critic_bwd_kernel, p, stream, what);
}

}  // namespace b200gan

using namespace b200gan;

extern "C" int b200gan_mlp_critic_fwd(const b200gan_mlp_critic_desc *d, const float *x, const float *W1,
                                      const float *b1, const float *W2, const float *b2, const float *W3,
                                      const float *b3, float *out, float *m1, float *a1, float *m2, float *a2,
                                      void *stream) {
  return critic_fwd(d, x, W1, b1, W2, b2, W3, b3, out, m1, a1, m2, a2, 0, stream, "mlp_critic_fwd");
}

extern "C" size_t b200gan_mlp_critic_bwd_workspace_floats(const b200gan_mlp_critic_desc *d) {
  if (!d) return 0;
  return (size_t)d->N * ((size_t)d->H1 + d->H2);
}

extern "C" int b200gan_mlp_critic_bwd(const b200gan_mlp_critic_desc *d, const float *dout, const float *x,
                                      const float *W1, const float *W2, const float *W3, const float *m1,
                                      const float *a1, const float *m2, const float *a2, float *dx, float *dW1,
                                      float *db1, float *dW2, float *db2, float *dW3, float *db3, float *U1, float *U2,
                                      float *workspace, void *stream) {
  return critic_bwd(d, dout, nullptr, x, W1, W2, W3, m1, a1, m2, a2, dx, dW1, db1, dW2, db2, dW3, db3, U1, U2,
                    workspace, stream, "mlp_critic_bwd");
}

extern "C" size_t b200gan_mlp_critic_dbwd_workspace_floats(const b200gan_mlp_critic_desc *d) {
  if (!d) return 0;
  return (size_t)d->N * ((size_t)d->H1 + d->H2);
}

extern "C" int b200gan_mlp_critic_dbwd(const b200gan_mlp_critic_desc *d, const float *u, const float *dout,
                                       const float *U1, const float *U2, const float *m1, const float *m2,
                                       const float *W1, const float *W2, const float *W3, float *dW1, float *dW2,
                                       float *dW3, float *ddout, float *workspace, void *stream) {
  B2_CHECK_ARG(d && u && dout && U1 && U2 && m1 && m2 && W1 && W2 && W3 && workspace,
               "mlp_critic_dbwd: null pointer");
  B2_CHECK_ARG(dims_ok(d), "mlp_critic_dbwd: bad dims");
  McDbwdP p;
  p.N = d->N; p.Din = d->Din; p.H1 = d->H1; p.H2 = d->H2;
  p.u = u; p.dout = dout; p.U1 = U1; p.U2 = U2; p.m1 = m1; p.m2 = m2; p.W1 = W1; p.W2 = W2; p.W3 = W3;
  p.dW1 = dW1; p.dW2 = dW2; p.dW3 = dW3; p.ddout = ddout;
  p.t = workspace;
  p.s = workspace + (size_t)d->N * d->H1;
  return launch_coop(mlp_critic_dbwd_kernel, p, stream, "mlp_critic_dbwd");
}

extern "C" int b200gan_mlp_disc_fwd(const b200gan_mlp_critic_desc *d, const float *x, const float *W1, const float *b1,
                                    const float *W2, const float *b2, const float *W3, const float *b3, float *y,
                                    float *m1, float *a1, float *m2, float *a2, void *stream) {
  return critic_fwd(d, x, W1, b1, W2, b2, W3, b3, y, m1, a1, m2, a2, 1, stream, "mlp_disc_fwd");
}

extern "C" size_t b200gan_mlp_disc_bwd_workspace_floats(const b200gan_mlp_critic_desc *d) {
  if (!d) return 0;
  return (size_t)d->N * ((size_t)d->H1 + d->H2 + 1);
}

extern "C" int b200gan_mlp_disc_bwd(const b200gan_mlp_critic_desc *d, const float *dout, const float *y,
                                    const float *x, const float *W1, const float *W2, const float *W3,
                                    const float *m1, const float *a1, const float *m2, const float *a2, float *dx,
                                    float *dW1, float *db1, float *dW2, float *db2, float *dW3, float *db3,
                                    float *workspace, void *stream) {
  B2_CHECK_ARG(y && workspace, "mlp_disc_bwd: null pointer");
  return critic_bwd(d, dout, y, x, W1, W2, W3, m1, a1, m2, a2, dx, dW1, db1, dW2, db2, dW3, db3, nullptr, nullptr,
                    workspace, stream, "mlp_disc_bwd");
}

extern "C" size_t b200gan_critic_step_workspace_floats(const b200gan_mlp_critic_desc *d) {
  if (!d) return 0;
  const size_t R = (size_t)3 * d->N;
  return R * ((size_t)d->Din + 3 * (size_t)d->H1 + 3 * (size_t)d->H2 + 1) + d->N + 64;
}

extern "C" int b200gan_critic_step_mlp(const b200gan_mlp_critic_desc *d, float lambda_gp, const float *real,
                                       const float *fake, const float *alpha, const float *W1, const float *b1,
                                       const float *W2, const float *b2, const float *W3, const float *b3,
                                       float *losses, float *dW1, float *db1, float *dW2, float *db2, float *dW3,
                                       float *db3, float *workspace, void *stream) {
  B2_CHECK_ARG(d && real && fake && alpha && W1 && b1 && W2 && b2 && W3 && b3 && losses && dW1 && db1 && dW2 && db2 &&
                   dW3 && db3 && workspace, "critic_step_mlp: null pointer");
  B2_CHECK_ARG(dims_ok(d), "critic_step_mlp: bad dims");
  CsP p;
  p.N = d->N; p.Din = d->Din; p.H1 = d->H1; p.H2 = d->H2; p.slope = d->slope; p.lambda_gp = lambda_gp;
  p.real = real; p.fake = fake; p.alpha = alpha; p.W1 = W1; p.b1 = b1; p.W2 = W2; p.b2 = b2; p.W3 = W3; p.b3 = b3;
  p.losses = losses; p.dW1 = dW1; p.db1 = db1; p.dW2 = dW2; p.db2 = db2; p.dW3 = dW3; p.db3 = db3;
  const size_t R = (size_t)3 * d->N;
  float *w = workspace;
  p.X3 = w; w += R * d->Din;
  p.A1 = w; w += R * d->H1; p.U1 = w; w += R * d->H1; p.M1 = w; w += R * d->H1;
  p.A2 = w; w += R * d->H2; p.U2 = w; w += R * d->H2; p.M2 = w; w += R * d->H2;
  p.dout = w; w += R;
  p.coef = w;
  return launch_coop(critic_step_kernel, p, stream, "critic_step_mlp");
}
