// mlp_critic.cu -- autograd of the MLP critic (wgan_gp.py:72-78, wgan_div.py:72-78) as three cooperative kernels:
//   D(x) = W3 lrelu(W2 lrelu(W1 x + b1) + b2) + b3,      Din -> H1 -> H2 -> 1, one LeakyReLU slope.
// Unlike gp_mlp.cu, no penalty is built in: the forward, the first-order backward for an arbitrary output gradient
// dout, and the double backward of the input gradient for an arbitrary upstream gradient u = dL/d(dD/dx) are separate
// entry points, so a script's own penalty arithmetic (||g|| - 1)^2, ||g||^p, ... stays in its autograd graph while every
// critic GEMM runs here.
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
#include "common.cuh"
#include "tile_gemm.cuh"
#include <cooperative_groups.h>

namespace cg = cooperative_groups;

namespace b200gan {

struct McFwdP {
  int N, Din, H1, H2;
  float slope;
  const float *x, *W1, *b1, *W2, *b2, *W3, *b3;
  float *out, *m1, *a1, *m2, *a2;
};

struct McBwdP {
  int N, Din, H1, H2;
  const float *dout, *x, *W1, *W2, *W3, *m1, *a1, *m2, *a2;
  float *dx, *dW1, *db1, *dW2, *db2, *dW3, *db3, *U1, *U2;
};

struct McDbwdP {
  int N, Din, H1, H2;
  const float *u, *dout, *U1, *U2, *m1, *m2, *W1, *W2, *W3;
  float *dW1, *dW2, *dW3, *ddout, *t, *s;
};

// out[r] = sum_c A[r][c] * w[c] (+ bias), one warp per row
__device__ __forceinline__ void row_dots(const float *A, const float *w, const float *bias, float *out, int R, int C) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int r = blockIdx.x * 8 + warp; r < R; r += gridDim.x * 8) {
    float s = 0.f;
    for (int c = lane; c < C; c += 32) s = fmaf(A[(size_t)r * C + c], w[c], s);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (lane == 0) out[r] = bias ? s + bias[0] : s;
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

__global__ void __launch_bounds__(256) mlp_critic_fwd_kernel(McFwdP p) {
  __shared__ float As[GT][GT + 1];
  __shared__ float Bs[GT][GT + 1];
  cg::grid_group grid = cg::this_grid();
  const int N = p.N, Din = p.Din, H1 = p.H1, H2 = p.H2;
  const int nb = gridDim.x, bid = blockIdx.x;
  // P1: h1 = x W1^T + b1
  for (int t = bid; t < ntiles(N, H1); t += nb)
    tile_gemm(p.x, Din, 1, p.W1, 1, Din, N, H1, Din, t,
              [&](int n, int j, float acc) {
                const float h = acc + p.b1[j];
                const float m = h > 0.f ? 1.f : p.slope;
                p.m1[(size_t)n * H1 + j] = m;
                p.a1[(size_t)n * H1 + j] = h * m;
              }, As, Bs);
  grid.sync();
  // P2: h2 = a1 W2^T + b2
  for (int t = bid; t < ntiles(N, H2); t += nb)
    tile_gemm(p.a1, H1, 1, p.W2, 1, H1, N, H2, H1, t,
              [&](int n, int j, float acc) {
                const float h = acc + p.b2[j];
                const float m = h > 0.f ? 1.f : p.slope;
                p.m2[(size_t)n * H2 + j] = m;
                p.a2[(size_t)n * H2 + j] = h * m;
              }, As, Bs);
  grid.sync();
  // P3: out = a2 W3^T + b3
  row_dots(p.a2, p.W3, p.b3, p.out, N, H2);
}

__global__ void __launch_bounds__(256) mlp_critic_bwd_kernel(McBwdP p) {
  __shared__ float As[GT][GT + 1];
  __shared__ float Bs[GT][GT + 1];
  cg::grid_group grid = cg::this_grid();
  const int N = p.N, Din = p.Din, H1 = p.H1, H2 = p.H2;
  const int nb = gridDim.x, bid = blockIdx.x;
  const int64_t gtid = (int64_t)bid * blockDim.x + threadIdx.x, gthreads = (int64_t)nb * blockDim.x;
  // P1: U2 = dout W3 * m2;  dW3 = dout^T a2;  db3 = sum dout
  for (int64_t i = gtid; i < (int64_t)N * H2; i += gthreads) {
    const int n = (int)(i / H2), j = (int)(i % H2);
    p.U2[i] = p.dout[n] * p.W3[j] * p.m2[i];
  }
  if (p.dW3) col_sums(p.a2, p.dout, p.dW3, N, H2);
  if (p.db3 && gtid == 0) {
    float s = 0.f;
    for (int n = 0; n < N; ++n) s += p.dout[n];
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

}  // namespace b200gan

using namespace b200gan;

extern "C" int b200gan_mlp_critic_fwd(const b200gan_mlp_critic_desc *d, const float *x, const float *W1,
                                      const float *b1, const float *W2, const float *b2, const float *W3,
                                      const float *b3, float *out, float *m1, float *a1, float *m2, float *a2,
                                      void *stream) {
  B2_CHECK_ARG(d && x && W1 && b1 && W2 && b2 && W3 && b3 && out && m1 && a1 && m2 && a2,
               "mlp_critic_fwd: null pointer");
  B2_CHECK_ARG(dims_ok(d), "mlp_critic_fwd: bad dims");
  McFwdP p;
  p.N = d->N; p.Din = d->Din; p.H1 = d->H1; p.H2 = d->H2; p.slope = d->slope;
  p.x = x; p.W1 = W1; p.b1 = b1; p.W2 = W2; p.b2 = b2; p.W3 = W3; p.b3 = b3;
  p.out = out; p.m1 = m1; p.a1 = a1; p.m2 = m2; p.a2 = a2;
  return launch_coop(mlp_critic_fwd_kernel, p, stream, "mlp_critic_fwd");
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
  B2_CHECK_ARG(d && dout && W2 && W3 && m1 && m2, "mlp_critic_bwd: null pointer");
  B2_CHECK_ARG(dims_ok(d), "mlp_critic_bwd: bad dims");
  B2_CHECK_ARG(!dx || W1, "mlp_critic_bwd: dx needs W1");
  B2_CHECK_ARG(!dW1 || x, "mlp_critic_bwd: dW1 needs x");
  B2_CHECK_ARG(!dW2 || a1, "mlp_critic_bwd: dW2 needs a1");
  B2_CHECK_ARG(!dW3 || a2, "mlp_critic_bwd: dW3 needs a2");
  B2_CHECK_ARG((U1 && U2) || workspace, "mlp_critic_bwd: U1/U2 need a workspace when not requested");
  McBwdP p;
  p.N = d->N; p.Din = d->Din; p.H1 = d->H1; p.H2 = d->H2;
  p.dout = dout; p.x = x; p.W1 = W1; p.W2 = W2; p.W3 = W3; p.m1 = m1; p.a1 = a1; p.m2 = m2; p.a2 = a2;
  p.dx = dx; p.dW1 = dW1; p.db1 = db1; p.dW2 = dW2; p.db2 = db2; p.dW3 = dW3; p.db3 = db3;
  p.U1 = U1 ? U1 : workspace;
  p.U2 = U2 ? U2 : workspace + (size_t)d->N * d->H1;
  return launch_coop(mlp_critic_bwd_kernel, p, stream, "mlp_critic_bwd");
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
