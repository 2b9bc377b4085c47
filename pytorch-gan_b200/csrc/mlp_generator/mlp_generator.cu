// mlp_generator.cu -- the MLP generator of wgan_gp.py:42-65 / gan.py:38-61 as two cooperative kernels:
//   [Linear -> (BatchNorm1d)? -> LeakyReLU(s)] x (L - 1), Linear -> Tanh       (include/b200gan.h: b200gan_mlp_gen_*)
//   forward    per layer: h = a W^T + b;  norm: column mean / biased variance, xhat = (h - mean) rstd,
//              y = gamma xhat + beta, running statistics;  a = lrelu(y);   out = tanh(a W^T + b)
//   backward   g = dout (1 - out^2);  per layer, top down: dW = g^T a_in, db = sum_n g, da = g W;  dy = da lrelu'(a);
//              norm: dbeta = sum_n dy, dgamma = sum_n dy xhat, dh = gamma rstd (dy - dbeta / N - xhat dgamma / N)
// At N = 64 every layer is a few MFLOP and latency bound, so each pass is ONE persistent cooperative launch whose
// dependent phases are separated by grid.sync(); the GEMM phases spread 32x32 fp32 FFMA output tiles (tile_gemm.cuh)
// over the grid, the column phases run one thread per column over the rows in order: the results are deterministic and
// independent of the grid size.  The LeakyReLU derivative is read from the sign of the stored activation a (slope >= 0:
// a > 0 exactly where y > 0), as torch's in-place LeakyReLU backward does.
#include "../common.cuh"
#include "../tile_gemm.cuh"
#include <cooperative_groups.h>

namespace cg = cooperative_groups;

namespace b200gan {

constexpr int MGL = B200GAN_MLP_GEN_MAX_LAYERS;

struct MgFwdP {
  int L, N;
  int w[MGL + 1];
  int norm[MGL];
  float slope, eps, momentum;
  const float *z, *W[MGL], *b[MGL], *gamma[MGL], *beta[MGL];
  float *rm[MGL], *rv[MGL];
  int64_t *nbt[MGL];
  float *out, *h;
  float *act[MGL], *xhat[MGL], *rstd[MGL];  // xhat / rstd NULL: no backward follows
};

struct MgBwdP {
  int L, N;
  int w[MGL + 1];
  int norm[MGL];
  int need_g[MGL];  // the gradient w.r.t. h_l is formed
  int prop[MGL];    // ... and multiplied back through W_l (dz for l = 0)
  float slope;
  const float *dout, *z, *out, *W[MGL], *gamma[MGL], *act[MGL], *xhat[MGL], *rstd[MGL];
  float *dz, *dW[MGL], *db[MGL], *dgamma[MGL], *dbeta[MGL];
  float *g0, *g1;
};

__device__ __forceinline__ float lrelu(float v, float slope) { return v > 0.f ? v : v * slope; }

// BatchNorm1d over the columns of h [N][C], one thread per column: statistics, running statistics, normalise, LeakyReLU
__device__ __forceinline__ void norm_fwd(const MgFwdP &p, int l, const float *h, float *a, int N, int C) {
  const float *gam = p.gamma[l], *bet = p.beta[l];
  float *xh = p.xhat[l], *rs = p.rstd[l], *rm = p.rm[l], *rv = p.rv[l];
  for (int c = blockIdx.x * blockDim.x + threadIdx.x; c < C; c += gridDim.x * blockDim.x) {
    float s = 0.f;
#pragma unroll 8
    for (int r = 0; r < N; ++r) s += h[(size_t)r * C + c];
    const float mean = s / (float)N;
    float q = 0.f;
#pragma unroll 8
    for (int r = 0; r < N; ++r) {
      const float d = h[(size_t)r * C + c] - mean;
      q = fmaf(d, d, q);
    }
    const float var = q / (float)N;
    const float rstd = 1.f / sqrtf(var + p.eps);
    const float gm = gam[c], bt = bet[c];
#pragma unroll 4
    for (int r = 0; r < N; ++r) {
      const float x = (h[(size_t)r * C + c] - mean) * rstd;
      if (xh) xh[(size_t)r * C + c] = x;
      a[(size_t)r * C + c] = lrelu(fmaf(x, gm, bt), p.slope);
    }
    if (rs) rs[c] = rstd;
    if (rm) {
      rm[c] = (1.f - p.momentum) * rm[c] + p.momentum * mean;
      rv[c] = (1.f - p.momentum) * rv[c] + p.momentum * (q / (float)(N - 1));
    }
  }
  if (p.nbt[l] && blockIdx.x == 0 && threadIdx.x == 0) p.nbt[l][0] += 1;
}

__global__ void __launch_bounds__(256) mlp_gen_fwd_kernel(const __grid_constant__ MgFwdP p) {
  __shared__ float As[GT][GT + 1];
  __shared__ float Bs[GT][GT + 1];
  cg::grid_group grid = cg::this_grid();
  const int N = p.N, L = p.L;
  const float slope = p.slope;
  const float *x = p.z;
  for (int l = 0; l < L; ++l) {
    const int K = p.w[l], J = p.w[l + 1];
    const float *W = p.W[l], *b = p.b[l];
    const bool last = l == L - 1, norm = p.norm[l] != 0;
    float *y = last ? p.out : (norm ? p.h : p.act[l]);
    // h = x W^T + b, with the bias, LeakyReLU (no norm) or Tanh (last layer) in the epilogue
    for (int t = blockIdx.x; t < ntiles(N, J); t += gridDim.x)
      tile_gemm(x, K, 1, W, 1, K, N, J, K, t,
                [&](int r, int j, float acc) {
                  const float v = acc + b[j];
                  y[(size_t)r * J + j] = last ? tanhf(v) : (norm ? v : lrelu(v, slope));
                }, As, Bs);
    if (last) break;
    grid.sync();
    if (norm) {
      norm_fwd(p, l, p.h, p.act[l], N, J);
      grid.sync();
    }
    x = p.act[l];
  }
}

__global__ void __launch_bounds__(256) mlp_gen_bwd_kernel(const __grid_constant__ MgBwdP p) {
  __shared__ float As[GT][GT + 1];
  __shared__ float Bs[GT][GT + 1];
  cg::grid_group grid = cg::this_grid();
  const int N = p.N, L = p.L;
  const float slope = p.slope;
  const int64_t gtid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x, gthreads = (int64_t)gridDim.x * blockDim.x;
  if (!p.need_g[L - 1]) return;  // nothing asked for (uniform over the grid)
  // P0: g = dout * tanh'
  for (int64_t i = gtid; i < (int64_t)N * p.w[L]; i += gthreads) {
    const float o = p.out[i];
    p.g0[i] = p.dout[i] * (1.f - o * o);
  }
  grid.sync();
  float *g = p.g0, *gn = p.g1;
  for (int l = L - 1; l >= 0 && p.need_g[l]; --l) {
    const int K = p.w[l], J = p.w[l + 1];
    const float *ain = l == 0 ? p.z : p.act[l - 1];
    float *dW = p.dW[l], *db = p.db[l];
    const bool prop = p.prop[l] != 0;
    // dW = g^T a_in;  da = g W, times lrelu'(a_in) below the first layer (dz at the first);  db = sum_n g
    const int ta = dW ? ntiles(J, K) : 0, tb = prop ? ntiles(N, K) : 0;
    for (int t = blockIdx.x; t < ta + tb; t += gridDim.x) {
      if (t < ta)
        tile_gemm(g, 1, J, ain, K, 1, J, K, N, t, [&](int j, int i, float acc) { dW[(size_t)j * K + i] = acc; }, As,
                  Bs);
      else
        tile_gemm(g, J, 1, p.W[l], K, 1, N, K, J, t - ta,
                  [&](int n, int i, float acc) {
                    const size_t e = (size_t)n * K + i;
                    if (l == 0)
                      p.dz[e] = acc;
                    else
                      gn[e] = ain[e] > 0.f ? acc : acc * slope;
                  }, As, Bs);
    }
    if (db)
      for (int c = (int)gtid; c < J; c += (int)gthreads) {
        float s = 0.f;
#pragma unroll 8
        for (int r = 0; r < N; ++r) s += g[(size_t)r * J + c];
        db[c] = s;
      }
    if (!prop || l == 0) break;
    grid.sync();
    if (p.norm[l - 1]) {
      // BatchNorm1d backward over the columns of dy (in gn, overwritten by dh)
      const float *xh = p.xhat[l - 1], *rs = p.rstd[l - 1], *gam = p.gamma[l - 1];
      float *dgam = p.dgamma[l - 1], *dbet = p.dbeta[l - 1];
      const bool want_dh = p.need_g[l - 1] != 0;
      for (int c = (int)gtid; c < K; c += (int)gthreads) {
        float s1 = 0.f, s2 = 0.f;
#pragma unroll 8
        for (int r = 0; r < N; ++r) {
          const float dy = gn[(size_t)r * K + c];
          s1 += dy;
          s2 = fmaf(dy, xh[(size_t)r * K + c], s2);
        }
        if (dbet) dbet[c] = s1;
        if (dgam) dgam[c] = s2;
        if (want_dh) {
          const float k = gam[c] * rs[c], m1 = s1 / (float)N, m2 = s2 / (float)N;
#pragma unroll 4
          for (int r = 0; r < N; ++r) {
            const size_t e = (size_t)r * K + c;
            gn[e] = k * (gn[e] - m1 - xh[e] * m2);
          }
        }
      }
      grid.sync();
    }
    float *tmp = g;
    g = gn;
    gn = tmp;
  }
}

// one persistent cooperative launch: the grid is what the device holds resident, at most two blocks per SM
template <class P>
static int launch_gen(void (*kernel)(const P), const P &p, void *stream, const char *what) {
  int dev = 0, coop = 0, per_sm = 0;
  B2_CUDA(cudaGetDevice(&dev));
  B2_CUDA(cudaDeviceGetAttribute(&coop, cudaDevAttrCooperativeLaunch, dev));
  if (!coop) B2_UNSUPPORTED("%s: the device does not support cooperative launches", what);
  B2_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, 256, 0));
  if (per_sm < 1) B2_UNSUPPORTED("%s: kernel cannot be made resident", what);
  const int grid = num_sms() * (per_sm > 2 ? 2 : per_sm);
  void *args[] = {const_cast<P *>(&p)};
  B2_CUDA(cudaLaunchCooperativeKernel((const void *)kernel, dim3(grid), dim3(256), args, 0, as_stream(stream)));
  return B200GAN_OK;
}

static bool has_any_norm(const b200gan_mlp_gen_desc *d) {
  for (int l = 0; l + 1 < d->L; ++l)
    if (d->has_norm[l]) return true;
  return false;
}

// the sizes the kernels take (what the size queries need)
static int check_dims(const b200gan_mlp_gen_desc *d, const char *what) {
  B2_CHECK_ARG(d, "%s: null descriptor", what);
  B2_CHECK_ARG(d->L >= 1 && d->L <= MGL, "%s: L = %d outside [1, %d]", what, d->L, MGL);
  B2_CHECK_ARG(d->N >= 1 && d->N <= B200GAN_MLP_GEN_MAX_N, "%s: N = %d outside [1, %d]", what, d->N,
               B200GAN_MLP_GEN_MAX_N);
  for (int l = 0; l <= d->L; ++l)
    B2_CHECK_ARG(d->width[l] >= 1 && d->width[l] <= B200GAN_MLP_GEN_MAX_WIDTH, "%s: width[%d] = %d outside [1, %d]",
                 what, l, d->width[l], B200GAN_MLP_GEN_MAX_WIDTH);
  B2_CHECK_ARG(!d->has_norm[d->L - 1], "%s: the last layer (Linear -> Tanh) has no norm", what);
  B2_CHECK_ARG(!has_any_norm(d) || d->N >= 2, "%s: BatchNorm1d in training needs more than 1 value per channel (N = %d)",
               what, d->N);
  return B200GAN_OK;
}

static int check_desc(const b200gan_mlp_gen_desc *d, const char *what) {
  const int rc = check_dims(d, what);
  if (rc != B200GAN_OK) return rc;
  B2_CHECK_ARG(d->slope >= 0.f, "%s: negative LeakyReLU slope", what);
  for (int l = 0; l < d->L; ++l) {
    B2_CHECK_ARG(d->W[l], "%s: null W[%d]", what, l);
    if (l + 1 < d->L && d->has_norm[l]) {
      B2_CHECK_ARG(d->gamma[l] && d->beta[l], "%s: null gamma / beta of norm layer %d", what, l);
      const bool any = d->running_mean[l] || d->running_var[l] || d->num_batches_tracked[l];
      const bool all = d->running_mean[l] && d->running_var[l] && d->num_batches_tracked[l];
      B2_CHECK_ARG(any == all, "%s: running statistics of layer %d are partly NULL", what, l);
    }
  }
  return B200GAN_OK;
}

static size_t max_width(const b200gan_mlp_gen_desc *d) {
  size_t m = 0;
  for (int l = 1; l <= d->L; ++l) m = d->width[l] > (int)m ? (size_t)d->width[l] : m;
  return m;
}

// the saved region's pointers (act, xhat, rstd per layer; NULL where a layer has none)
static void saved_layout(const b200gan_mlp_gen_desc *d, float *saved, float **act, float **xhat, float **rstd) {
  float *q = saved;
  for (int l = 0; l < MGL; ++l) act[l] = xhat[l] = rstd[l] = nullptr;
  for (int l = 0; l + 1 < d->L; ++l) {
    act[l] = q;
    q += (size_t)d->N * d->width[l + 1];
  }
  for (int l = 0; l + 1 < d->L; ++l)
    if (d->has_norm[l]) {
      xhat[l] = q;
      q += (size_t)d->N * d->width[l + 1];
    }
  for (int l = 0; l + 1 < d->L; ++l)
    if (d->has_norm[l]) {
      rstd[l] = q;
      q += d->width[l + 1];
    }
}

}  // namespace b200gan

using namespace b200gan;

extern "C" size_t b200gan_mlp_gen_saved_floats(const b200gan_mlp_gen_desc *d) {
  if (check_dims(d, "mlp_gen_saved_floats") != B200GAN_OK) return 0;
  size_t n = 0;
  for (int l = 0; l + 1 < d->L; ++l) n += (size_t)(d->has_norm[l] ? 2 * d->N + 1 : d->N) * d->width[l + 1];
  return n;
}

extern "C" size_t b200gan_mlp_gen_workspace_floats(const b200gan_mlp_gen_desc *d) {
  if (check_dims(d, "mlp_gen_workspace_floats") != B200GAN_OK) return 0;
  return 3 * (size_t)d->N * max_width(d);
}

extern "C" int b200gan_mlp_gen_fwd(const b200gan_mlp_gen_desc *d, const float *z, float *out, float *saved,
                                   float *workspace, void *stream) {
  int rc = check_desc(d, "mlp_gen_fwd");
  if (rc != B200GAN_OK) return rc;
  B2_CHECK_ARG(z && out && workspace, "mlp_gen_fwd: null z, out or workspace");
  for (int l = 0; l < d->L; ++l) B2_CHECK_ARG(d->b[l], "mlp_gen_fwd: null b[%d]", l);
  MgFwdP p = {};
  p.L = d->L; p.N = d->N; p.slope = d->slope; p.eps = d->eps; p.momentum = d->momentum;
  const size_t slab = (size_t)d->N * max_width(d);
  p.h = workspace;
  if (saved) {
    saved_layout(d, saved, p.act, p.xhat, p.rstd);
  } else {  // no backward: the activations ping-pong through the workspace
    for (int l = 0; l + 1 < d->L; ++l) p.act[l] = workspace + (1 + (l & 1)) * slab;
  }
  for (int l = 0; l <= d->L; ++l) p.w[l] = d->width[l];
  for (int l = 0; l < d->L; ++l) {
    p.norm[l] = l + 1 < d->L && d->has_norm[l];
    p.W[l] = d->W[l]; p.b[l] = d->b[l];
    if (p.norm[l]) {
      p.gamma[l] = d->gamma[l]; p.beta[l] = d->beta[l];
      p.rm[l] = d->running_mean[l]; p.rv[l] = d->running_var[l]; p.nbt[l] = d->num_batches_tracked[l];
    }
  }
  p.z = z;
  p.out = out;
  return launch_gen(mlp_gen_fwd_kernel, p, stream, "mlp_gen_fwd");
}

extern "C" int b200gan_mlp_gen_bwd(const b200gan_mlp_gen_desc *d, const float *dout, const float *z, const float *out,
                                   const float *saved, float *dz, const b200gan_mlp_gen_grads *grads, float *workspace,
                                   void *stream) {
  int rc = check_desc(d, "mlp_gen_bwd");
  if (rc != B200GAN_OK) return rc;
  B2_CHECK_ARG(dout && out && grads && workspace && (saved || d->L == 1), "mlp_gen_bwd: null pointer");
  B2_CHECK_ARG(!grads->dW[0] || z, "mlp_gen_bwd: dW[0] needs z");
  MgBwdP p = {};
  p.L = d->L; p.N = d->N; p.slope = d->slope;
  float *act[MGL], *xhat[MGL], *rstd[MGL];
  saved_layout(d, const_cast<float *>(saved), act, xhat, rstd);
  for (int l = 0; l <= d->L; ++l) p.w[l] = d->width[l];
  // which gradients w.r.t. h_l are formed, and which are multiplied back through W_l, from the bottom up
  for (int l = 0; l < d->L; ++l) {
    p.norm[l] = l + 1 < d->L && d->has_norm[l];
    if (l == 0)
      p.prop[l] = dz != nullptr;
    else
      p.prop[l] = p.need_g[l - 1] || (p.norm[l - 1] && (grads->dgamma[l - 1] || grads->dbeta[l - 1]));
    p.need_g[l] = p.prop[l] || grads->dW[l] || grads->db[l];
    p.W[l] = d->W[l];
    p.act[l] = act[l]; p.xhat[l] = xhat[l]; p.rstd[l] = rstd[l];
    p.dW[l] = grads->dW[l]; p.db[l] = grads->db[l];
    if (p.norm[l]) {
      B2_CHECK_ARG(d->gamma[l], "mlp_gen_bwd: null gamma[%d]", l);
      p.gamma[l] = d->gamma[l]; p.dgamma[l] = grads->dgamma[l]; p.dbeta[l] = grads->dbeta[l];
    }
  }
  p.dout = dout; p.z = z; p.out = out; p.dz = dz;
  const size_t slab = (size_t)d->N * max_width(d);
  p.g0 = workspace;
  p.g1 = workspace + slab;
  return launch_gen(mlp_gen_bwd_kernel, p, stream, "mlp_gen_bwd");
}
