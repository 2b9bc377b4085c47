// norm.cu -- BatchNorm2d (training mode) and InstanceNorm2d on NHWC fp32 tensors.
//
// Reference call sites: nn.BatchNorm2d(128) / (C, 0.8) dcgan.py:53,56,60,80 (second positional
// argument is eps = 0.8, momentum stays 0.1); nn.InstanceNorm2d(C) pix2pix/models.py:25,40,117,
// cyclegan/models.py:29,33,51,61,76,108 (affine=False, no running stats, eps 1e-5).
// Statistics are kept per "group": g = c (BatchNorm) or n*C + c (InstanceNorm).  Normalisation
// uses the biased variance; running_var is updated with the unbiased one (torch semantics).
// All kernels are HBM-bound streaming passes with fp64 accumulation only at the final atomic.  The
// statistics are [sum x, sum x^2] per group, and the variance E[x^2]-E[x]^2 is formed from them in
// fp64.  fp32 partial sums taken from zero round relative to mean^2 + var, and the subtraction loses
// the variance in proportion to (mean / std)^2: a channel far from zero, or constant, would get an
// rstd wrong by O(1).  So every producer of those sums (norm_stats_kernel here, the conv_tc.cu and
// narrow_block.cu epilogues) sums x - p and (x - p)^2 around a pivot p taken from the group's own
// data and adds n p + sum(x - p) and sum(x - p)^2 + 2 p sum(x - p) + n p^2 in fp64; norm_stats and
// the conv epilogues add their plain sums instead where a block's mean is near zero
// (stats_plain_ok, common.cuh).
// Each pass has one kernel for every C: the
// apply and backward kernels are templated on the vector width (float4 along C, or scalar when C
// is not a multiple of 4 or an operand is not 16-byte aligned), and the backward always recomputes
// a LeakyReLU / ReLU mask from x when scale_shift is given.
#include "common.cuh"
#include <initializer_list>
#include <stdlib.h>

namespace b200gan {

// ---- statistics ---------------------------------------------------------------------------
// grid: (ceil(C/32), row_blocks, N or 1).  block (32, 8).
__global__ void __launch_bounds__(256)
norm_stats_kernel(const float *__restrict__ x, double *__restrict__ stats, int C, int64_t rows,
                  int64_t rows_per_block, int G, int per_sample) {
  __shared__ float s1[8][33], s2[8][33], s3[8][33], s4[8][33];
  const int c = blockIdx.x * 32 + threadIdx.x;
  const int64_t base_row = per_sample ? (int64_t)blockIdx.z * rows : 0;
  int64_t r0 = (int64_t)blockIdx.y * rows_per_block;
  int64_t r1 = r0 + rows_per_block;
  if (r1 > rows) r1 = rows;
  // plain sums a = sum x, b = sum x^2, and around the column's first row of the block, p: d = sum (x - p),
  // e = sum (x - p)^2, whose rounding is relative to the spread of the group rather than to its mean (stats_plain_ok)
  float a = 0.f, b = 0.f, d = 0.f, e = 0.f, p = 0.f;
  if (c < C) {
    const float *xp = x + (base_row + r0) * C + c;
    p = __ldg(xp);
    for (int64_t r = r0 + threadIdx.y; r < r1; r += 8) {
      const float v = __ldg(xp + (r - r0) * C), w = v - p;
      a += v;
      b = fmaf(v, v, b);
      d += w;
      e = fmaf(w, w, e);
    }
  }
  s1[threadIdx.y][threadIdx.x] = a;
  s2[threadIdx.y][threadIdx.x] = b;
  s3[threadIdx.y][threadIdx.x] = d;
  s4[threadIdx.y][threadIdx.x] = e;
  __syncthreads();
  if (threadIdx.y == 0 && c < C) {
    double ta = 0.0, tb = 0.0, td = 0.0, te = 0.0;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      ta += (double)s1[i][threadIdx.x];
      tb += (double)s2[i][threadIdx.x];
      td += (double)s3[i][threadIdx.x];
      te += (double)s4[i][threadIdx.x];
    }
    // the pivoted sums back to [sum x, sum x^2] in fp64: n p + d and e + 2 p d + n p^2 over the block's n rows
    const double n = (double)(r1 - r0), pd = (double)p;
    const double pa = fma(n, pd, td), pb = fma(n * pd, pd, fma(2.0 * pd, td, te));
    const bool plain = stats_plain_ok(pa, pb, n);
    int g = per_sample ? blockIdx.z * C + c : c;
    atomicAdd(stats + g, plain ? ta : pa);
    atomicAdd(stats + G + g, plain ? tb : pb);
  }
}

__global__ void norm_finalize_kernel(double *__restrict__ stats, const float *__restrict__ gamma,
                                     const float *__restrict__ beta, float *__restrict__ mean_rstd,
                                     float *__restrict__ scale_shift, float *running_mean,
                                     float *running_var, int64_t *nbt, int G, int C, double count,
                                     float eps, float momentum) {
  int g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g == 0 && nbt) *nbt += 1;
  if (g >= G) return;
  double mean = stats[g] / count;
  double var = stats[G + g] / count - mean * mean;
  stats[g] = 0.0;      // the accumulator is consumed: leave it zeroed for its next use (no memset launch needed)
  stats[G + g] = 0.0;
  if (var < 0.0) var = 0.0;
  float rstd = (float)(1.0 / sqrt(var + (double)eps));
  int c = g % C;
  float ga = gamma ? gamma[c] : 1.f;
  float be = beta ? beta[c] : 0.f;
  mean_rstd[g] = (float)mean;
  mean_rstd[G + g] = rstd;
  float sc = ga * rstd;
  scale_shift[g] = sc;
  scale_shift[G + g] = be - (float)mean * sc;
  if (running_mean) {
    double unbiased = count > 1.0 ? var * count / (count - 1.0) : var;
    running_mean[g] = (1.f - momentum) * running_mean[g] + momentum * (float)mean;
    running_var[g] = (1.f - momentum) * running_var[g] + momentum * (float)unbiased;
  }
}

// ---- apply and backward: one kernel per pass, templated on the vector width ---------------------------------------
// VEC = 4 (float4 along C) when C % 4 == 0 and the streamed operands are 16-byte aligned, else VEC = 1.  A thread keeps
// ONE channel group of VEC channels for its whole loop, so there is no index arithmetic beyond an add per row.
// grid = (row blocks, samples, channel slices): blockIdx.y selects the sample for per-sample (InstanceNorm) groups,
// else gridDim.y == 1; blockIdx.z selects a slice of at most 256 channel groups (C > 1024 at VEC 4, C > 256 at VEC 1).
// A block covers 256 / CVs rows of its slice's CVs groups; the 256 % CVs threads left over load nothing.
template <int VEC> struct vec_of;
template <> struct vec_of<4> { using type = float4; };
template <> struct vec_of<1> { using type = float; };

__device__ __forceinline__ void unpack(float4 v, float (&a)[4]) { a[0] = v.x; a[1] = v.y; a[2] = v.z; a[3] = v.w; }
__device__ __forceinline__ void unpack(float v, float (&a)[1]) { a[0] = v; }
__device__ __forceinline__ float4 pack(const float (&a)[4]) { return make_float4(a[0], a[1], a[2], a[3]); }
__device__ __forceinline__ float pack(const float (&a)[1]) { return a[0]; }

// this thread's place in the block's channel slice
struct GroupSlice {
  int CV;    // channel groups per row
  int cv;    // this thread's group: channels cv * VEC .. cv * VEC + VEC - 1
  int CVs;   // groups in the slice
  int rpb;   // rows per block
  int row;   // this thread's row within the block; == rpb for the threads left over
  __device__ __forceinline__ GroupSlice(int C, int vec) {
    CV = vec == 4 ? C >> 2 : C;  // a shift: C / 4 would be a signed division
    const int c0 = blockIdx.z * 256;
    CVs = min(CV - c0, 256);
    cv = c0 + threadIdx.x % CVs;
    rpb = 256 / CVs;
    row = threadIdx.x / CVs;
  }
  // first row of this thread (rows: none for a thread left over)
  __device__ __forceinline__ int64_t first_row(int64_t rows) const {
    return row < rpb ? (int64_t)blockIdx.x * rpb + row : rows;
  }
};

// y = act(x*scale + shift)
template <int VEC>
__global__ void __launch_bounds__(256)
norm_apply_kernel(const float *__restrict__ x, const float *__restrict__ scale_shift, float *__restrict__ y,
                  int64_t rows, int C, int G, int act, float slope, int rtf) {
  using V = typename vec_of<VEC>::type;
  const GroupSlice s(C, VEC);
  const int gbase = (gridDim.y > 1 ? blockIdx.y * C : 0) + s.cv * VEC;
  float sc[VEC], sh[VEC];
  unpack(__ldg(reinterpret_cast<const V *>(scale_shift + gbase)), sc);
  unpack(__ldg(reinterpret_cast<const V *>(scale_shift + G + gbase)), sh);
  const int64_t base = (gridDim.y > 1 ? (int64_t)blockIdx.y * rows : 0);
  const V *xv = reinterpret_cast<const V *>(x) + base * s.CV + s.cv;
  V *yv = reinterpret_cast<V *>(y) + base * s.CV + s.cv;
  const int CV = s.CV;
  const int64_t step = (int64_t)gridDim.x * s.rpb;
#pragma unroll 4
  for (int64_t r = s.first_row(rows); r < rows; r += step) {
    float v[VEC], o[VEC];
    unpack(__ldg(xv + r * CV), v);
#pragma unroll
    for (int j = 0; j < VEC; ++j) o[j] = apply_act(fmaf(v[j], sc[j], sh[j]), act, slope);
    if (rtf) {
#pragma unroll
      for (int j = 0; j < VEC; ++j) o[j] = round_tf32(o[j]);
    }
    yv[r * CV] = pack(o);
  }
}

// derivative of the fused activation: from the pre-activation value recomputed from x (scale_shift given: LeakyReLU /
// ReLU masks need no saved output) or from the saved output y
__device__ __forceinline__ float norm_act_grad(float xv, float sc, float sh, float yv, bool from_x, int act, float slope) {
  if (act == B200GAN_ACT_NONE) return 1.f;
  if (from_x) {
    const float pre = fmaf(xv, sc, sh);
    return act == B200GAN_ACT_LRELU ? (pre > 0.f ? 1.f : slope) : (pre > 0.f ? 1.f : 0.f);
  }
  return act_grad_from_out(yv, act, slope);
}

// the block's per-thread partials red[t][0 .. n) summed per group in fp64 and added to out[j * G + g], j < n
template <int VEC>
__device__ __forceinline__ void norm_block_sums(float (&red)[256][2 * VEC], const GroupSlice &s, int gbase, int G,
                                                int n, double *__restrict__ out) {
  __syncthreads();
  if (threadIdx.x < s.CVs) {
    for (int k = 0; k < n; ++k) {
      double t = 0.0;
      for (int r = 0; r < s.rpb; ++r) t += (double)red[r * s.CVs + threadIdx.x][k];
      atomicAdd(out + (k / VEC) * G + gbase + k % VEC, t);
    }
  }
}

// double-backward mode of pass 1 (u given, act none / LeakyReLU / ReLU with the mask from x): sums[g] += sum u,
// sums[G+g] += sum u * xhat, sums[2G+g] += sum u * dy'.  The third sum goes through the shared slots after the first two.
template <int VEC>
__device__ __forceinline__ void norm_dbwd_reduce(float (&red)[256][2 * VEC], const GroupSlice &s, int gbase,
                                                 const float *__restrict__ dy, const float *__restrict__ x,
                                                 const float *__restrict__ u, const float (&mean)[VEC],
                                                 const float (&rstd)[VEC], const float (&sc)[VEC],
                                                 const float (&sh)[VEC], double *__restrict__ sums, int64_t rows,
                                                 int G, int act, float slope) {
  using V = typename vec_of<VEC>::type;
  const int64_t base = (gridDim.y > 1 ? (int64_t)blockIdx.y * rows : 0);
  const V *dyv = reinterpret_cast<const V *>(dy) + base * s.CV + s.cv;
  const V *xv = reinterpret_cast<const V *>(x) + base * s.CV + s.cv;
  const V *uv = reinterpret_cast<const V *>(u) + base * s.CV + s.cv;
  float su[VEC], st[VEC], sq[VEC];
#pragma unroll
  for (int j = 0; j < VEC; ++j) su[j] = st[j] = sq[j] = 0.f;
  const int CV = s.CV;
  const int64_t step = (int64_t)gridDim.x * s.rpb;
#pragma unroll 2
  for (int64_t r = s.first_row(rows); r < rows; r += step) {
    float dd[VEC], xx[VEC], uu[VEC];
    unpack(__ldg(dyv + r * CV), dd);
    unpack(__ldg(xv + r * CV), xx);
    unpack(__ldg(uv + r * CV), uu);
#pragma unroll
    for (int j = 0; j < VEC; ++j) {
      const float g = dd[j] * norm_act_grad(xx[j], sc[j], sh[j], 0.f, true, act, slope);
      su[j] += uu[j];
      st[j] = fmaf(uu[j], (xx[j] - mean[j]) * rstd[j], st[j]);
      sq[j] = fmaf(uu[j], g, sq[j]);
    }
  }
#pragma unroll
  for (int j = 0; j < VEC; ++j) {
    red[threadIdx.x][j] = su[j];
    red[threadIdx.x][VEC + j] = st[j];
  }
  norm_block_sums<VEC>(red, s, gbase, G, 2 * VEC, sums);
  __syncthreads();
#pragma unroll
  for (int j = 0; j < VEC; ++j) red[threadIdx.x][j] = sq[j];
  norm_block_sums<VEC>(red, s, gbase, G, VEC, sums + 2 * G);
}

// pass 1: sums[g] += sum dy', sums[G+g] += sum dy' * xhat   with dy' = dy * act'
// (u != NULL: the double-backward mode norm_dbwd_reduce, into sums[0 .. 3G))
template <int VEC>
__global__ void __launch_bounds__(256)
norm_bwd_reduce_kernel(const float *__restrict__ dy, const float *__restrict__ x, const float *__restrict__ y,
                       const float *__restrict__ mean_rstd, const float *__restrict__ scale_shift,
                       double *__restrict__ sums, int64_t rows, int C, int G, int act, float slope,
                       const float *__restrict__ u) {
  using V = typename vec_of<VEC>::type;
  __shared__ float red[256][2 * VEC];
  const GroupSlice s(C, VEC);
  const int gbase = (gridDim.y > 1 ? blockIdx.y * C : 0) + s.cv * VEC;
  const bool from_x = scale_shift != nullptr && (act == B200GAN_ACT_LRELU || act == B200GAN_ACT_RELU);
  float mean[VEC], rstd[VEC], sc[VEC], sh[VEC];
#pragma unroll
  for (int j = 0; j < VEC; ++j) {
    mean[j] = __ldg(mean_rstd + gbase + j);
    rstd[j] = __ldg(mean_rstd + G + gbase + j);
    sc[j] = from_x ? __ldg(scale_shift + gbase + j) : 1.f;
    sh[j] = from_x ? __ldg(scale_shift + G + gbase + j) : 0.f;
  }
  if (u != nullptr) {
    norm_dbwd_reduce<VEC>(red, s, gbase, dy, x, u, mean, rstd, sc, sh, sums, rows, G, act, slope);
    return;
  }
  const int64_t base = (gridDim.y > 1 ? (int64_t)blockIdx.y * rows : 0);
  const V *dyv = reinterpret_cast<const V *>(dy) + base * s.CV + s.cv;
  const V *xv = reinterpret_cast<const V *>(x) + base * s.CV + s.cv;
  const V *yv = reinterpret_cast<const V *>(y) + base * s.CV + s.cv;
  const bool need_y = act != B200GAN_ACT_NONE && !from_x;
  float a[VEC], b[VEC];
#pragma unroll
  for (int j = 0; j < VEC; ++j) a[j] = b[j] = 0.f;
  const int CV = s.CV;
  const int64_t step = (int64_t)gridDim.x * s.rpb;
#pragma unroll 4
  for (int64_t r = s.first_row(rows); r < rows; r += step) {
    float dd[VEC], xx[VEC], yy[VEC];
    unpack(__ldg(dyv + r * CV), dd);
    unpack(__ldg(xv + r * CV), xx);
    unpack(need_y ? __ldg(yv + r * CV) : V{}, yy);
#pragma unroll
    for (int j = 0; j < VEC; ++j) {
      const float dz = dd[j] * norm_act_grad(xx[j], sc[j], sh[j], yy[j], from_x, act, slope);
      a[j] += dz;
      b[j] = fmaf(dz, (xx[j] - mean[j]) * rstd[j], b[j]);
    }
  }
  // the slots of the threads left over hold zeros and are never read
#pragma unroll
  for (int j = 0; j < VEC; ++j) {
    red[threadIdx.x][j] = a[j];
    red[threadIdx.x][VEC + j] = b[j];
  }
  __syncthreads();
  if (threadIdx.x < s.CVs) {
    double t[2 * VEC];
#pragma unroll
    for (int j = 0; j < 2 * VEC; ++j) t[j] = 0.0;
    for (int r = 0; r < s.rpb; ++r)
#pragma unroll
      for (int j = 0; j < 2 * VEC; ++j) t[j] += (double)red[r * s.CVs + threadIdx.x][j];
#pragma unroll
    for (int j = 0; j < VEC; ++j) {
      atomicAdd(sums + gbase + j, t[j]);
      atomicAdd(sums + G + gbase + j, t[VEC + j]);
    }
  }
}

// double-backward mode of pass 2.  sums[5][G] = S1 = sum g, S2 = sum g * xhat, U = sum u, T = sum u * xhat,
// Q = sum u * g over the m elements of a group, with g = dy * act'; A = S1/m, B = S2/m.  Per element
//   gdy = act' * (gamma r (u - U/m - xhat T/m) + ugamma xhat + ubeta)
//   gx  = ugamma r (g - A - xhat B) - (gamma r^2 / m) (xhat (Q - A U - 3 B T) + T (g - A) + B (m u - U))
// written as gx = c1 g + c2 x + c3 u + c4 and gdy = act' (c5 u + c6 x + c7), the per-group constants formed in fp64
// (xhat = x r - mean r is folded into c2, c4 and c6, c7).  c5 = gamma r is the forward's scale (the same fp32
// product), so it shares the mask's register.  gx, gdy: either may be NULL.
template <int VEC>
__device__ __forceinline__ void norm_dbwd_apply(const GroupSlice &s, int gbase, const float *__restrict__ dy,
                                                const float *__restrict__ x, const float *__restrict__ u,
                                                const float *__restrict__ mean_rstd,
                                                const float *__restrict__ scale_shift, const float *__restrict__ gamma,
                                                const float *__restrict__ ugb, const double *__restrict__ sums,
                                                float *__restrict__ gx, float *__restrict__ gdy, int64_t rows, int C,
                                                int G, float inv_count, int act, float slope) {
  using V = typename vec_of<VEC>::type;
  const bool masked = act != B200GAN_ACT_NONE;
  float k1[VEC], k2[VEC], k3[VEC], k4[VEC], k6[VEC], k7[VEC], sc[VEC], sh[VEC];
#pragma unroll
  for (int j = 0; j < VEC; ++j) {
    const int g = gbase + j, c = s.cv * VEC + j;  // gamma and ugamma / ubeta are per channel, not per group
    const double m = (double)rows, r = __ldg(mean_rstd + G + g), mu = __ldg(mean_rstd + g);
    const double ga = gamma ? __ldg(gamma + c) : 1.0;
    const double ug = ugb ? __ldg(ugb + c) : 0.0, ub = ugb ? __ldg(ugb + C + c) : 0.0;
    const double A = sums[g] / m, B = sums[G + g] / m, Um = sums[2 * G + g] / m, Tm = sums[3 * G + g] / m;
    const double Qm = sums[4 * G + g] / m;
    const double gr = ga * r, gr2 = gr * r;
    const double c1 = ug * r - gr2 * Tm;
    const double c2 = -ug * r * B - gr2 * (Qm - A * Um - 3.0 * B * Tm);  // multiplies xhat
    const double c6 = ug - gr * Tm;                                        // multiplies xhat
    k1[j] = (float)c1;
    k2[j] = (float)(c2 * r);
    k3[j] = (float)(-gr2 * B);
    k4[j] = (float)(-A * c1 + gr2 * B * Um - c2 * r * mu);
    k6[j] = (float)(c6 * r);
    k7[j] = (float)(ub - gr * Um - c6 * r * mu);
    sc[j] = masked ? __ldg(scale_shift + g) : (float)gr;
    sh[j] = masked ? __ldg(scale_shift + G + g) : 0.f;
  }
  const int64_t base = (gridDim.y > 1 ? (int64_t)blockIdx.y * rows : 0);
  const V *dyv = reinterpret_cast<const V *>(dy) + base * s.CV + s.cv;
  const V *xv = reinterpret_cast<const V *>(x) + base * s.CV + s.cv;
  const V *uv = reinterpret_cast<const V *>(u) + base * s.CV + s.cv;
  V *gxv = reinterpret_cast<V *>(gx) + base * s.CV + s.cv;
  V *gdyv = reinterpret_cast<V *>(gdy) + base * s.CV + s.cv;
  const int CV = s.CV;
  const int64_t step = (int64_t)gridDim.x * s.rpb;
#pragma unroll 1
  for (int64_t r = s.first_row(rows); r < rows; r += step) {
    float dd[VEC], xx[VEC], uu[VEC], o[VEC], p[VEC];
    unpack(__ldg(xv + r * CV), xx);
    unpack(__ldg(uv + r * CV), uu);
    unpack(gx ? __ldg(dyv + r * CV) : V{}, dd);
#pragma unroll
    for (int j = 0; j < VEC; ++j) {
      const float ap = norm_act_grad(xx[j], sc[j], sh[j], 0.f, true, act, slope);
      o[j] = fmaf(k1[j], dd[j] * ap, fmaf(k2[j], xx[j], fmaf(k3[j], uu[j], k4[j])));
      p[j] = ap * fmaf(sc[j], uu[j], fmaf(k6[j], xx[j], k7[j]));
    }
    if (gx) gxv[r * CV] = pack(o);
    if (gdy) gdyv[r * CV] = pack(p);
  }
}

// pass 2: dx = gamma*rstd * (dy' - mean(dy') - xhat * mean(dy' xhat))
// (u != NULL: the double-backward mode norm_dbwd_apply, dx = gx)
template <int VEC>
__global__ void __launch_bounds__(256)
norm_bwd_apply_kernel(const float *__restrict__ dy, const float *__restrict__ x, const float *__restrict__ y,
                      const float *__restrict__ mean_rstd, const float *__restrict__ scale_shift,
                      const float *__restrict__ gamma, const double *__restrict__ sums, float *__restrict__ dx,
                      int64_t rows, int C, int G, float inv_count, int act, float slope, int rtf,
                      const float *__restrict__ u, const float *__restrict__ ugb, float *__restrict__ gdy) {
  using V = typename vec_of<VEC>::type;
  const GroupSlice s(C, VEC);
  const int gbase = (gridDim.y > 1 ? blockIdx.y * C : 0) + s.cv * VEC;
  if (u != nullptr) {
    norm_dbwd_apply<VEC>(s, gbase, dy, x, u, mean_rstd, scale_shift, gamma, ugb, sums, dx, gdy, rows, C, G, inv_count,
                         act, slope);
    return;
  }
  const bool from_x = scale_shift != nullptr && (act == B200GAN_ACT_LRELU || act == B200GAN_ACT_RELU);
  float mean[VEC], rstd[VEC], gr[VEC], m1[VEC], m2[VEC], sc[VEC], sh[VEC];
#pragma unroll
  for (int j = 0; j < VEC; ++j) {
    mean[j] = __ldg(mean_rstd + gbase + j);
    rstd[j] = __ldg(mean_rstd + G + gbase + j);
    gr[j] = (gamma ? __ldg(gamma + s.cv * VEC + j) : 1.f) * rstd[j];  // gamma is per channel, not per group
    m1[j] = (float)sums[gbase + j] * inv_count;
    m2[j] = (float)sums[G + gbase + j] * inv_count;
    sc[j] = from_x ? __ldg(scale_shift + gbase + j) : 1.f;
    sh[j] = from_x ? __ldg(scale_shift + G + gbase + j) : 0.f;
  }
  const int64_t base = (gridDim.y > 1 ? (int64_t)blockIdx.y * rows : 0);
  const V *dyv = reinterpret_cast<const V *>(dy) + base * s.CV + s.cv;
  const V *xv = reinterpret_cast<const V *>(x) + base * s.CV + s.cv;
  const V *yv = reinterpret_cast<const V *>(y) + base * s.CV + s.cv;
  V *dxv = reinterpret_cast<V *>(dx) + base * s.CV + s.cv;
  const bool need_y = act != B200GAN_ACT_NONE && !from_x;
  const int CV = s.CV;
  const int64_t step = (int64_t)gridDim.x * s.rpb;
#pragma unroll 4
  for (int64_t r = s.first_row(rows); r < rows; r += step) {
    float dd[VEC], xx[VEC], yy[VEC], o[VEC];
    unpack(__ldg(dyv + r * CV), dd);
    unpack(__ldg(xv + r * CV), xx);
    unpack(need_y ? __ldg(yv + r * CV) : V{}, yy);
#pragma unroll
    for (int j = 0; j < VEC; ++j) {
      const float dz = dd[j] * norm_act_grad(xx[j], sc[j], sh[j], yy[j], from_x, act, slope);
      const float v = gr[j] * (dz - m1[j] - ((xx[j] - mean[j]) * rstd[j]) * m2[j]);
      o[j] = rtf ? round_tf32(v) : v;
    }
    dxv[r * CV] = pack(o);
  }
}

// pass 3: dgamma / dbeta per group; hands the workspace back zeroed.  Double-backward mode (mean_rstd given, sums[5][G]
// as norm_dbwd_apply reads it): ggamma[g] = r (Q - S1 U / m - S2 T / m) (ggamma may be NULL)
__global__ void norm_bwd_params_kernel(double *__restrict__ sums, float *__restrict__ dgb, int G,
                                       const float *__restrict__ mean_rstd, float *__restrict__ ggamma, double count) {
  int g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= G) return;
  if (mean_rstd) {
    if (ggamma)
      ggamma[g] = (float)((double)mean_rstd[G + g] *
                          (sums[4 * G + g] - (sums[g] * sums[2 * G + g] + sums[G + g] * sums[3 * G + g]) / count));
    for (int k = 0; k < 5; ++k) sums[k * G + g] = 0.0;
    return;
  }
  if (dgb) {
    dgb[g] = (float)sums[G + g];  // dgamma = sum dy' * xhat
    dgb[G + g] = (float)sums[g];  // dbeta  = sum dy'
  }
  sums[g] = 0.0;  // workspace handed back zeroed
  sums[G + g] = 0.0;
}

// 4 when C % 4 == 0 and every float4 operand is 16-byte aligned, else 1
static int vec_width(int C, std::initializer_list<const void *> streamed) {
  uintptr_t bits = 0;
  for (const void *p : streamed) bits |= (uintptr_t)p;
  return C % 4 == 0 && (bits & 15) == 0 ? 4 : 1;
}
// (row blocks, samples, channel slices) with ~8 blocks per SM in total
static dim3 slice_grid(const b200gan_norm_desc *d, int vec, int64_t &rows) {
  rows = d->per_sample ? (int64_t)d->HW : (int64_t)d->N * d->HW;
  const int CV = d->C / vec;
  const int64_t ny = d->per_sample ? d->N : 1, nz = ceil_div(CV, 256);
  const int rpb = 256 / (CV < 256 ? CV : 256);
  int64_t want = (num_sms() * 8 + ny * nz - 1) / (ny * nz);
  int64_t maxb = ceil_div64(rows, (int64_t)rpb * 4);
  if (want > maxb) want = maxb;
  if (want < 1) want = 1;
  return dim3((unsigned)want, (unsigned)ny, (unsigned)nz);
}

static void reduce_grid(const b200gan_norm_desc *d, dim3 &grid, int64_t &rows, int64_t &rpb) {
  rows = d->per_sample ? (int64_t)d->HW : (int64_t)d->N * d->HW;
  int xb = ceil_div(d->C, 32);
  int zb = d->per_sample ? d->N : 1;
  int64_t want = (num_sms() * 8) / ((int64_t)xb * zb);
  if (want < 1) want = 1;
  rpb = ceil_div64(rows, want);
  if (rpb < 32) rpb = 32;
  int64_t yb = ceil_div64(rows, rpb);
  grid = dim3((unsigned)xb, (unsigned)yb, (unsigned)zb);
}

static int check_desc(const b200gan_norm_desc *d) {
  B2_CHECK_ARG(d != nullptr, "norm: null descriptor");
  B2_CHECK_ARG(d->N > 0 && d->HW > 0 && d->C > 0, "norm: bad dims N=%d HW=%d C=%d", d->N, d->HW, d->C);
  B2_CHECK_ARG(!d->per_sample || d->N <= 65535, "norm: N too large for per-sample grid");
  return B200GAN_OK;
}

// passes 2 and 3 of the backward, once `sums` holds sum dy' and sum dy' * xhat (hands the workspace back zeroed)
static int norm_bwd_apply_params(const b200gan_norm_desc *d, const float *dy, const float *x, const float *y,
                                 const float *mean_rstd, const float *scale_shift, const float *gamma, double *sums,
                                 float *dx, float *dgamma_dbeta, int vec, dim3 grid, int64_t rows, cudaStream_t st) {
  const int G = d->per_sample ? d->N * d->C : d->C;
  const float inv = (float)(1.0 / (d->per_sample ? (double)d->HW : (double)d->N * (double)d->HW));
  auto apply = vec == 4 ? norm_bwd_apply_kernel<4> : norm_bwd_apply_kernel<1>;
  apply<<<grid, 256, 0, st>>>(dy, x, y, mean_rstd, scale_shift, gamma, sums, dx, rows, d->C, G, inv, d->act, d->slope,
                              d->round_tf32, nullptr, nullptr, nullptr);
  B2_LAUNCH_CHECK();
  norm_bwd_params_kernel<<<ceil_div(G, 128), 128, 0, st>>>(sums, dgamma_dbeta, G, nullptr, nullptr, 0.0);
  B2_LAUNCH_CHECK();
  return B200GAN_OK;
}

}  // namespace b200gan

using namespace b200gan;

extern "C" int b200gan_norm_stats(const b200gan_norm_desc *d, const float *x, double *stats,
                                  void *stream) {
  if (int e = check_desc(d)) return e;
  B2_CHECK_ARG(x && stats, "norm_stats: null pointer");
  dim3 grid;
  int64_t rows, rpb;
  reduce_grid(d, grid, rows, rpb);
  int G = d->per_sample ? d->N * d->C : d->C;
  norm_stats_kernel<<<grid, dim3(32, 8), 0, as_stream(stream)>>>(x, stats, d->C, rows, rpb, G,
                                                                 d->per_sample);
  B2_LAUNCH_CHECK();
  return B200GAN_OK;
}

extern "C" int b200gan_norm_finalize(const b200gan_norm_desc *d, double *stats,
                                     const float *gamma, const float *beta, float *mean_rstd,
                                     float *scale_shift, float *running_mean, float *running_var,
                                     int64_t *num_batches_tracked, void *stream) {
  if (int e = check_desc(d)) return e;
  B2_CHECK_ARG(stats && mean_rstd && scale_shift, "norm_finalize: null pointer");
  B2_CHECK_ARG(!(running_mean && d->per_sample), "norm_finalize: running stats with per-sample norm");
  B2_CHECK_ARG((running_mean == nullptr) == (running_var == nullptr),
               "norm_finalize: running_mean/var must both be given");
  int G = d->per_sample ? d->N * d->C : d->C;
  double count = d->per_sample ? (double)d->HW : (double)d->N * (double)d->HW;
  norm_finalize_kernel<<<ceil_div(G, 128), 128, 0, as_stream(stream)>>>(
      stats, gamma, beta, mean_rstd, scale_shift, running_mean, running_var, num_batches_tracked, G,
      d->C, count, d->eps, d->momentum);
  B2_LAUNCH_CHECK();
  return B200GAN_OK;
}

extern "C" int b200gan_norm_apply(const b200gan_norm_desc *d, const float *x,
                                  const float *scale_shift, float *y, void *stream) {
  if (int e = check_desc(d)) return e;
  B2_CHECK_ARG(x && scale_shift && y, "norm_apply: null pointer");
  const int G = d->per_sample ? d->N * d->C : d->C;
  const int vec = vec_width(d->C, {x, y, scale_shift});
  int64_t rows;
  const dim3 grid = slice_grid(d, vec, rows);
  auto kernel = vec == 4 ? norm_apply_kernel<4> : norm_apply_kernel<1>;
  kernel<<<grid, 256, 0, as_stream(stream)>>>(x, scale_shift, y, rows, d->C, G, d->act, d->slope, d->round_tf32);
  B2_LAUNCH_CHECK();
  return B200GAN_OK;
}

extern "C" int b200gan_norm_bwd(const b200gan_norm_desc *d, const float *dy, const float *x,
                                const float *y, const float *mean_rstd, const float *scale_shift,
                                const float *gamma, double *sums, float *dx, float *dgamma_dbeta, void *stream) {
  if (int e = check_desc(d)) return e;
  B2_CHECK_ARG(dy && x && mean_rstd && sums && dx, "norm_bwd: null pointer");
  const bool from_x = scale_shift && (d->act == B200GAN_ACT_LRELU || d->act == B200GAN_ACT_RELU);
  B2_CHECK_ARG(d->act == B200GAN_ACT_NONE || from_x || y != nullptr,
               "norm_bwd: fused activation needs the saved output y (or scale_shift for LeakyReLU / ReLU)");
  cudaStream_t st = as_stream(stream);
  const int G = d->per_sample ? d->N * d->C : d->C;
  const float *yy = y ? y : x;  // never dereferenced when the mask comes from x
  const int vec = vec_width(d->C, {dy, x, dx, yy});
  int64_t rows;
  const dim3 grid = slice_grid(d, vec, rows);
  auto reduce = vec == 4 ? norm_bwd_reduce_kernel<4> : norm_bwd_reduce_kernel<1>;
  reduce<<<grid, 256, 0, st>>>(dy, x, yy, mean_rstd, scale_shift, sums, rows, d->C, G, d->act, d->slope, nullptr);
  B2_LAUNCH_CHECK();
  return norm_bwd_apply_params(d, dy, x, yy, mean_rstd, scale_shift, gamma, sums, dx, dgamma_dbeta, vec, grid, rows, st);
}

extern "C" int b200gan_norm_bwd_from_sums(const b200gan_norm_desc *d, const float *dy, const float *x,
                                          const float *mean_rstd, const float *scale_shift, const float *gamma,
                                          double *sums, float *dx, float *dgamma_dbeta, void *stream) {
  if (int e = check_desc(d)) return e;
  B2_CHECK_ARG(dy && x && mean_rstd && sums && dx, "norm_bwd_from_sums: null pointer");
  B2_CHECK_ARG(d->act == B200GAN_ACT_NONE || ((d->act == B200GAN_ACT_LRELU || d->act == B200GAN_ACT_RELU) && scale_shift),
               "norm_bwd_from_sums: activation must be none, or LeakyReLU / ReLU with scale_shift");
  const int vec = vec_width(d->C, {dy, x, dx});
  int64_t rows;
  const dim3 grid = slice_grid(d, vec, rows);
  return norm_bwd_apply_params(d, dy, x, x, mean_rstd, scale_shift, gamma, sums, dx, dgamma_dbeta, vec, grid, rows,
                               as_stream(stream));
}

extern "C" int b200gan_norm_dbwd(const b200gan_norm_desc *d, const float *dy, const float *x, const float *mean_rstd,
                                 const float *scale_shift, const float *gamma, const float *u, const float *ugamma_ubeta,
                                 double *sums, float *gx, float *gdy, float *ggamma_per_group, void *stream) {
  if (int e = check_desc(d)) return e;
  if (d->act != B200GAN_ACT_NONE && d->act != B200GAN_ACT_LRELU && d->act != B200GAN_ACT_RELU)
    B2_UNSUPPORTED("norm_dbwd: a fused Tanh / Sigmoid has a second-order term of its own (activation %d)", d->act);
  B2_CHECK_ARG(dy && x && mean_rstd && u && sums, "norm_dbwd: null pointer");
  B2_CHECK_ARG(d->act == B200GAN_ACT_NONE || scale_shift, "norm_dbwd: LeakyReLU / ReLU needs scale_shift for the mask");
  cudaStream_t st = as_stream(stream);
  const int G = d->per_sample ? d->N * d->C : d->C;
  const float *ss = d->act == B200GAN_ACT_NONE ? nullptr : scale_shift;
  const int vec = vec_width(d->C, {dy, x, u, gx, gdy});
  int64_t rows;
  const dim3 grid = slice_grid(d, vec, rows);
  auto reduce = vec == 4 ? norm_bwd_reduce_kernel<4> : norm_bwd_reduce_kernel<1>;
  // S1, S2 as the first-order backward forms them, then U, T, Q
  reduce<<<grid, 256, 0, st>>>(dy, x, x, mean_rstd, ss, sums, rows, d->C, G, d->act, d->slope, nullptr);
  B2_LAUNCH_CHECK();
  reduce<<<grid, 256, 0, st>>>(dy, x, x, mean_rstd, ss, sums + 2 * (int64_t)G, rows, d->C, G, d->act, d->slope, u);
  B2_LAUNCH_CHECK();
  if (gx || gdy) {
    auto apply = vec == 4 ? norm_bwd_apply_kernel<4> : norm_bwd_apply_kernel<1>;
    apply<<<grid, 256, 0, st>>>(dy, x, x, mean_rstd, ss, gamma, sums, gx, rows, d->C, G, 0.f, d->act, d->slope, 0, u,
                                ugamma_ubeta, gdy);
    B2_LAUNCH_CHECK();
  }
  const double count = d->per_sample ? (double)d->HW : (double)d->N * (double)d->HW;
  norm_bwd_params_kernel<<<ceil_div(G, 128), 128, 0, st>>>(sums, nullptr, G, mean_rstd, ggamma_per_group, count);
  B2_LAUNCH_CHECK();
  return B200GAN_OK;
}
