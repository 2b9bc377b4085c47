// head.cu -- the Discriminator head and the adversarial loss of the DCGAN step as single small kernels.
//
// Reference call sites:
//   self.adv_layer = nn.Sequential(nn.Linear(128 * ds_size ** 2, 1), nn.Sigmoid())      dcgan.py:92
//   adversarial_loss = torch.nn.BCELoss()                                                dcgan.py:103
//   g_loss = adversarial_loss(discriminator(gen_imgs), valid)                            dcgan.py:166, 178-180
// Stock torch runs these as a cuBLASLt GEMV (+ split-K reduce + bias epilogue), a sigmoid kernel, a BCE kernel and a
// mean reduction forward, and five more backward -- ~12 launches per discriminator pass for 128 x 2048 numbers.
// Here: one kernel per direction for Linear(K -> 1) [+ Sigmoid], one per direction for the BCE mean.
//
// The auxiliary-classifier head of the class-conditional scripts and its loss are run-time modes of the same four kernels:
//   self.aux_layer = nn.Sequential(nn.Linear(128 * ds_size ** 2, opt.n_classes), nn.Softmax())  acgan.py:100, sgan.py:99
//   auxiliary_loss = torch.nn.CrossEntropyLoss()                                                   acgan.py:113
// linear1_{fwd,bwd}_kernel with nout >= 2 are Linear(K -> nout) + Softmax over the nout outputs; bce_{fwd,bwd}_kernel
// with C >= 1 are CrossEntropyLoss(reduction='mean') with class-index targets.  nout == 1 and C == 0 are the paths above.
#include <math.h>

#include "common.cuh"

namespace b200gan {

__device__ __forceinline__ float block_sum_128(float v, float *red) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (lane == 0) red[warp] = v;
  __syncthreads();
  float t = 0.f;
  const int nw = blockDim.x >> 5;
  for (int i = 0; i < nw; ++i) t += red[i];
  __syncthreads();
  return t;
}

constexpr int kMaxClasses = 32;  // one warp holds a row's logits

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// y[r][0..nout) = softmax(x[r] W^T + b), 2 <= nout <= 32.  One block (128 threads) per row: each thread streams its
// slice of x[r] once against the nout rows of W (small: they stay in L2), the per-class partials are reduced over the
// warp by a fixed butterfly and over the 4 warps in warp order, and warp 0 takes the softmax with one class per lane.
__device__ __forceinline__ void class_head_fwd_row(const float *__restrict__ x, const float *__restrict__ w,
                                                   const float *__restrict__ b, float *__restrict__ y, int K,
                                                   int nout) {
  __shared__ float part[4][kMaxClasses];
  const float *xr = x + (int64_t)blockIdx.x * K;
  float acc[kMaxClasses];
#pragma unroll
  for (int j = 0; j < kMaxClasses; ++j) acc[j] = 0.f;
  if ((K & 3) == 0 && (((uintptr_t)x | (uintptr_t)w) & 15) == 0) {
    const float4 *x4 = reinterpret_cast<const float4 *>(xr), *w4 = reinterpret_cast<const float4 *>(w);
    const int K4 = K >> 2;
    for (int i = threadIdx.x; i < K4; i += 128) {
      const float4 a = __ldg(x4 + i);
#pragma unroll
      for (int j = 0; j < kMaxClasses; ++j) {
        if (j < nout) {
          const float4 c = __ldg(w4 + (int64_t)j * K4 + i);
          acc[j] += a.x * c.x + a.y * c.y + a.z * c.z + a.w * c.w;
        }
      }
    }
  } else {
    for (int i = threadIdx.x; i < K; i += 128) {
      const float a = __ldg(xr + i);
#pragma unroll
      for (int j = 0; j < kMaxClasses; ++j)
        if (j < nout) acc[j] = fmaf(a, __ldg(w + (int64_t)j * K + i), acc[j]);
    }
  }
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
#pragma unroll
  for (int j = 0; j < kMaxClasses; ++j) {
    if (j < nout) {
      const float v = warp_sum(acc[j]);
      if (lane == 0) part[warp][j] = v;
    }
  }
  __syncthreads();
  if (warp != 0) return;
  const bool on = lane < nout;
  float z = -INFINITY;
  if (on) z = part[0][lane] + part[1][lane] + part[2][lane] + part[3][lane] + (b ? __ldg(b + lane) : 0.f);
  const float m = warp_max(z);
  const float e = on ? expf(z - m) : 0.f;
  const float s = warp_sum(e);
  if (on) y[(int64_t)blockIdx.x * nout + lane] = e / s;
}

// y[n] = act(dot(x[n], w) + b).  One block (128 threads) per sample.  nout >= 2: class_head_fwd_row.
__global__ void __launch_bounds__(128)
linear1_fwd_kernel(const float *__restrict__ x, const float *__restrict__ w, const float *__restrict__ b,
                   float *__restrict__ y, int K, int act, int nout) {
  if (nout > 1) {
    class_head_fwd_row(x, w, b, y, K, nout);
    return;
  }
  __shared__ float red[4];
  const float *xr = x + (int64_t)blockIdx.x * K;
  float s = 0.f;
  if ((K & 3) == 0 && (((uintptr_t)x | (uintptr_t)w) & 15) == 0) {
    const float4 *x4 = reinterpret_cast<const float4 *>(xr), *w4 = reinterpret_cast<const float4 *>(w);
    for (int i = threadIdx.x; i < (K >> 2); i += 128) {
      const float4 a = __ldg(x4 + i), c = __ldg(w4 + i);
      s += a.x * c.x + a.y * c.y + a.z * c.z + a.w * c.w;
    }
  } else {
    for (int i = threadIdx.x; i < K; i += 128) s = fmaf(__ldg(xr + i), __ldg(w + i), s);
  }
  s = block_sum_128(s, red);
  if (threadIdx.x == 0) y[blockIdx.x] = apply_act(s + (b ? __ldg(b) : 0.f), act, 0.f);
}

// Backward of class_head_fwd_row.  Every block first forms dz[r][j] = y (dy - sum_i y_i dy_i) (torch's softmax backward)
// for all N rows in shared memory, one row per thread, the sum in class order; then thread k reads x[r][k] once per row
// and accumulates dw[j][k] = sum_r dz[r][j] x[r][k] in registers, and writes dx[r][k] = sum_j dz[r][j] w[j][k].  Block 0
// writes db[j] = sum_r dz[r][j], summed in row order.  N * nout <= B200GAN_CLASS_HEAD_BWD_MAX_ELEMS: dz and the 16 bytes
// of the kernel's own block reduction fit the 48 KB a launch may take without opting in to more.
__device__ __forceinline__ void class_head_bwd(const float *__restrict__ x, const float *__restrict__ w,
                                               const float *__restrict__ y, const float *__restrict__ dy,
                                               float *__restrict__ dx, float *__restrict__ dw, float *__restrict__ db,
                                               int N, int K, int nout, float *dz) {
  for (int r = threadIdx.x; r < N; r += 128) {
    const float *yr = y + (int64_t)r * nout, *dyr = dy + (int64_t)r * nout;
    float s = 0.f;
    for (int j = 0; j < nout; ++j) s = fmaf(__ldg(yr + j), __ldg(dyr + j), s);
    for (int j = 0; j < nout; ++j) dz[r * nout + j] = __ldg(yr + j) * (__ldg(dyr + j) - s);
  }
  __syncthreads();
  if (db && blockIdx.x == 0 && threadIdx.x < nout) {
    float t = 0.f;
    for (int r = 0; r < N; ++r) t += dz[r * nout + threadIdx.x];
    db[threadIdx.x] = t;
  }
  const int k = blockIdx.x * 128 + threadIdx.x;
  if (k >= K) return;
  float wk[kMaxClasses], acc[kMaxClasses];
#pragma unroll
  for (int j = 0; j < kMaxClasses; ++j) {
    wk[j] = j < nout ? __ldg(w + (int64_t)j * K + k) : 0.f;
    acc[j] = 0.f;
  }
  for (int r = 0; r < N; ++r) {
    const float xv = __ldg(x + (int64_t)r * K + k);
    const float *d = dz + r * nout;
    float s = 0.f;
#pragma unroll
    for (int j = 0; j < kMaxClasses; ++j) {
      if (j < nout) {
        const float dj = d[j];
        acc[j] = fmaf(dj, xv, acc[j]);
        s = fmaf(dj, wk[j], s);
      }
    }
    if (dx) dx[(int64_t)r * K + k] = s;
  }
#pragma unroll
  for (int j = 0; j < kMaxClasses; ++j)
    if (j < nout) dw[(int64_t)j * K + k] = acc[j];
}

// dl[n] = dy[n] * act'(y[n]);  dw[k] = sum_n dl[n] x[n][k];  dx[n][k] = dl[n] w[k];  db = sum_n dl[n].
// grid = ceil(K / 128); thread = one k.  N <= 4096 (dl staged in shared memory).  nout >= 2: class_head_bwd.
__global__ void __launch_bounds__(128)
linear1_bwd_kernel(const float *__restrict__ x, const float *__restrict__ w, const float *__restrict__ y,
                   const float *__restrict__ dy, float *__restrict__ dx, float *__restrict__ dw,
                   float *__restrict__ db, int N, int K, int act, int nout) {
  extern __shared__ float dl[];  // [N], or [N][nout]
  if (nout > 1) {
    class_head_bwd(x, w, y, dy, dx, dw, db, N, K, nout, dl);
    return;
  }
  __shared__ float red[4];
  float part = 0.f;
  for (int n = threadIdx.x; n < N; n += 128) {
    const float v = __ldg(dy + n) * act_grad_from_out(__ldg(y + n), act, 0.f);
    dl[n] = v;
    part += v;
  }
  __syncthreads();
  if (db && blockIdx.x == 0) {
    const float t = block_sum_128(part, red);
    if (threadIdx.x == 0) *db = t;
  }
  const int k = blockIdx.x * 128 + threadIdx.x;
  if (k >= K) return;
  const float wk = __ldg(w + k);
  float acc = 0.f;
  for (int n = 0; n < N; ++n) {
    const float d = dl[n];
    acc = fmaf(d, __ldg(x + (int64_t)n * K + k), acc);
    if (dx) dx[(int64_t)n * K + k] = d * wk;
  }
  dw[k] = acc;
}

// Row r of CrossEntropyLoss: the max m and the sum s of expf(x - m) over the C logits, lanes striding the row.  Both
// reductions are fixed butterflies, so a row's m and s do not depend on the launch.
__device__ __forceinline__ void ce_row_stats(const float *__restrict__ xr, int C, int lane, float &m, float &s) {
  float mx = -INFINITY;
  for (int j = lane; j < C; j += 32) mx = fmaxf(mx, __ldg(xr + j));
  m = warp_max(mx);
  float e = 0.f;
  for (int j = lane; j < C; j += 32) e += expf(__ldg(xr + j) - m);
  s = warp_sum(e);
}

// torch.nn.CrossEntropyLoss(reduction='mean') with class indices: out2[0] = sum over the rows not ignored of
// logsumexp(x[r]) - x[r][t[r]], divided by their count, which goes to out2[1].  A target outside [0, C) that is not
// ignore_index makes its term NaN; no element outside the row is read.  One block of kCeFwdThreads, a warp per row in
// turn; each warp sums its terms in row order in fp64, and thread 0 adds the warps in warp order: bit-identical from
// call to call.  All rows ignored: 0 / 0 = NaN, as in torch.
constexpr int kCeFwdThreads = 1024;
__device__ __forceinline__ void cross_entropy_fwd(const float *__restrict__ x, const int64_t *__restrict__ target,
                                                  float *__restrict__ out2, int64_t N, int C, int64_t ignore_index) {
  constexpr int kWarps = kCeFwdThreads / 32;
  __shared__ double tot[kWarps];
  __shared__ int64_t cnt[kWarps];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  double acc = 0.0;
  int64_t count = 0;
  for (int64_t r = warp; r < N; r += kWarps) {
    const int64_t t = __ldg(target + r);
    if (t == ignore_index) continue;
    const float *xr = x + r * C;
    float m, s;
    ce_row_stats(xr, C, lane, m, s);
    const float term = (t >= 0 && t < C) ? (m - __ldg(xr + t)) + logf(s) : NAN;
    acc += (double)term;
    ++count;
  }
  if (lane == 0) {
    tot[warp] = acc;
    cnt[warp] = count;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    double sum = 0.0;
    int64_t n = 0;
    for (int i = 0; i < kWarps; ++i) {
      sum += tot[i];
      n += cnt[i];
    }
    out2[0] = (float)(sum / (double)n);
    out2[1] = (float)n;
  }
}

// d loss / d x[r][j] = g / count * (softmax(x[r])_j - [j == t[r]]), with g = gout[0] and count = out2[1] read on the
// device; zero rows for ignored targets, NaN rows for targets outside [0, C).  A warp per row.
__device__ __forceinline__ void cross_entropy_bwd(const float *__restrict__ x, const int64_t *__restrict__ target,
                                                  const float *__restrict__ out2, const float *__restrict__ gout,
                                                  float *__restrict__ dx, int64_t N, int C, int64_t ignore_index) {
  const int64_t r = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (r >= N) return;
  const float *xr = x + r * C;
  float *dr = dx + r * C;
  const int64_t t = __ldg(target + r);
  if (t == ignore_index) {
    for (int j = lane; j < C; j += 32) dr[j] = 0.f;
    return;
  }
  if (t < 0 || t >= C) {
    for (int j = lane; j < C; j += 32) dr[j] = NAN;
    return;
  }
  float m, s;
  ce_row_stats(xr, C, lane, m, s);
  const float g = __ldg(gout) / __ldg(out2 + 1);
  for (int j = lane; j < C; j += 32) {
    const float p = expf(__ldg(xr + j) - m) / s;
    dr[j] = g * (j == t ? p - 1.f : p);
  }
}

// torch.nn.BCELoss(reduction='mean'): log terms clamped at -100 (torch/aten binary_cross_entropy semantics).
// C >= 1: cross_entropy_fwd of the [n][C] logits v, on kCeFwdThreads threads.
__global__ void __launch_bounds__(kCeFwdThreads)
bce_fwd_kernel(const float *__restrict__ v, const float *__restrict__ t, float *__restrict__ loss, int64_t n,
               const int64_t *__restrict__ target, int C, int64_t ignore_index) {
  if (C > 0) {
    cross_entropy_fwd(v, target, loss, n, C, ignore_index);
    return;
  }
  __shared__ float red[4];
  float s = 0.f;
  for (int64_t i = threadIdx.x; i < n; i += 128) {
    const float p = __ldg(v + i), y = __ldg(t + i);
    const float lp = fmaxf(logf(p), -100.f), lq = fmaxf(log1pf(-p), -100.f);
    s += (y - 1.f) * lq - y * lp;
  }
  s = block_sum_128(s, red);
  if (threadIdx.x == 0) *loss = s / (float)n;
}
// d loss / d v = gout / n * (v - t) / max((1 - v) v, 1e-12).  C >= 1: cross_entropy_bwd of the [n][C] logits v, with
// the forward's out2 passed as t.
__global__ void bce_bwd_kernel(const float *__restrict__ v, const float *__restrict__ t, const float *__restrict__ gout,
                               float *__restrict__ dv, int64_t n, const int64_t *__restrict__ target, int C,
                               int64_t ignore_index) {
  if (C > 0) {
    cross_entropy_bwd(v, target, t, gout, dv, n, C, ignore_index);
    return;
  }
  const float g = __ldg(gout) / (float)n;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const float p = __ldg(v + i), y = __ldg(t + i);
    dv[i] = g * (p - y) / fmaxf((1.f - p) * p, 1e-12f);
  }
}

}  // namespace b200gan

using namespace b200gan;

extern "C" int b200gan_linear1_fwd(const float *x, const float *w, const float *b, float *y, int32_t N, int32_t K,
                                   int32_t act, void *stream) {
  B2_CHECK_ARG(x && w && y && N >= 0 && K > 0, "linear1_fwd: bad arguments");
  if (N == 0) return B200GAN_OK;
  linear1_fwd_kernel<<<(unsigned)N, 128, 0, as_stream(stream)>>>(x, w, b, y, K, act, 1);
  B2_LAUNCH_CHECK();
  return B200GAN_OK;
}

extern "C" int b200gan_linear1_bwd(const float *x, const float *w, const float *y, const float *dy, float *dx, float *dw,
                                   float *db, int32_t N, int32_t K, int32_t act, void *stream) {
  B2_CHECK_ARG(x && w && y && dy && dw && N > 0 && K > 0, "linear1_bwd: bad arguments");
  B2_CHECK_ARG(N <= 4096, "linear1_bwd: batch %d > 4096", N);
  linear1_bwd_kernel<<<(unsigned)ceil_div(K, 128), 128, (size_t)N * sizeof(float), as_stream(stream)>>>(
      x, w, y, dy, dx, dw, db, N, K, act, 1);
  B2_LAUNCH_CHECK();
  return B200GAN_OK;
}

extern "C" int b200gan_bce_fwd(const float *v, const float *t, float *loss, int64_t n, void *stream) {
  B2_CHECK_ARG(v && t && loss && n > 0, "bce_fwd: bad arguments");
  bce_fwd_kernel<<<1, 128, 0, as_stream(stream)>>>(v, t, loss, n, nullptr, 0, 0);
  B2_LAUNCH_CHECK();
  return B200GAN_OK;
}

extern "C" int b200gan_bce_bwd(const float *v, const float *t, const float *gout, float *dv, int64_t n, void *stream) {
  B2_CHECK_ARG(v && t && gout && dv && n > 0, "bce_bwd: bad arguments");
  int64_t blocks = ceil_div64(n, 256);
  if (blocks > 1184) blocks = 1184;
  bce_bwd_kernel<<<(unsigned)blocks, 256, 0, as_stream(stream)>>>(v, t, gout, dv, n, nullptr, 0, 0);
  B2_LAUNCH_CHECK();
  return B200GAN_OK;
}

extern "C" int b200gan_class_head_fwd(const float *x, const float *w, const float *b, float *y, int32_t N, int32_t K,
                                      int32_t nout, void *stream) {
  B2_CHECK_ARG(x && w && y && N >= 1 && K > 0, "class_head_fwd: bad arguments");
  B2_CHECK_ARG(nout >= 2 && nout <= kMaxClasses, "class_head_fwd: %d classes, 2..%d supported", nout, kMaxClasses);
  linear1_fwd_kernel<<<(unsigned)N, 128, 0, as_stream(stream)>>>(x, w, b, y, K, B200GAN_ACT_NONE, nout);
  B2_LAUNCH_CHECK();
  return B200GAN_OK;
}

extern "C" int b200gan_class_head_bwd(const float *x, const float *w, const float *y, const float *dy, float *dx,
                                      float *dw, float *db, int32_t N, int32_t K, int32_t nout, void *stream) {
  B2_CHECK_ARG(x && w && y && dy && dw && N >= 1 && K > 0, "class_head_bwd: bad arguments");
  B2_CHECK_ARG(nout >= 2 && nout <= kMaxClasses, "class_head_bwd: %d classes, 2..%d supported", nout, kMaxClasses);
  B2_CHECK_ARG((int64_t)N * nout <= B200GAN_CLASS_HEAD_BWD_MAX_ELEMS, "class_head_bwd: N * nout = %lld > %d",
               (long long)N * nout, B200GAN_CLASS_HEAD_BWD_MAX_ELEMS);
  linear1_bwd_kernel<<<(unsigned)ceil_div(K, 128), 128, (size_t)N * nout * sizeof(float), as_stream(stream)>>>(
      x, w, y, dy, dx, dw, db, N, K, B200GAN_ACT_NONE, nout);
  B2_LAUNCH_CHECK();
  return B200GAN_OK;
}

extern "C" int b200gan_cross_entropy_fwd(const float *x, const int64_t *target, float *out2, int32_t N, int32_t C,
                                         int64_t ignore_index, void *stream) {
  B2_CHECK_ARG(x && target && out2 && N >= 1, "cross_entropy_fwd: bad arguments");
  B2_CHECK_ARG(C >= 1 && C <= B200GAN_CROSS_ENTROPY_MAX_CLASSES, "cross_entropy_fwd: %d classes, 1..%d supported", C,
               B200GAN_CROSS_ENTROPY_MAX_CLASSES);
  bce_fwd_kernel<<<1, kCeFwdThreads, 0, as_stream(stream)>>>(x, nullptr, out2, N, target, C, ignore_index);
  B2_LAUNCH_CHECK();
  return B200GAN_OK;
}

extern "C" int b200gan_cross_entropy_bwd(const float *x, const int64_t *target, const float *out2, const float *gout,
                                         float *dx, int32_t N, int32_t C, int64_t ignore_index, void *stream) {
  B2_CHECK_ARG(x && target && out2 && gout && dx && N >= 1, "cross_entropy_bwd: bad arguments");
  B2_CHECK_ARG(C >= 1 && C <= B200GAN_CROSS_ENTROPY_MAX_CLASSES, "cross_entropy_bwd: %d classes, 1..%d supported", C,
               B200GAN_CROSS_ENTROPY_MAX_CLASSES);
  bce_bwd_kernel<<<(unsigned)ceil_div(N, 8), 256, 0, as_stream(stream)>>>(x, out2, gout, dx, N, target, C,
                                                                           ignore_index);
  B2_LAUNCH_CHECK();
  return B200GAN_OK;
}
