// index_ops.cu -- shape/index kernels (bit-exact data movement), element-wise activation,
// epilogue backward and the flat Adam step.  All are streaming HBM-bound passes.
//
// Reference modules replaced when they cannot be folded into a neighbouring kernel:
//   nn.Upsample(scale_factor=2)  dcgan.py:54,58   (nearest: dst -> src = dst // 2)
//   nn.ZeroPad2d((1,0,1,0))      pix2pix/models.py:78,126  (left & top only)
//   nn.ReflectionPad2d(k)        cyclegan/models.py:27,31,49,81 (edge pixel not repeated)
//   nn.LeakyReLU/ReLU/Tanh       dcgan.py:57,63 ...
//   nn.Dropout / nn.Dropout2d    mask drawn by torch (same RNG stream as the reference), applied here
//   torch.optim.Adam             dcgan.py:134-135
#include "common.cuh"

namespace b200gan {

// ---- NCHW <-> NHWC ----------------------------------------------------------------------------
// per image: [C][HW] <-> [HW][C]: classic 32x32 smem tile transpose. grid (HW/32, C/32, N)
__global__ void transpose_kernel(const float *__restrict__ x, float *__restrict__ y, int rows, int cols) {
  // x: [rows][cols] -> y: [cols][rows], per blockIdx.z image
  __shared__ float tile[32][33];
  const int64_t img = (int64_t)blockIdx.z * rows * cols;
  int c = blockIdx.x * 32 + threadIdx.x;
  int r0 = blockIdx.y * 32;
  for (int i = threadIdx.y; i < 32; i += 8) {
    int r = r0 + i;
    if (r < rows && c < cols) tile[i][threadIdx.x] = x[img + (int64_t)r * cols + c];
  }
  __syncthreads();
  int r = r0 + threadIdx.x;
  int c0 = blockIdx.x * 32;
  for (int i = threadIdx.y; i < 32; i += 8) {
    int cc = c0 + i;
    if (r < rows && cc < cols) y[img + (int64_t)cc * rows + r] = tile[threadIdx.x][i];
  }
}

static int launch_transpose(const float *x, float *y, int N, int rows, int cols, cudaStream_t st) {
  if (N == 0 || rows == 0 || cols == 0) return B200GAN_OK;
  if (rows == 1 || cols == 1) {
    B2_CUDA(cudaMemcpyAsync(y, x, (size_t)N * rows * cols * sizeof(float), cudaMemcpyDeviceToDevice, st));
    return B200GAN_OK;
  }
  B2_CHECK_ARG(N <= 65535 && ceil_div(rows, 32) <= 65535, "transpose: dims too large");
  dim3 grid(ceil_div(cols, 32), ceil_div(rows, 32), N);
  transpose_kernel<<<grid, dim3(32, 8), 0, st>>>(x, y, rows, cols);
  B2_LAUNCH_CHECK();
  return B200GAN_OK;
}

// ---- nearest x2 upsample ---------------------------------------------------------------------
__global__ void upsample2x_fwd_kernel(const float *__restrict__ x, float *__restrict__ y, int64_t total,
                                      int H, int W, int C) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (int64_t)gridDim.x * blockDim.x) {
    int c = (int)(i % C);
    int64_t t = i / C;
    int ow = (int)(t % (2 * W));
    t /= (2 * W);
    int oh = (int)(t % (2 * H));
    int n = (int)(t / (2 * H));
    y[i] = __ldg(x + (((int64_t)n * H + (oh >> 1)) * W + (ow >> 1)) * C + c);
  }
}
__global__ void upsample2x_bwd_kernel(const float *__restrict__ dy, float *__restrict__ dx, int64_t total,
                                      int H, int W, int C) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (int64_t)gridDim.x * blockDim.x) {
    int c = (int)(i % C);
    int64_t t = i / C;
    int w = (int)(t % W);
    t /= W;
    int h = (int)(t % H);
    int n = (int)(t / H);
    const float *p = dy + (((int64_t)n * 2 * H + 2 * h) * 2 * W + 2 * w) * C + c;
    int64_t rs = (int64_t)2 * W * C;
    dx[i] = (__ldg(p) + __ldg(p + C)) + (__ldg(p + rs) + __ldg(p + rs + C));
  }
}

// ---- padding ------------------------------------------------------------------------------------
__global__ void pad2d_fwd_kernel(const float *__restrict__ x, float *__restrict__ y, int64_t total, int H,
                                 int W, int C, int Ho, int Wo, int pad_t, int pad_l, int mode, int rtf) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (int64_t)gridDim.x * blockDim.x) {
    int c = (int)(i % C);
    int64_t t = i / C;
    int ow = (int)(t % Wo);
    t /= Wo;
    int oh = (int)(t % Ho);
    int n = (int)(t / Ho);
    int ih = oh - pad_t, iw = ow - pad_l;
    float v = 0.f;
    if (mode == B200GAN_PAD_REFLECT) {
      ih = reflect_idx(ih, H);
      iw = reflect_idx(iw, W);
      v = __ldg(x + (((int64_t)n * H + ih) * W + iw) * C + c);
    } else if (ih >= 0 && ih < H && iw >= 0 && iw < W) {
      v = __ldg(x + (((int64_t)n * H + ih) * W + iw) * C + c);
    }
    y[i] = rtf ? round_tf32(v) : v;
  }
}
// gradient: zero pad -> crop; reflect -> each input pixel sums the (<= 4) padded pixels that mirror
// onto it.  Gather formulation (deterministic, no atomics).
__global__ void pad2d_bwd_kernel(const float *__restrict__ dy, float *__restrict__ dx, int64_t total, int H,
                                 int W, int C, int Ho, int Wo, int pad_t, int pad_l, int pad_b, int pad_r,
                                 int mode) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (int64_t)gridDim.x * blockDim.x) {
    int c = (int)(i % C);
    int64_t t = i / C;
    int w = (int)(t % W);
    t /= W;
    int h = (int)(t % H);
    int n = (int)(t / H);
    const float *base = dy + (int64_t)n * Ho * Wo * C + c;
    // candidate padded rows mapping onto h: h+pad_t (interior), pad_t-h (top mirror, h in [1,pad_t]),
    // pad_t + 2(H-1) - h (bottom mirror, H-1-h in [1,pad_b])
    int rows[3], nr = 0, cols[3], nc = 0;
    rows[nr++] = h + pad_t;
    cols[nc++] = w + pad_l;
    if (mode == B200GAN_PAD_REFLECT) {
      if (h >= 1 && h <= pad_t) rows[nr++] = pad_t - h;
      if (H - 1 - h >= 1 && H - 1 - h <= pad_b) rows[nr++] = pad_t + 2 * (H - 1) - h;
      if (w >= 1 && w <= pad_l) cols[nc++] = pad_l - w;
      if (W - 1 - w >= 1 && W - 1 - w <= pad_r) cols[nc++] = pad_l + 2 * (W - 1) - w;
    }
    float s = 0.f;
    for (int a = 0; a < nr; ++a)
      for (int b = 0; b < nc; ++b) s += __ldg(base + ((int64_t)rows[a] * Wo + cols[b]) * C);
    dx[i] = s;
  }
}

// float4 along the channels (C % 4 == 0, fewer than 2^31 float4s): 32-bit index arithmetic, 16-byte accesses.  The scalar
// kernels above moved 69 MB in 56 us (cyclegan's ReflectionPad2d(1) in front of every residual conv, models.py:18-25).
__global__ void __launch_bounds__(256)
pad2d_fwd_v4_kernel(const float4 *__restrict__ x, float4 *__restrict__ y, unsigned total4, int H, int W, int C4, int Ho,
                    int Wo, int pad_t, int pad_l, int mode, int rtf) {
  for (unsigned i = blockIdx.x * 256u + threadIdx.x; i < total4; i += gridDim.x * 256u) {
    const unsigned pix = i / (unsigned)C4, c4 = i - pix * (unsigned)C4;
    const unsigned row = pix / (unsigned)Wo, ow = pix - row * (unsigned)Wo;
    const unsigned n = row / (unsigned)Ho, oh = row - n * (unsigned)Ho;
    int ih = (int)oh - pad_t, iw = (int)ow - pad_l;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    bool ok = true;
    if (mode == B200GAN_PAD_REFLECT) {
      ih = reflect_idx(ih, H);
      iw = reflect_idx(iw, W);
    } else {
      ok = ih >= 0 && ih < H && iw >= 0 && iw < W;
    }
    if (ok) v = __ldg(x + ((size_t)(n * H + ih) * W + iw) * C4 + c4);
    if (rtf) { v.x = round_tf32(v.x); v.y = round_tf32(v.y); v.z = round_tf32(v.z); v.w = round_tf32(v.w); }
    y[i] = v;
  }
}
__global__ void __launch_bounds__(256)
pad2d_bwd_v4_kernel(const float4 *__restrict__ dy, float4 *__restrict__ dx, unsigned total4, int H, int W, int C4, int Ho,
                    int Wo, int pad_t, int pad_l, int pad_b, int pad_r, int mode) {
  for (unsigned i = blockIdx.x * 256u + threadIdx.x; i < total4; i += gridDim.x * 256u) {
    const unsigned pix = i / (unsigned)C4, c4 = i - pix * (unsigned)C4;
    const unsigned row = pix / (unsigned)W;
    const int w = (int)(pix - row * (unsigned)W);
    const unsigned n = row / (unsigned)H;
    const int h = (int)(row - n * (unsigned)H);
    const float4 *base = dy + (size_t)n * Ho * Wo * C4 + c4;
    int rows[3], nr = 0, cols[3], nc = 0;
    rows[nr++] = h + pad_t;
    cols[nc++] = w + pad_l;
    if (mode == B200GAN_PAD_REFLECT) {
      if (h >= 1 && h <= pad_t) rows[nr++] = pad_t - h;
      if (H - 1 - h >= 1 && H - 1 - h <= pad_b) rows[nr++] = pad_t + 2 * (H - 1) - h;
      if (w >= 1 && w <= pad_l) cols[nc++] = pad_l - w;
      if (W - 1 - w >= 1 && W - 1 - w <= pad_r) cols[nc++] = pad_l + 2 * (W - 1) - w;
    }
    float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int a = 0; a < nr; ++a)
      for (int b = 0; b < nc; ++b) {
        const float4 v = __ldg(base + ((size_t)rows[a] * Wo + cols[b]) * C4);
        s.x += v.x; s.y += v.y; s.z += v.z; s.w += v.w;
      }
    dx[i] = s;
  }
}

// ---- activation (+ mask) --------------------------------------------------------------------------
__global__ void act_fwd_kernel(const float *__restrict__ x, const float *__restrict__ mask, int mask_pc,
                               int act, float slope, int64_t n, int C, int64_t HW, float *__restrict__ y) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n;
       i += (int64_t)gridDim.x * blockDim.x) {
    float v = apply_act(__ldg(x + i), act, slope);
    if (mask) {
      if (mask_pc) {
        int c = (int)(i % C);
        int64_t img = i / ((int64_t)C * HW);
        v *= __ldg(mask + img * C + c);
      } else {
        v *= __ldg(mask + i);
      }
    }
    y[i] = v;
  }
}

__global__ void epilogue_bwd_kernel(const float *__restrict__ dy, const float *__restrict__ y,
                                    const float *__restrict__ chan_scale, int act, float slope, int64_t n,
                                    int K, int64_t PQ, int rtf, float *__restrict__ dz) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n;
       i += (int64_t)gridDim.x * blockDim.x) {
    float d = __ldg(dy + i);
    float cs = 1.f;
    if (chan_scale) {
      int k = (int)(i % K);
      int64_t img = i / ((int64_t)K * PQ);
      cs = __ldg(chan_scale + img * K + k);
      d *= cs;
    }
    if (act != B200GAN_ACT_NONE) {
      // y = cs * act(z): recover act(z) for the derivative.  cs == 0 (dropped channel) gives d == 0
      // already; for LReLU/ReLU only the sign of y matters (cs >= 0).
      float yv = __ldg(y + i);
      if (chan_scale && (act == B200GAN_ACT_TANH || act == B200GAN_ACT_SIGMOID))
        yv = cs != 0.f ? yv / cs : 0.f;
      d *= act_grad_from_out(yv, act, slope);
    }
    dz[i] = rtf ? round_tf32(d) : d;
  }
}

// bias gradient of a fused conv block from unrounded values: db[k] = sum_m dy[m][k] act'(y[m][k]) cs[n(m)][k]
__global__ void __launch_bounds__(256)
bias_grad_kernel(const float *__restrict__ dy, const float *__restrict__ y, const float *__restrict__ chan_scale, int act,
                 float slope, int64_t M, int K, int64_t PQ, int64_t rows_per_block, float *__restrict__ db) {
  __shared__ float red[8][33];
  const int k = blockIdx.x * 32 + threadIdx.x;
  int64_t r0 = (int64_t)blockIdx.y * rows_per_block, r1 = r0 + rows_per_block;
  if (r1 > M) r1 = M;
  float s = 0.f;
  if (k < K)
    for (int64_t r = r0 + threadIdx.y; r < r1; r += 8) {
      float d = __ldg(dy + r * K + k);
      float cs = 1.f;
      if (chan_scale) {
        cs = __ldg(chan_scale + (r / PQ) * K + k);
        d *= cs;
      }
      if (act != B200GAN_ACT_NONE) {
        float yv = __ldg(y + r * K + k);
        if (chan_scale && (act == B200GAN_ACT_TANH || act == B200GAN_ACT_SIGMOID)) yv = cs != 0.f ? yv / cs : 0.f;
        d *= act_grad_from_out(yv, act, slope);
      }
      s += d;
    }
  red[threadIdx.y][threadIdx.x] = s;
  __syncthreads();
  if (threadIdx.y == 0 && k < K) {
    float t = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) t += red[i][threadIdx.x];
    atomicAdd(db + k, t);
  }
}

// ---- Adam ---------------------------------------------------------------------------------------------
// torch.optim.Adam (no amsgrad, no weight decay), arithmetic of _single_tensor_adam: the hyper-parameters, the bias
// corrections 1 - beta^t and the step size lr / (1 - beta1^t) are Python doubles that are cast to fp32 only where they
// meet a tensor -- (float)(1 - 0.999) is not 1.f - 0.999f (1.3e-5 apart), so they arrive here as doubles too.
//   m = b1 m + (1-b1) g;  v = b2 v + (1-b2) g^2;  p -= step_size * m / (sqrt(v) / sqrt(1 - b2^t) + eps)
// The step count lives on the device (CUDA-graph capturable).
__global__ void adam_step_inc_kernel(float *step) { *step += 1.f; }

// ONE launch updates every parameter tensor of an optimizer.  The tensor table travels as a kernel
// argument (no device-side table to maintain; addresses are whatever autograd produced this step, or the fixed
// addresses of a captured CUDA graph).  Block b works on chunk (b - block_begin[t]) of tensor t; the last block to
// finish (atomicInc ticket, self-resetting) advances the device-side step count, so there is no second launch.
constexpr int ADAM_MAX_TENSORS = 48;
constexpr int ADAM_CHUNK = 256 * 16;  // elements per block
struct AdamTable {
  float *p[ADAM_MAX_TENSORS];
  const float *g[ADAM_MAX_TENSORS];
  float *m[ADAM_MAX_TENSORS];
  float *v[ADAM_MAX_TENSORS];
  long long n[ADAM_MAX_TENSORS];
  int block_begin[ADAM_MAX_TENSORS + 1];
  int count;
};
__global__ void __launch_bounds__(256)
adam_multi_kernel(const __grid_constant__ AdamTable tb, double lr, double b1, double b2, double eps, float gscale,
                  float *__restrict__ step, int advance) {
  const double t = (double)step[0] + 1.0;
  const float neg_step_size = (float)(-(lr / (1.0 - pow(b1, t))));
  const float bc2_sqrt = (float)sqrt(1.0 - pow(b2, t));
  const float b1f = (float)b1, omb1 = (float)(1.0 - b1), b2f = (float)b2, omb2 = (float)(1.0 - b2);
  const float epsf = (float)eps;
  int lo = 0, hi = tb.count;  // tensor of this block: largest ti with block_begin[ti] <= blockIdx.x
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (tb.block_begin[mid] <= (int)blockIdx.x) lo = mid; else hi = mid;
  }
  const int ti = lo;
  float *__restrict__ p = tb.p[ti];
  const float *__restrict__ g = tb.g[ti];
  float *__restrict__ m = tb.m[ti];
  float *__restrict__ v = tb.v[ti];
  const long long n = tb.n[ti];
  const long long i0 = (long long)((int)blockIdx.x - tb.block_begin[ti]) * ADAM_CHUNK;
  long long i1 = i0 + ADAM_CHUNK;
  if (i1 > n) i1 = n;
  for (long long i = i0 + threadIdx.x; i < i1; i += 256) {
    const float gi = g[i] * gscale;
    const float mi = b1f * m[i] + omb1 * gi;
    const float vi = b2f * v[i] + omb2 * gi * gi;
    m[i] = mi;
    v[i] = vi;
    const float denom = sqrtf(vi) / bc2_sqrt + epsf;
    p[i] += neg_step_size * (mi / denom);
  }
  if (advance) {
    __syncthreads();  // every thread of this block has read step[0]
    if (threadIdx.x == 0) {
      __threadfence();
      unsigned *ticket = reinterpret_cast<unsigned *>(step + 1);
      if (atomicInc(ticket, gridDim.x - 1) == gridDim.x - 1) step[0] = (float)t;  // last block; ticket wrapped to 0
    }
  }
}

static unsigned stream_blocks(int64_t n) {
  int64_t b = ceil_div64(n, 256);
  if (b > num_sms() * 16) b = num_sms() * 16;
  if (b < 1) b = 1;
  return (unsigned)b;
}

}  // namespace b200gan

using namespace b200gan;

extern "C" int b200gan_nchw_to_nhwc(const float *x, float *y, int32_t N, int32_t C, int32_t HW, void *stream) {
  B2_CHECK_ARG(x && y, "nchw_to_nhwc: null pointer");
  return launch_transpose(x, y, N, C, HW, as_stream(stream));
}
extern "C" int b200gan_nhwc_to_nchw(const float *x, float *y, int32_t N, int32_t C, int32_t HW, void *stream) {
  B2_CHECK_ARG(x && y, "nhwc_to_nchw: null pointer");
  return launch_transpose(x, y, N, HW, C, as_stream(stream));
}

extern "C" int b200gan_upsample2x_fwd(const float *x, float *y, int32_t N, int32_t H, int32_t W, int32_t C,
                                      void *stream) {
  B2_CHECK_ARG(x && y, "upsample2x_fwd: null pointer");
  int64_t total = (int64_t)N * 4 * H * W * C;
  if (total == 0) return B200GAN_OK;
  upsample2x_fwd_kernel<<<stream_blocks(total), 256, 0, as_stream(stream)>>>(x, y, total, H, W, C);
  B2_LAUNCH_CHECK();
  return B200GAN_OK;
}
extern "C" int b200gan_upsample2x_bwd(const float *dy, float *dx, int32_t N, int32_t H, int32_t W, int32_t C,
                                      void *stream) {
  B2_CHECK_ARG(dy && dx, "upsample2x_bwd: null pointer");
  int64_t total = (int64_t)N * H * W * C;
  if (total == 0) return B200GAN_OK;
  upsample2x_bwd_kernel<<<stream_blocks(total), 256, 0, as_stream(stream)>>>(dy, dx, total, H, W, C);
  B2_LAUNCH_CHECK();
  return B200GAN_OK;
}

extern "C" int b200gan_pad2d_fwd(const float *x, float *y, int32_t N, int32_t H, int32_t W, int32_t C,
                                 int32_t pad_t, int32_t pad_l, int32_t pad_b, int32_t pad_r, int32_t mode,
                                 int32_t round_tf32_, void *stream) {
  B2_CHECK_ARG(x && y, "pad2d_fwd: null pointer");
  B2_CHECK_ARG(mode != B200GAN_PAD_REFLECT || (pad_t < H && pad_b < H && pad_l < W && pad_r < W),
               "pad2d_fwd: reflection pad must be smaller than the input");
  int Ho = H + pad_t + pad_b, Wo = W + pad_l + pad_r;
  int64_t total = (int64_t)N * Ho * Wo * C;
  if (total == 0) return B200GAN_OK;
  if ((C & 3) == 0 && total / 4 < (int64_t)0x7fffffff && (((uintptr_t)x | (uintptr_t)y) & 15) == 0) {
    pad2d_fwd_v4_kernel<<<stream_blocks(total / 4), 256, 0, as_stream(stream)>>>(
        reinterpret_cast<const float4 *>(x), reinterpret_cast<float4 *>(y), (unsigned)(total / 4), H, W, C / 4, Ho, Wo, pad_t,
        pad_l, mode, round_tf32_);
    B2_LAUNCH_CHECK();
    return B200GAN_OK;
  }
  pad2d_fwd_kernel<<<stream_blocks(total), 256, 0, as_stream(stream)>>>(x, y, total, H, W, C, Ho, Wo, pad_t,
                                                                         pad_l, mode, round_tf32_);
  B2_LAUNCH_CHECK();
  return B200GAN_OK;
}
extern "C" int b200gan_pad2d_bwd(const float *dy, float *dx, int32_t N, int32_t H, int32_t W, int32_t C,
                                 int32_t pad_t, int32_t pad_l, int32_t pad_b, int32_t pad_r, int32_t mode,
                                 void *stream) {
  B2_CHECK_ARG(dy && dx, "pad2d_bwd: null pointer");
  B2_CHECK_ARG(mode != B200GAN_PAD_REFLECT || (pad_t < H && pad_b < H && pad_l < W && pad_r < W),
               "pad2d_bwd: reflection pad must be smaller than the input");
  int Ho = H + pad_t + pad_b, Wo = W + pad_l + pad_r;
  int64_t total = (int64_t)N * H * W * C;
  if (total == 0) return B200GAN_OK;
  if ((C & 3) == 0 && total / 4 < (int64_t)0x7fffffff && (((uintptr_t)dy | (uintptr_t)dx) & 15) == 0) {
    pad2d_bwd_v4_kernel<<<stream_blocks(total / 4), 256, 0, as_stream(stream)>>>(
        reinterpret_cast<const float4 *>(dy), reinterpret_cast<float4 *>(dx), (unsigned)(total / 4), H, W, C / 4, Ho, Wo,
        pad_t, pad_l, pad_b, pad_r, mode);
    B2_LAUNCH_CHECK();
    return B200GAN_OK;
  }
  pad2d_bwd_kernel<<<stream_blocks(total), 256, 0, as_stream(stream)>>>(dy, dx, total, H, W, C, Ho, Wo, pad_t,
                                                                         pad_l, pad_b, pad_r, mode);
  B2_LAUNCH_CHECK();
  return B200GAN_OK;
}

extern "C" int b200gan_act_fwd(const float *x, const float *mask, int32_t mask_per_channel, int32_t act,
                               float slope, int64_t n, int32_t C, int64_t HW, float *y, void *stream) {
  B2_CHECK_ARG(x && y, "act_fwd: null pointer");
  if (n == 0) return B200GAN_OK;
  act_fwd_kernel<<<stream_blocks(n), 256, 0, as_stream(stream)>>>(x, mask, mask_per_channel, act, slope, n, C,
                                                                   HW, y);
  B2_LAUNCH_CHECK();
  return B200GAN_OK;
}

extern "C" int b200gan_epilogue_bwd(const float *dy, const float *y, const float *chan_scale, int32_t act,
                                    float slope, int64_t n, int32_t K, int64_t PQ, int32_t round_tf32_,
                                    float *dz, void *stream) {
  B2_CHECK_ARG(dy && dz, "epilogue_bwd: null pointer");
  B2_CHECK_ARG(act == B200GAN_ACT_NONE || y != nullptr, "epilogue_bwd: activation needs saved output");
  if (n == 0) return B200GAN_OK;
  epilogue_bwd_kernel<<<stream_blocks(n), 256, 0, as_stream(stream)>>>(dy, y, chan_scale, act, slope, n, K, PQ,
                                                                        round_tf32_, dz);
  B2_LAUNCH_CHECK();
  return B200GAN_OK;
}

extern "C" int b200gan_adam_multi(const b200gan_adam_tensor *tensors, int32_t count, double lr, double beta1,
                                  double beta2, double eps, float grad_scale, float *step, void *stream) {
  B2_CHECK_ARG(step != nullptr && (count == 0 || tensors != nullptr) && count >= 0, "adam_multi: bad arguments");
  // the whole table before the first launch: a refused call updates no tensor
  for (int i = 0; i < count; ++i) {
    const b200gan_adam_tensor &t = tensors[i];
    B2_CHECK_ARG(t.p && t.g && t.m && t.v && t.n > 0, "adam_multi: tensor %d has a null pointer or no elements", i);
  }
  cudaStream_t st = as_stream(stream);
  if (count == 0) {
    adam_step_inc_kernel<<<1, 1, 0, st>>>(step);
    B2_LAUNCH_CHECK();
    return B200GAN_OK;
  }
  for (int base = 0; base < count; base += ADAM_MAX_TENSORS) {
    AdamTable tb;
    const int c = count - base < ADAM_MAX_TENSORS ? count - base : ADAM_MAX_TENSORS;
    int blocks = 0;
    for (int i = 0; i < c; ++i) {
      const b200gan_adam_tensor &t = tensors[base + i];
      tb.p[i] = t.p; tb.g[i] = t.g; tb.m[i] = t.m; tb.v[i] = t.v; tb.n[i] = t.n;
      tb.block_begin[i] = blocks;
      blocks += (int)ceil_div64(t.n, ADAM_CHUNK);
    }
    tb.block_begin[c] = blocks;
    tb.count = c;
    const int last = base + c >= count;
    adam_multi_kernel<<<(unsigned)blocks, 256, 0, st>>>(tb, lr, beta1, beta2, eps, grad_scale, step, last);
    B2_LAUNCH_CHECK();
  }
  return B200GAN_OK;
}

extern "C" int b200gan_bias_grad(const float *dy, const float *y, const float *chan_scale, int32_t act, float slope,
                                 int64_t rows, int32_t K, int64_t PQ, float *db, void *stream) {
  B2_CHECK_ARG(dy && db, "bias_grad: null pointer");
  B2_CHECK_ARG(act == B200GAN_ACT_NONE || y != nullptr, "bias_grad: activation needs the saved output");
  cudaStream_t st = as_stream(stream);
  B2_CUDA(cudaMemsetAsync(db, 0, (size_t)K * sizeof(float), st));
  if (rows == 0) return B200GAN_OK;
  int64_t yb = num_sms() * 8 / ceil_div(K, 32);
  if (yb < 1) yb = 1;
  int64_t rpb = ceil_div64(rows, yb);
  if (rpb < 64) rpb = 64;
  yb = ceil_div64(rows, rpb);
  bias_grad_kernel<<<dim3((unsigned)ceil_div(K, 32), (unsigned)yb), dim3(32, 8), 0, st>>>(dy, y, chan_scale, act, slope, rows,
                                                                                       K, PQ, rpb, db);
  B2_LAUNCH_CHECK();
  return B200GAN_OK;
}
