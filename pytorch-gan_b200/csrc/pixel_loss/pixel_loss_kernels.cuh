// pixel_loss_kernels.cuh -- the two kernels of the MSE / L1 losses and their device helpers (pixel_loss.cu holds the C
// entry points that launch them).  The fp64 conformance cases of both kernels are the table of
// tests/test_gpu_pixel_loss_conformance.py; tests/test_cpu_pixel_loss.py holds every __global__ under csrc/, in .cu files
// and headers at any depth, to a case.
#pragma once
#include "../common.cuh"

namespace b200gan {

constexpr int PL_THREADS = 256;
constexpr int PL_PER_THREAD = 8;       // elements per thread in one pass of the forward grid
constexpr int PL_MAX_BLOCKS = 1024;    // bound of the forward grid: the last block stages the partials in shared memory
constexpr int PL_TICKET_BYTES = 16;    // workspace: [ticket (unsigned) | pad][double partial per block]

struct PixelLossArgs {
  const float *a, *b;
  int32_t n, C, H, W;
  int32_t mode, same;   // same: both operands in one layout
  int32_t a_nhwc;       // layout of a (b has the other one when !same)
  int32_t vec;          // same layout and both pointers 16-byte aligned: float4 loads
};

// offset in b of the element at offset i of a (layouts differ)
__device__ __forceinline__ uint32_t pl_b_offset(uint32_t i, const PixelLossArgs &p) {
  const uint32_t C = p.C, H = p.H, W = p.W;
  if (p.a_nhwc) {  // a NHWC -> b NCHW
    const uint32_t c = i % C, t = i / C, w = t % W, t2 = t / W, h = t2 % H, nn = t2 / H;
    return ((nn * C + c) * H + h) * W + w;
  }
  const uint32_t w = i % W, t = i / W, h = t % H, t2 = t / H, c = t2 % C, nn = t2 / C;  // a NCHW -> b NHWC
  return ((nn * H + h) * W + w) * C + c;
}

__device__ __forceinline__ float pl_term(float a, float b, int mode) {
  const float d = a - b;
  return mode == B200GAN_PIXEL_LOSS_MSE ? d * d : fabsf(d);
}

// torch.sign semantics: 0 at 0
__device__ __forceinline__ float pl_sign(float d) { return (float)((d > 0.f) - (d < 0.f)); }

// loss = sum(term(a - b)) / n.  Block k sums elements [k * chunk, (k + 1) * chunk) in fp32 per thread, reduces the
// block in fp64 and stores the partial; the last block to finish (atomicInc ticket, which wraps back to 0) adds the
// partials in index order in fp64.  The grid depends on n and the SM count only: bit-identical from run to run.
__global__ void __launch_bounds__(PL_THREADS)
pixel_loss_fwd_kernel(const PixelLossArgs p, int32_t chunk, void *__restrict__ workspace, float *__restrict__ loss) {
  __shared__ double red[PL_THREADS / 32];
  __shared__ double parts[PL_MAX_BLOCKS];
  __shared__ int is_last;
  unsigned *ticket = reinterpret_cast<unsigned *>(workspace);
  double *partials = reinterpret_cast<double *>(reinterpret_cast<char *>(workspace) + PL_TICKET_BYTES);
  const int tid = threadIdx.x;
  const int64_t lo = (int64_t)blockIdx.x * chunk;
  const int64_t hi = min(lo + chunk, (int64_t)p.n);  // <= lo for a trailing empty block
  float s = 0.f;
  if (p.vec) {  // chunk is a multiple of 4: lo is float4-aligned; the last block may end in 1-3 scalars
    const int64_t hv = hi > lo ? lo + ((hi - lo) & ~3ll) : lo;
    const float4 *a4 = reinterpret_cast<const float4 *>(p.a), *b4 = reinterpret_cast<const float4 *>(p.b);
    for (int64_t i = lo + 4 * tid; i < hv; i += 4 * PL_THREADS) {
      const float4 x = __ldg(a4 + (i >> 2)), y = __ldg(b4 + (i >> 2));
      s += pl_term(x.x, y.x, p.mode);
      s += pl_term(x.y, y.y, p.mode);
      s += pl_term(x.z, y.z, p.mode);
      s += pl_term(x.w, y.w, p.mode);
    }
    for (int64_t i = hv + tid; i < hi; i += PL_THREADS) s += pl_term(__ldg(p.a + i), __ldg(p.b + i), p.mode);
  } else if (p.same) {
    for (int64_t i = lo + tid; i < hi; i += PL_THREADS) s += pl_term(__ldg(p.a + i), __ldg(p.b + i), p.mode);
  } else {
    for (int64_t i = lo + tid; i < hi; i += PL_THREADS)
      s += pl_term(__ldg(p.a + i), __ldg(p.b + pl_b_offset((uint32_t)i, p)), p.mode);
  }
  double v = (double)s;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  if ((tid & 31) == 0) red[tid >> 5] = v;
  __syncthreads();
  if (tid == 0) {
    double t = 0.0;
#pragma unroll
    for (int w = 0; w < PL_THREADS / 32; ++w) t += red[w];
    partials[blockIdx.x] = t;
    __threadfence();
    is_last = atomicInc(ticket, gridDim.x - 1) == gridDim.x - 1;  // the last block wraps the ticket back to 0
  }
  __syncthreads();
  if (!is_last) return;
  __threadfence();
  for (int k = tid; k < (int)gridDim.x; k += PL_THREADS) parts[k] = __ldcg(partials + k);
  __syncthreads();
  if (tid == 0) {
    double t = 0.0;
    for (int k = 0; k < (int)gridDim.x; ++k) t += parts[k];
    *loss = (float)(t / (double)p.n);
  }
}

// d_a = 2 (a - b) g / n (MSE) or sign(a - b) g / n (L1), written in a's layout; d_b = -d_a in b's layout (when db).
// g = *gout is read on the device: no host synchronisation.
__global__ void __launch_bounds__(PL_THREADS)
pixel_loss_bwd_kernel(const PixelLossArgs p, const float *__restrict__ gout, float *__restrict__ da,
                      float *__restrict__ db) {
  const double g = (double)__ldg(gout);
  const float scale = (float)((p.mode == B200GAN_PIXEL_LOSS_MSE ? 2.0 : 1.0) * g / (double)p.n);
  const bool mse = p.mode == B200GAN_PIXEL_LOSS_MSE;
  const int64_t stride = (int64_t)gridDim.x * PL_THREADS;
  const int64_t first = (int64_t)blockIdx.x * PL_THREADS + threadIdx.x;
  int64_t scalar_from = 0;
  if (p.vec) {
    const int64_t nv = p.n >> 2;
    const float4 *a4 = reinterpret_cast<const float4 *>(p.a), *b4 = reinterpret_cast<const float4 *>(p.b);
    for (int64_t i = first; i < nv; i += stride) {
      const float4 x = __ldg(a4 + i), y = __ldg(b4 + i);
      float4 d;
      d.x = mse ? (x.x - y.x) * scale : pl_sign(x.x - y.x) * scale;
      d.y = mse ? (x.y - y.y) * scale : pl_sign(x.y - y.y) * scale;
      d.z = mse ? (x.z - y.z) * scale : pl_sign(x.z - y.z) * scale;
      d.w = mse ? (x.w - y.w) * scale : pl_sign(x.w - y.w) * scale;
      reinterpret_cast<float4 *>(da)[i] = d;
      if (db) reinterpret_cast<float4 *>(db)[i] = make_float4(-d.x, -d.y, -d.z, -d.w);
    }
    scalar_from = nv << 2;
  }
  for (int64_t i = scalar_from + first; i < p.n; i += stride) {
    const uint32_t j = p.same ? (uint32_t)i : pl_b_offset((uint32_t)i, p);
    const float diff = __ldg(p.a + i) - __ldg(p.b + j);
    const float d = mse ? diff * scale : pl_sign(diff) * scale;
    da[i] = d;
    if (db) db[j] = -d;
  }
}

}  // namespace b200gan
