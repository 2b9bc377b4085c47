// conv_narrow.cu -- launchers of the narrow-layer convolution kernels (EXPERIMENTAL: B200GAN_NARROW=1).
//
// Per-thread bodies and their rationale: conv_narrow.cuh.  They are checked on CPU by an emulator built from the same
// source (tests/test_cpu_narrow_emulation.py); on the GPU they are exercised by tests/test_gpu_y_narrow.py, which only
// runs when B200GAN_NARROW=1.  Until they have been validated and timed on hardware the generic kernels of
// conv_simt.cu stay the default for these layers (dcgan.py:62,77-88).
#include <stdlib.h>
#include "common.cuh"
#include "conv_narrow.cuh"

namespace b200gan {

template <int KT>
__global__ void __launch_bounds__(256)
narrow_gather_kernel(const narrow::Geom g, const float *__restrict__ x, const float *__restrict__ wp, float *__restrict__ y) {
  int64_t m;
  int kg;
  narrow::gather_coords(g, KT, (int64_t)blockIdx.x * blockDim.x + threadIdx.x, &m, &kg);
  narrow::gather_thread<KT>(g, x, wp, y, m, kg, (int)blockIdx.z);
}

template <int DT>
__global__ void __launch_bounds__(256)
narrow_wgrad_kernel(const narrow::Geom g, const float *__restrict__ xg, const float *__restrict__ dn, float *__restrict__ dw,
                    int Cd, int64_t m_per_split) {
  const int64_t o = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t mb = (int64_t)blockIdx.y * m_per_split;
  narrow::wgrad_thread<DT>(g, xg, dn, dw, Cd, o, mb, mb + m_per_split, [](float *p, float v) { atomicAdd(p, v); });
}

bool narrow_enabled() {
  static const bool on = [] {
    const char *e = getenv("B200GAN_NARROW");
    return e && atoi(e) != 0;
  }();
  return on;
}

static bool aligned16(const void *p) { return ((uintptr_t)p & 15) == 0; }

// Which launches the narrow kernels take: zero padding, no folded upsample, stride 1 or 2, at most 64 channels on either
// side and a weight matrix that stays in L1 (<= 96 KB).
bool narrow_gather_ok(int C, int K, int R, int S, int stride, int pad_mode, int up, const void *x, const void *wp,
                      const void *y) {
  if (pad_mode != B200GAN_PAD_ZERO || up != 1 || (stride != 1 && stride != 2)) return false;
  if (C < 1 || K < 1 || C > 64 || K > 64) return false;
  if ((int64_t)R * S * C * K * 4 > 96 * 1024) return false;
  // one thread per pixel reading > 64 B of channels: a warp's 16-byte loads scatter over 32 lines and the L1 becomes
  // the bottleneck (estimate for the 64 -> 1 output conv: 2.5x slower than the lane-per-channel kernels)
  if (K < 4 && C > 16) return false;
  return aligned16(x) && aligned16(wp) && aligned16(y);
}

int narrow_gather(int N, int H, int W, int C, int P, int Q, int K, int R, int S, int stride, int pad_t, int pad_l, int mode,
                  const b200gan_epilogue *ep, const float *x, const float *wp, float *y, cudaStream_t st) {
  narrow::Geom g;
  g.N = N; g.H = H; g.W = W; g.C = C; g.P = P; g.Q = Q; g.K = K; g.R = R; g.S = S;
  g.stride = stride; g.pad_t = pad_t; g.pad_l = pad_l; g.mode = mode;
  g.bias = ep ? ep->bias : nullptr;
  g.chan_scale = ep ? ep->chan_scale : nullptr;
  g.act = ep ? ep->act : 0;
  g.slope = ep ? ep->slope : 0.f;
  g.rtf = ep ? ep->round_tf32 : 0;
  if ((int64_t)N * P * Q == 0) return B200GAN_OK;
  const int KT = (K % 8 == 0) ? 8 : ((K % 4 == 0) ? 4 : 1);
  const int ncls = narrow::num_classes(g);
  const int64_t threads = narrow::gather_threads(g, KT, 0);  // class 0 is the largest
  dim3 grid((unsigned)ceil_div64(threads, 256), 1, (unsigned)ncls);
  if (KT == 8) narrow_gather_kernel<8><<<grid, 256, 0, st>>>(g, x, wp, y);
  else if (KT == 4) narrow_gather_kernel<4><<<grid, 256, 0, st>>>(g, x, wp, y);
  else narrow_gather_kernel<1><<<grid, 256, 0, st>>>(g, x, wp, y);
  B2_LAUNCH_CHECK();
  return B200GAN_OK;
}

bool narrow_wgrad_ok(int64_t gathered_floats, int Cg, int Cd, int R, int S, int pad_mode, int up, const void *xg,
                     const void *dn) {
  if (pad_mode != B200GAN_PAD_ZERO || up != 1) return false;
  if (Cg < 1 || Cd < 1 || Cg > 64 || Cd > 64 || R * S > 49) return false;
  // every tap is its own set of threads, so the gathered tensor is read R*S times: it has to sit in L2
  if (gathered_floats * 4 > (int64_t)32 << 20) return false;
  return aligned16(xg) && aligned16(dn);
}

// dw [Cd][Cg][R][S] must be zero on entry (simt_wgrad clears it).
int narrow_wgrad(int N, int H, int W, int Cg, int P, int Q, int Cd, int R, int S, int stride, int pad_t, int pad_l,
                 const float *xg, const float *dn, float *dw, cudaStream_t st) {
  narrow::Geom g;
  g.N = N; g.H = H; g.W = W; g.C = Cg; g.P = P; g.Q = Q; g.K = Cd; g.R = R; g.S = S;
  g.stride = stride; g.pad_t = pad_t; g.pad_l = pad_l; g.mode = 0;
  g.bias = nullptr; g.chan_scale = nullptr; g.act = 0; g.slope = 0.f; g.rtf = 0;
  const int64_t M = (int64_t)N * P * Q;
  if (M == 0) return B200GAN_OK;
  const int DT = (Cd % 4 == 0) ? 4 : 1;
  const int64_t nout = (int64_t)R * S * Cg * (Cd / DT);
  // ~150k threads in total (half of what the SMs hold), at least 64 pixels per thread
  int64_t splits = ceil_div64(150000, nout);
  if (splits > ceil_div64(M, 64)) splits = ceil_div64(M, 64);
  if (splits < 1) splits = 1;
  if (splits > 65535) splits = 65535;
  const int64_t per = ceil_div64(M, splits);
  splits = ceil_div64(M, per);
  dim3 grid((unsigned)ceil_div64(nout, 256), (unsigned)splits);
  if (DT == 4) narrow_wgrad_kernel<4><<<grid, 256, 0, st>>>(g, xg, dn, dw, Cd, per);
  else narrow_wgrad_kernel<1><<<grid, 256, 0, st>>>(g, xg, dn, dw, Cd, per);
  B2_LAUNCH_CHECK();
  return B200GAN_OK;
}

}  // namespace b200gan
