// conv_simt.cu -- fp32 FFMA implicit-GEMM convolution kernels (any geometry).
//
// These kernels serve (1) the HBM-bound layers with tiny channel counts where tensor cores
// cannot be fed (DCGAN discriminator 1->16->32->64->128 k3 s2, dcgan.py:77-88; the 64->1
// output conv dcgan.py:62; pix2pix/cyclegan C=3 edge layers) and (2) every other geometry as
// the always-correct fp32 path that the wgmma kernels are validated against on the GPU.
//
// One gather function maps an output pixel + filter tap to the stored input pixel, covering
// stride, zero / reflection padding (cyclegan/models.py:27,49), a folded nearest x2 upsample
// (dcgan.py:54,58) and the transposed ("fractionally strided") form used for
// ConvTranspose2d fprop (pix2pix/models.py:39) and Conv2d dgrad.
#include "common.cuh"

namespace b200gan {

struct GatherP {
  int N, H, W, C;      // stored (gathered) tensor dims, NHWC
  int P, Q;            // output pixel grid
  int R, S;
  int stride, pad_t, pad_l;
  int pad_mode, up;    // only for mode 0
  int Hv, Wv;          // H*up, W*up
  int mode;            // 0: ih = p*stride - pad + r ; 1: ih = (p + pad - r)/stride (if divisible)
  int cls;             // mode 1, stride > 1: blockIdx.z enumerates the stride^2 output parity classes, each with
                       // its own compact tap set (no work on taps that can never divide); 1 = off
};

// returns element offset of pixel (n, ih, iw) in the stored tensor or -1 if it contributes 0
__device__ __forceinline__ int64_t gather_pixel(const GatherP &g, int n, int p, int q, int r, int s) {
  int ih, iw;
  if (g.mode == 0) {
    int vh = p * g.stride - g.pad_t + r;
    int vw = q * g.stride - g.pad_l + s;
    if (g.pad_mode == B200GAN_PAD_REFLECT) {
      vh = reflect_idx(vh, g.Hv);
      vw = reflect_idx(vw, g.Wv);
    } else if (vh < 0 || vh >= g.Hv || vw < 0 || vw >= g.Wv) {
      return -1;
    }
    ih = g.up == 2 ? (vh >> 1) : vh;
    iw = g.up == 2 ? (vw >> 1) : vw;
  } else {
    int th = p + g.pad_t - r;
    int tw = q + g.pad_l - s;
    if (th < 0 || tw < 0) return -1;
    if (g.stride > 1) {
      if (th % g.stride != 0 || tw % g.stride != 0) return -1;
      th /= g.stride;
      tw /= g.stride;
    }
    if (th >= g.H || tw >= g.W) return -1;
    ih = th;
    iw = tw;
  }
  return ((int64_t)(n * g.H + ih) * g.W + iw) * g.C;
}

struct EpiP {
  const float *bias;
  const float *chan_scale;
  int act;
  float slope;
  int round_tf32;
};

// ------------------------------------------------------------------------------------------
// y[M][K] = A[M][RSC] * B[RSC][K],  M = N*P*Q.  64x64 tile, BK = 16, 256 threads, 4x4 / thread.
// ------------------------------------------------------------------------------------------
constexpr int FBM = 64, FBN = 64, FBK = 16, FPAD = 4;

__global__ void __launch_bounds__(256)
conv_gather_gemm_kernel(GatherP g, EpiP ep, const float *__restrict__ x,
                        const float *__restrict__ wp, float *__restrict__ y, int K) {
  __shared__ __align__(16) float As[FBK][FBM + FPAD];
  __shared__ __align__(16) float Bs[FBK][FBN + FPAD];
  const int tid = threadIdx.x;
  const int tm = tid >> 4, tn = tid & 15;
  // parity-class decomposition of the transposed gather (stride-2 dgrad: 9 taps -> 1/2/2/4 per class)
  const int cls = g.cls;
  int pa = 0, pb = 0, r0 = 0, s0 = 0, Rc = g.R, Sc = g.S, Pc = g.P, Qc = g.Q;
  if (cls > 1) {
    pa = blockIdx.z / cls;
    pb = blockIdx.z % cls;
    r0 = (pa + g.pad_t) % cls;
    s0 = (pb + g.pad_l) % cls;
    Rc = r0 < g.R ? (g.R - r0 + cls - 1) / cls : 0;
    Sc = s0 < g.S ? (g.S - s0 + cls - 1) / cls : 0;
    Pc = pa < g.P ? (g.P - pa + cls - 1) / cls : 0;
    Qc = pb < g.Q ? (g.Q - pb + cls - 1) / cls : 0;
  }
  const int64_t M = (int64_t)g.N * Pc * Qc;
  const int Ktot = Rc * Sc * g.C;
  const int64_t m0 = (int64_t)blockIdx.x * FBM;
  const int n0 = blockIdx.y * FBN;
  if (m0 >= M) return;

  // the 4 A rows this thread gathers: rows (tid>>4) + 16*i, column kk = tid & 15
  const int a_kk = tid & 15;
  int a_n[4], a_p[4], a_q[4];
  bool a_ok[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    int64_t m = m0 + (tid >> 4) + 16 * i;
    a_ok[i] = m < M;
    int64_t mm = a_ok[i] ? m : 0;
    a_q[i] = pb + cls * (int)(mm % Qc);
    int64_t t = mm / Qc;
    a_p[i] = pa + cls * (int)(t % Pc);
    a_n[i] = (int)(t / Pc);
  }
  const int b_n = tid & 63, b_k = tid >> 6;

  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

  for (int k0 = 0; k0 < Ktot; k0 += FBK) {
    {  // A tile
      int k = k0 + a_kk;
      bool kok = k < Ktot;
      int c = 0, r = 0, s = 0;
      if (kok) {
        c = k % g.C;
        int t = k / g.C;
        s = s0 + cls * (t % Sc);
        r = r0 + cls * (t / Sc);
      }
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        float v = 0.f;
        if (kok && a_ok[i]) {
          int64_t off = gather_pixel(g, a_n[i], a_p[i], a_q[i], r, s);
          if (off >= 0) v = __ldg(x + off + c);
        }
        As[a_kk][(tid >> 4) + 16 * i] = v;
      }
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) {  // B tile
      int k = k0 + b_k + 4 * i;
      int n = n0 + b_n;
      float v = 0.f;
      if (k < Ktot && n < K) {
        if (cls == 1) {
          v = __ldg(wp + (int64_t)k * K + n);
        } else {
          int c = k % g.C;
          int t = k / g.C;
          int s = s0 + cls * (t % Sc), r = r0 + cls * (t / Sc);
          v = __ldg(wp + ((int64_t)(r * g.S + s) * g.C + c) * K + n);
        }
      }
      Bs[b_k + 4 * i][b_n] = v;
    }
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < FBK; ++kk) {
      float4 a4 = *reinterpret_cast<const float4 *>(&As[kk][tm * 4]);
      float4 b4 = *reinterpret_cast<const float4 *>(&Bs[kk][tn * 4]);
      float a[4] = {a4.x, a4.y, a4.z, a4.w};
      float b[4] = {b4.x, b4.y, b4.z, b4.w};
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    __syncthreads();
  }

#pragma unroll
  for (int i = 0; i < 4; ++i) {
    int64_t m = m0 + tm * 4 + i;
    if (m >= M) continue;
    const int q = pb + cls * (int)(m % Qc);
    const int64_t t = m / Qc;
    const int pp = pa + cls * (int)(t % Pc);
    const int64_t n_img = t / Pc;
    const int64_t mfull = (n_img * g.P + pp) * g.Q + q;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      int k = n0 + tn * 4 + j;
      if (k >= K) continue;
      float v = acc[i][j];
      if (ep.bias) v += __ldg(ep.bias + k);
      v = apply_act(v, ep.act, ep.slope);
      if (ep.chan_scale) v *= __ldg(ep.chan_scale + n_img * K + k);
      if (ep.round_tf32) v = round_tf32(v);
      y[mfull * K + k] = v;
    }
  }
}

// ------------------------------------------------------------------------------------------
// Few output channels (K <= 4): one warp per output pixel, lanes stride the (r,s,c) reduction.
// dcgan.py:62 (64->1), pix2pix/models.py:79 (128->3), cyclegan/models.py:82 (64->3),
// PatchGAN heads 512->1.
// ------------------------------------------------------------------------------------------
template <int KMAX>
__global__ void __launch_bounds__(256)
conv_gather_smallk_kernel(GatherP g, EpiP ep, const float *__restrict__ x,
                          const float *__restrict__ wp, float *__restrict__ y, int K) {
  extern __shared__ float wsm[];  // [Ktot][K]
  const int Ktot = g.R * g.S * g.C;
  for (int i = threadIdx.x; i < Ktot * K; i += blockDim.x) wsm[i] = wp[i];
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const int warp = threadIdx.x >> 5;
  const int64_t M = (int64_t)g.N * g.P * g.Q;
  const int64_t PQ = (int64_t)g.P * g.Q;
  for (int64_t m = (int64_t)blockIdx.x * 8 + warp; m < M; m += (int64_t)gridDim.x * 8) {
    int q = (int)(m % g.Q);
    int64_t t = m / g.Q;
    int p = (int)(t % g.P);
    int n = (int)(t / g.P);
    float acc[KMAX];
#pragma unroll
    for (int j = 0; j < KMAX; ++j) acc[j] = 0.f;
    for (int r = 0; r < g.R; ++r)
      for (int s = 0; s < g.S; ++s) {
        int64_t off = gather_pixel(g, n, p, q, r, s);
        if (off < 0) continue;
        const float *xp = x + off;
        const float *wr = wsm + (int64_t)((r * g.S + s) * g.C) * K;
        for (int c = lane; c < g.C; c += 32) {
          float xv = __ldg(xp + c);
#pragma unroll
          for (int j = 0; j < KMAX; ++j)
            if (j < K) acc[j] = fmaf(xv, wr[c * K + j], acc[j]);
        }
      }
#pragma unroll
    for (int j = 0; j < KMAX; ++j)
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) acc[j] += __shfl_xor_sync(0xffffffffu, acc[j], o);
    if (lane == 0) {
      int64_t n_img = m / PQ;
#pragma unroll
      for (int j = 0; j < KMAX; ++j) {
        if (j >= K) break;
        float v = acc[j];
        if (ep.bias) v += __ldg(ep.bias + j);
        v = apply_act(v, ep.act, ep.slope);
        if (ep.chan_scale) v *= __ldg(ep.chan_scale + n_img * K + j);
        if (ep.round_tf32) v = round_tf32(v);
        y[m * K + j] = v;
      }
    }
  }
}

// ------------------------------------------------------------------------------------------
// Weight gradient:  Wg[(r,s,cg)][cd] = sum_m Agather[m][(r,s,cg)] * D[m][cd]
//   Conv2d         : gathered = x (mode 0), dense D = dz[N][P][Q][K]   -> dW[K][C][R][S]
//   ConvTranspose2d: gathered = dy (mode 0 over dy), dense D = x        -> dW[C][K][R][S]
// Output element index = ((cd * Cg + cg) * R + r) * S + s  (both cases).
// 64 x 64 tile, reduction over pixels split across blockIdx.z, atomicAdd into zeroed dw.
// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
conv_wgrad_kernel(GatherP g, const float *__restrict__ xg, const float *__restrict__ dn,
                  float *__restrict__ dw, int Cd, int64_t m_per_split) {
  __shared__ __align__(16) float As[FBK][FBM + FPAD];  // [pixel][kdim]
  __shared__ __align__(16) float Ds[FBK][FBN + FPAD];  // [pixel][cd]
  const int tid = threadIdx.x;
  const int tk = tid >> 4, td = tid & 15;
  const int64_t M = (int64_t)g.N * g.P * g.Q;
  const int Ktot = g.R * g.S * g.C;
  const int kd0 = blockIdx.x * FBM;
  const int cd0 = blockIdx.y * FBN;
  const int64_t m_begin = (int64_t)blockIdx.z * m_per_split;
  int64_t m_end = m_begin + m_per_split;
  if (m_end > M) m_end = M;

  // this thread gathers column kd = kd0 + (tid & 63) for pixels (tid >> 6) + 4*i
  const int a_kd = kd0 + (tid & 63);
  const bool a_kok = a_kd < Ktot;
  int a_c = 0, a_r = 0, a_s = 0;
  if (a_kok) {
    a_c = a_kd % g.C;
    int t = a_kd / g.C;
    a_s = t % g.S;
    a_r = t / g.S;
  }
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

  for (int64_t mb = m_begin; mb < m_end; mb += FBK) {
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      int mm = (tid >> 6) + 4 * i;
      int64_t m = mb + mm;
      float av = 0.f, dv = 0.f;
      if (m < m_end) {
        if (a_kok) {
          int q = (int)(m % g.Q);
          int64_t t = m / g.Q;
          int p = (int)(t % g.P);
          int n = (int)(t / g.P);
          int64_t off = gather_pixel(g, n, p, q, a_r, a_s);
          if (off >= 0) av = __ldg(xg + off + a_c);
        }
        int cd = cd0 + (tid & 63);
        if (cd < Cd) dv = __ldg(dn + m * Cd + cd);
      }
      As[mm][tid & 63] = av;
      Ds[mm][tid & 63] = dv;
    }
    __syncthreads();
#pragma unroll
    for (int mm = 0; mm < FBK; ++mm) {
      float4 a4 = *reinterpret_cast<const float4 *>(&As[mm][tk * 4]);
      float4 d4 = *reinterpret_cast<const float4 *>(&Ds[mm][td * 4]);
      float a[4] = {a4.x, a4.y, a4.z, a4.w};
      float d[4] = {d4.x, d4.y, d4.z, d4.w};
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], d[j], acc[i][j]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    int kd = kd0 + tk * 4 + i;
    if (kd >= Ktot) continue;
    int cg = kd % g.C;
    int t = kd / g.C;
    int s = t % g.S, r = t / g.S;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      int cd = cd0 + td * 4 + j;
      if (cd >= Cd) continue;
      atomicAdd(dw + (((int64_t)cd * g.C + cg) * g.R + r) * g.S + s, acc[i][j]);
    }
  }
}


// ------------------------------------------------------------------------------------------
// Few output channels (K <= 4), C % 4 == 0: L lanes (float4 each) cover the channels of one pixel,
// 32/L pixel groups per warp, PIX pixels per group in flight (independent loads for latency hiding).
// Weights sit in shared memory as [k][tap][C] so a lane reads float4 weights next to float4 inputs.
// HBM-bound: dcgan.py:62 (64->1) reads 134 MB of activations per call.
// ------------------------------------------------------------------------------------------
template <int L, int PIX>
__global__ void __launch_bounds__(256)
conv_smallk_vec_kernel(GatherP g, EpiP ep, const float *__restrict__ x, const float *__restrict__ wp,
                       float *__restrict__ y, int K) {
  extern __shared__ __align__(16) float wsm[];  // [K][R*S][C]
  const int taps = g.R * g.S;
  for (int i = threadIdx.x; i < taps * g.C * K; i += blockDim.x) {
    int k = i % K;
    int tc = i / K;  // tap * C + c
    wsm[(size_t)k * taps * g.C + tc] = wp[i];
  }
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const int sl = lane % L, sg = lane / L;
  constexpr int GROUPS = 32 / L;
  const int64_t M = (int64_t)g.N * g.P * g.Q;
  const int64_t PQ = (int64_t)g.P * g.Q;
  const int64_t warp_global = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int64_t warps_total = (int64_t)gridDim.x * (blockDim.x >> 5);
  for (int64_t base = warp_global * (GROUPS * PIX); base < M; base += warps_total * (GROUPS * PIX)) {
    int pn[PIX], pp[PIX], pq[PIX];
    bool ok[PIX];
    float acc[PIX][4];
#pragma unroll
    for (int i = 0; i < PIX; ++i) {
      int64_t m = base + sg * PIX + i;
      ok[i] = m < M;
      int64_t mm = ok[i] ? m : 0;
      pq[i] = (int)(mm % g.Q);
      int64_t t = mm / g.Q;
      pp[i] = (int)(t % g.P);
      pn[i] = (int)(t / g.P);
#pragma unroll
      for (int k = 0; k < 4; ++k) acc[i][k] = 0.f;
    }
    for (int r = 0; r < g.R; ++r)
      for (int s = 0; s < g.S; ++s) {
        int64_t off[PIX];
#pragma unroll
        for (int i = 0; i < PIX; ++i) off[i] = ok[i] ? gather_pixel(g, pn[i], pp[i], pq[i], r, s) : -1;
        const float *wt = wsm + (size_t)(r * g.S + s) * g.C;
        for (int c0 = sl * 4; c0 < g.C; c0 += L * 4) {
          float4 xv[PIX];
#pragma unroll
          for (int i = 0; i < PIX; ++i)
            xv[i] = off[i] >= 0 ? __ldg(reinterpret_cast<const float4 *>(x + off[i] + c0)) : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
          for (int k = 0; k < 4; ++k) {
            if (k < K) {
              float4 w4 = *reinterpret_cast<const float4 *>(wt + (size_t)k * taps * g.C + c0);
#pragma unroll
              for (int i = 0; i < PIX; ++i)
                acc[i][k] += xv[i].x * w4.x + xv[i].y * w4.y + xv[i].z * w4.z + xv[i].w * w4.w;
            }
          }
        }
      }
#pragma unroll
    for (int i = 0; i < PIX; ++i)
#pragma unroll
      for (int k = 0; k < 4; ++k)
#pragma unroll
        for (int o = L / 2; o > 0; o >>= 1) acc[i][k] += __shfl_xor_sync(0xffffffffu, acc[i][k], o);
    if (sl == 0) {
#pragma unroll
      for (int i = 0; i < PIX; ++i) {
        if (!ok[i]) continue;
        int64_t m = base + sg * PIX + i;
        int64_t n_img = m / PQ;
        for (int k = 0; k < K; ++k) {
          float v = acc[i][k];
          if (ep.bias) v += __ldg(ep.bias + k);
          v = apply_act(v, ep.act, ep.slope);
          if (ep.chan_scale) v *= __ldg(ep.chan_scale + n_img * K + k);
          if (ep.round_tf32) v = round_tf32(v);
          y[m * K + k] = v;
        }
      }
    }
  }
}

// ------------------------------------------------------------------------------------------
// Few gathered channels (C <= 8), K % 4 == 0: one thread per (output pixel, 4 output channels).
// Output-write bound: DCGAN D block 1 (1->16, dcgan.py:84), the data gradient of the 64->1 output conv
// (dcgan.py:62), pix2pix/cyclegan first layers (3->64).  Weights [R*S*C][K] live in shared memory.
// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
conv_smallc_kernel(GatherP g, EpiP ep, const float *__restrict__ x, const float *__restrict__ wp,
                   float *__restrict__ y, int K) {
  extern __shared__ __align__(16) float wsm[];  // [R*S*C][K]
  const int taps = g.R * g.S;
  for (int i = threadIdx.x; i < taps * g.C * K; i += blockDim.x) wsm[i] = wp[i];
  __syncthreads();
  const int KQ = K >> 2;
  const int64_t M = (int64_t)g.N * g.P * g.Q;
  const int64_t PQ = (int64_t)g.P * g.Q;
  const int64_t total = M * KQ;
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (int64_t)gridDim.x * blockDim.x) {
    const int kq = (int)(idx % KQ);
    const int64_t m = idx / KQ;
    const int q = (int)(m % g.Q);
    const int64_t t = m / g.Q;
    const int p = (int)(t % g.P);
    const int n = (int)(t / g.P);
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int r = 0; r < g.R; ++r)
      for (int s = 0; s < g.S; ++s) {
        int64_t off = gather_pixel(g, n, p, q, r, s);
        if (off < 0) continue;
        const float *wt = wsm + (size_t)((r * g.S + s) * g.C) * K + kq * 4;
        for (int c = 0; c < g.C; ++c) {
          float xv = __ldg(x + off + c);
          float4 w4 = *reinterpret_cast<const float4 *>(wt + (size_t)c * K);
          acc.x = fmaf(xv, w4.x, acc.x);
          acc.y = fmaf(xv, w4.y, acc.y);
          acc.z = fmaf(xv, w4.z, acc.z);
          acc.w = fmaf(xv, w4.w, acc.w);
        }
      }
    float v[4] = {acc.x, acc.y, acc.z, acc.w};
    const int64_t n_img = m / PQ;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      int k = kq * 4 + j;
      if (ep.bias) v[j] += __ldg(ep.bias + k);
      v[j] = apply_act(v[j], ep.act, ep.slope);
      if (ep.chan_scale) v[j] *= __ldg(ep.chan_scale + n_img * K + k);
      if (ep.round_tf32) v[j] = round_tf32(v[j]);
    }
    *reinterpret_cast<float4 *>(y + m * K + kq * 4) = make_float4(v[0], v[1], v[2], v[3]);
  }
}

// ------------------------------------------------------------------------------------------
// Weight gradient with few dense channels (Cd <= 4): thread per (r,s,cg) column, loop over a pixel range,
// block-wide partial sums -> atomicAdd.  dcgan.py:62 (64->1): a 524288-pixel reduction reading 134 MB.
// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
conv_wgrad_smallcd_kernel(GatherP g, const float *__restrict__ xg, const float *__restrict__ dn,
                          float *__restrict__ dw, int Cd, int64_t m_per_block) {
  const int Ktot = g.R * g.S * g.C;
  const int kd = blockIdx.y * blockDim.x + threadIdx.x;
  const bool kok = kd < Ktot;
  int c = 0, r = 0, s = 0;
  if (kok) {
    c = kd % g.C;
    int t = kd / g.C;
    s = t % g.S;
    r = t / g.S;
  }
  const int64_t M = (int64_t)g.N * g.P * g.Q;
  const int64_t m0 = (int64_t)blockIdx.x * m_per_block;
  int64_t m1 = m0 + m_per_block;
  if (m1 > M) m1 = M;
  float acc[4] = {0.f, 0.f, 0.f, 0.f};
  if (kok) {
    int q = (int)(m0 % g.Q);
    int64_t t = m0 / g.Q;
    int p = (int)(t % g.P);
    int n = (int)(t / g.P);
    for (int64_t m = m0; m < m1; ++m) {
      int64_t off = gather_pixel(g, n, p, q, r, s);
      if (off >= 0) {
        float xv = __ldg(xg + off + c);
#pragma unroll
        for (int j = 0; j < 4; ++j)
          if (j < Cd) acc[j] = fmaf(xv, __ldg(dn + m * Cd + j), acc[j]);
      }
      if (++q == g.Q) {
        q = 0;
        if (++p == g.P) {
          p = 0;
          ++n;
        }
      }
    }
    for (int j = 0; j < Cd; ++j) atomicAdd(dw + (((int64_t)j * g.C + c) * g.R + r) * g.S + s, acc[j]);
  }
}


// ==========================================================================================
// Lean kernels for the HBM-bound 3x3 / stride-1 / zero-pad layers with one tiny channel side
// (dcgan.py:62: Conv2d(64, 1, 3, 1, 1) on [128,64,64,64] -- 134 MB of activations per pass).
// No generic gather: rows/cols are walked incrementally, every input element is loaded once per
// pixel group and reused from registers across the taps.
// ==========================================================================================

// fprop, K <= 4 output channels: L lanes x float4 cover the C channels of a pixel; each lane group
// produces PX = 4 consecutive output pixels of one row from a (3 x 6) window of input pixels.
template <int L, int KK>
__global__ void __launch_bounds__(256)
conv3x3s1_smallk_kernel(const float *__restrict__ x, const float *__restrict__ wp, float *__restrict__ y, EpiP ep,
                        int N, int H, int W, int C, int dir) {
  // wp: [3][3][C][KK] (SIMT fprop pack).  dir = +1: y[p] = sum x[p + r - 1] w[r] (conv fprop, pad 1);
  // dir = -1: taps mirrored (transposed gather: y[p] = sum x[p + 1 - r] w[r]).
  extern __shared__ __align__(16) float wsm[];  // [KK][9][C]
  for (int i = threadIdx.x; i < 9 * C * KK; i += blockDim.x) {
    int k = i % KK, tc = i / KK;
    wsm[(size_t)k * 9 * C + tc] = wp[i];
  }
  __syncthreads();
  constexpr int PX = 4, GROUPS = 32 / L;
  const int lane = threadIdx.x & 31, sl = lane % L, sg = lane / L;
  const int QG = (W + PX - 1) / PX;
  const int64_t ngroups = (int64_t)N * H * QG;
  const int64_t gstride = (int64_t)gridDim.x * (blockDim.x >> 5) * GROUPS;
  for (int64_t gi = ((int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5)) * GROUPS + sg;
       gi - sg < ngroups; gi += gstride) {  // whole warp iterates together (shuffles below)
    const bool gok = gi < ngroups;
    const int64_t g2 = gok ? gi : 0;
    const int q0 = (int)(g2 % QG) * PX;
    const int64_t t = g2 / QG;
    const int p = (int)(t % H), n = (int)(t / H);
    float acc[PX][KK];
#pragma unroll
    for (int o = 0; o < PX; ++o)
#pragma unroll
      for (int k = 0; k < KK; ++k) acc[o][k] = 0.f;
    for (int c0 = sl * 4; c0 < C; c0 += L * 4) {
#pragma unroll
      for (int r = 0; r < 3; ++r) {
        const int ih = p + dir * (r - 1);
        if (!gok || ih < 0 || ih >= H) continue;
        const float *xrow = x + ((int64_t)(n * H + ih) * W) * C + c0;
        float4 xv[PX + 2];
#pragma unroll
        for (int j = 0; j < PX + 2; ++j) {
          const int iw = q0 + j - 1;
          xv[j] = (iw >= 0 && iw < W) ? __ldg(reinterpret_cast<const float4 *>(xrow + (int64_t)iw * C))
                                      : make_float4(0.f, 0.f, 0.f, 0.f);
        }
#pragma unroll
        for (int sx = 0; sx < 3; ++sx) {
          // input column offset sx-1 relative to the output pixel  <->  filter column s = 1 + dir*(sx-1)
          const int s = 1 + dir * (sx - 1);
#pragma unroll
          for (int k = 0; k < KK; ++k) {
            const float4 w4 = *reinterpret_cast<const float4 *>(wsm + (size_t)k * 9 * C + (size_t)(r * 3 + s) * C + c0);
#pragma unroll
            for (int o = 0; o < PX; ++o) {
              const float4 v = xv[o + sx];
              acc[o][k] += v.x * w4.x + v.y * w4.y + v.z * w4.z + v.w * w4.w;
            }
          }
        }
      }
    }
#pragma unroll
    for (int o = 0; o < PX; ++o)
#pragma unroll
      for (int k = 0; k < KK; ++k)
#pragma unroll
        for (int d = L / 2; d > 0; d >>= 1) acc[o][k] += __shfl_xor_sync(0xffffffffu, acc[o][k], d);
    if (gok && sl == 0) {
#pragma unroll
      for (int o = 0; o < PX; ++o) {
        if (q0 + o >= W) continue;
        const int64_t m = ((int64_t)(n * H + p) * W) + q0 + o;
#pragma unroll
        for (int k = 0; k < KK; ++k) {
          float v = acc[o][k];
          if (ep.bias) v += __ldg(ep.bias + k);
          v = apply_act(v, ep.act, ep.slope);
          if (ep.chan_scale) v *= __ldg(ep.chan_scale + (int64_t)n * KK + k);
          if (ep.round_tf32) v = round_tf32(v);
          y[m * KK + k] = v;
        }
      }
    }
  }
}

// few gathered channels (CG <= 4), many outputs (K % 8 == 0): thread = (pixel, 8 output channels).
template <int CG>
__global__ void __launch_bounds__(256)
conv3x3s1_smallc_kernel(const float *__restrict__ x, const float *__restrict__ wp, float *__restrict__ y, EpiP ep,
                        int N, int H, int W, int K, int dir) {
  extern __shared__ __align__(16) float wsm[];  // [9][CG][K]
  for (int i = threadIdx.x; i < 9 * CG * K; i += blockDim.x) wsm[i] = wp[i];
  __syncthreads();
  const int KO = K >> 3;
  const int64_t total = (int64_t)N * H * W * KO;
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (int64_t)gridDim.x * blockDim.x) {
    const int ko = (int)(idx % KO);
    const int64_t m = idx / KO;
    const int q = (int)(m % W);
    const int64_t t = m / W;
    const int p = (int)(t % H), n = (int)(t / H);
    float acc[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] = 0.f;
#pragma unroll
    for (int r = 0; r < 3; ++r) {
      const int ih = p + dir * (r - 1);
      if (ih < 0 || ih >= H) continue;
      const float *xrow = x + ((int64_t)(n * H + ih) * W) * CG;
#pragma unroll
      for (int s = 0; s < 3; ++s) {
        const int iw = q + dir * (s - 1);
        if (iw < 0 || iw >= W) continue;
        const float *wt = wsm + (size_t)((r * 3 + s) * CG) * K + ko * 8;
#pragma unroll
        for (int c = 0; c < CG; ++c) {
          const float xv = __ldg(xrow + (int64_t)iw * CG + c);
          const float4 a = *reinterpret_cast<const float4 *>(wt + (size_t)c * K);
          const float4 b = *reinterpret_cast<const float4 *>(wt + (size_t)c * K + 4);
          acc[0] = fmaf(xv, a.x, acc[0]); acc[1] = fmaf(xv, a.y, acc[1]);
          acc[2] = fmaf(xv, a.z, acc[2]); acc[3] = fmaf(xv, a.w, acc[3]);
          acc[4] = fmaf(xv, b.x, acc[4]); acc[5] = fmaf(xv, b.y, acc[5]);
          acc[6] = fmaf(xv, b.z, acc[6]); acc[7] = fmaf(xv, b.w, acc[7]);
        }
      }
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int k = ko * 8 + j;
      if (ep.bias) acc[j] += __ldg(ep.bias + k);
      acc[j] = apply_act(acc[j], ep.act, ep.slope);
      if (ep.chan_scale) acc[j] *= __ldg(ep.chan_scale + (int64_t)n * K + k);
      if (ep.round_tf32) acc[j] = round_tf32(acc[j]);
    }
    float4 *dst = reinterpret_cast<float4 *>(y + m * K + ko * 8);
    dst[0] = make_float4(acc[0], acc[1], acc[2], acc[3]);
    dst[1] = make_float4(acc[4], acc[5], acc[6], acc[7]);
  }
}

// weight gradient with ONE dense channel (Cd == 1): stream the gathered tensor once (L lanes x float4 per pixel),
// multiply by the 9 neighbouring dz scalars, keep 9 x 4 accumulators per lane; block partials -> atomicAdd.
// dw[0][c][r][s] += sum_pix x[pix][c] * dz[pix + pad - (r,s)]      (mode 0, stride 1, pad 1)
template <int L>
__global__ void __launch_bounds__(256)
conv3x3s1_wgrad_cd1_kernel(const float *__restrict__ x, const float *__restrict__ dz, float *__restrict__ dw, int N,
                           int H, int W, int C, int64_t pix_per_block) {
  __shared__ float red[9 * 128];  // C <= 128
  for (int i = threadIdx.x; i < 9 * C; i += blockDim.x) red[i] = 0.f;
  __syncthreads();
  constexpr int GROUPS = 32 / L;
  const int lane = threadIdx.x & 31, sl = lane % L, sg = lane / L;
  const int gid = (threadIdx.x >> 5) * GROUPS + sg;           // pixel lane within the block
  const int gcount = (blockDim.x >> 5) * GROUPS;
  const int64_t M = (int64_t)N * H * W;
  const int64_t m0 = (int64_t)blockIdx.x * pix_per_block;
  int64_t m1 = m0 + pix_per_block;
  if (m1 > M) m1 = M;
  const int c0 = sl * 4;
  float4 acc[9];
#pragma unroll
  for (int t = 0; t < 9; ++t) acc[t] = make_float4(0.f, 0.f, 0.f, 0.f);
  if (c0 < C) {
    for (int64_t m = m0 + gid; m < m1; m += gcount) {
      const int w = (int)(m % W);
      const int64_t t2 = m / W;
      const int h = (int)(t2 % H);
      const float4 xv = __ldg(reinterpret_cast<const float4 *>(x + m * C + c0));
      const float *dzc = dz + m;  // same (n,h,w) in the output grid (P == H, Q == W)
#pragma unroll
      for (int r = 0; r < 3; ++r) {
        const int oh = h + 1 - r;
        if (oh < 0 || oh >= H) continue;
#pragma unroll
        for (int s = 0; s < 3; ++s) {
          const int ow = w + 1 - s;
          if (ow < 0 || ow >= W) continue;
          const float d = __ldg(dzc + (1 - r) * W + (1 - s));
          float4 &a = acc[r * 3 + s];
          a.x = fmaf(xv.x, d, a.x); a.y = fmaf(xv.y, d, a.y); a.z = fmaf(xv.z, d, a.z); a.w = fmaf(xv.w, d, a.w);
        }
      }
    }
#pragma unroll
    for (int t = 0; t < 9; ++t) {
      atomicAdd(&red[t * C + c0 + 0], acc[t].x);
      atomicAdd(&red[t * C + c0 + 1], acc[t].y);
      atomicAdd(&red[t * C + c0 + 2], acc[t].z);
      atomicAdd(&red[t * C + c0 + 3], acc[t].w);
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < 9 * C; i += blockDim.x) {
    const int c = i % C, t = i / C;
    atomicAdd(dw + (int64_t)c * 9 + t, red[i]);  // dw[0][c][r][s], t = r*3+s
  }
}

// column sums: out[c] += sum_m x[m][c]   (bias gradient). out zeroed by caller.
__global__ void __launch_bounds__(256)
colsum_kernel(const float *__restrict__ x, float *__restrict__ out, int64_t M, int C,
              int64_t rows_per_block) {
  // blockDim = (32, 8): x = channel lane, y = row lane
  __shared__ float red[8][33];
  int c = blockIdx.x * 32 + threadIdx.x;
  int64_t r0 = (int64_t)blockIdx.y * rows_per_block;
  int64_t r1 = r0 + rows_per_block;
  if (r1 > M) r1 = M;
  float s = 0.f;
  if (c < C)
    for (int64_t r = r0 + threadIdx.y; r < r1; r += 8) s += __ldg(x + r * C + c);
  red[threadIdx.y][threadIdx.x] = s;
  __syncthreads();
  if (threadIdx.y == 0 && c < C) {
    float t = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) t += red[i][threadIdx.x];
    atomicAdd(out + c, t);
  }
}

// ------------------------------------------------------------------------------------------
// host launchers (called from conv_api.cu)
// ------------------------------------------------------------------------------------------
static GatherP make_gather(int N, int H, int W, int C, int P, int Q, int R, int S, int stride,
                           int pad_t, int pad_l, int pad_mode, int up, int mode) {
  GatherP g;
  g.N = N; g.H = H; g.W = W; g.C = C; g.P = P; g.Q = Q; g.R = R; g.S = S;
  g.stride = stride; g.pad_t = pad_t; g.pad_l = pad_l; g.pad_mode = pad_mode; g.up = up;
  g.Hv = H * up; g.Wv = W * up; g.mode = mode; g.cls = 1;
  return g;
}

int simt_gather_gemm(int N, int H, int W, int C, int P, int Q, int K, int R, int S, int stride,
                     int pad_t, int pad_l, int pad_mode, int up, int mode,
                     const b200gan_epilogue *ep, const float *x, const float *wp, float *y,
                     cudaStream_t st) {
  GatherP g = make_gather(N, H, W, C, P, Q, R, S, stride, pad_t, pad_l, pad_mode, up, mode);
  EpiP e;
  e.bias = ep ? ep->bias : nullptr;
  e.chan_scale = ep ? ep->chan_scale : nullptr;
  e.act = ep ? ep->act : 0;
  e.slope = ep ? ep->slope : 0.f;
  e.round_tf32 = ep ? ep->round_tf32 : 0;
  int64_t M = (int64_t)N * P * Q;
  if (M == 0 || K == 0) return B200GAN_OK;
  int Ktot = R * S * C;
  size_t wbytes = (size_t)Ktot * K * sizeof(float);
  const bool aligned = ((uintptr_t)x % 16 == 0) && ((uintptr_t)y % 16 == 0);
  // lean 3x3 / stride 1 / pad 1 kernels (mode 0: conv fprop; mode 1: transposed gather with mirrored taps)
  const bool s3 = R == 3 && S == 3 && stride == 1 && pad_t == 1 && pad_l == 1 && up == 1 && pad_mode == B200GAN_PAD_ZERO &&
                  P == H && Q == W && aligned;
  const int dir = mode == 0 ? 1 : -1;
  if (s3 && K <= 4 && C % 4 == 0 && C >= 16 && C <= 512 && wbytes <= 48 * 1024) {
    const int L = C >= 128 ? 32 : (C >= 64 ? 16 : (C >= 32 ? 8 : 4));
    const int64_t ngroups = (int64_t)N * H * ((W + 3) / 4);
    int64_t blocks = ceil_div64(ngroups, 8 * (32 / L));
    if (blocks > num_sms() * 16) blocks = num_sms() * 16;
#define LAUNCH_SK(LL, KK_) conv3x3s1_smallk_kernel<LL, KK_><<<(unsigned)blocks, 256, wbytes, st>>>(x, wp, y, e, N, H, W, C, dir)
#define LAUNCH_SK_L(KK_) \
  do { if (L == 32) LAUNCH_SK(32, KK_); else if (L == 16) LAUNCH_SK(16, KK_); else if (L == 8) LAUNCH_SK(8, KK_); else LAUNCH_SK(4, KK_); } while (0)
    if (K == 1) LAUNCH_SK_L(1); else if (K == 2) LAUNCH_SK_L(2); else if (K == 3) LAUNCH_SK_L(3); else LAUNCH_SK_L(4);
#undef LAUNCH_SK_L
#undef LAUNCH_SK
    B2_LAUNCH_CHECK();
    return B200GAN_OK;
  }
  if (s3 && C <= 4 && K % 8 == 0 && wbytes <= 48 * 1024) {
    int64_t blocks = ceil_div64(M * (K / 8), 256);
    if (blocks > num_sms() * 32) blocks = num_sms() * 32;
    if (C == 1) conv3x3s1_smallc_kernel<1><<<(unsigned)blocks, 256, wbytes, st>>>(x, wp, y, e, N, H, W, K, dir);
    else if (C == 2) conv3x3s1_smallc_kernel<2><<<(unsigned)blocks, 256, wbytes, st>>>(x, wp, y, e, N, H, W, K, dir);
    else if (C == 3) conv3x3s1_smallc_kernel<3><<<(unsigned)blocks, 256, wbytes, st>>>(x, wp, y, e, N, H, W, K, dir);
    else conv3x3s1_smallc_kernel<4><<<(unsigned)blocks, 256, wbytes, st>>>(x, wp, y, e, N, H, W, K, dir);
    B2_LAUNCH_CHECK();
    return B200GAN_OK;
  }
  if (K <= 4 && C % 4 == 0 && C >= 16 && wbytes <= 48 * 1024 && aligned) {
    // few output channels: lanes over channels (float4), several pixels in flight per lane group
    const int64_t blocks_max = num_sms() * 8;
    if (C >= 128) {
      int64_t blocks = ceil_div64(M, 8 * 1 * 4);
      if (blocks > blocks_max) blocks = blocks_max;
      conv_smallk_vec_kernel<32, 4><<<(unsigned)blocks, 256, wbytes, st>>>(g, e, x, wp, y, K);
    } else if (C >= 64) {
      int64_t blocks = ceil_div64(M, 8 * 2 * 4);
      if (blocks > blocks_max) blocks = blocks_max;
      conv_smallk_vec_kernel<16, 4><<<(unsigned)blocks, 256, wbytes, st>>>(g, e, x, wp, y, K);
    } else if (C >= 32) {
      int64_t blocks = ceil_div64(M, 8 * 4 * 4);
      if (blocks > blocks_max) blocks = blocks_max;
      conv_smallk_vec_kernel<8, 4><<<(unsigned)blocks, 256, wbytes, st>>>(g, e, x, wp, y, K);
    } else {
      int64_t blocks = ceil_div64(M, 8 * 8 * 4);
      if (blocks > blocks_max) blocks = blocks_max;
      conv_smallk_vec_kernel<4, 4><<<(unsigned)blocks, 256, wbytes, st>>>(g, e, x, wp, y, K);
    }
  } else if (K <= 4 && C >= 32 && wbytes <= 48 * 1024) {
    int64_t blocks = ceil_div64(M, 8);
    if (blocks > num_sms() * 64) blocks = num_sms() * 64;
    conv_gather_smallk_kernel<4><<<(unsigned)blocks, 256, wbytes, st>>>(g, e, x, wp, y, K);
  } else if (C <= 8 && K % 4 == 0 && K >= 8 && wbytes <= 48 * 1024 && aligned) {
    int64_t blocks = ceil_div64(M * (K / 4), 256);
    if (blocks > num_sms() * 32) blocks = num_sms() * 32;
    conv_smallc_kernel<<<(unsigned)blocks, 256, wbytes, st>>>(g, e, x, wp, y, K);
  } else {
    if (mode == 1 && stride > 1 && stride <= 4) {
      g.cls = stride;
      int64_t mc = (int64_t)N * ceil_div(P, stride) * ceil_div(Q, stride);
      dim3 grid((unsigned)ceil_div64(mc, FBM), (unsigned)ceil_div(K, FBN), (unsigned)(stride * stride));
      conv_gather_gemm_kernel<<<grid, 256, 0, st>>>(g, e, x, wp, y, K);
    } else {
      dim3 grid((unsigned)ceil_div64(M, FBM), (unsigned)ceil_div(K, FBN));
      conv_gather_gemm_kernel<<<grid, 256, 0, st>>>(g, e, x, wp, y, K);
    }
  }
  B2_LAUNCH_CHECK();
  return B200GAN_OK;
}

// dw must hold Cd*Cg*R*S floats; it is zeroed here.
int simt_wgrad(int N, int H, int W, int Cg, int P, int Q, int Cd, int R, int S, int stride,
               int pad_t, int pad_l, int pad_mode, int up, const float *xg, const float *dn,
               float *dw, cudaStream_t st) {
  GatherP g = make_gather(N, H, W, Cg, P, Q, R, S, stride, pad_t, pad_l, pad_mode, up, 0);
  int64_t M = (int64_t)N * P * Q;
  int Ktot = R * S * Cg;
  B2_CUDA(cudaMemsetAsync(dw, 0, (size_t)Ktot * Cd * sizeof(float), st));
  if (M == 0) return B200GAN_OK;
  if (Cd == 1 && R == 3 && S == 3 && stride == 1 && pad_t == 1 && pad_l == 1 && up == 1 && pad_mode == B200GAN_PAD_ZERO &&
      P == H && Q == W && Cg % 4 == 0 && Cg >= 16 && Cg <= 128 && ((uintptr_t)xg % 16 == 0)) {
    const int L = Cg >= 128 ? 32 : (Cg >= 64 ? 16 : (Cg >= 32 ? 8 : 4));
    int64_t blocks = num_sms() * 4;
    int64_t ppb = ceil_div64(M, blocks);
    if (ppb < 256) ppb = 256;
    blocks = ceil_div64(M, ppb);
    if (L == 32) conv3x3s1_wgrad_cd1_kernel<32><<<(unsigned)blocks, 256, 0, st>>>(xg, dn, dw, N, H, W, Cg, ppb);
    else if (L == 16) conv3x3s1_wgrad_cd1_kernel<16><<<(unsigned)blocks, 256, 0, st>>>(xg, dn, dw, N, H, W, Cg, ppb);
    else if (L == 8) conv3x3s1_wgrad_cd1_kernel<8><<<(unsigned)blocks, 256, 0, st>>>(xg, dn, dw, N, H, W, Cg, ppb);
    else conv3x3s1_wgrad_cd1_kernel<4><<<(unsigned)blocks, 256, 0, st>>>(xg, dn, dw, N, H, W, Cg, ppb);
    B2_LAUNCH_CHECK();
    return B200GAN_OK;
  }
  if (Cd <= 4) {
    int yb = ceil_div(Ktot, 256);
    int64_t xb = (num_sms() * 8) / yb;
    if (xb < 1) xb = 1;
    int64_t m_per_block = ceil_div64(M, xb);
    if (m_per_block < 64) m_per_block = 64;
    xb = ceil_div64(M, m_per_block);
    conv_wgrad_smallcd_kernel<<<dim3((unsigned)xb, (unsigned)yb), 256, 0, st>>>(g, xg, dn, dw, Cd, m_per_block);
    B2_LAUNCH_CHECK();
    return B200GAN_OK;
  }
  int tiles = ceil_div(Ktot, FBM) * ceil_div(Cd, FBN);
  int64_t splits = (num_sms() * 4 + tiles - 1) / tiles;
  int64_t max_splits = ceil_div64(M, 128);
  if (splits > max_splits) splits = max_splits;
  if (splits < 1) splits = 1;
  if (splits > 65535) splits = 65535;
  int64_t m_per = ceil_div64(ceil_div64(M, splits), FBK) * FBK;
  splits = ceil_div64(M, m_per);
  dim3 grid((unsigned)ceil_div(Ktot, FBM), (unsigned)ceil_div(Cd, FBN), (unsigned)splits);
  conv_wgrad_kernel<<<grid, 256, 0, st>>>(g, xg, dn, dw, Cd, m_per);
  B2_LAUNCH_CHECK();
  return B200GAN_OK;
}

int simt_colsum(const float *x, float *out, int64_t M, int C, cudaStream_t st) {
  B2_CUDA(cudaMemsetAsync(out, 0, (size_t)C * sizeof(float), st));
  if (M == 0) return B200GAN_OK;
  int64_t yb = num_sms() * 8 / ceil_div(C, 32);
  if (yb < 1) yb = 1;
  int64_t rows = ceil_div64(M, yb);
  if (rows < 64) rows = 64;
  yb = ceil_div64(M, rows);
  dim3 grid((unsigned)ceil_div(C, 32), (unsigned)yb);
  colsum_kernel<<<grid, dim3(32, 8), 0, st>>>(x, out, M, C, rows);
  B2_LAUNCH_CHECK();
  return B200GAN_OK;
}

}  // namespace b200gan
