// conv_simt.cu -- fp32 FFMA implicit-GEMM convolution kernels for any geometry.
//
// The any-geometry fp32 path: the gather GEMM (forward, and the data gradient as a transposed gather), the
// weight-gradient GEMM and the bias-gradient column sum.  They run every convolution pass that the tensor-core
// (conv_tc.cu, wgrad_tc.cu), few-output-channel (fewk.cu) and staged (narrow_block.cu) kernels do not take, whether by
// geometry or because B200GAN_ALGO=simt sets the tensor cores aside.  Their fp32 results are what the wgmma kernels
// are validated against on the GPU.
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
  if (mode == 1 && stride > 1 && stride <= 4) {
    g.cls = stride;
    int64_t mc = (int64_t)N * ceil_div(P, stride) * ceil_div(Q, stride);
    dim3 grid((unsigned)ceil_div64(mc, FBM), (unsigned)ceil_div(K, FBN), (unsigned)(stride * stride));
    conv_gather_gemm_kernel<<<grid, 256, 0, st>>>(g, e, x, wp, y, K);
  } else {
    dim3 grid((unsigned)ceil_div64(M, FBM), (unsigned)ceil_div(K, FBN));
    conv_gather_gemm_kernel<<<grid, 256, 0, st>>>(g, e, x, wp, y, K);
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
