// fewk.cu -- stride-1 convolutions with a handful of OUTPUT channels (K <= 4): the image-producing last layer of the
// generators and the 1-channel patch output of the discriminators.
//
// Reference: pix2pix/models.py:97-102   nn.Upsample(scale_factor=2), nn.ZeroPad2d((1, 0, 1, 0)), nn.Conv2d(128, 3, 4, padding=1), nn.Tanh()
//            pix2pix/models.py:131-132  nn.ZeroPad2d((1, 0, 1, 0)), nn.Conv2d(512, 1, 4, padding=1, bias=False)
//            cyclegan/models.py:88-90   nn.ReflectionPad2d(3), nn.Conv2d(64, 3, 7), nn.Tanh()
//            cyclegan/models.py:124-125 nn.ZeroPad2d((1, 0, 1, 0)), nn.Conv2d(512, 1, 4, padding=1)
// These layers are 0.5 - 13 GFLOP with a GEMM N of 1..3: a tensor-core tile would spend its time staging A tiles that
// are used for one 8-wide column, and a pixel-per-thread SIMT kernel reads its input with one cache line per lane
// (measured: 2.3 ms forward, 2.4 ms + 0.2 ms data gradient, 5.6 ms weight gradient for the pix2pix layer at batch 16).
// Here the LANES of a warp span the input channels (float4 each: a pixel's 128 channels are one 512-byte coalesced
// load), a lane group register-tiles 8 pixels of a row, and the weights come from shared memory as one LDS.128 per 32
// FMAs:
//   fewk_fprop  dot products over channels finished with a butterfly across the lanes of a group
//   fewk_dgrad  dx[h, w, 4c] accumulated from a register window of dz (uniform loads)
//   fewk_wgrad  a warp owns one filter row and streams output rows; per-block slabs + the fixed-order reduce kernel
// A nearest-neighbour x2 upsample in front of a zero-padded 3x3 / 4x4 conv runs on folded filters (the *_up2 kernels
// below; the data gradient's upsample backward is part of their accumulation).  Elsewhere (forward and weight gradient
// with reflection padding or 7x7) the upsample only changes the address computation (source pixel = index >> 1).
#include "tc_common.cuh"
#include <string.h>

namespace b200gan {

struct FewkP {
  const float *x;    // [N][H][W][C]
  const float *w;    // fprop: PACK_SIMT_FPROP [tap][C][K]; dgrad: PACK_SIMT_DGRAD [tap][K][C]
  const float *bias, *dy;
  float *y, *dx, *ws;
  int N, H, W, C, P, Q, R, pad_t, pad_l, up, reflect, act;
  float slope;
  int CL, G;         // lanes per pixel group (channels / 4, at most 32) and groups per warp
  int HU, WU;        // H * up, W * up
  int dw_elems;
};

constexpr int FK_PX = 8;   // pixels of a row per lane group
__host__ __device__ __forceinline__ int fk_cdiv(int a, int b) { return (a + b - 1) / b; }

__device__ __forceinline__ float dot4(const float4 &a, const float4 &b, float acc) {
  acc = fmaf(a.x, b.x, acc);
  acc = fmaf(a.y, b.y, acc);
  acc = fmaf(a.z, b.z, acc);
  return fmaf(a.w, b.w, acc);
}
__device__ __forceinline__ void axpy4(float4 &acc, float a, const float4 &b) {
  acc.x = fmaf(a, b.x, acc.x);
  acc.y = fmaf(a, b.y, acc.y);
  acc.z = fmaf(a, b.z, acc.z);
  acc.w = fmaf(a, b.w, acc.w);
}

// source row / column of virtual (upsampled, padded) index i; -1: zero padding
__device__ __forceinline__ int fk_src(int i, int n_virtual, int up, int reflect) {
  if (reflect) i = reflect_idx(i, n_virtual);
  if (i < 0 || i >= n_virtual) return -1;
  return up == 2 ? (i >> 1) : i;
}

// ---- forward --------------------------------------------------------------------------------------------------------
// block = 8 warps = 8 consecutive output rows x (G * 8) columns; dynamic smem: w [R*S][K][C]
template <int S, int K>
__global__ void __launch_bounds__(256)
fewk_fprop_kernel(const __grid_constant__ FewkP p) {
  extern __shared__ __align__(16) float w_s[];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int taps = p.R * S;
  for (int i = tid; i < taps * K * p.C; i += 256) {
    const int c = i % p.C, k = (i / p.C) % K, t = i / (p.C * K);
    w_s[i] = __ldg(p.w + ((int64_t)t * p.C + c) * K + k);
  }
  __syncthreads();
  const int grp = lane / p.CL, cl = lane % p.CL;
  const int tiles_q = fk_cdiv(p.Q, p.G * FK_PX), tiles_p = fk_cdiv(p.P, 8);
  const int ntiles = p.N * tiles_p * tiles_q;
  const int chunk = p.CL * 4;
  for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const int tq = tile % tiles_q, tp = (tile / tiles_q) % tiles_p, n = tile / (tiles_q * tiles_p);
    const int prow = tp * 8 + warp, q0 = (tq * p.G + grp) * FK_PX;
    const bool live = prow < p.P && q0 < p.Q;
    float acc[FK_PX][K];
#pragma unroll
    for (int px = 0; px < FK_PX; ++px)
#pragma unroll
      for (int k = 0; k < K; ++k) acc[px][k] = 0.f;
    if (live) {
      for (int cb = 0; cb < p.C; cb += chunk) {
#pragma unroll 1
        for (int r = 0; r < p.R; ++r) {
          const int ihs = fk_src(prow + r - p.pad_t, p.HU, p.up, p.reflect);
          if (ihs < 0) continue;
          const float *xrow = p.x + ((int64_t)(n * p.H + ihs) * p.W) * p.C + cb + cl * 4;
          float4 xw[FK_PX + S - 1];
#pragma unroll
          for (int j = 0; j < FK_PX + S - 1; ++j) {
            const int iws = fk_src(q0 + j - p.pad_l, p.WU, p.up, p.reflect);
            xw[j] = iws >= 0 ? __ldg(reinterpret_cast<const float4 *>(xrow + (int64_t)iws * p.C)) : make_float4(0.f, 0.f, 0.f, 0.f);
          }
#pragma unroll
          for (int s = 0; s < S; ++s) {
#pragma unroll
            for (int k = 0; k < K; ++k) {
              const float4 w4 = *reinterpret_cast<const float4 *>(w_s + ((r * S + s) * K + k) * p.C + cb + cl * 4);
#pragma unroll
              for (int px = 0; px < FK_PX; ++px) acc[px][k] = dot4(xw[px + s], w4, acc[px][k]);
            }
          }
        }
      }
    }
    // sum over the lanes of the group (all 32 lanes take part: dead groups hold zeros)
    for (int off = p.CL >> 1; off > 0; off >>= 1) {
#pragma unroll
      for (int px = 0; px < FK_PX; ++px)
#pragma unroll
        for (int k = 0; k < K; ++k) acc[px][k] += __shfl_xor_sync(0xffffffffu, acc[px][k], off);
    }
    if (live) {
      float *yo = p.y + ((int64_t)(n * p.P + prow) * p.Q + q0) * K;
      for (int v = cl; v < FK_PX * K; v += p.CL) {
        float val = 0.f;
#pragma unroll
        for (int i = 0; i < FK_PX * K; ++i)
          if (v == i) val = acc[i / K][i % K];
        const int px = v / K, k = v % K;
        if (q0 + px < p.Q) {
          if (p.bias) val += __ldg(p.bias + k);
          yo[v] = apply_act(val, p.act, p.slope);
        }
      }
    }
  }
}

// ---- data gradient --------------------------------------------------------------------------------------------------
// thread group = 8 pixels of a row x 4 channels per lane; zero padding, no upsample (fewk_dgrad_up2_kernel folds it).
// dynamic smem: w [R*S][K][C]
template <int S, int K>
__global__ void __launch_bounds__(256)
fewk_dgrad_kernel(const __grid_constant__ FewkP p) {
  extern __shared__ __align__(16) float w_s[];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int taps = p.R * S;
  for (int i = tid; i < taps * K * p.C; i += 256) w_s[i] = __ldg(p.w + i);
  __syncthreads();
  const int grp = lane / p.CL, cl = lane % p.CL;
  const int tiles_w = fk_cdiv(p.W, p.G * FK_PX), tiles_h = fk_cdiv(p.H, 8);
  const int ntiles = p.N * tiles_h * tiles_w;
  const int chunk = p.CL * 4;
  constexpr int WIN = FK_PX + S - 1;   // dz columns a row of 8 pixels touches
  for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const int tw = tile % tiles_w, th = (tile / tiles_w) % tiles_h, n = tile / (tiles_w * tiles_h);
    const int h = th * 8 + warp, w0 = (tw * p.G + grp) * FK_PX;
    if (h >= p.H || w0 >= p.W) continue;
    for (int cb = 0; cb < p.C; cb += chunk) {
      float4 acc[FK_PX];
#pragma unroll
      for (int px = 0; px < FK_PX; ++px) acc[px] = make_float4(0.f, 0.f, 0.f, 0.f);
      const int qstart = w0 + p.pad_l - (S - 1);
#pragma unroll 1
      for (int r = 0; r < p.R; ++r) {
        const int prow = h + p.pad_t - r;   // output row whose tap r reads row h
        if (prow < 0 || prow >= p.P) continue;
        const float *drow = p.dy + ((int64_t)(n * p.P + prow) * p.Q) * K;
        float dzw[WIN][K];
#pragma unroll
        for (int j = 0; j < WIN; ++j) {
          const int q = qstart + j;
          const bool ok = q >= 0 && q < p.Q;
#pragma unroll
          for (int k = 0; k < K; ++k) dzw[j][k] = ok ? __ldg(drow + (int64_t)q * K + k) : 0.f;
        }
#pragma unroll
        for (int s = 0; s < S; ++s) {
#pragma unroll
          for (int k = 0; k < K; ++k) {
            const float4 w4 = *reinterpret_cast<const float4 *>(w_s + ((r * S + s) * K + k) * p.C + cb + cl * 4);
#pragma unroll
            for (int px = 0; px < FK_PX; ++px) axpy4(acc[px], dzw[px + (S - 1) - s][k], w4);
          }
        }
      }
      float *dxo = p.dx + ((int64_t)(n * p.H + h) * p.W + w0) * p.C + cb + cl * 4;
#pragma unroll
      for (int px = 0; px < FK_PX; ++px)
        if (w0 + px < p.W) *reinterpret_cast<float4 *>(dxo + (int64_t)px * p.C) = acc[px];
    }
  }
}

// ---- weight gradient ------------------------------------------------------------------------------------------------
// A lane group owns filter row r = (global group index) % R and streams the output rows of its strip: per 8 output
// pixels, 8 + S - 1 coalesced float4 loads of x and 8 * K uniform loads of dz feed S * 8 * K * 4 FMAs into
// acc[s][k][4 channels].  Groups of one block are summed through shared memory in a fixed order, the block writes its
// slab [K][C][R][S] of the workspace, nbk_wgrad_reduce_kernel adds the slabs.  dynamic smem: blk [R][S][K][C]
template <int S, int K>
__global__ void __launch_bounds__(256)
fewk_wgrad_kernel(const __grid_constant__ FewkP p) {
  extern __shared__ __align__(16) float blk[];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int grp = lane / p.CL, cl = lane % p.CL;
  const int nchunks = p.C / (p.CL * 4);
  const int groups_per_block = 8 * p.G;
  for (int i = tid; i < p.R * S * K * p.C; i += 256) blk[i] = 0.f;
  // virtual group id -> (channel chunk, filter row, strip)
  const int64_t gid = (int64_t)blockIdx.x * groups_per_block + warp * p.G + grp;
  const int64_t ngroups = (int64_t)gridDim.x * groups_per_block;
  const int per = p.R * nchunks;
  const int r = (int)(gid % p.R), cb = (int)((gid / p.R) % nchunks) * p.CL * 4;
  const int64_t strip = gid / per, nstrips = ngroups / per;
  float4 acc[S][K];
#pragma unroll
  for (int s = 0; s < S; ++s)
#pragma unroll
    for (int k = 0; k < K; ++k) acc[s][k] = make_float4(0.f, 0.f, 0.f, 0.f);
  const int qtiles = fk_cdiv(p.Q, FK_PX);
  const int64_t nitems = (int64_t)p.N * p.P * qtiles;
  if (strip < nstrips) {
    for (int64_t it = strip; it < nitems; it += nstrips) {
      const int tq = (int)(it % qtiles);
      const int prow = (int)((it / qtiles) % p.P), n = (int)(it / ((int64_t)qtiles * p.P));
      const int ihs = fk_src(prow + r - p.pad_t, p.HU, p.up, p.reflect);
      if (ihs < 0) continue;
      const int q0 = tq * FK_PX;
      const float *xrow = p.x + ((int64_t)(n * p.H + ihs) * p.W) * p.C + cb + cl * 4;
      const float *drow = p.dy + ((int64_t)(n * p.P + prow) * p.Q + q0) * K;
      float4 xw[FK_PX + S - 1];
#pragma unroll
      for (int j = 0; j < FK_PX + S - 1; ++j) {
        const int iws = fk_src(q0 + j - p.pad_l, p.WU, p.up, p.reflect);
        xw[j] = iws >= 0 ? __ldg(reinterpret_cast<const float4 *>(xrow + (int64_t)iws * p.C)) : make_float4(0.f, 0.f, 0.f, 0.f);
      }
      float dz[FK_PX][K];
#pragma unroll
      for (int px = 0; px < FK_PX; ++px)
#pragma unroll
        for (int k = 0; k < K; ++k) dz[px][k] = (q0 + px < p.Q) ? __ldg(drow + px * K + k) : 0.f;
#pragma unroll
      for (int s = 0; s < S; ++s)
#pragma unroll
        for (int px = 0; px < FK_PX; ++px)
#pragma unroll
          for (int k = 0; k < K; ++k) axpy4(acc[s][k], dz[px][k], xw[px + s]);
    }
  }
  __syncthreads();
  // fixed-order accumulation of the block's groups: one group at a time adds its row into blk
  for (int turn = 0; turn < groups_per_block; ++turn) {
    if (turn == warp * p.G + grp && strip < nstrips) {
#pragma unroll
      for (int s = 0; s < S; ++s)
#pragma unroll
        for (int k = 0; k < K; ++k) {
          float4 *dst = reinterpret_cast<float4 *>(blk + ((size_t)(r * S + s) * K + k) * p.C + cb + cl * 4);
          float4 v = *dst;
          v.x += acc[s][k].x; v.y += acc[s][k].y; v.z += acc[s][k].z; v.w += acc[s][k].w;
          *dst = v;
        }
    }
    __syncthreads();
  }
  // slab in parameter layout dw[k][c][r][s]
  float *slab = p.ws + (size_t)blockIdx.x * p.dw_elems;
  const int RS = p.R * S;
  for (int i = tid; i < p.dw_elems; i += 256) {
    const int t = i % RS, c = (i / RS) % p.C, k = i / (RS * p.C);
    slab[i] = blk[((size_t)t * K + k) * p.C + c];
  }
}

// =====================================================================================================================
// Folded x2 upsample (g->up == 2): an output pixel at distance e = o - pad from the virtual origin reads, per dimension,
// virtual positions e + t (t < S), i.e. source positions floor((e + t) / 2) = m + floor((b + t) / 2) with b = e & 1,
// m = floor(e / 2): only NF(b) = floor((b + S - 1) / 2) + 1 DISTINCT source positions.  Summing the taps that share a
// source position ("folded taps" f = floor((b + t) / 2)) gives a filter per output parity with NF(0) x/+ NF(1) taps per
// dimension -- (2 + 3)^2 = 25 folded tap pairs instead of 4 x 16 for the 4x4 filter: 2.56x fewer FMAs in all three
// passes (the kernels are FMA-issue bound: profiles/r2_ncu_full_pix2pix_edge_kernels_c13.txt).  Zero padding is exact:
// virtual positions 2m and 2m + 1 are inside or outside the tensor together.
template <int S> struct Fold {
  static constexpr int NF0 = (S - 1) / 2 + 1, NF1 = S / 2 + 1, NFT = NF0 + NF1, NFM = NF1 > NF0 ? NF1 : NF0;
  __host__ __device__ static constexpr int nf(int b) { return b ? NF1 : NF0; }
  __host__ __device__ static constexpr int off(int b) { return b ? NF0 : 0; }
  __host__ __device__ static constexpr int slot(int a, int fr, int b, int fs) { return (off(a) + fr) * NFT + off(b) + fs; }
  __host__ __device__ static constexpr int fold(int b, int t) { return (b + t) >> 1; }   // folded tap of original tap t
};

// folded filter table in shared memory: wf[slot][k][C]; raw: order 0 = [tap][C][K] (fprop pack), 1 = [tap][K][C] (dgrad pack)
template <int S, int K>
__device__ __forceinline__ void fold_weights(float *wf, const float *__restrict__ raw, int C, int order, int tid) {
  using F = Fold<S>;
  for (int i = tid; i < F::NFT * F::NFT * K * C; i += 256) {
    const int c = i % C, k = (i / C) % K, sl = i / (C * K);
    const int ra = sl / F::NFT, cb = sl % F::NFT;          // row slot (a, fr), column slot (b, fs)
    const int a = ra >= F::NF0, fr = ra - F::off(a), b = cb >= F::NF0, fs = cb - F::off(b);
    float v = 0.f;
    for (int r = 0; r < S; ++r) {
      if (F::fold(a, r) != fr) continue;
      for (int q = 0; q < S; ++q) {
        if (F::fold(b, q) != fs) continue;
        const int t = r * S + q;
        v += __ldg(raw + (order == 0 ? ((int64_t)t * C + c) * K + k : ((int64_t)t * K + k) * C + c));
      }
    }
    wf[i] = v;
  }
}

// forward.  PAR = parity of -pad_l (of e0 = q0 - pad_l for the 8-pixel groups, q0 % 8 == 0)
template <int S, int K, int PAR>
__global__ void __launch_bounds__(256)
fewk_fprop_up2_kernel(const __grid_constant__ FewkP p) {
  using F = Fold<S>;
  extern __shared__ __align__(16) float w_s[];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  fold_weights<S, K>(w_s, p.w, p.C, 0, tid);
  __syncthreads();
  const int grp = lane / p.CL, cl = lane % p.CL;
  const int tiles_q = fk_cdiv(p.Q, p.G * FK_PX), tiles_p = fk_cdiv(p.P, 8);
  const int ntiles = p.N * tiles_p * tiles_q;
  const int chunk = p.CL * 4;
  constexpr int WINF = ((PAR + FK_PX - 1) >> 1) + F::NFM;     // source columns a group of 8 pixels touches
  for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const int tq = tile % tiles_q, tp = (tile / tiles_q) % tiles_p, n = tile / (tiles_q * tiles_p);
    const int prow = tp * 8 + warp, q0 = (tq * p.G + grp) * FK_PX;
    const bool live = prow < p.P && q0 < p.Q;
    float acc[FK_PX][K];
#pragma unroll
    for (int px = 0; px < FK_PX; ++px)
#pragma unroll
      for (int k = 0; k < K; ++k) acc[px][k] = 0.f;
    if (live) {
      const int er = prow - p.pad_t, a = er & 1, mr = (er - a) >> 1;
      const int m0 = (q0 - p.pad_l - PAR) >> 1;               // floor((q0 - pad_l) / 2)
      const int nfr = F::nf(a);
      for (int cb = 0; cb < p.C; cb += chunk) {
#pragma unroll 1
        for (int fr = 0; fr < nfr; ++fr) {
          const int ih = mr + fr;
          if (ih < 0 || ih >= p.H) continue;
          const float *xrow = p.x + ((int64_t)(n * p.H + ih) * p.W) * p.C + cb + cl * 4;
          float4 xw[WINF];
#pragma unroll
          for (int j = 0; j < WINF; ++j) {
            const int iw = m0 + j;
            xw[j] = (iw >= 0 && iw < p.W) ? __ldg(reinterpret_cast<const float4 *>(xrow + (int64_t)iw * p.C))
                                          : make_float4(0.f, 0.f, 0.f, 0.f);
          }
          const float *wrow = w_s + (size_t)((F::off(a) + fr) * F::NFT) * K * p.C + cb + cl * 4;
#pragma unroll
          for (int b = 0; b < 2; ++b) {
#pragma unroll
            for (int fs = 0; fs < F::nf(b); ++fs) {
#pragma unroll
              for (int k = 0; k < K; ++k) {
                const float4 w4 = *reinterpret_cast<const float4 *>(wrow + (size_t)((F::off(b) + fs) * K + k) * p.C);
#pragma unroll
                for (int px = 0; px < FK_PX; ++px)
                  if (((PAR + px) & 1) == b) acc[px][k] = dot4(xw[((PAR + px) >> 1) + fs], w4, acc[px][k]);
              }
            }
          }
        }
      }
    }
    for (int off = p.CL >> 1; off > 0; off >>= 1) {
#pragma unroll
      for (int px = 0; px < FK_PX; ++px)
#pragma unroll
        for (int k = 0; k < K; ++k) acc[px][k] += __shfl_xor_sync(0xffffffffu, acc[px][k], off);
    }
    if (live) {
      float *yo = p.y + ((int64_t)(n * p.P + prow) * p.Q + q0) * K;
      for (int v = cl; v < FK_PX * K; v += p.CL) {
        float val = 0.f;
#pragma unroll
        for (int i = 0; i < FK_PX * K; ++i)
          if (v == i) val = acc[i / K][i % K];
        const int px = v / K, k = v % K;
        if (q0 + px < p.Q) {
          if (p.bias) val += __ldg(p.bias + k);
          yo[v] = apply_act(val, p.act, p.slope);
        }
      }
    }
  }
}

// data gradient of the SOURCE tensor: dx[h][w] = sum over (a, fr), (b, fs), k of dz[2(h - fr) + a + pad_t][2(w - fs) + b + pad_l][k]
// * Wf[a][fr][b][fs][k]
template <int S, int K>
__global__ void __launch_bounds__(256)
fewk_dgrad_up2_kernel(const __grid_constant__ FewkP p) {
  using F = Fold<S>;
  extern __shared__ __align__(16) float w_s[];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  fold_weights<S, K>(w_s, p.w, p.C, 1, tid);
  __syncthreads();
  const int grp = lane / p.CL, cl = lane % p.CL;
  const int tiles_w = fk_cdiv(p.W, p.G * FK_PX), tiles_h = fk_cdiv(p.H, 8);
  const int ntiles = p.N * tiles_h * tiles_w;
  const int chunk = p.CL * 4;
  constexpr int WIN = 2 * FK_PX + 2 * (F::NFM - 1);   // dz columns 2(w0 - (NFM-1)) + pad_l .. 2(w0 + 7) + 1 + pad_l
  for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const int tw = tile % tiles_w, th = (tile / tiles_w) % tiles_h, n = tile / (tiles_w * tiles_h);
    const int h = th * 8 + warp, w0 = (tw * p.G + grp) * FK_PX;
    if (h >= p.H || w0 >= p.W) continue;
    const int qstart = 2 * (w0 - (F::NFM - 1)) + p.pad_l;
    for (int cb = 0; cb < p.C; cb += chunk) {
      float4 acc[FK_PX];
#pragma unroll
      for (int px = 0; px < FK_PX; ++px) acc[px] = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll 1
      for (int ra = 0; ra < F::NFT; ++ra) {                    // row slot (a, fr)
        const int a = ra >= F::NF0, fr = ra - F::off(a);
        const int prow = 2 * (h - fr) + a + p.pad_t;
        if (prow < 0 || prow >= p.P) continue;
        const float *drow = p.dy + ((int64_t)(n * p.P + prow) * p.Q) * K;
        float dzw[WIN][K];
#pragma unroll
        for (int j = 0; j < WIN; ++j) {
          const int q = qstart + j;
          const bool ok = q >= 0 && q < p.Q;
#pragma unroll
          for (int k = 0; k < K; ++k) dzw[j][k] = ok ? __ldg(drow + (int64_t)q * K + k) : 0.f;
        }
        const float *wrow = w_s + (size_t)(ra * F::NFT) * K * p.C + cb + cl * 4;
#pragma unroll
        for (int b = 0; b < 2; ++b) {
#pragma unroll
          for (int fs = 0; fs < F::nf(b); ++fs) {
#pragma unroll
            for (int k = 0; k < K; ++k) {
              const float4 w4 = *reinterpret_cast<const float4 *>(wrow + (size_t)((F::off(b) + fs) * K + k) * p.C);
#pragma unroll
              for (int px = 0; px < FK_PX; ++px)   // q = 2(w0 + px - fs) + b + pad_l -> window index 2(px - fs + NFM - 1) + b
                axpy4(acc[px], dzw[2 * (px - fs + F::NFM - 1) + b][k], w4);
            }
          }
        }
      }
      float *dxo = p.dx + ((int64_t)(n * p.H + h) * p.W + w0) * p.C + cb + cl * 4;
#pragma unroll
      for (int px = 0; px < FK_PX; ++px)
        if (w0 + px < p.W) *reinterpret_cast<float4 *>(dxo + (int64_t)px * p.C) = acc[px];
    }
  }
}

// weight gradient: a lane group owns a folded ROW slot (a, fr) and streams the output rows of parity a; acc[column slot][k]
template <int S, int K, int PAR>
__global__ void __launch_bounds__(256)
fewk_wgrad_up2_kernel(const __grid_constant__ FewkP p) {
  using F = Fold<S>;
  extern __shared__ __align__(16) float blk[];                 // [NFT row slots][NFT column slots][K][C]
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int grp = lane / p.CL, cl = lane % p.CL;
  const int nchunks = p.C / (p.CL * 4);
  const int groups_per_block = 8 * p.G;
  for (int i = tid; i < F::NFT * F::NFT * K * p.C; i += 256) blk[i] = 0.f;
  const int64_t gid = (int64_t)blockIdx.x * groups_per_block + warp * p.G + grp;
  const int64_t ngroups = (int64_t)gridDim.x * groups_per_block;
  const int per = F::NFT * nchunks;
  const int ra = (int)(gid % F::NFT), cb = (int)((gid / F::NFT) % nchunks) * p.CL * 4;
  const int a = ra >= F::NF0, fr = ra - F::off(a);
  const int64_t strip = gid / per, nstrips = ngroups / per;
  float4 acc[F::NFT][K];
#pragma unroll
  for (int cs = 0; cs < F::NFT; ++cs)
#pragma unroll
    for (int k = 0; k < K; ++k) acc[cs][k] = make_float4(0.f, 0.f, 0.f, 0.f);
  constexpr int WINF = ((PAR + FK_PX - 1) >> 1) + F::NFM;
  const int qtiles = fk_cdiv(p.Q, FK_PX);
  // output rows of parity a: p - pad_t = 2 j + a
  const int pfirst = ((a - p.pad_t) & 1) ? 1 : 0;              // smallest p >= 0 with (p - pad_t) & 1 == a
  const int nrows = p.P > pfirst ? (p.P - pfirst + 1) / 2 : 0;
  const int64_t nitems = (int64_t)p.N * nrows * qtiles;
  if (strip < nstrips) {
    for (int64_t it = strip; it < nitems; it += nstrips) {
      const int tq = (int)(it % qtiles);
      const int prow = pfirst + 2 * (int)((it / qtiles) % nrows), n = (int)(it / ((int64_t)qtiles * nrows));
      const int ih = ((prow - p.pad_t - a) >> 1) + fr;
      if (ih < 0 || ih >= p.H) continue;
      const int q0 = tq * FK_PX;
      const int m0 = (q0 - p.pad_l - PAR) >> 1;
      const float *xrow = p.x + ((int64_t)(n * p.H + ih) * p.W) * p.C + cb + cl * 4;
      const float *drow = p.dy + ((int64_t)(n * p.P + prow) * p.Q + q0) * K;
      float4 xw[WINF];
#pragma unroll
      for (int j = 0; j < WINF; ++j) {
        const int iw = m0 + j;
        xw[j] = (iw >= 0 && iw < p.W) ? __ldg(reinterpret_cast<const float4 *>(xrow + (int64_t)iw * p.C))
                                      : make_float4(0.f, 0.f, 0.f, 0.f);
      }
      float dz[FK_PX][K];
#pragma unroll
      for (int px = 0; px < FK_PX; ++px)
#pragma unroll
        for (int k = 0; k < K; ++k) dz[px][k] = (q0 + px < p.Q) ? __ldg(drow + px * K + k) : 0.f;
#pragma unroll
      for (int px = 0; px < FK_PX; ++px) {
        const int b = (PAR + px) & 1;
#pragma unroll
        for (int fs = 0; fs < F::NFM; ++fs) {
          if (fs < F::nf(b)) {
#pragma unroll
            for (int k = 0; k < K; ++k) axpy4(acc[F::off(b) + fs][k], dz[px][k], xw[((PAR + px) >> 1) + fs]);
          }
        }
      }
    }
  }
  __syncthreads();
  for (int turn = 0; turn < groups_per_block; ++turn) {
    if (turn == warp * p.G + grp && strip < nstrips) {
#pragma unroll
      for (int cs = 0; cs < F::NFT; ++cs)
#pragma unroll
        for (int k = 0; k < K; ++k) {
          float4 *dst = reinterpret_cast<float4 *>(blk + ((size_t)(ra * F::NFT + cs) * K + k) * p.C + cb + cl * 4);
          float4 v = *dst;
          v.x += acc[cs][k].x; v.y += acc[cs][k].y; v.z += acc[cs][k].z; v.w += acc[cs][k].w;
          *dst = v;
        }
    }
    __syncthreads();
  }
  // un-fold into the parameter layout: dw[k][c][r][s] = sum over (a, b) of dWf[a][fold(a, r)][b][fold(b, s)]
  float *slab = p.ws + (size_t)blockIdx.x * p.dw_elems;
  for (int i = tid; i < p.dw_elems; i += 256) {
    const int t = i % (S * S), c = (i / (S * S)) % p.C, k = i / (S * S * p.C);
    const int r = t / S, q = t % S;
    float v = 0.f;
#pragma unroll
    for (int aa = 0; aa < 2; ++aa)
#pragma unroll
      for (int bb = 0; bb < 2; ++bb) v += blk[((size_t)F::slot(aa, F::fold(aa, r), bb, F::fold(bb, q)) * K + k) * p.C + c];
    slab[i] = v;
  }
}

// narrow_block.cu: dw[e] = sum over the slabs, fixed order
int nb_wgrad_reduce(const float *ws, float *dw, int elems, int nslabs, cudaStream_t st);

static bool fewk_geom_ok(const b200gan_conv_geom *g) {
  if (!g || g->transposed || g->stride != 1) return false;
  if (g->up != 1 && g->up != 2) return false;
  if (g->K < 1 || g->K > 4) return false;
  if (g->R != g->S || (g->S != 3 && g->S != 4 && g->S != 7)) return false;
  if (g->C < 32 || (g->C <= 128 ? 128 % g->C != 0 : g->C % 128 != 0)) return false;
  if ((size_t)g->R * g->S * g->K * g->C * sizeof(float) > 160 * 1024) return false;
  return true;
}
// pas: 0 fprop, 1 dgrad, 2 wgrad
bool fewk_ok(const b200gan_conv_geom *g, int pas) {
  if (!fewk_geom_ok(g)) return false;
  if (pas == 1 && g->pad_mode != B200GAN_PAD_ZERO) return false;   // the mirrored border folds back in pad2d_bwd
  if (pas == 1 && g->S == 7 && g->up == 2) return false;
  return true;
}

static void fewk_fill(FewkP &p, const b200gan_conv_geom *g) {
  memset(&p, 0, sizeof(p));
  p.N = g->N; p.H = g->H; p.W = g->W; p.C = g->C; p.P = g->P; p.Q = g->Q; p.R = g->R;
  p.pad_t = g->pad_t; p.pad_l = g->pad_l; p.up = g->up; p.reflect = g->pad_mode == B200GAN_PAD_REFLECT ? 1 : 0;
  p.CL = g->C >= 128 ? 32 : g->C / 4;
  p.G = 32 / p.CL;
  p.HU = g->H * g->up; p.WU = g->W * g->up;
  p.dw_elems = g->K * g->C * g->R * g->S;
}


static bool fewk_fold_on(const b200gan_conv_geom *g) {
  return g->up == 2 && g->pad_mode == B200GAN_PAD_ZERO && (g->S == 3 || g->S == 4);
}
template <int S> static size_t fewk_fold_smem(const b200gan_conv_geom *g) {
  return (size_t)Fold<S>::NFT * Fold<S>::NFT * g->K * g->C * sizeof(float);
}
#define FEWK_LAUNCH(KERN, GRID)                                                                   \
  {                                                                                               \
    static std::atomic<uint64_t> done{0};                                                         \
    if (int e = ensure_dynamic_smem(KERN, 160 * 1024, done)) return e;                            \
    KERN<<<GRID, 256, smem, st>>>(p);                                                             \
    B2_LAUNCH_CHECK();                                                                            \
    return B200GAN_OK;                                                                            \
  }
template <int S, int PAR>
static int fewk_fprop_up2_launch(const FewkP &p, int K, int grid, size_t smem, cudaStream_t st) {
  if (K == 1) FEWK_LAUNCH((fewk_fprop_up2_kernel<S, 1, PAR>), grid)
  if (K == 2) FEWK_LAUNCH((fewk_fprop_up2_kernel<S, 2, PAR>), grid)
  if (K == 3) FEWK_LAUNCH((fewk_fprop_up2_kernel<S, 3, PAR>), grid)
  FEWK_LAUNCH((fewk_fprop_up2_kernel<S, 4, PAR>), grid)
}
template <int S>
static int fewk_dgrad_up2_launch(const FewkP &p, int K, int grid, size_t smem, cudaStream_t st) {
  if (K == 1) FEWK_LAUNCH((fewk_dgrad_up2_kernel<S, 1>), grid)
  if (K == 2) FEWK_LAUNCH((fewk_dgrad_up2_kernel<S, 2>), grid)
  if (K == 3) FEWK_LAUNCH((fewk_dgrad_up2_kernel<S, 3>), grid)
  FEWK_LAUNCH((fewk_dgrad_up2_kernel<S, 4>), grid)
}
template <int S, int PAR>
static int fewk_wgrad_up2_launch(const FewkP &p, int K, int grid, size_t smem, cudaStream_t st) {
  if (K == 1) FEWK_LAUNCH((fewk_wgrad_up2_kernel<S, 1, PAR>), grid)
  if (K == 2) FEWK_LAUNCH((fewk_wgrad_up2_kernel<S, 2, PAR>), grid)
  if (K == 3) FEWK_LAUNCH((fewk_wgrad_up2_kernel<S, 3, PAR>), grid)
  FEWK_LAUNCH((fewk_wgrad_up2_kernel<S, 4, PAR>), grid)
}

template <int S>
static int fewk_fprop_launch(const FewkP &p, int K, int grid, size_t smem, cudaStream_t st) {
  static std::atomic<uint64_t> d1{0}, d2{0}, d3{0}, d4{0};
  switch (K) {
    case 1: if (int e = ensure_dynamic_smem(fewk_fprop_kernel<S, 1>, 160 * 1024, d1)) return e;
            fewk_fprop_kernel<S, 1><<<grid, 256, smem, st>>>(p); break;
    case 2: if (int e = ensure_dynamic_smem(fewk_fprop_kernel<S, 2>, 160 * 1024, d2)) return e;
            fewk_fprop_kernel<S, 2><<<grid, 256, smem, st>>>(p); break;
    case 3: if (int e = ensure_dynamic_smem(fewk_fprop_kernel<S, 3>, 160 * 1024, d3)) return e;
            fewk_fprop_kernel<S, 3><<<grid, 256, smem, st>>>(p); break;
    default: if (int e = ensure_dynamic_smem(fewk_fprop_kernel<S, 4>, 160 * 1024, d4)) return e;
            fewk_fprop_kernel<S, 4><<<grid, 256, smem, st>>>(p); break;
  }
  B2_LAUNCH_CHECK();
  return B200GAN_OK;
}

int fewk_fprop(const b200gan_conv_geom *g, const b200gan_epilogue *ep, const float *x, const float *packed, float *y,
               cudaStream_t st) {
  B2_CHECK_ARG(fewk_ok(g, 0), "fewk_fprop: unsupported geometry");
  B2_CHECK_ARG(!ep || (!ep->chan_scale && !ep->stats && !ep->round_tf32), "fewk_fprop: epilogue option not supported");
  if ((int64_t)g->N * g->P * g->Q == 0) return B200GAN_OK;
  FewkP p;
  fewk_fill(p, g);
  p.x = x; p.w = packed; p.y = y;
  p.bias = ep ? ep->bias : nullptr;
  p.act = ep ? ep->act : B200GAN_ACT_NONE;
  p.slope = ep ? ep->slope : 0.f;
  const size_t smem = (size_t)g->R * g->S * g->K * g->C * sizeof(float);
  const int64_t ntiles = (int64_t)g->N * ceil_div(g->P, 8) * ceil_div(g->Q, p.G * FK_PX);
  const int grid = (int)(ntiles < num_sms() * 4 ? ntiles : num_sms() * 4);
  if (fewk_fold_on(g)) {   // folded x2 upsample: parity-specific filters with 2..3 taps per dimension
    const int par = g->pad_l & 1;
    if (g->S == 3) return par ? fewk_fprop_up2_launch<3, 1>(p, g->K, grid, fewk_fold_smem<3>(g), st)
                              : fewk_fprop_up2_launch<3, 0>(p, g->K, grid, fewk_fold_smem<3>(g), st);
    return par ? fewk_fprop_up2_launch<4, 1>(p, g->K, grid, fewk_fold_smem<4>(g), st)
               : fewk_fprop_up2_launch<4, 0>(p, g->K, grid, fewk_fold_smem<4>(g), st);
  }
  if (g->S == 3) return fewk_fprop_launch<3>(p, g->K, grid, smem, st);
  if (g->S == 4) return fewk_fprop_launch<4>(p, g->K, grid, smem, st);
  return fewk_fprop_launch<7>(p, g->K, grid, smem, st);
}

template <int S>
static int fewk_dgrad_launch(const FewkP &p, int K, int grid, size_t smem, cudaStream_t st) {
  static std::atomic<uint64_t> d1{0}, d2{0}, d3{0}, d4{0};
  switch (K) {
    case 1: if (int e = ensure_dynamic_smem(fewk_dgrad_kernel<S, 1>, 160 * 1024, d1)) return e;
            fewk_dgrad_kernel<S, 1><<<grid, 256, smem, st>>>(p); break;
    case 2: if (int e = ensure_dynamic_smem(fewk_dgrad_kernel<S, 2>, 160 * 1024, d2)) return e;
            fewk_dgrad_kernel<S, 2><<<grid, 256, smem, st>>>(p); break;
    case 3: if (int e = ensure_dynamic_smem(fewk_dgrad_kernel<S, 3>, 160 * 1024, d3)) return e;
            fewk_dgrad_kernel<S, 3><<<grid, 256, smem, st>>>(p); break;
    default: if (int e = ensure_dynamic_smem(fewk_dgrad_kernel<S, 4>, 160 * 1024, d4)) return e;
            fewk_dgrad_kernel<S, 4><<<grid, 256, smem, st>>>(p); break;
  }
  B2_LAUNCH_CHECK();
  return B200GAN_OK;
}

// dx [N][H][W][C] (the SOURCE tensor: the upsample's backward is folded in), OVERWRITTEN
int fewk_dgrad(const b200gan_conv_geom *g, const float *dy, const float *packed, float *dx, cudaStream_t st) {
  B2_CHECK_ARG(fewk_ok(g, 1), "fewk_dgrad: unsupported geometry");
  if ((int64_t)g->N * g->H * g->W == 0) return B200GAN_OK;
  FewkP p;
  fewk_fill(p, g);
  p.dy = dy; p.w = packed; p.dx = dx;
  const size_t smem = (size_t)g->R * g->S * g->K * g->C * sizeof(float);
  const int64_t ntiles = (int64_t)g->N * ceil_div(g->H, 8) * ceil_div(g->W, p.G * FK_PX);
  const int grid = (int)(ntiles < num_sms() * 4 ? ntiles : num_sms() * 4);
  if (fewk_fold_on(g)) {
    if (g->S == 3) return fewk_dgrad_up2_launch<3>(p, g->K, grid, fewk_fold_smem<3>(g), st);
    return fewk_dgrad_up2_launch<4>(p, g->K, grid, fewk_fold_smem<4>(g), st);
  }
  if (g->S == 3) return fewk_dgrad_launch<3>(p, g->K, grid, smem, st);
  if (g->S == 4) return fewk_dgrad_launch<4>(p, g->K, grid, smem, st);
  return fewk_dgrad_launch<7>(p, g->K, grid, smem, st);
}

static int fk_wg_blocks() { return num_sms() * 2; }
size_t fewk_wgrad_workspace_floats(const b200gan_conv_geom *g) {
  return (size_t)fk_wg_blocks() * g->K * g->C * g->R * g->S;
}

template <int S>
static int fewk_wgrad_launch(const FewkP &p, int K, size_t smem, cudaStream_t st) {
  static std::atomic<uint64_t> d1{0}, d2{0}, d3{0}, d4{0};
  switch (K) {
    case 1: if (int e = ensure_dynamic_smem(fewk_wgrad_kernel<S, 1>, 160 * 1024, d1)) return e;
            fewk_wgrad_kernel<S, 1><<<fk_wg_blocks(), 256, smem, st>>>(p); break;
    case 2: if (int e = ensure_dynamic_smem(fewk_wgrad_kernel<S, 2>, 160 * 1024, d2)) return e;
            fewk_wgrad_kernel<S, 2><<<fk_wg_blocks(), 256, smem, st>>>(p); break;
    case 3: if (int e = ensure_dynamic_smem(fewk_wgrad_kernel<S, 3>, 160 * 1024, d3)) return e;
            fewk_wgrad_kernel<S, 3><<<fk_wg_blocks(), 256, smem, st>>>(p); break;
    default: if (int e = ensure_dynamic_smem(fewk_wgrad_kernel<S, 4>, 160 * 1024, d4)) return e;
            fewk_wgrad_kernel<S, 4><<<fk_wg_blocks(), 256, smem, st>>>(p); break;
  }
  B2_LAUNCH_CHECK();
  return B200GAN_OK;
}

int fewk_wgrad(const b200gan_conv_geom *g, const float *x, const float *dy, float *dw, float *workspace, cudaStream_t st) {
  B2_CHECK_ARG(fewk_ok(g, 2), "fewk_wgrad: unsupported geometry");
  B2_CHECK_ARG(workspace, "fewk_wgrad: workspace required");
  const int dw_elems = g->K * g->C * g->R * g->S;
  if ((int64_t)g->N * g->P * g->Q == 0) {
    B2_CUDA(cudaMemsetAsync(dw, 0, (size_t)dw_elems * sizeof(float), st));
    return B200GAN_OK;
  }
  FewkP p;
  fewk_fill(p, g);
  p.x = x; p.dy = dy; p.ws = workspace;
  const size_t smem = (size_t)dw_elems * sizeof(float);
  int rc;
  if (fewk_fold_on(g)) {
    const int par = g->pad_l & 1;
    if (g->S == 3) rc = par ? fewk_wgrad_up2_launch<3, 1>(p, g->K, fk_wg_blocks(), fewk_fold_smem<3>(g), st)
                            : fewk_wgrad_up2_launch<3, 0>(p, g->K, fk_wg_blocks(), fewk_fold_smem<3>(g), st);
    else rc = par ? fewk_wgrad_up2_launch<4, 1>(p, g->K, fk_wg_blocks(), fewk_fold_smem<4>(g), st)
                  : fewk_wgrad_up2_launch<4, 0>(p, g->K, fk_wg_blocks(), fewk_fold_smem<4>(g), st);
    if (rc) return rc;
    return nb_wgrad_reduce(workspace, dw, dw_elems, fk_wg_blocks(), st);
  }
  if (g->S == 3) rc = fewk_wgrad_launch<3>(p, g->K, smem, st);
  else if (g->S == 4) rc = fewk_wgrad_launch<4>(p, g->K, smem, st);
  else rc = fewk_wgrad_launch<7>(p, g->K, smem, st);
  if (rc) return rc;
  return nb_wgrad_reduce(workspace, dw, dw_elems, fk_wg_blocks(), st);
}

}  // namespace b200gan
