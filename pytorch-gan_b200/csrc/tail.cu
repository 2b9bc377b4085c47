// tail.cu -- the Generator "tail": BatchNorm2d -> LeakyReLU/ReLU -> Conv2d(C, K<=3, 3, 1, 1) -> Tanh as fused kernels
// that never materialise the normalised activation, its gradient, or the conv's data gradient.
//
// Reference call site: dcgan.py:60-63
//     nn.BatchNorm2d(64, 0.8), nn.LeakyReLU(0.2, inplace=True), nn.Conv2d(64, opt.channels, 3, stride=1, padding=1), nn.Tanh()
// on a = the raw output of the preceding conv, [128, 64, 64, 64] = 134 MB at the BASELINE config.  Un-fused this tail
// costs: norm apply (read a, write y), conv fprop (read y), conv dgrad (write dy), norm backward (read dy, a, y twice,
// write da), conv wgrad (read y): ~1.6 GB of HBM traffic.  Fused:
//   tail_fprop_tc_kernel   reads a once (134 MB).  A tile of 128 pixels is loaded with coalesced 16-byte loads,
//                          normalised + activated in registers, stored TF32-rounded into shared memory in the K-major
//                          128B-swizzled wgmma layout, and multiplied with wgmma (two warpgroups x M64 x N16/32 x K8,
//                          TF32) by the [taps x C] filter matrix: D[pixel][tap] in registers.  Every thread writes its
//                          accumulator fragment as tap partials into the band's rows in shared memory (the 3x3
//                          stencil is gathered at the end), then bias + Tanh + one coalesced store.  HBM-bound by
//                          design: the SM does ~300 instructions per pixel.
//   tail_bwd_reduce_kernel reads a once: recomputes the conv's data gradient from the 2 MB output gradient (9 FMAs per
//                          channel), applies the activation mask, accumulates the BatchNorm backward sums AND the conv's
//                          weight gradient (y recomputed from a) in registers; lane <-> 4 channels, so there is no
//                          cross-lane reduction until the end of the block.
//   tail_bwd_apply_kernel  reads a, writes da (the gradient w.r.t. the preceding conv's output).
// = 134 + 134 + 268 MB.
#include "tc_common.cuh"

namespace b200gan {

constexpr int TL_TH = 14;        // output rows per band (TH + 2 input rows = a whole number of 128-pixel tiles)
constexpr int TL_THREADS = 256;

struct TailP {
  const float *a;            // [N][H][W][C]
  const float *scale_shift;  // [2][C]
  const float *w;            // [K][C][3][3] (parameter layout)
  const float *bias;         // [K] or null
  float *out;                // [N][H][W][K]
  int N, H, W, C, K;
  int w_log2;                // W is a power of two
  int act_mid;
  float slope;
  int act_out;
};

__device__ __forceinline__ float mid_act(float v, int act, float slope) {
  if (act == B200GAN_ACT_LRELU) return v > 0.f ? v : v * slope;
  if (act == B200GAN_ACT_RELU) return fmaxf(v, 0.f);
  return v;
}
__device__ __forceinline__ float mid_act_grad(float pre, int act, float slope) {
  if (act == B200GAN_ACT_LRELU) return pre > 0.f ? 1.f : slope;
  if (act == B200GAN_ACT_RELU) return pre > 0.f ? 1.f : 0.f;
  return 1.f;
}

// ---- forward ------------------------------------------------------------------------------------------------
__device__ __forceinline__ void st_shared_v4(uint32_t addr, float4 v) {
  asm volatile("st.shared.v4.f32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}
__device__ __forceinline__ void st_shared_f32(uint32_t addr, float v) {
  asm volatile("st.shared.f32 [%0], %1;" ::"r"(addr), "f"(v) : "memory");
}
__device__ __forceinline__ float ld_shared_f32(uint32_t addr) {
  float v;
  asm volatile("ld.shared.f32 %0, [%1];" : "=f"(v) : "r"(addr));
  return v;
}

// grid (bands per image, N); block 256.  C4 = C/4 float4 per pixel (8, 16 or 32), NB = MMA N (16: K = 1; 32: K <= 3).
// Shared memory: A tile (KC x 16 KB, wgmma K-major SW128) | filter matrix B | T[(TH+2) rows][W][9K] tap
// partials of every input pixel of the band (+1 halo row each side).  No atomics: the 3x3 stencil is a gather over T at
// the end of the band (shared-memory fp32 atomics are CAS loops on this architecture).
template <int C4, int NB>
__global__ void __launch_bounds__(TL_THREADS, C4 == 32 ? 2 : 3)
tail_fprop_tc_kernel(const __grid_constant__ TailP p) {
  constexpr int KC = C4 / 8;                // 32-channel k-chunks
  constexpr int A_BYTES = KC * 16384;       // 128 pixels x 128 B per k-chunk
  constexpr int B_CHUNK = NB * 128;
  constexpr int IT = 128 * C4 / TL_THREADS; // float4 per thread per tile
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw = smem_u32(smem_raw);
  const uint32_t sA = (raw + 1023u) & ~1023u;   // shared-space byte addresses
  const uint32_t sB = sA + A_BYTES;
  const uint32_t sT = sB + KC * B_CHUNK;

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int wg = tid >> 7;  // warpgroup: MMA rows (pixels) [64 * wg, +64) of the tile
  const int W = p.W, H = p.H, K = p.K;
  const int n = blockIdx.y;
  const int p0 = blockIdx.x * TL_TH;
  const int th_eff = min(TL_TH, H - p0);
  const int RT = 128 >> p.w_log2;           // image rows per 128-pixel tile
  const int K9 = 9 * K;

  // filter matrix B[row = k*9 + tap][c] (zero rows above 9K), TF32-rounded, K-major SW128
  for (int i = tid; i < NB * C4 * 4; i += TL_THREADS) {
    const int c = i % (C4 * 4), row = i / (C4 * 4);
    float v = 0.f;
    if (row < K9) {
      const int k = row / 9, tap = row % 9;
      v = round_tf32(__ldg(p.w + ((int64_t)k * (C4 * 4) + c) * 9 + tap));
    }
    const int kc = c >> 5, cc = c & 31;
    st_shared_f32(sB + kc * B_CHUNK + row * 128 + (((cc >> 2) ^ (row & 7)) << 4) + (cc & 3) * 4, v);
  }
  // per-thread channel constants: this thread always handles float4 column (tid % C4) of a pixel
  const int c4 = tid % C4;
  float sc[4], sh[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    sc[j] = __ldg(p.scale_shift + c4 * 4 + j);
    sh[j] = __ldg(p.scale_shift + C4 * 4 + c4 * 4 + j);
  }
  const int act_mid = p.act_mid;
  const float slope = p.slope;
  fence_proxy_async();
  __syncthreads();

  // tiles of RT input rows starting at row p0 - 1; only those with a valid row that reaches the band are processed
  int t_lo = 0, t_hi = (TL_TH + 2) / RT;
  while (t_lo < t_hi && p0 - 1 + t_lo * RT + RT <= 0) ++t_lo;
  while (t_hi > t_lo && (p0 - 1 + (t_hi - 1) * RT >= H || p0 - 1 + (t_hi - 1) * RT > p0 + th_eff)) --t_hi;

  float4 v[IT];
  auto load_tile = [&](int t) {
    const int r0 = p0 - 1 + t * RT;
    const float4 *src = reinterpret_cast<const float4 *>(p.a) + ((int64_t)(n * H + r0) * W) * C4;
#pragma unroll
    for (int it = 0; it < IT; ++it) {
      const int idx = it * TL_THREADS + tid;
      const int row = r0 + ((idx / C4) >> p.w_log2);
      v[it] = (row >= 0 && row < H) ? __ldg(src + idx) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
  };
  if (t_lo < t_hi) load_tile(t_lo);

  for (int t = t_lo; t < t_hi; ++t) {
    const int r0 = p0 - 1 + t * RT;
#pragma unroll
    for (int it = 0; it < IT; ++it) {
      const int idx = it * TL_THREADS + tid;
      const int m = idx / C4;
      const int row = r0 + (m >> p.w_log2);
      float4 o = make_float4(0.f, 0.f, 0.f, 0.f);
      if (row >= 0 && row < H) {
        o.x = round_tf32(mid_act(fmaf(v[it].x, sc[0], sh[0]), act_mid, slope));
        o.y = round_tf32(mid_act(fmaf(v[it].y, sc[1], sh[1]), act_mid, slope));
        o.z = round_tf32(mid_act(fmaf(v[it].z, sc[2], sh[2]), act_mid, slope));
        o.w = round_tf32(mid_act(fmaf(v[it].w, sc[3], sh[3]), act_mid, slope));
      }
      const int kc = c4 >> 3, j = c4 & 7;
      st_shared_v4(sA + kc * 16384 + m * 128 + ((j ^ (m & 7)) << 4), o);
    }
    fence_proxy_async();  // generic-proxy smem writes -> visible to the tensor core (async proxy)
    __syncthreads();
    float d[NB / 2];
    wgmma_fence();
#pragma unroll
    for (int kc = 0; kc < KC; ++kc)
#pragma unroll
      for (int k = 0; k < 4; ++k)
        wgmma_tf32<NB>(d, gmma_desc_sw128(sA + kc * 16384 + wg * 8192 + k * 32), gmma_desc_sw128(sB + kc * B_CHUNK + k * 32),
                       (kc > 0 || k > 0) ? 1u : 0u);
    wgmma_commit();
    if (t + 1 < t_hi) load_tile(t + 1);  // in flight while the tensor core works on tile t
    wgmma_wait<0>();
    wgmma_fence_regs<NB / 2>(d);
    // D[m][k*9 + r*3 + s] is the (r,s) tap partial of INPUT pixel m of the tile; this thread holds rows m0 and m0 + 8
#pragma unroll
    for (int hr = 0; hr < 2; ++hr) {
      const int m = wg * 64 + (warp & 3) * 16 + (lane >> 2) + hr * 8;
      const int h = r0 + (m >> p.w_log2), w = m & (W - 1);
      if (h >= 0 && h < H) {
        const uint32_t dst = sT + (uint32_t)(((h - (p0 - 1)) * W + w) * K9) * 4;
#pragma unroll
        for (int j = 0; j < NB / 8; ++j)
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int col = j * 8 + (lane & 3) * 2 + e;
            if (col < K9) st_shared_f32(dst + col * 4, d[4 * j + 2 * hr + e]);
          }
      }
    }
    __syncthreads();  // both warpgroups' MMAs have retired: sA may be overwritten
  }
  {
    // out[p][q][k] = act(bias[k] + sum_{r,s} T[p + r - 1][q + s - 1][k*9 + r*3 + s])
    float *dst = p.out + ((int64_t)(n * H + p0) * W) * K;
    const int act_out = p.act_out;
    for (int i = tid; i < th_eff * W * K; i += TL_THREADS) {
      const int k = i % K, pq = i / K;
      const int qo = pq & (W - 1), po = pq >> p.w_log2;
      float acc = p.bias ? __ldg(p.bias + k) : 0.f;
#pragma unroll
      for (int r = 0; r < 3; ++r) {
        const int hh = p0 + po + r - 1;  // input row
        if (hh < 0 || hh >= H) continue;
#pragma unroll
        for (int s2 = 0; s2 < 3; ++s2) {
          const int ww = qo + s2 - 1;
          if (ww < 0 || ww >= W) continue;
          acc += ld_shared_f32(sT + (uint32_t)(((hh - (p0 - 1)) * W + ww) * K9 + k * 9 + r * 3 + s2) * 4);
        }
      }
      dst[i] = apply_act(acc, act_out, 0.f);
    }
  }
}

// ---- backward -------------------------------------------------------------------------------------------------
struct TailBwdP {
  const float *a;            // [N][H][W][C]
  const float *mean_rstd;    // [2][C]
  const float *scale_shift;  // [2][C]
  const float *w;            // [K][C][3][3]
  const float *g;            // [N][H][W][K]  gradient w.r.t. the conv's pre-activation output
  double *sums;              // [2][C]   sum dz, sum dz * xhat      (workspace, zero on entry of the reduce kernel)
  float *dw_acc;             // [K][C][3][3] (workspace, zero on entry)
  float *db_acc;             // [K]          (workspace, zero on entry)
  float *da;                 // [N][H][W][C]
  float *dgamma_dbeta;       // [2][C] or null
  float *dw;                 // [K][C][3][3]
  float *db;                 // [K] or null
  int N, H, W, C, K;
  int act_mid;
  float slope;
  int rtf;                   // round da to TF32 (it feeds the tensor-core dgrad / wgrad of the preceding conv)
  int64_t px_per_block;
};

// ---- streaming skeleton of the two backward passes ---------------------------------------------------------------
// `a` is read exactly once per pass, so the passes are pure HBM streams: a producer warp moves CHUNK-pixel pieces of the
// block's contiguous pixel range into a ring of shared-memory stages with 1-D bulk copies (cp.async.bulk, the TMA engine;
// completion on an mbarrier), eight consumer warps read their float4 from the ring (lane <-> 4 channels: conflict-free)
// and release the stage through an `empty` mbarrier.  Bytes in flight do not depend on registers or occupancy.
constexpr int RB_STAGES = 6;
constexpr int RB_CHUNK = 64;             // pixels per stage
constexpr int RB_CONSUMERS = 8;          // consumer warps
constexpr int RB_THREADS = (RB_CONSUMERS + 1) * 32;

__device__ __forceinline__ void bulk_g2s(uint32_t dst, const void *src, uint32_t bytes, uint64_t *bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst),
               "l"(reinterpret_cast<uint64_t>(src)), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
__device__ __forceinline__ float4 ld_shared_v4(uint32_t addr) {
  float4 v;
  asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(addr));
  return v;
}

// producer warp: streams pixels [b0, b1) of `a` (C floats each) through the ring
template <int C>
__device__ __forceinline__ void ring_produce(const float *__restrict__ a, int64_t b0, int64_t b1, uint32_t ring,
                                             uint64_t *full, uint64_t *empty) {
  if ((threadIdx.x & 31) != 0) return;
  const int64_t nchunks = (b1 - b0 + RB_CHUNK - 1) / RB_CHUNK;
  for (int64_t i = 0; i < nchunks; ++i) {
    const int stage = (int)(i % RB_STAGES);
    if (i >= RB_STAGES) mbar_wait(&empty[stage], (uint32_t)((i / RB_STAGES - 1) & 1));
    const int64_t px0 = b0 + i * RB_CHUNK;
    const int64_t npx = (b1 - px0) < RB_CHUNK ? (b1 - px0) : RB_CHUNK;
    const uint32_t bytes = (uint32_t)(npx * C * 4);
    mbar_arrive_expect_tx(&full[stage], bytes);
    bulk_g2s(ring + stage * (RB_CHUNK * C * 4), a + px0 * C, bytes, &full[stage]);
  }
}

// (h, w) of the pixel `off` columns after column 0 of row h0 -- 32-bit arithmetic (a shift when W is a power of two).
// The first version took pix % W and (pix / W) % H in 64 bits for every pixel: over half of the kernels' instructions.
__device__ __forceinline__ void tail_hw(int off, int h0, int W, int H, int wsh, int &w, int &h) {
  int q;
  if (wsh >= 0) { q = off >> wsh; w = off & (W - 1); }
  else { q = (int)((unsigned)off / (unsigned)W); w = off - q * W; }
  h = h0 + q;
  if (h >= H) h = (int)((unsigned)h % (unsigned)H);
}

__device__ __forceinline__ void tail_advance(int &w0, int &h0, int step, int W, int H, int wsh) {
  w0 += step;
  const int q = wsh >= 0 ? (w0 >> wsh) : (int)((unsigned)w0 / (unsigned)W);
  w0 -= q * W;
  h0 += q;
  if (h0 >= H) h0 = (int)((unsigned)h0 % (unsigned)H);
}

// the nine neighbours g[h + 1 - r][w + 1 - s] (zero outside the image) of channel k
template <int KK>
__device__ __forceinline__ void load_gn(const float *__restrict__ g, int64_t pix, int h, int w, int H, int W,
                                        float (&gn)[KK][9]) {
#pragma unroll
  for (int r = 0; r < 3; ++r) {
    const int hh = h + 1 - r;
#pragma unroll
    for (int s = 0; s < 3; ++s) {
      const int ww = w + 1 - s;
      const bool ok = hh >= 0 && hh < H && ww >= 0 && ww < W;
      const int64_t off = pix + (int64_t)(1 - r) * W + (1 - s);
#pragma unroll
      for (int k = 0; k < KK; ++k) gn[k][r * 3 + s] = ok ? __ldg(g + off * KK + k) : 0.f;
    }
  }
}

// (Tried: lane t < 9 of the pixel's lane group loads tap t and a shuffle hands it round -- one guarded load instead of nine
// per lane.  Measured slower, 250 vs 224 us for the backward pair: the nine dependent shuffles sit on the load latency.)
// pass 1: BatchNorm-backward sums + the conv's weight / bias gradient.  C4 lanes cover one pixel (float4 each).
template <int C4, int KK>
__global__ void __launch_bounds__(RB_THREADS, KK == 1 ? 2 : 1)
tail_bwd_reduce_kernel(const __grid_constant__ TailBwdP p) {
  constexpr int PPW = 32 / C4;                  // pixels per warp per pass
  constexpr int PPB = PPW * RB_CONSUMERS;       // pixels per block per pass
  constexpr int C = C4 * 4;
  extern __shared__ __align__(128) uint8_t dsm[];
  const uint32_t ring = smem_u32(dsm);                                   // RB_STAGES x RB_CHUNK x C floats
  float *wsm = reinterpret_cast<float *>(dsm + RB_STAGES * RB_CHUNK * C * 4);  // [KK*9][C] filter, tap-major
  float *red = wsm + KK * 9 * C;                                         // [KK*9 dw | s1 | s2][C]
  float *red_db = red + (KK * 9 + 2) * C;                                // [KK] (padded to 4)
  uint64_t *full = reinterpret_cast<uint64_t *>(red_db + 4);
  uint64_t *empty = full + RB_STAGES;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  for (int i = tid; i < KK * 9 * C; i += RB_THREADS) {
    const int c = i % C, kt = i / C;
    wsm[i] = __ldg(p.w + ((int64_t)(kt / 9) * C + c) * 9 + (kt % 9));
  }
  for (int i = tid; i < (KK * 9 + 2) * C + 4; i += RB_THREADS) red[i] = 0.f;
  if (tid == 0) {
    for (int s = 0; s < RB_STAGES; ++s) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], RB_CONSUMERS);
    }
    fence_barrier_init();
  }
  __syncthreads();

  const int H = p.H, W = p.W;
  const int64_t total = (int64_t)p.N * H * W;
  const int64_t b0 = (int64_t)blockIdx.x * p.px_per_block;
  int64_t b1 = b0 + p.px_per_block;
  if (b1 > total) b1 = total;
  if (warp == RB_CONSUMERS) {
    ring_produce<C>(p.a, b0, b1, ring, full, empty);
  } else {
    const int c4 = lane % C4, ps = lane / C4;
    float dwa[KK][9][4];
    float sc[4], sh[4], mean[4], rstd[4], s1[4], s2[4], dba[KK];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int c = c4 * 4 + j;
      sc[j] = __ldg(p.scale_shift + c);
      sh[j] = __ldg(p.scale_shift + C + c);
      mean[j] = __ldg(p.mean_rstd + c);
      rstd[j] = __ldg(p.mean_rstd + C + c);
      s1[j] = s2[j] = 0.f;
#pragma unroll
      for (int k = 0; k < KK; ++k)
#pragma unroll
        for (int t = 0; t < 9; ++t) dwa[k][t][j] = 0.f;
    }
#pragma unroll
    for (int k = 0; k < KK; ++k) dba[k] = 0.f;
    const int act_mid = p.act_mid;
    const float slope = p.slope;
    const uint32_t wsm_a = smem_u32(wsm) + c4 * 16;
    const int64_t nchunks = (b1 - b0 + RB_CHUNK - 1) / RB_CHUNK;
    int cw0 = (int)(b0 % W), ch0 = (int)((b0 / W) % H);   // (w, h) of the chunk\'s first pixel, advanced per chunk
    const int wsh = (W & (W - 1)) == 0 ? 31 - __clz(W) : -1;
    for (int64_t i = 0; i < nchunks; ++i) {
      const int stage = (int)(i % RB_STAGES);
      mbar_wait(&full[stage], (uint32_t)((i / RB_STAGES) & 1));
      const int64_t px0 = b0 + i * RB_CHUNK;
      const uint32_t sbase = ring + stage * (RB_CHUNK * C * 4) + c4 * 16;
#pragma unroll 1
      for (int lp = warp * PPW + ps; lp < RB_CHUNK; lp += PPB) {
        const int64_t pix = px0 + lp;
        if (pix >= b1) break;
        const float4 av = ld_shared_v4(sbase + lp * (C * 4));
        int w, h;
        tail_hw(cw0 + lp, ch0, W, H, wsh, w, h);
        float gn[KK][9];
        load_gn<KK>(p.g, pix, h, w, H, W, gn);
        const float x[4] = {av.x, av.y, av.z, av.w};
        float pre[4], y[4], dy[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          pre[j] = fmaf(x[j], sc[j], sh[j]);
          y[j] = mid_act(pre[j], act_mid, slope);
        }
#pragma unroll
        for (int k = 0; k < KK; ++k)
#pragma unroll
          for (int t = 0; t < 9; ++t) {
            const float4 wv = ld_shared_v4(wsm_a + (k * 9 + t) * (C * 4));
            const float gv = gn[k][t];
            dy[0] = fmaf(gv, wv.x, dy[0]);
            dy[1] = fmaf(gv, wv.y, dy[1]);
            dy[2] = fmaf(gv, wv.z, dy[2]);
            dy[3] = fmaf(gv, wv.w, dy[3]);
#pragma unroll
            for (int j = 0; j < 4; ++j) dwa[k][t][j] = fmaf(y[j], gv, dwa[k][t][j]);
          }
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const float dz = dy[j] * mid_act_grad(pre[j], act_mid, slope);
          const float xh = (x[j] - mean[j]) * rstd[j];
          s1[j] += dz;
          s2[j] = fmaf(dz, xh, s2[j]);
        }
        if (c4 == 0) {
#pragma unroll
          for (int k = 0; k < KK; ++k) dba[k] += gn[k][4];  // centre tap = g at this pixel
        }
      }
      tail_advance(cw0, ch0, RB_CHUNK, W, H, wsh);
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty[stage]);
    }
    // block reduction through shared-memory atomics (once per block)
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int c = c4 * 4 + j;
#pragma unroll
      for (int k = 0; k < KK; ++k)
#pragma unroll
        for (int t = 0; t < 9; ++t) atomicAdd(&red[(k * 9 + t) * C + c], dwa[k][t][j]);
      atomicAdd(&red[(KK * 9) * C + c], s1[j]);
      atomicAdd(&red[(KK * 9 + 1) * C + c], s2[j]);
    }
    if (c4 == 0) {
#pragma unroll
      for (int k = 0; k < KK; ++k) atomicAdd(&red_db[k], dba[k]);
    }
  }
  __syncthreads();
  for (int i = tid; i < KK * 9 * C; i += RB_THREADS) {
    const int c = i % C, kt = i / C;  // kt = k*9 + tap
    atomicAdd(p.dw_acc + ((int64_t)(kt / 9) * C + c) * 9 + (kt % 9), red[i]);
  }
  for (int i = tid; i < 2 * C; i += RB_THREADS) atomicAdd(p.sums + i, (double)red[KK * 9 * C + i]);
  if (tid < KK) atomicAdd(p.db_acc + tid, red_db[tid]);
}

// pass 2: da = scale * (dz - mean(dz) - xhat * mean(dz * xhat)); block 0 also publishes the parameter gradients
template <int C4, int KK>
__global__ void __launch_bounds__(RB_THREADS, KK == 1 ? 2 : 1)
tail_bwd_apply_kernel(const __grid_constant__ TailBwdP p) {
  constexpr int PPW = 32 / C4;
  constexpr int PPB = PPW * RB_CONSUMERS;
  constexpr int C = C4 * 4;
  extern __shared__ __align__(128) uint8_t dsm[];
  const uint32_t ring = smem_u32(dsm);
  float *wsm = reinterpret_cast<float *>(dsm + RB_STAGES * RB_CHUNK * C * 4);  // [KK*9][C]
  uint64_t *full = reinterpret_cast<uint64_t *>(wsm + KK * 9 * C);
  uint64_t *empty = full + RB_STAGES;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int H = p.H, W = p.W;
  const int64_t total = (int64_t)p.N * H * W;
  const float inv_count = (float)(1.0 / (double)total);

  if (blockIdx.x == 0) {
    if (p.dgamma_dbeta)
      for (int i = tid; i < C; i += RB_THREADS) {
        p.dgamma_dbeta[i] = (float)p.sums[C + i];  // dgamma = sum dz * xhat
        p.dgamma_dbeta[C + i] = (float)p.sums[i];  // dbeta  = sum dz
      }
    for (int i = tid; i < KK * C * 9; i += RB_THREADS) p.dw[i] = p.dw_acc[i];
    if (p.db && tid < KK) p.db[tid] = p.db_acc[tid];
  }
  for (int i = tid; i < KK * 9 * C; i += RB_THREADS) {
    const int c = i % C, kt = i / C;
    wsm[i] = __ldg(p.w + ((int64_t)(kt / 9) * C + c) * 9 + (kt % 9));
  }
  if (tid == 0) {
    for (int s = 0; s < RB_STAGES; ++s) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], RB_CONSUMERS);
    }
    fence_barrier_init();
  }
  __syncthreads();

  const int64_t b0 = (int64_t)blockIdx.x * p.px_per_block;
  int64_t b1 = b0 + p.px_per_block;
  if (b1 > total) b1 = total;
  if (warp == RB_CONSUMERS) {
    ring_produce<C>(p.a, b0, b1, ring, full, empty);
    return;
  }
  const int c4 = lane % C4, ps = lane / C4;
  float sc[4], sh[4], mean[4], rstd[4], m1[4], m2[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const int c = c4 * 4 + j;
    sc[j] = __ldg(p.scale_shift + c);
    sh[j] = __ldg(p.scale_shift + C + c);
    mean[j] = __ldg(p.mean_rstd + c);
    rstd[j] = __ldg(p.mean_rstd + C + c);
    m1[j] = (float)p.sums[c] * inv_count;
    m2[j] = (float)p.sums[C + c] * inv_count;
  }
  const int act_mid = p.act_mid, rtf = p.rtf;
  const float slope = p.slope;
  const uint32_t wsm_a = smem_u32(wsm) + c4 * 16;
  float4 *da4 = reinterpret_cast<float4 *>(p.da);
  const int64_t nchunks = (b1 - b0 + RB_CHUNK - 1) / RB_CHUNK;
  int cw0 = (int)(b0 % W), ch0 = (int)((b0 / W) % H);   // (w, h) of the chunk\'s first pixel, advanced per chunk
  const int wsh = (W & (W - 1)) == 0 ? 31 - __clz(W) : -1;
  for (int64_t i = 0; i < nchunks; ++i) {
    const int stage = (int)(i % RB_STAGES);
    mbar_wait(&full[stage], (uint32_t)((i / RB_STAGES) & 1));
    const int64_t px0 = b0 + i * RB_CHUNK;
    const uint32_t sbase = ring + stage * (RB_CHUNK * C * 4) + c4 * 16;
#pragma unroll 2
    for (int lp = warp * PPW + ps; lp < RB_CHUNK; lp += PPB) {
      const int64_t pix = px0 + lp;
      if (pix >= b1) break;
      const float4 av = ld_shared_v4(sbase + lp * (C * 4));
      int w, h;
      tail_hw(cw0 + lp, ch0, W, H, wsh, w, h);
      float gn[KK][9];
      load_gn<KK>(p.g, pix, h, w, H, W, gn);
      const float x[4] = {av.x, av.y, av.z, av.w};
      float dy[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
      for (int k = 0; k < KK; ++k)
#pragma unroll
        for (int t = 0; t < 9; ++t) {
          const float4 wv = ld_shared_v4(wsm_a + (k * 9 + t) * (C * 4));
          const float gv = gn[k][t];
          dy[0] = fmaf(gv, wv.x, dy[0]);
          dy[1] = fmaf(gv, wv.y, dy[1]);
          dy[2] = fmaf(gv, wv.z, dy[2]);
          dy[3] = fmaf(gv, wv.w, dy[3]);
        }
      float o[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float pre = fmaf(x[j], sc[j], sh[j]);
        const float dz = dy[j] * mid_act_grad(pre, act_mid, slope);
        const float xh = (x[j] - mean[j]) * rstd[j];
        const float v = sc[j] * (dz - m1[j] - xh * m2[j]);
        o[j] = rtf ? round_tf32(v) : v;
      }
      da4[pix * C4 + c4] = make_float4(o[0], o[1], o[2], o[3]);
    }
    tail_advance(cw0, ch0, RB_CHUNK, W, H, wsh);
    __syncwarp();
    if (lane == 0) mbar_arrive(&empty[stage]);
  }
}

static int ilog2_exact(int v) {
  int l = 0;
  while ((1 << l) < v) ++l;
  return (1 << l) == v ? l : -1;
}

template <int C4, int NB>
static int launch_tail_fprop(const TailP &p, cudaStream_t st) {
  const int smem = 1024 + (C4 / 8) * (16384 + NB * 128) + (TL_TH + 2) * p.W * 9 * p.K * 4;
  static std::atomic<uint64_t> done{0};
  B2_CHECK_ARG(smem <= 227 * 1024, "tail_fprop: W=%d K=%d C=%d needs %d bytes of shared memory", p.W, p.K, p.C, smem);
  if (int e = ensure_dynamic_smem(tail_fprop_tc_kernel<C4, NB>, 227 * 1024, done)) return e;
  dim3 grid((unsigned)ceil_div(p.H, TL_TH), (unsigned)p.N);
  tail_fprop_tc_kernel<C4, NB><<<grid, TL_THREADS, smem, st>>>(p);
  B2_LAUNCH_CHECK();
  return B200GAN_OK;
}

template <int C4, int KK>
static int launch_tail_bwd(TailBwdP &p, cudaStream_t st) {
  constexpr int C = C4 * 4;
  const int64_t total = (int64_t)p.N * p.H * p.W;
  const int ring_bytes = RB_STAGES * RB_CHUNK * C * 4;
  const int smem_reduce = ring_bytes + (KK * 9 * C + (KK * 9 + 2) * C + 4) * 4 + 2 * RB_STAGES * 8;
  const int smem_apply = ring_bytes + KK * 9 * C * 4 + 2 * RB_STAGES * 8;
  static std::atomic<uint64_t> done_r{0}, done_a{0};
  if (int e = ensure_dynamic_smem(tail_bwd_reduce_kernel<C4, KK>, smem_reduce, done_r)) return e;
  if (int e = ensure_dynamic_smem(tail_bwd_apply_kernel<C4, KK>, smem_apply, done_a)) return e;
  const int per_sm = (KK == 1 && C4 <= 16) ? 2 : 1;
  // contiguous pixel ranges, a whole number of ring chunks each, one block per resident slot
  int64_t per = ceil_div64(ceil_div64(total, (int64_t)num_sms() * per_sm), RB_CHUNK) * RB_CHUNK;
  p.px_per_block = per;
  const unsigned blocks = (unsigned)ceil_div64(total, per);
  tail_bwd_reduce_kernel<C4, KK><<<blocks, RB_THREADS, smem_reduce, st>>>(p);
  B2_LAUNCH_CHECK();
  tail_bwd_apply_kernel<C4, KK><<<blocks, RB_THREADS, smem_apply, st>>>(p);
  B2_LAUNCH_CHECK();
  return B200GAN_OK;
}

static int check_tail(const b200gan_tail_desc *d) {
  B2_CHECK_ARG(d != nullptr, "tail: null descriptor");
  B2_CHECK_ARG(d->N > 0 && d->H > 0 && d->W > 0, "tail: bad dims");
  if (!b200gan_tail_supported(d)) B2_UNSUPPORTED("tail: unsupported geometry (C in {32,64,128}, K in 1..3, W a power of two in 16..128)");
  return B200GAN_OK;
}

}  // namespace b200gan

using namespace b200gan;

extern "C" int b200gan_tail_supported(const b200gan_tail_desc *d) {
  if (!d) return 0;
  if (!(d->C == 32 || d->C == 64 || d->C == 128)) return 0;
  if (d->K < 1 || d->K > 3) return 0;
  const int wl = ilog2_exact(d->W);
  if (wl < 4 || wl > 7) return 0;
  if (d->H < 1 || d->N < 1 || d->N > 65535) return 0;
  if (!(d->act_mid == B200GAN_ACT_NONE || d->act_mid == B200GAN_ACT_LRELU || d->act_mid == B200GAN_ACT_RELU)) return 0;
  return 1;
}

extern "C" size_t b200gan_tail_bwd_workspace_bytes(const b200gan_tail_desc *d) {
  if (!d) return 0;
  return (size_t)2 * d->C * sizeof(double) + ((size_t)d->K * d->C * 9 + 4) * sizeof(float);
}

extern "C" int b200gan_tail_fprop(const b200gan_tail_desc *d, const float *a, const float *scale_shift, const float *w,
                                  const float *bias, float *out, void *stream) {
  if (int e = check_tail(d)) return e;
  B2_CHECK_ARG(a && scale_shift && w && out, "tail_fprop: null pointer");
  B2_CHECK_ARG((uintptr_t)a % 16 == 0, "tail_fprop: activation pointer must be 16-byte aligned");
  TailP p;
  p.a = a; p.scale_shift = scale_shift; p.w = w; p.bias = bias; p.out = out;
  p.N = d->N; p.H = d->H; p.W = d->W; p.C = d->C; p.K = d->K;
  p.w_log2 = ilog2_exact(d->W);
  p.act_mid = d->act_mid; p.slope = d->slope; p.act_out = d->act_out;
  cudaStream_t st = as_stream(stream);
  const bool wide = d->K > 1;
  if (d->C == 64) return wide ? launch_tail_fprop<16, 32>(p, st) : launch_tail_fprop<16, 16>(p, st);
  if (d->C == 128) return wide ? launch_tail_fprop<32, 32>(p, st) : launch_tail_fprop<32, 16>(p, st);
  return wide ? launch_tail_fprop<8, 32>(p, st) : launch_tail_fprop<8, 16>(p, st);
}

extern "C" int b200gan_tail_bwd(const b200gan_tail_desc *d, const float *a, const float *mean_rstd,
                                const float *scale_shift, const float *w, const float *g, void *workspace, float *da,
                                float *dgamma_dbeta, float *dw, float *db, int32_t round_tf32, void *stream) {
  if (int e = check_tail(d)) return e;
  B2_CHECK_ARG(a && mean_rstd && scale_shift && w && g && workspace && da && dw, "tail_bwd: null pointer");
  B2_CHECK_ARG(((uintptr_t)a | (uintptr_t)da | (uintptr_t)workspace) % 16 == 0, "tail_bwd: pointers must be 16-byte aligned");
  cudaStream_t st = as_stream(stream);
  B2_CUDA(cudaMemsetAsync(workspace, 0, b200gan_tail_bwd_workspace_bytes(d), st));
  TailBwdP p;
  p.a = a; p.mean_rstd = mean_rstd; p.scale_shift = scale_shift; p.w = w; p.g = g;
  p.sums = reinterpret_cast<double *>(workspace);
  p.dw_acc = reinterpret_cast<float *>(p.sums + 2 * d->C);
  p.db_acc = p.dw_acc + (size_t)d->K * d->C * 9;
  p.da = da; p.dgamma_dbeta = dgamma_dbeta; p.dw = dw; p.db = db;
  p.N = d->N; p.H = d->H; p.W = d->W; p.C = d->C; p.K = d->K;
  p.act_mid = d->act_mid; p.slope = d->slope; p.rtf = round_tf32; p.px_per_block = 0;
#define TAIL_BWD(C4)                                              \
  do {                                                            \
    if (d->K == 1) return launch_tail_bwd<C4, 1>(p, st);          \
    if (d->K == 2) return launch_tail_bwd<C4, 2>(p, st);          \
    return launch_tail_bwd<C4, 3>(p, st);                         \
  } while (0)
  if (d->C == 64) TAIL_BWD(16);
  if (d->C == 128) TAIL_BWD(32);
  TAIL_BWD(8);
#undef TAIL_BWD
}
