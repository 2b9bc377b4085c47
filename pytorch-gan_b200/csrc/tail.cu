// tail.cu -- the Generator "tail": BatchNorm2d -> LeakyReLU/ReLU -> Conv2d(C, K<=3, 3, 1, 1) -> Tanh as fused kernels
// that never materialise the normalised activation, its gradient, or the conv's data gradient.
//
// Reference call site: dcgan.py:60-63
//     nn.BatchNorm2d(64, 0.8), nn.LeakyReLU(0.2, inplace=True), nn.Conv2d(64, opt.channels, 3, stride=1, padding=1), nn.Tanh()
// on a = the raw output of the preceding conv, [128, 64, 64, 64] = 134 MB at the BASELINE config.  Un-fused this tail
// costs: norm apply (read a, write y), conv fprop (read y), conv dgrad (write dy), norm backward (read dy, a, y twice,
// write da), conv wgrad (read y): ~1.6 GB of HBM traffic.  Fused:
//   tail_fprop_tc_kernel   reads a once (134 MB), persistent: one block per resident slot streams a contiguous range of
//                          the N*H image rows (ranges cross image boundaries; only the two halo rows of each range are
//                          read twice).  A tile of 128 pixels is loaded with coalesced 16-byte loads one tile ahead,
//                          normalised + activated in registers, stored TF32-rounded into shared memory in the K-major
//                          128B-swizzled wgmma layout, and multiplied with wgmma (two warpgroups x M64 x N16/32 x K8,
//                          TF32) by the [taps x C] filter matrix: D[pixel][tap] in registers.  Every thread writes its
//                          accumulator fragment as tap partials into a ring of RT + 2 rows in shared memory; each output
//                          row is gathered (3x3 stencil, bias, Tanh, coalesced store) as soon as the row below it has
//                          been multiplied, while the next tile's loads are in flight.
//   tail_bwd_reduce_kernel reads a once: recomputes the conv's data gradient from the 2 MB output gradient (9 FMAs per
//                          channel, neighbours from a zero-padded copy of g in shared memory), applies the activation
//                          mask, accumulates the BatchNorm backward sums AND the conv's weight gradient (y recomputed
//                          from a) in registers; lane <-> 4 channels, so there is no cross-lane reduction until the end
//                          of the block.
//   tail_bwd_apply_kernel  reads a, writes da (the gradient w.r.t. the preceding conv's output); walks each block's
//                          range backwards, so that it starts on what the reduce pass left in L2.
// = 134 + 134 + 268 MB.
#include "tc_common.cuh"

namespace b200gan {

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
  int rows_per_block;         // output rows of the N*H rows per block
};

__device__ __forceinline__ float mid_act(float v, int act, float slope) {
  if (act == B200GAN_ACT_LRELU) return v > 0.f ? v : v * slope;
  if (act == B200GAN_ACT_RELU) return fmaxf(v, 0.f);
  return v;
}
// The backward passes use the activation through its slope below zero (LeakyReLU: slope, ReLU: 0, none: 1), so the
// pixel loops hold no branch on the activation kind.
__device__ __forceinline__ float mid_neg_slope(int act, float slope) {
  return act == B200GAN_ACT_LRELU ? slope : act == B200GAN_ACT_RELU ? 0.f : 1.f;
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

// Persistent: grid = one block per resident slot; block b owns output rows [b * rows_per_block, +rows_per_block) of
// the N*H rows of all images (a range may cross image boundaries) and streams input rows from one row above its range
// to one row below it in tiles of RT = 128 / W rows.  C4 = C/4 float4 per pixel (8, 16 or 32), NB = MMA N (16: K = 1;
// 32: K <= 3).  Shared memory: A tile (KC x 16 KB, wgmma K-major SW128) | filter matrix B | T, a ring of RT + 2 rows
// [W][9K] of tap partials.  After tile t, every output row whose three input rows are in T is gathered (bias, then r,
// then s) and stored while the next tile's loads are in flight.  No atomics (shared-memory fp32 atomics are CAS loops on
// this architecture).
// Blocks per SM: three (two at C = 128); one fewer for the N = 32 accumulator at C >= 64, which would spill otherwise.
template <int C4, int NB>
constexpr int tail_fprop_blocks() { return (C4 == 32 ? 2 : 3) - (NB == 32 && C4 >= 16 ? 1 : 0); }

template <int C4, int NB>
__global__ void __launch_bounds__(TL_THREADS, tail_fprop_blocks<C4, NB>())
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
  const int W = p.W, H = p.H, K = p.K, wl = p.w_log2;
  const int NH = p.N * H;
  const int P0 = blockIdx.x * p.rows_per_block;
  const int P1 = min(P0 + p.rows_per_block, NH);   // output rows [P0, P1)
  const int RT = 128 >> wl;                 // image rows per 128-pixel tile
  const int TR = RT + 2;                    // rows of the T ring
  const int K9 = 9 * K;
  const int ntiles = (P1 + 1 - (P0 - 1) + RT - 1) / RT;

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
  const int act_mid = p.act_mid, act_out = p.act_out;
  const float slope = p.slope;
  fence_proxy_async();
  __syncthreads();

  float4 v[IT];
  auto load_tile = [&](int t) {
    const int r0 = P0 - 1 + t * RT;
    const float4 *src = reinterpret_cast<const float4 *>(p.a) + (int64_t)r0 * W * C4;
#pragma unroll
    for (int it = 0; it < IT; ++it) {
      const int idx = it * TL_THREADS + tid;
      const int row = r0 + ((idx / C4) >> wl);
      v[it] = (row >= 0 && row < NH) ? __ldg(src + idx) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
  };
  load_tile(0);

  int pg = P0;  // first output row not yet stored
  for (int t = 0; t < ntiles; ++t) {
    const int r0 = P0 - 1 + t * RT;
#pragma unroll
    for (int it = 0; it < IT; ++it) {
      const int idx = it * TL_THREADS + tid;
      const int m = idx / C4;
      const int row = r0 + (m >> wl);
      float4 o = make_float4(0.f, 0.f, 0.f, 0.f);
      if (row >= 0 && row < NH) {
        o.x = round_tf32(mid_act(fmaf(v[it].x, sc[0], sh[0]), act_mid, slope));
        o.y = round_tf32(mid_act(fmaf(v[it].y, sc[1], sh[1]), act_mid, slope));
        o.z = round_tf32(mid_act(fmaf(v[it].z, sc[2], sh[2]), act_mid, slope));
        o.w = round_tf32(mid_act(fmaf(v[it].w, sc[3], sh[3]), act_mid, slope));
      }
      const int kc = c4 >> 3, j = c4 & 7;
      st_shared_v4(sA + kc * 16384 + m * 128 + ((j ^ (m & 7)) << 4), o);
    }
    fence_proxy_async();  // generic-proxy smem writes -> visible to the tensor core (async proxy)
    __syncthreads();      // also: the previous tile's gather is done with the T rows this tile overwrites
    float d[NB / 2];
    wgmma_fence();
#pragma unroll
    for (int kc = 0; kc < KC; ++kc)
#pragma unroll
      for (int k = 0; k < 4; ++k)
        wgmma_tf32<NB>(d, gmma_desc_sw128(sA + kc * 16384 + wg * 8192 + k * 32), gmma_desc_sw128(sB + kc * B_CHUNK + k * 32),
                       (kc > 0 || k > 0) ? 1u : 0u);
    wgmma_commit();
    if (t + 1 < ntiles) load_tile(t + 1);  // in flight while the tensor core works on tile t and T is gathered
    wgmma_wait<0>();
    wgmma_fence_regs<NB / 2>(d);
    // D[m][k*9 + r*3 + s] is the (r,s) tap partial of INPUT pixel m of the tile; this thread holds rows m0 and m0 + 8
#pragma unroll
    for (int hr = 0; hr < 2; ++hr) {
      const int m = wg * 64 + (warp & 3) * 16 + (lane >> 2) + hr * 8;
      const int row = r0 + (m >> wl), w = m & (W - 1);
      if (row >= 0 && row < NH) {
        const uint32_t dst = sT + (uint32_t)((((unsigned)row % (unsigned)TR) * W + w) * K9) * 4;
#pragma unroll
        for (int j = 0; j < NB / 8; ++j)
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int col = j * 8 + (lane & 3) * 2 + e;
            if (col < K9) st_shared_f32(dst + col * 4, d[4 * j + 2 * hr + e]);
          }
      }
    }
    __syncthreads();  // both warpgroups' MMAs have retired: sA may be overwritten; T rows of tile t are visible
    // output rows [pg, pe) now have all three input rows in T:
    // out[P][q][k] = act(bias[k] + sum_{r,s} T[P + r - 1][q + s - 1][k*9 + r*3 + s])
    const int pe = t + 1 == ntiles ? P1 : max(pg, min(P1, r0 + RT - 1));
    float *dst = p.out + (int64_t)pg * W * K;
    for (int i = tid; i < (pe - pg) * W * K; i += TL_THREADS) {
      const int k = i % K, pq = i / K;
      const int qo = pq & (W - 1), P = pg + (pq >> wl);
      const int h = P % H;
      float acc = p.bias ? __ldg(p.bias + k) : 0.f;
#pragma unroll
      for (int r = 0; r < 3; ++r) {
        const int hh = h + r - 1;  // input row within the image
        if (hh < 0 || hh >= H) continue;
        const uint32_t trow = sT + (uint32_t)(((unsigned)(P + r - 1) % (unsigned)TR) * W * K9 + k * 9 + r * 3) * 4;
#pragma unroll
        for (int s2 = 0; s2 < 3; ++s2) {
          const int ww = qo + s2 - 1;
          if (ww < 0 || ww >= W) continue;
          acc += ld_shared_f32(trow + (uint32_t)(ww * K9 + s2) * 4);
        }
      }
      dst[i] = apply_act(acc, act_out, 0.f);
    }
    pg = pe;
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
  int tab_rows;               // rows a block's range can touch (row table entries)
  int slab_rows;              // rows of the zero-padded g slab
};

// ---- streaming skeleton of the two backward passes ---------------------------------------------------------------
// `a` is read exactly once per pass, so the passes are pure HBM streams.  Each block owns a contiguous pixel range and
// moves it in RB_STAGE_BYTES pieces through a ring of shared-memory stages with 1-D bulk copies (cp.async.bulk, the TMA
// engine; completion on an mbarrier).  All eight warps consume (lane <-> 4 channels: conflict-free float4 reads); the
// last warp to finish with a stage refills it (a shared counter per stage), so there is no producer warp, the block is
// 256 threads, and no warp ever waits for a free stage.  Bytes in flight do not depend on registers or occupancy.
//
// The output gradient g of the block's rows (+1 halo row each side) sits in shared memory as a zero-padded slab: one
// zero column on each side of every row and one zero row between images.  The nine neighbours of a pixel are then
// plain shared-memory loads at fixed offsets from its centre, with no bounds checks and no global loads in the pixel
// loop.  A per-row table holds the slab address of each of the block's rows.
constexpr int RB_STAGES = 5;
constexpr int RB_STAGE_BYTES = 16384;    // C=32: 128 pixels, C=64: 64, C=128: 32
constexpr int RB_WARPS = 8;
constexpr int RB_THREADS = RB_WARPS * 32;
constexpr int RB_SMEM_2CTA = 110 * 1024; // per-block budget for two blocks per SM
constexpr int RB_SMEM_1CTA = 220 * 1024;

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
__device__ __forceinline__ int ld_shared_s32(uint32_t addr) {
  int v;
  asm volatile("ld.shared.s32 %0, [%1];" : "=r"(v) : "r"(addr));
  return v;
}
__device__ __forceinline__ int64_t floor_div(int64_t a, int64_t b) { return a >= 0 ? a / b : -((-a + b - 1) / b); }

// shared-memory layout of both passes: ring | filter [KK*9][C] (KK > 1 only; KK = 1 keeps it in registers) |
// reduction [KK*9 dw | s1 | s2][C] + [4] db (reduce pass only) | full[RB_STAGES] | count[RB_STAGES] | row table | slab
template <int C4, int KK, bool REDUCE>
struct TailBwdSmem {
  static constexpr int C = C4 * 4;
  static constexpr bool WREG = KK == 1;
  static constexpr int RING = RB_STAGES * RB_STAGE_BYTES;
  static constexpr int WSM = WREG ? 0 : KK * 9 * C * 4;
  static constexpr int RED = REDUCE ? ((KK * 9 + 2) * C + 4) * 4 : 0;
  static constexpr int BARS = RING + WSM + RED;
  static constexpr int FIXED = BARS + (RB_STAGES * 12 + 15) / 16 * 16;
  static_assert(FIXED % 16 == 0, "row table alignment");
  static int bytes(int tab_rows, int slab_rows, int W) {
    return FIXED + (tab_rows * 4 + 15) / 16 * 16 + slab_rows * (W + 2) * KK * 4;
  }
};

// Everything a block needs to walk its range: ring, slab, row table.  `sweep` runs the block's pixels through body(pix,
// row-table entry, x) in chunk order (forward, or backward when REV) and keeps the ring full.
template <int C4, int KK, bool REDUCE>
struct TailBwdBlock {
  using L = TailBwdSmem<C4, KK, REDUCE>;
  static constexpr int C = C4 * 4;
  static constexpr int CHUNK = RB_STAGE_BYTES / (C * 4);  // pixels per stage
  uint32_t ring, tab, slab;
  uint64_t *full;
  unsigned *count;
  int64_t b0;
  int npx, nchunks, c0, rowf;  // c0: column of the first pixel; rowf: floats per slab row

  __device__ void init(const TailBwdP &p, uint8_t *dsm) {
    const int tid = threadIdx.x;
    ring = smem_u32(dsm);
    full = reinterpret_cast<uint64_t *>(dsm + L::BARS);
    count = reinterpret_cast<unsigned *>(full + RB_STAGES);
    tab = smem_u32(dsm + L::FIXED);
    slab = tab + (p.tab_rows * 4 + 15) / 16 * 16;
    const int64_t total = (int64_t)p.N * p.H * p.W;
    b0 = (int64_t)blockIdx.x * p.px_per_block;
    npx = (int)((total - b0) < p.px_per_block ? (total - b0) : p.px_per_block);
    nchunks = (npx + CHUNK - 1) / CHUNK;
    rowf = (p.W + 2) * KK;
    if (tid == 0) {
      for (int s = 0; s < RB_STAGES; ++s) {
        mbar_init(&full[s], 1);
        count[s] = 0;
      }
      fence_barrier_init();
    }
    float *sl = reinterpret_cast<float *>(dsm + (slab - ring));
    for (int i = tid; i < p.slab_rows * rowf; i += RB_THREADS) sl[i] = 0.f;
  }

  template <bool REV>
  __device__ __forceinline__ void issue(const float *a, int i) {
    const int stage = i % RB_STAGES;
    const int j = REV ? nchunks - 1 - i : i;
    const int n = min(CHUNK, npx - j * CHUNK);
    const uint32_t bytes = (uint32_t)(n * C * 4);
    mbar_arrive_expect_tx(&full[stage], bytes);
    bulk_g2s(ring + stage * RB_STAGE_BYTES, a + (b0 + (int64_t)j * CHUNK) * C, bytes, &full[stage]);
  }

  // after init's __syncthreads: start the ring, then fill the slab and the row table (overlapping the first loads)
  template <bool REV>
  __device__ void start(const TailBwdP &p, uint8_t *dsm) {
    const int tid = threadIdx.x, W = p.W, H = p.H;
    if (tid == 0)
      for (int i = 0; i < min(RB_STAGES, nchunks); ++i) issue<REV>(p.a, i);
    const int64_t R0 = b0 / W, NH = (int64_t)p.N * H;
    c0 = (int)(b0 - R0 * W);
    const int nq = (c0 + npx + W - 1) / W;  // rows of the range
    const int64_t sep0 = floor_div(R0 - 1, H);
    // slab row of global row R >= R0 - 1: its distance from R0 - 1 plus the image starts in (R0 - 1, R]
    auto slab_row = [&](int64_t R) { return (int)(R - R0 + 1 + floor_div(R, H) - sep0); };
    float *sl = reinterpret_cast<float *>(dsm + (slab - ring));
    const int WK = W * KK;
    for (int i = tid; i < (nq + 2) * WK; i += RB_THREADS) {
      const int rr = i / WK, e = i - rr * WK;
      const int64_t R = R0 - 1 + rr;
      if (R >= 0 && R < NH) sl[slab_row(R) * rowf + KK + e] = __ldg(p.g + R * WK + e);
    }
    for (int q = tid; q < nq; q += RB_THREADS)
      reinterpret_cast<int *>(dsm + (tab - ring))[q] = (int)slab + (slab_row(R0 + q) * rowf + KK) * 4;
  }

  // the stage of sequence number i is no longer read by this warp; the last of the eight warps refills it
  template <bool REV>
  __device__ __forceinline__ void release(const float *a, int i) {
    __syncwarp();
    if ((threadIdx.x & 31) == 0) {
      __threadfence_block();
      const unsigned done = atomicAdd(&count[i % RB_STAGES], 1u) + 1u;
      if (done == (unsigned)(i / RB_STAGES + 1) * RB_WARPS && i + RB_STAGES < nchunks) {
        __threadfence_block();
        fence_proxy_async();  // the generic-proxy reads of the stage are ordered before the bulk copy that overwrites it
        issue<REV>(a, i + RB_STAGES);
      }
    }
  }

  // the nine neighbours g[h + 1 - r][w + 1 - s] of channel k (zero outside the image): `ctr` is the pixel's slab address
  __device__ __forceinline__ void gather(uint32_t ctr, float (&gn)[KK][9]) const {
#pragma unroll
    for (int r = 0; r < 3; ++r)
#pragma unroll
      for (int s = 0; s < 3; ++s)
#pragma unroll
        for (int k = 0; k < KK; ++k)
          gn[k][r * 3 + s] = ld_shared_f32(ctr + (uint32_t)(((1 - r) * rowf + (1 - s) * KK + k) * 4));
  }
};

// pass 1: BatchNorm-backward sums + the conv's weight / bias gradient.  C4 lanes cover one pixel (float4 each).
template <int C4, int KK>
__global__ void __launch_bounds__(RB_THREADS, KK == 1 ? 2 : 1)
tail_bwd_reduce_kernel(const __grid_constant__ TailBwdP p) {
  using Blk = TailBwdBlock<C4, KK, true>;
  using L = TailBwdSmem<C4, KK, true>;
  constexpr int PPW = 32 / C4;                  // pixels per warp per pass
  constexpr int PPB = PPW * RB_WARPS;           // pixels per block per pass
  constexpr int C = C4 * 4;
  extern __shared__ __align__(128) uint8_t dsm[];
  float *wsm = reinterpret_cast<float *>(dsm + L::RING);  // [KK*9][C] filter, tap-major (KK > 1)
  float *red = reinterpret_cast<float *>(dsm + L::RING + L::WSM);  // [KK*9 dw | s1 | s2][C]
  float *red_db = red + (KK * 9 + 2) * C;                 // [KK] (padded to 4)
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  Blk blk;
  blk.init(p, dsm);
  if constexpr (!L::WREG)
    for (int i = tid; i < KK * 9 * C; i += RB_THREADS) {
      const int c = i % C, kt = i / C;
      wsm[i] = __ldg(p.w + ((int64_t)(kt / 9) * C + c) * 9 + (kt % 9));
    }
  for (int i = tid; i < (KK * 9 + 2) * C + 4; i += RB_THREADS) red[i] = 0.f;
  __syncthreads();
  blk.template start<false>(p, dsm);

  const int c4 = lane % C4, ps = lane / C4;
  float wr[L::WREG ? 9 : 1][4];
  if constexpr (L::WREG)
#pragma unroll
    for (int t = 0; t < 9; ++t)
#pragma unroll
      for (int j = 0; j < 4; ++j) wr[t][j] = __ldg(p.w + (c4 * 4 + j) * 9 + t);
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
  const float neg = mid_neg_slope(p.act_mid, p.slope);
  const uint32_t wsm_a = smem_u32(wsm) + c4 * 16;
  const int wsh = 31 - __clz(p.W), wmask = p.W - 1;
  __syncthreads();  // slab and row table are complete
  for (int i = 0; i < blk.nchunks; ++i) {
    const int stage = i % RB_STAGES;
    mbar_wait(&blk.full[stage], (uint32_t)((i / RB_STAGES) & 1));
    const int o0 = i * Blk::CHUNK;
    const int n = min(Blk::CHUNK, blk.npx - o0);
    const uint32_t sbase = blk.ring + stage * RB_STAGE_BYTES + c4 * 16;
#pragma unroll 1
    for (int lp = warp * PPW + ps; lp < n; lp += PPB) {
      const float4 av = ld_shared_v4(sbase + lp * (C * 4));
      const int off = blk.c0 + o0 + lp;
      const uint32_t ctr = (uint32_t)ld_shared_s32(blk.tab + (off >> wsh) * 4) + (uint32_t)((off & wmask) * KK * 4);
      float gn[KK][9];
      blk.gather(ctr, gn);
      const float x[4] = {av.x, av.y, av.z, av.w};
      float pre[4], y[4], dy[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        pre[j] = fmaf(x[j], sc[j], sh[j]);
        y[j] = pre[j] > 0.f ? pre[j] : pre[j] * neg;
      }
#pragma unroll
      for (int k = 0; k < KK; ++k)
#pragma unroll
        for (int t = 0; t < 9; ++t) {
          float4 wv;
          if constexpr (L::WREG) wv = make_float4(wr[t][0], wr[t][1], wr[t][2], wr[t][3]);
          else wv = ld_shared_v4(wsm_a + (k * 9 + t) * (C * 4));
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
        const float dz = dy[j] * (pre[j] > 0.f ? 1.f : neg);
        const float xh = (x[j] - mean[j]) * rstd[j];
        s1[j] += dz;
        s2[j] = fmaf(dz, xh, s2[j]);
      }
      if (c4 == 0) {
#pragma unroll
        for (int k = 0; k < KK; ++k) dba[k] += gn[k][4];  // centre tap = g at this pixel
      }
    }
    blk.template release<false>(p.a, i);
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
  __syncthreads();
  for (int i = tid; i < KK * 9 * C; i += RB_THREADS) {
    const int c = i % C, kt = i / C;  // kt = k*9 + tap
    atomicAdd(p.dw_acc + ((int64_t)(kt / 9) * C + c) * 9 + (kt % 9), red[i]);
  }
  for (int i = tid; i < 2 * C; i += RB_THREADS) atomicAdd(p.sums + i, (double)red[KK * 9 * C + i]);
  if (tid < KK) atomicAdd(p.db_acc + tid, red_db[tid]);
}

// pass 2: da = scale * (dz - mean(dz) - xhat * mean(dz * xhat)); block 0 also publishes the parameter gradients.
// Each block walks its range backwards: the reduce pass read the same range forwards just before, so the first chunks
// read here are the ones most likely still in L2.
template <int C4, int KK>
__global__ void __launch_bounds__(RB_THREADS, KK == 1 ? 2 : 1)
tail_bwd_apply_kernel(const __grid_constant__ TailBwdP p) {
  using Blk = TailBwdBlock<C4, KK, false>;
  using L = TailBwdSmem<C4, KK, false>;
  constexpr int PPW = 32 / C4;
  constexpr int PPB = PPW * RB_WARPS;
  constexpr int C = C4 * 4;
  extern __shared__ __align__(128) uint8_t dsm[];
  float *wsm = reinterpret_cast<float *>(dsm + L::RING);  // [KK*9][C] (KK > 1)
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int64_t total = (int64_t)p.N * p.H * p.W;
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
  Blk blk;
  blk.init(p, dsm);
  if constexpr (!L::WREG)
    for (int i = tid; i < KK * 9 * C; i += RB_THREADS) {
      const int c = i % C, kt = i / C;
      wsm[i] = __ldg(p.w + ((int64_t)(kt / 9) * C + c) * 9 + (kt % 9));
    }
  __syncthreads();
  blk.template start<true>(p, dsm);

  const int c4 = lane % C4, ps = lane / C4;
  float wr[L::WREG ? 9 : 1][4];
  if constexpr (L::WREG)
#pragma unroll
    for (int t = 0; t < 9; ++t)
#pragma unroll
      for (int j = 0; j < 4; ++j) wr[t][j] = __ldg(p.w + (c4 * 4 + j) * 9 + t);
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
  const int rtf = p.rtf;
  const float neg = mid_neg_slope(p.act_mid, p.slope);
  const uint32_t wsm_a = smem_u32(wsm) + c4 * 16;
  float4 *da4 = reinterpret_cast<float4 *>(p.da) + blk.b0 * C4 + c4;
  const int wsh = 31 - __clz(p.W), wmask = p.W - 1;
  __syncthreads();  // slab and row table are complete
  for (int i = 0; i < blk.nchunks; ++i) {
    const int stage = i % RB_STAGES;
    mbar_wait(&blk.full[stage], (uint32_t)((i / RB_STAGES) & 1));
    const int o0 = (blk.nchunks - 1 - i) * Blk::CHUNK;
    const int n = min(Blk::CHUNK, blk.npx - o0);
    const uint32_t sbase = blk.ring + stage * RB_STAGE_BYTES + c4 * 16;
#pragma unroll 2
    for (int lp = warp * PPW + ps; lp < n; lp += PPB) {
      const float4 av = ld_shared_v4(sbase + lp * (C * 4));
      const int off = blk.c0 + o0 + lp;
      const uint32_t ctr = (uint32_t)ld_shared_s32(blk.tab + (off >> wsh) * 4) + (uint32_t)((off & wmask) * KK * 4);
      float gn[KK][9];
      blk.gather(ctr, gn);
      const float x[4] = {av.x, av.y, av.z, av.w};
      float dy[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
      for (int k = 0; k < KK; ++k)
#pragma unroll
        for (int t = 0; t < 9; ++t) {
          float4 wv;
          if constexpr (L::WREG) wv = make_float4(wr[t][0], wr[t][1], wr[t][2], wr[t][3]);
          else wv = ld_shared_v4(wsm_a + (k * 9 + t) * (C * 4));
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
        const float dz = dy[j] * (pre > 0.f ? 1.f : neg);
        const float xh = (x[j] - mean[j]) * rstd[j];
        const float v = sc[j] * (dz - m1[j] - xh * m2[j]);
        o[j] = rtf ? round_tf32(v) : v;
      }
      da4[(int64_t)(o0 + lp) * C4] = make_float4(o[0], o[1], o[2], o[3]);
    }
    blk.template release<true>(p.a, i);
  }
}

static int ilog2_exact(int v) {
  int l = 0;
  while ((1 << l) < v) ++l;
  return (1 << l) == v ? l : -1;
}

template <int C4, int NB>
static int launch_tail_fprop(TailP &p, cudaStream_t st) {
  constexpr int per_sm = tail_fprop_blocks<C4, NB>();
  const int RT = 128 / p.W;
  const int smem = 1024 + (C4 / 8) * (16384 + NB * 128) + (RT + 2) * p.W * 9 * p.K * 4;
  static std::atomic<uint64_t> done{0};
  B2_CHECK_ARG(smem <= 227 * 1024, "tail_fprop: W=%d K=%d C=%d needs %d bytes of shared memory", p.W, p.K, p.C, smem);
  if (int e = ensure_dynamic_smem(tail_fprop_tc_kernel<C4, NB>, 227 * 1024, done)) return e;
  // one block per resident slot; a range's input rows (its rows + one halo row each side) fill whole tiles
  const int NH = p.N * p.H;
  const int share = ceil_div(NH, num_sms() * per_sm);
  p.rows_per_block = ceil_div(share + 2, RT) * RT - 2;
  tail_fprop_tc_kernel<C4, NB><<<(unsigned)ceil_div(NH, p.rows_per_block), TL_THREADS, smem, st>>>(p);
  B2_LAUNCH_CHECK();
  return B200GAN_OK;
}

template <int C4, int KK>
static int launch_tail_bwd(TailBwdP &p, cudaStream_t st) {
  using LR = TailBwdSmem<C4, KK, true>;
  using LA = TailBwdSmem<C4, KK, false>;
  constexpr int CHUNK = TailBwdBlock<C4, KK, true>::CHUNK;
  const int64_t total = (int64_t)p.N * p.H * p.W;
  const int per_sm = KK == 1 ? 2 : 1;
  const int budget = per_sm == 2 ? RB_SMEM_2CTA : RB_SMEM_1CTA;
  // rows a range of `per` pixels touches, and the slab rows they need (halo rows + one zero row per image start)
  auto tab_rows = [&](int64_t per) { return (int)(per / p.W + 2); };
  auto slab_rows = [&](int64_t per) { const int nq = tab_rows(per); return nq + 3 + (nq + 1) / p.H; };
  auto smem_of = [&](int64_t per) { return LR::bytes(tab_rows(per), slab_rows(per), p.W); };
  // contiguous pixel ranges, a whole number of ring chunks each, one block per resident slot -- or more, smaller ranges
  // when a slot's share of g would not fit in shared memory
  int64_t per = ceil_div64(ceil_div64(total, (int64_t)num_sms() * per_sm), CHUNK) * CHUNK;
  if (smem_of(per) > budget) {
    int64_t lo = CHUNK, hi = per;  // largest fitting multiple of CHUNK in [lo, hi)
    B2_CHECK_ARG(smem_of(lo) <= budget, "tail_bwd: W=%d K=%d C=%d does not fit in shared memory", p.W, p.K, p.C);
    while (hi - lo > CHUNK) {
      const int64_t mid = (lo + hi) / 2 / CHUNK * CHUNK;
      (smem_of(mid) <= budget ? lo : hi) = mid;
    }
    per = lo;
  }
  p.px_per_block = per;
  p.tab_rows = tab_rows(per);
  p.slab_rows = slab_rows(per);
  const int smem_reduce = smem_of(per);
  const int smem_apply = LA::bytes(p.tab_rows, p.slab_rows, p.W);
  static std::atomic<uint64_t> done_r{0}, done_a{0};
  if (int e = ensure_dynamic_smem(tail_bwd_reduce_kernel<C4, KK>, budget, done_r)) return e;
  if (int e = ensure_dynamic_smem(tail_bwd_apply_kernel<C4, KK>, budget, done_a)) return e;
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
  p.act_mid = d->act_mid; p.slope = d->slope; p.act_out = d->act_out; p.rows_per_block = 0;
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
  p.act_mid = d->act_mid; p.slope = d->slope; p.rtf = round_tf32;
  p.px_per_block = 0; p.tab_rows = p.slab_rows = 0;
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
