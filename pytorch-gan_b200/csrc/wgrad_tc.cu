// wgrad_tc.cu -- wgmma TF32 weight gradient of the stride-1 convolutions (sm_90a).
//
// dW[tap][k][c] = sum over output pixels o of  dy[o][k] * x[o + offset(tap)][c]
// (reference: autograd of nn.Conv2d, dcgan.py:168,182 -> cudnnConvolutionBackwardFilter).
//
// As a GEMM the contraction runs over PIXELS, so both operands arrive "MN-major": a TMA box {32 channels, BW, 1, BH,
// ipb} (32 pixels) lands in shared memory as 32 pixel rows x 128 B (128-byte swizzle).  wgmma takes TF32 operands from
// shared memory only K-major.  The operand with a multiple of 128 channels is A (M = 128: two warpgroups of 64 rows);
// it goes to wgmma as register fragments, loaded with 32-bit LDS straight from the TMA stage.  The other, B (N =
// 32..256), is transposed by the consumer warpgroups into a K-major 128B-swizzled tile (channel rows of 32 pixels;
// double-buffered, so that stage i+1 is prepared while the MMAs of stage i run).  Inside every 8-pixel k slice both
// operands take the pixels in the order 0 2 4 6 1 3 5 7 (wg_kpos), which makes the fragment loads free of bank
// conflicts.  Zero padding = TMA out-of-bounds fill on the shifted x box.  The upsample-folded convolution
// (dcgan.py:54-55,58-59) contributes 16 (phase, tap) jobs that read dy through the phase view {2K, Q/2, 2, P/2, N}; a
// second kernel folds them back into the 3x3 filter.
//
// Parallelisation: grid = (pixel splits, jobs, M-tiles x N-tiles).  Every CTA accumulates its pixel range in
// registers, stages the tile in shared memory and adds it into the job's [M'][N'] matrix with a TMA reduce-store
// (cp.reduce.async.bulk.tensor ... .add: the fp32 additions happen at L2); wgrad_reduce_kernel then folds the
// jobs into the parameter layout [K][C][R][S].
#include "tc_common.cuh"
#include <stdlib.h>

namespace b200gan {

constexpr int WG_THREADS = 384;  // producer warpgroup + two consumer warpgroups
constexpr int WG_MAX_JOBS = 52;
constexpr int WG_PIX = 32;       // pixels (GEMM-K) per pipeline stage
constexpr int WG_CHUNK_BYTES = WG_PIX * 128;  // one 32-channel chunk of one stage

// One job = one filter tap (or one (phase, tap) pair of the upsample fold).  "S" is the operand that is shifted by
// the tap (x for Conv2d, dy for ConvTranspose2d), "D" the one that is read at the loop pixel.
struct WgJob {
  int16_t s_dc, d_dc;  // channel base in the parity / phase view
  int8_t s_da, d_da;   // row-parity coordinate in the view
  int8_t s_dw, s_dh;   // shift of S in (view) pixels
};

struct WgParams {
  WgJob jobs[WG_MAX_JOBS];
  int32_t njobs;
  int32_t bw_log2, bh_log2;       // 32-pixel box = BW x BH
  int32_t tiles_w, tiles_h, N;    // pixel tiles per image
  int32_t imgs_per_box;           // 32 / (BW * BH)
  int32_t tiles_total, tiles_per_split;
  int32_t s_is_a;                 // 1: A = shifted operand S, B = D; 0: A = D, B = S
  int32_t mtiles, ntiles;         // tiles of the (M', N') output
  int32_t ldn;                    // N' total (row length of a partial matrix)
  int32_t mtotal;                 // M' total
  float *partial;                 // [job][M'][N'], zeroed by the host; splits accumulate with TMA reduce-add
};

// shared memory: TMA ring | two K-major B buffers; after the last MMA the front is the staging tile
template <int NB, int STAGES>
struct WgSmem {
  static constexpr int A_BYTES = 4 * WG_CHUNK_BYTES;            // 128 channels
  static constexpr int B_BYTES = (NB / 32) * WG_CHUNK_BYTES;
  static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  static constexpr int RING = STAGES * STAGE_BYTES;
  static constexpr int T_BYTES = NB * 128;                      // B^T: NB channel rows of 32 pixels
  static constexpr int STAGING = (NB / 32) * 16384;
  static constexpr int MAIN = RING + 2 * T_BYTES > STAGING ? RING + 2 * T_BYTES : STAGING;
  static constexpr int TOTAL = MAIN + 1024 + 256;
  static_assert(TOTAL <= 232448, "wgrad_tc_kernel: shared memory");
};

__device__ __forceinline__ void wg_consumers_sync() { asm volatile("bar.sync 1, 256;" ::: "memory"); }

// K position of pixel row p of a stage: inside each 8-pixel k slice, even pixels take positions 0..3 and odd ones 4..7.
// Thread (l%4) of an A fragment then reads pixels 2(l%4) and 2(l%4) + 1, whose rows have distinct 128-byte swizzle
// phases for the four values of l%4: the 32 lanes of one fragment load hit 32 different banks.
__device__ __forceinline__ int wg_kpos(int p) { return (p & ~7) | ((p & 7) >> 1) | ((p & 1) << 2); }

template <int NB, int STAGES>
__global__ void __launch_bounds__(WG_THREADS, 1)
wgrad_tc_kernel(const __grid_constant__ CUtensorMap tmX, const __grid_constant__ CUtensorMap tmY,
                const __grid_constant__ CUtensorMap tmP, const __grid_constant__ WgParams p) {
  using L = WgSmem<NB, STAGES>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t *smem = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint64_t *full = reinterpret_cast<uint64_t *>(smem + L::MAIN);
  uint64_t *empty = full + STAGES;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int split = blockIdx.x, job = blockIdx.y;
  const int mt = blockIdx.z / p.ntiles, nt = blockIdx.z % p.ntiles;
  const int t_begin = split * p.tiles_per_split;
  int t_end = t_begin + p.tiles_per_split;
  if (t_end > p.tiles_total) t_end = p.tiles_total;
  const int iters = t_end - t_begin;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmX);
    tma_prefetch_desc(&tmY);
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], 256);  // every consumer thread, once its fragment and transpose reads of the stage are done
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp < 4) {
    setmaxnreg_dec<40>();
    if (warp == 0 && lane == 0) {
      const WgJob jb = p.jobs[job];
      const CUtensorMap *mapA = p.s_is_a ? &tmX : &tmY;   // tmX = shifted operand S, tmY = dense operand D
      const CUtensorMap *mapB = p.s_is_a ? &tmY : &tmX;
      const int a_dc = p.s_is_a ? jb.s_dc : jb.d_dc, a_da = p.s_is_a ? jb.s_da : jb.d_da;
      const int a_dw = p.s_is_a ? jb.s_dw : 0, a_dh = p.s_is_a ? jb.s_dh : 0;
      const int b_dc = p.s_is_a ? jb.d_dc : jb.s_dc, b_da = p.s_is_a ? jb.d_da : jb.s_da;
      const int b_dw = p.s_is_a ? 0 : jb.s_dw, b_dh = p.s_is_a ? 0 : jb.s_dh;
      int stage = 0;
      uint32_t phase = 0;
      for (int it = 0; it < iters; ++it) {
        int t = t_begin + it;
        const int tw = t % p.tiles_w;
        t /= p.tiles_w;
        const int th = t % p.tiles_h;
        const int n = (t / p.tiles_h) * p.imgs_per_box;  // a box spans several images when H*W < WG_PIX
        const int w0 = tw << p.bw_log2, h0 = th << p.bh_log2;
        mbar_wait(&empty[stage], phase ^ 1);
        uint8_t *sa = smem + stage * L::STAGE_BYTES;
        uint8_t *sb = sa + L::A_BYTES;
        mbar_arrive_expect_tx(&full[stage], L::STAGE_BYTES);
#pragma unroll
        for (int c = 0; c < 4; ++c)
          tma_load_5d(sa + c * WG_CHUNK_BYTES, mapA, &full[stage], a_dc + (mt * 4 + c) * 32, w0 + a_dw, a_da,
                      h0 + a_dh, n);
#pragma unroll
        for (int c = 0; c < NB / 32; ++c)
          tma_load_5d(sb + c * WG_CHUNK_BYTES, mapB, &full[stage], b_dc + (nt * (NB / 32) + c) * 32, w0 + b_dw, b_da,
                      h0 + b_dh, n);
        if (++stage == STAGES) {
          stage = 0;
          phase ^= 1;
        }
      }
    }
  } else {
    setmaxnreg_inc<232>();  // 128 x 40 + 256 x 232 registers = the 384 x 168 the kernel starts with
    if (iters == 0) return;
    const int ct = threadIdx.x - 128;
    const int half = ct >> 7;           // MMA rows [64 * half, +64) of the 128 x NB tile
    const int tp = ct & 31, tq = ct >> 5;  // B transpose: pixel row tp, 16-byte column tq (4 channels) of every chunk
    const int tk = wg_kpos(tp);
    // A fragments (wgmma_tf32_rs): warp wq of this warpgroup holds channels 64 * half + 16 * wq + [0, 16), i.e.
    // channels ac, ac + 8 of 32-channel chunk 2 * half + wq / 2; its k slice j reads pixels 8j + 2(l%4) (+1)
    const int wq = tq & 3;
    const int ac = 16 * (wq & 1) + (lane >> 2), ap = 2 * (lane & 3);
    const int abase = (2 * half + (wq >> 1)) * WG_CHUNK_BYTES + ap * 128 + (ac & 3) * 4;
    const uint32_t aoff[4] = {
        (uint32_t)(abase + ((((ac >> 2)) ^ ap) << 4)),                  // a0: channel ac,     pixel ap
        (uint32_t)(abase + ((((ac >> 2) + 2) ^ ap) << 4)),              // a1: channel ac + 8, pixel ap
        (uint32_t)(abase + 128 + ((((ac >> 2)) ^ (ap + 1)) << 4)),      // a2: channel ac,     pixel ap + 1
        (uint32_t)(abase + 128 + ((((ac >> 2) + 2) ^ (ap + 1)) << 4))}; // a3: channel ac + 8, pixel ap + 1
    float acc[NB / 2];                  // the first MMA overwrites it (scale_d = 0)
    int stage = 0;
    uint32_t phase = 0;
    // stage `it` -> A fragments fa and the K-major B tile of buffer it & 1; the ring slot is released afterwards
    auto prepare = [&](int it, uint32_t(&fa)[16]) {
      uint8_t *tb = smem + L::RING + (it & 1) * L::T_BYTES;  // B^T: NB rows x 128 B
      mbar_wait(&full[stage], phase);
      wg_consumers_sync();  // both warpgroups' MMAs of iteration it-2 (which read this buffer) have retired
      const uint8_t *src = smem + stage * L::STAGE_BYTES;
#pragma unroll
      for (int k = 0; k < WG_PIX / 8; ++k)
#pragma unroll
        for (int j = 0; j < 4; ++j) fa[4 * k + j] = *reinterpret_cast<const uint32_t *>(src + aoff[j] + k * 1024);
#pragma unroll
      for (int c = 0; c < NB / 32; ++c) {
        const float4 v = *reinterpret_cast<const float4 *>(src + L::A_BYTES + c * WG_CHUNK_BYTES + tp * 128 +
                                                           ((tq ^ (tp & 7)) << 4));
        const float e[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const int r = c * 32 + tq * 4 + i;
          *reinterpret_cast<float *>(tb + r * 128 + (((tk >> 2) ^ (r & 7)) << 4) + (tk & 3) * 4) = e[i];
        }
      }
      mbar_arrive(&empty[stage]);
      fence_proxy_async();  // generic-proxy smem writes -> visible to wgmma
      wg_consumers_sync();
      if (++stage == STAGES) {
        stage = 0;
        phase ^= 1;
      }
    };
    auto mma = [&](int it, const uint32_t(&fa)[16]) {
      const uint32_t sb = smem_u32(smem + L::RING + (it & 1) * L::T_BYTES);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < WG_PIX / 8; ++k)
        wgmma_tf32_rs<NB>(acc, fa + 4 * k, gmma_desc_sw128(sb + k * 32), (it > 0 || k > 0) ? 1u : 0u);
      wgmma_commit();
    };
    // the MMAs of stage i run while stage i+1 is prepared into the other fragment set and B buffer; a wgmma's
    // register operands are all defined before it is issued, so ptxas keeps the wgmma pipeline asynchronous
    uint32_t fa0[16], fa1[16];
    prepare(0, fa0);
#pragma unroll 1
    for (int it = 0; it < iters; it += 2) {
      mma(it, fa0);
      if (it + 1 < iters) prepare(it + 1, fa1);
      wgmma_wait<0>();
      if (it + 1 < iters) {
        mma(it + 1, fa1);
        if (it + 2 < iters) prepare(it + 2, fa0);
        wgmma_wait<0>();
      }
    }
    wgmma_wait<0>();
    wgmma_fence_regs<NB / 2>(acc);
    wg_consumers_sync();  // every MMA has retired: ring and operand buffers are free for the staging tile
    // registers -> 128B-swizzled staging tile -> TMA reduce-add of the partial tile into partial[job][m'][n']
    store_acc_sw128<NB>(smem, acc, half * 64);
    fence_proxy_async();
    wg_consumers_sync();
    if (ct == 0) {
      // all pixel splits of a job accumulate into the same [job][M'][N'] tile: TMA reduce-add (fp32 add at L2)
      const int row0 = job * p.mtotal + mt * 128;
#pragma unroll 1
      for (int c = 0; c < NB; c += 32) tma_reduce_add_2d(&tmP, smem + (c >> 5) * 16384, nt * NB + c, row0);
      tma_store_commit_and_wait_read();
    }
  }
}

// dw = fold of partial[job][m'][n'] into the parameter layout (Conv2d [K][C][R][S], ConvTranspose2d [C][K][R][S]).
struct WgReduceP {
  int32_t K, C, R, S, njobs, s_is_a, up2, transposed;
  int32_t mtotal, ldn;
};
__device__ __forceinline__ bool up2_contrib(int r, int a, int d) {
  // r in Rset(a,d): Rset(0,0)={0} Rset(0,1)={1,2} Rset(1,0)={0,1} Rset(1,1)={2}
  if (a == 0) return d == 0 ? r == 0 : r >= 1;
  return d == 0 ? r <= 1 : r == 2;
}
__global__ void wgrad_reduce_kernel(const float *__restrict__ partial, float *__restrict__ dw, WgReduceP p) {
  int64_t total = (int64_t)p.K * p.C * p.R * p.S;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (int64_t)gridDim.x * blockDim.x) {
    // c fastest so that reads of partial[..][k][c] (or [c][k]) stay reasonably coalesced
    int c = (int)(i % p.C);
    int64_t t = i / p.C;
    int k = (int)(t % p.K);
    t /= p.K;
    int s = (int)(t % p.S), r = (int)(t / p.S);
    const int sch = p.transposed ? k : c;   // channel index inside the shifted operand S
    const int dch = p.transposed ? c : k;   // channel index inside the dense operand D
    int64_t elem = p.s_is_a ? (int64_t)sch * p.ldn + dch : (int64_t)dch * p.ldn + sch;
    int64_t job_stride = (int64_t)p.mtotal * p.ldn;
    const float *base = partial + elem;
    float acc = 0.f;
    if (!p.up2) {
      acc = __ldg(base + (int64_t)(r * p.S + s) * job_stride);
    } else {
      for (int j = 0; j < 16; ++j) {
        int ph = j >> 2, tp = j & 3;
        if (up2_contrib(r, ph >> 1, tp >> 1) && up2_contrib(s, ph & 1, tp & 1)) acc += __ldg(base + j * job_stride);
      }
    }
    const int64_t o = p.transposed ? (((int64_t)c * p.K + k) * p.R + r) * p.S + s
                                   : (((int64_t)k * p.C + c) * p.R + r) * p.S + s;
    dw[o] = acc;
  }
}


// Tile version: the partial matrices are contiguous along one channel dimension ("col"), the parameter layout along the
// taps and then the OTHER or the same channel dimension -- element-wise, consecutive threads wrote 4 bytes every R*S*4
// bytes (28 us per U-Net layer, 0.57 ms per Pix2Pix step).  A block moves a 32 (col) x 8 (row) x taps tile through shared
// memory: 128-byte reads per (row, tap), contiguous runs of 8*R*S or 32*R*S floats out.
constexpr int WR_COL = 32, WR_ROW = 8, WR_TAPS = 16;
__global__ void __launch_bounds__(256)
wgrad_reduce_tile_kernel(const float *__restrict__ partial, float *__restrict__ dw, WgReduceP p) {
  __shared__ float s[WR_ROW][WR_COL][WR_TAPS + 1];
  const int RS = p.R * p.S;
  const int tin = p.up2 ? 16 : RS;                       // partial matrices (jobs) per weight
  // partial[job][row][col]: (row, col) = (sch, dch) if s_is_a else (dch, sch); sch = transposed ? k : c, dch = transposed ? c : k
  const bool col_is_k = (p.s_is_a != 0) != (p.transposed != 0);   // s_is_a: col = dch = (transposed ? c : k)
  const int ncol = col_is_k ? p.K : p.C, nrow = col_is_k ? p.C : p.K;
  const int tiles_col = (ncol + WR_COL - 1) / WR_COL;
  const int col0 = (blockIdx.x % tiles_col) * WR_COL, row0 = (blockIdx.x / tiles_col) * WR_ROW;
  const int64_t job_stride = (int64_t)p.mtotal * p.ldn;
  const int tid = threadIdx.x;
  for (int e = tid; e < WR_COL * WR_ROW * tin; e += 256) {
    const int cl = e % WR_COL, rw = (e / WR_COL) % WR_ROW, j = e / (WR_COL * WR_ROW);
    float v = 0.f;
    if (col0 + cl < ncol && row0 + rw < nrow) v = __ldg(partial + j * job_stride + (int64_t)(row0 + rw) * p.ldn + col0 + cl);
    s[rw][cl][j] = v;
  }
  __syncthreads();
  // dw[(A * NB + B) * RS + t]: (A, B) = (k, c) for Conv2d, (c, k) for ConvTranspose2d
  const bool col_is_b = col_is_k == (p.transposed != 0);          // inner output dimension B = transposed ? k : c
  const int nb = p.transposed ? p.K : p.C;
  for (int e = tid; e < WR_COL * WR_ROW * RS; e += 256) {
    const int t = e % RS;
    int cl, rw;
    if (col_is_b) { cl = (e / RS) % WR_COL; rw = e / (RS * WR_COL); }   // runs of 32 * RS floats
    else          { rw = (e / RS) % WR_ROW; cl = e / (RS * WR_ROW); }   // runs of 8 * RS floats
    const int col = col0 + cl, row = row0 + rw;
    if (col >= ncol || row >= nrow) continue;
    float acc;
    if (!p.up2) {
      acc = s[rw][cl][t];
    } else {
      const int r = t / 3, q = t % 3;
      acc = 0.f;
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        const int ph = j >> 2, tp = j & 3;
        if (up2_contrib(r, ph >> 1, tp >> 1) && up2_contrib(q, ph & 1, tp & 1)) acc += s[rw][cl][j];
      }
    }
    const int a = col_is_b ? row : col, b = col_is_b ? col : row;
    dw[((int64_t)a * nb + b) * RS + t] = acc;
  }
}

// ---- host -------------------------------------------------------------------------------------------
static int ilog2c(int v) {
  int l = 0;
  while ((1 << l) < v) ++l;
  return l;
}

struct WgPlan {
  int s_is_a, NB, mtiles, ntiles, mtotal, ldn, njobs, bwl, bhl, tiles_w, tiles_h, tiles_total, nsplits, tps, Ho, Wo;
  int sch, dch;  // channels of the shifted / dense operand
  int ipb;
};

static bool wg_plan(const b200gan_conv_geom *g, WgPlan &pl) {
  if (g->pad_mode != B200GAN_PAD_ZERO || g->N < 1) return false;
  if (g->stride != 1 && g->stride != 2) return false;
  if (g->C % 32 || g->K % 32 || 2 * g->C > 32767 || 2 * g->K > 32767) return false;
  const bool up2 = g->up == 2;
  if (up2 && (g->transposed || g->stride != 1 ||
              !(g->R == 3 && g->S == 3 && g->pad_t == 1 && g->pad_l == 1 && g->pad_b == 1 && g->pad_r == 1)))
    return false;
  if (g->R * g->S > WG_MAX_JOBS || g->R > 15 || g->S > 15 || g->pad_t > 15 || g->pad_l > 15) return false;
  // shifted operand S (x / dy for ConvTranspose2d) and dense operand D
  pl.sch = g->transposed ? g->K : g->C;
  pl.dch = g->transposed ? g->C : g->K;
  if (g->stride == 2) {
    const int Hf = g->transposed ? g->P : g->H, Wf = g->transposed ? g->Q : g->W;  // S is the full-resolution side
    if ((Hf & 1) || (Wf & 1)) return false;
  }
  // A = the operand with a multiple of 128 channels; B = the other (multiple of 32)
  if (pl.dch % 128 == 0) pl.s_is_a = 0;
  else if (pl.sch % 128 == 0) pl.s_is_a = 1;
  else return false;
  const int mch = pl.s_is_a ? pl.sch : pl.dch, nch = pl.s_is_a ? pl.dch : pl.sch;
  pl.NB = nch % 128 == 0 ? 128 : (nch % 64 == 0 ? 64 : 32);
  // 128 x 256 output tiles: the 128-channel operand is re-read and re-transposed half as often (a 256 -> 256 3x3 layer
  // pulls 9 jobs x 4 tiles x 33 MB = 1.2 GB through L2 with 128 x 128 tiles)
  if (nch % 256 == 0) pl.NB = 256;
  pl.mtotal = mch;
  pl.ldn = nch;
  pl.mtiles = mch / 128;
  pl.ntiles = nch / pl.NB;
  pl.njobs = up2 ? 16 : g->R * g->S;
  // pixel grid the contraction runs over = grid of the dense operand (low-res grid for the upsample fold)
  pl.Ho = up2 ? g->H : (g->transposed ? g->H : g->P);
  pl.Wo = up2 ? g->W : (g->transposed ? g->W : g->Q);
  const int pl2 = 5;  // log2(WG_PIX)
  pl.bwl = ilog2c(pl.Wo);
  if (pl.bwl > pl2) pl.bwl = pl2;
  pl.bhl = ilog2c(pl.Ho);
  if (pl.bhl > pl2 - pl.bwl) pl.bhl = pl2 - pl.bwl;
  pl.tiles_w = ceil_div(pl.Wo, 1 << pl.bwl);
  pl.tiles_h = ceil_div(pl.Ho, 1 << pl.bhl);
  pl.ipb = WG_PIX >> (pl.bwl + pl.bhl);  // images per box (>1 only when the whole map has fewer pixels than a stage)
  int64_t tt = (int64_t)ceil_div(g->N, pl.ipb) * pl.tiles_w * pl.tiles_h;
  if (tt > (1 << 30)) return false;
  pl.tiles_total = (int)tt;
  // pixel splits: one CTA per SM fits (shared memory), so the kernel takes waves x (stages per CTA + fill and epilogue,
  // about 8 stages).  Pick the split count with the least of that; a last wave that is nearly empty costs as much as a
  // full one (16 jobs x 17 splits on 132 SMs ran 3 waves where 16 x 8 runs one of twice the length).
  const int64_t ctas_per_split = (int64_t)pl.njobs * pl.mtiles * pl.ntiles;
  int max_ns = pl.tiles_total / 8;
  if (max_ns < 1) max_ns = 1;
  if (max_ns > 4 * num_sms()) max_ns = 4 * num_sms();
  int ns = 1;
  int64_t best = -1;
  for (int s = 1; s <= max_ns; ++s) {
    const int64_t waves = ceil_div64(s * ctas_per_split, num_sms());
    const int64_t cost = waves * (ceil_div(pl.tiles_total, s) + 8);
    if (best < 0 || cost < best) {
      best = cost;
      ns = s;
    }
  }
  pl.tps = ceil_div(pl.tiles_total, ns);
  pl.nsplits = ceil_div(pl.tiles_total, pl.tps);
  return true;
}

int tc_wgrad_supported(const b200gan_conv_geom *g) {
  WgPlan pl;
  return wg_plan(g, pl) ? 1 : 0;
}

size_t tc_wgrad_workspace_floats(const b200gan_conv_geom *g) {
  WgPlan pl;
  if (!wg_plan(g, pl)) return 0;
  return (size_t)pl.njobs * pl.mtotal * pl.ldn;
}

template <int NB, int STAGES>
static int launch_wg(const CUtensorMap &tmX, const CUtensorMap &tmY, const CUtensorMap &tmP, const WgParams &p, dim3 grid,
                     cudaStream_t st) {
  constexpr int SMEM = WgSmem<NB, STAGES>::TOTAL;
  static std::atomic<uint64_t> attr_done{0};
  if (int e = ensure_dynamic_smem(wgrad_tc_kernel<NB, STAGES>, SMEM, attr_done)) return e;
  wgrad_tc_kernel<NB, STAGES><<<grid, WG_THREADS, SMEM, st>>>(tmX, tmY, tmP, p);
  B2_LAUNCH_CHECK();
  return B200GAN_OK;
}

int tc_wgrad(const b200gan_conv_geom *g, const float *x, const float *dy, float *dw, float *ws, cudaStream_t st) {
  WgPlan pl;
  if (!wg_plan(g, pl)) B2_UNSUPPORTED("tensor-core wgrad: geometry not supported");
  B2_CHECK_ARG(ws != nullptr, "tensor-core wgrad: workspace required");
  B2_CHECK_ARG(((uintptr_t)x % 16 == 0) && ((uintptr_t)dy % 16 == 0) && ((uintptr_t)ws % 16 == 0),
               "tensor-core wgrad: pointers must be 16-byte aligned");
  const bool up2 = g->up == 2;
  const int st2 = g->stride == 2;
  WgParams p;
  memset(&p, 0, sizeof(p));
  p.njobs = pl.njobs;
  if (up2) {
    // S = x (plain, shifted), D = dy through the phase view {2K, Q/2, 2, P/2, N}
    for (int ph = 0; ph < 4; ++ph)
      for (int tp = 0; tp < 4; ++tp) {
        int a = ph >> 1, b = ph & 1, dr = tp >> 1, ds = tp & 1;
        WgJob &j = p.jobs[ph * 4 + tp];
        j.d_dc = (int16_t)(b * g->K); j.d_da = (int8_t)a; j.s_dh = (int8_t)(a - 1 + dr); j.s_dw = (int8_t)(b - 1 + ds);
      }
  } else {
    for (int r = 0; r < g->R; ++r)
      for (int s2 = 0; s2 < g->S; ++s2) {
        WgJob &j = p.jobs[r * g->S + s2];
        const int eh = r - g->pad_t, ew = s2 - g->pad_l;
        if (!st2) {
          j.s_dh = (int8_t)eh; j.s_dw = (int8_t)ew;
        } else {  // S[2p + e] through the parity view {2Cs, Wf/2, 2, Hf/2, N}
          j.s_dh = (int8_t)(eh >= 0 ? eh / 2 : -((-eh + 1) / 2)); j.s_da = (int8_t)(eh & 1);
          j.s_dw = (int8_t)(ew >= 0 ? ew / 2 : -((-ew + 1) / 2)); j.s_dc = (int16_t)((ew & 1) * pl.sch);
        }
      }
  }
  p.bw_log2 = pl.bwl; p.bh_log2 = pl.bhl;
  p.tiles_w = pl.tiles_w; p.tiles_h = pl.tiles_h; p.N = g->N; p.imgs_per_box = pl.ipb;
  p.tiles_total = pl.tiles_total; p.tiles_per_split = pl.tps;
  p.s_is_a = pl.s_is_a; p.mtiles = pl.mtiles; p.ntiles = pl.ntiles; p.ldn = pl.ldn; p.mtotal = pl.mtotal;
  p.partial = ws;

  // operand tensors: Conv2d: S = x [N][H][W][C], D = dy [N][P][Q][K]; ConvTranspose2d: S = dy, D = x
  const float *sptr = g->transposed ? dy : x, *dptr = g->transposed ? x : dy;
  const uint64_t Hs = g->transposed ? g->P : g->H, Ws = g->transposed ? g->Q : g->W, Cs = pl.sch;
  const uint64_t Hd = g->transposed ? g->H : g->P, Wd = g->transposed ? g->W : g->Q, Cd = pl.dch;
  CUtensorMap tmX, tmY;
  const uint32_t box[5] = {32, (uint32_t)(1 << pl.bwl), 1, (uint32_t)(1 << pl.bhl), (uint32_t)pl.ipb};
  {
    uint64_t dims[5], strides[4];
    if (!st2) {
      dims[0] = Cs; dims[1] = Ws; dims[2] = 1; dims[3] = Hs; dims[4] = g->N;
      strides[0] = Cs * 4; strides[1] = Ws * Cs * 4; strides[2] = Ws * Cs * 4; strides[3] = Hs * Ws * Cs * 4;
    } else {
      dims[0] = 2 * Cs; dims[1] = Ws / 2; dims[2] = 2; dims[3] = Hs / 2; dims[4] = g->N;
      strides[0] = 2 * Cs * 4; strides[1] = Ws * Cs * 4; strides[2] = 2 * Ws * Cs * 4; strides[3] = Hs * Ws * Cs * 4;
    }
    if (int e = make_tmap_f32(&tmX, sptr, 5, dims, strides, box)) return e;
  }
  {
    uint64_t dims[5], strides[4];
    if (!up2) {
      dims[0] = Cd; dims[1] = Wd; dims[2] = 1; dims[3] = Hd; dims[4] = g->N;
      strides[0] = Cd * 4; strides[1] = Wd * Cd * 4; strides[2] = Wd * Cd * 4; strides[3] = Hd * Wd * Cd * 4;
    } else {
      dims[0] = 2 * Cd; dims[1] = Wd / 2; dims[2] = 2; dims[3] = Hd / 2; dims[4] = g->N;
      strides[0] = 2 * Cd * 4; strides[1] = Wd * Cd * 4; strides[2] = 2 * Wd * Cd * 4; strides[3] = Hd * Wd * Cd * 4;
    }
    if (int e = make_tmap_f32(&tmY, dptr, 5, dims, strides, box)) return e;
  }
  CUtensorMap tmP;
  {
    uint64_t dims[2] = {(uint64_t)pl.ldn, (uint64_t)pl.njobs * pl.mtotal};
    uint64_t strides[1] = {(uint64_t)pl.ldn * 4};
    uint32_t pbox[2] = {32, 128};
    if (int e = make_tmap_f32(&tmP, ws, 2, dims, strides, pbox)) return e;
  }
  B2_CUDA(cudaMemsetAsync(ws, 0, (size_t)pl.njobs * pl.mtotal * pl.ldn * sizeof(float), st));
  dim3 grid((unsigned)pl.nsplits, (unsigned)pl.njobs, (unsigned)(pl.mtiles * pl.ntiles));
  int rc = pl.NB == 256 ? launch_wg<256, 3>(tmX, tmY, tmP, p, grid, st)
           : pl.NB == 128 ? launch_wg<128, 6>(tmX, tmY, tmP, p, grid, st)
           : pl.NB == 64 ? launch_wg<64, 8>(tmX, tmY, tmP, p, grid, st)
                         : launch_wg<32, 8>(tmX, tmY, tmP, p, grid, st);
  if (rc) return rc;
  WgReduceP rp;
  rp.K = g->K; rp.C = g->C; rp.R = g->R; rp.S = g->S; rp.njobs = pl.njobs;
  rp.s_is_a = pl.s_is_a; rp.up2 = up2 ? 1 : 0; rp.transposed = g->transposed ? 1 : 0; rp.mtotal = pl.mtotal; rp.ldn = pl.ldn;
  int64_t total = (int64_t)g->K * g->C * g->R * g->S;
  if (g->R * g->S <= WR_TAPS && g->K >= 32 && g->C >= 32) {
    const bool col_is_k = (pl.s_is_a != 0) != (g->transposed != 0);
    const int ncol = col_is_k ? g->K : g->C, nrow = col_is_k ? g->C : g->K;
    const unsigned tiles = (unsigned)(ceil_div(ncol, WR_COL) * ceil_div(nrow, WR_ROW));
    wgrad_reduce_tile_kernel<<<tiles, 256, 0, st>>>(ws, dw, rp);
    B2_LAUNCH_CHECK();
    return B200GAN_OK;
  }
  unsigned blocks = (unsigned)(ceil_div64(total, 256) > num_sms() * 16 ? num_sms() * 16 : ceil_div64(total, 256));
  wgrad_reduce_kernel<<<blocks, 256, 0, st>>>(ws, dw, rp);
  B2_LAUNCH_CHECK();
  return B200GAN_OK;
}

}  // namespace b200gan
