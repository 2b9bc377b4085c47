// conv_tc.cu -- wgmma TF32 implicit-GEMM convolution (fprop and dgrad) for sm_90a.
//
// Hot path of the reference: the big Generator convolutions
//   Upsample(x2) -> Conv2d(128,128,3,1,1)   dcgan.py:54-55
//   Upsample(x2) -> Conv2d(128, 64,3,1,1)   dcgan.py:58-59
// and every other stride-1 convolution with >= 32 input channels (cyclegan/models.py:28,32,75).
//
// Formulation.  y[m][k] = sum_taps sum_c A_tap[m][c] * B_tap[k][c], m = output pixel, accumulated in registers by
// wgmma (TF32, M = 64 per warpgroup, N = BN).  No im2col buffer ever exists: the A tile of a tap is a rank-5 TMA box
// {32 channels, BW, 1, BH, BNn} of the NHWC activation tensor shifted by the tap offset; TMA zero-fills out-of-bounds
// coordinates, which *is* the zero padding.  The box lands in shared memory as 128 rows x 128 B with the 128-byte
// swizzle -- exactly the K-major wgmma operand layout.  B tiles come from the packed weight matrix [tap][Cout][Cin]
// (tf32-rounded at pack time).
//
// A nearest x2 upsample in front of a 3x3 conv is folded into four 2x2 "phase" convolutions on the
// low-resolution input (B200GAN_PACK_TC_*_UP2): the 4x larger upsampled tensor is never written and
// 2.25x fewer MACs are executed.  The data gradient of that composite runs through the same kernel:
// 16 taps over a rank-5 phase view {2K, Q/2, 2, P/2, N} of dy.
//
// Warp roles (384 threads): warpgroup 0 = TMA producer (one thread), warpgroups 1-2 = consumers, each issuing the
// wgmma of one 64-pixel half of the 128-pixel tile.  smem ring of STAGES x (A 16 KB + B BN*128 B), full/empty
// mbarriers.  Epilogue: the consumers write their accumulators into the 128B-swizzled staging tile (the idle pipeline
// buffers), then each thread takes one pixel row of a 32-channel chunk (bias / activation / Dropout2d scale /
// BatchNorm partial sums) and one thread issues the TMA bulk tensor stores.
#include "tc_common.cuh"
#include <mutex>
#include <stdlib.h>

namespace b200gan {

// ---- tensor map encoder ----------------------------------------------------------------------
PFN_encodeTiled get_encode_tiled() {
  static PFN_encodeTiled fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void *p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPointByVersion("cuTensorMapEncodeTiled", &p, 12000, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<PFN_encodeTiled>(p);
  });
  return fn;
}

int make_tmap_f32(CUtensorMap *map, const void *base, int rank, const uint64_t *dims, const uint64_t *strides_bytes,
                  const uint32_t *box) {
  PFN_encodeTiled enc = get_encode_tiled();
  if (!enc) {
    set_error("cuTensorMapEncodeTiled entry point not available");
    return B200GAN_E_CUDA;
  }
  cuuint64_t gd[5], gs[4];
  cuuint32_t bx[5], es[5];
  for (int i = 0; i < rank; ++i) {
    gd[i] = dims[i];
    bx[i] = box[i];
    es[i] = 1;
  }
  for (int i = 0; i < rank - 1; ++i) gs[i] = strides_bytes[i];
  CUresult r = enc(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, (cuuint32_t)rank, const_cast<void *>(base), gd, gs, bx, es,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                   CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled failed (%d): rank %d dims [%llu %llu %llu %llu %llu] box [%u %u %u %u %u]", (int)r,
              rank, (unsigned long long)gd[0], (unsigned long long)(rank > 1 ? gd[1] : 0),
              (unsigned long long)(rank > 2 ? gd[2] : 0), (unsigned long long)(rank > 3 ? gd[3] : 0),
              (unsigned long long)(rank > 4 ? gd[4] : 0), bx[0], rank > 1 ? bx[1] : 0, rank > 2 ? bx[2] : 0,
              rank > 3 ? bx[3] : 0, rank > 4 ? bx[4] : 0);
    return B200GAN_E_CUDA;
  }
  return B200GAN_OK;
}

// ---- kernel ------------------------------------------------------------------------------------
constexpr int TC_BM = 128;
constexpr int TC_BK = 32;  // fp32 elements = 128 bytes = one swizzle row
constexpr int TC_A_BYTES = TC_BM * TC_BK * 4;
constexpr int TC_MAX_TAPS = 52;
constexpr int TC_THREADS = 384;  // producer warpgroup + two consumer warpgroups

struct TcTap {
  int16_t dc;  // channel base offset in the A view (selects the w-parity half of a phase view)
  int8_t dw, da, dh;
  int8_t bt;   // row block of this tap in the packed weight matrix (B rows = bt * Kout + ...)
  int8_t pad_[2];
};

struct TcParams {
  int32_t tap_begin[5];  // taps of phase z: [tap_begin[z], tap_begin[z+1])
  TcTap taps[TC_MAX_TAPS];
  int32_t kout_total;  // rows of the packed B matrix per tap
  int32_t kchunks;     // contraction channels / 32
  int32_t bw_log2, bh_log2;  // box width / height (powers of two), BW*BH*BNn = 128
  int32_t tiles_w, tiles_h;
  int32_t N, Ho, Wo;         // logical output grid of one phase
  int32_t out_dc[4], out_da[4];  // per phase: channel base / phase-row coordinate in the output tensor map
  int32_t ldk;               // channels of the output tensor (row length)
  const float *bias;
  const float *chan_scale;
  double *stats;
  int32_t stats_groups;  // G: ldk (BatchNorm) or N*ldk (InstanceNorm: per-sample groups, tile = one image)
  int32_t stats_per_sample;
  int32_t act;
  float slope;
  int32_t rtf;
  float *y;
  int32_t narrow_k;  // 0, or the real number of output channels (< 32) of a layer whose B rows are zero-padded to 32 by
                     // TMA out-of-bounds fill (cyclegan/models.py:82, Conv2d(64, 3, 7)): direct stores, no TMA store
  int32_t ksplit;    // > 1: the (tap, k-chunk) loop is split over `ksplit` CTAs; raw partial tiles are added into a zeroed
                     // output with TMA reduce-stores (layers with few output pixels: pix2pix/models.py:62-73 at 1x1..8x8)
  long long *trace;  // bring-up: per-CTA clock64 timeline (64 slots per CTA) or nullptr
};

#define TC_TRACE(slot)                                                   \
  do {                                                                   \
    if (p.trace) p.trace[((size_t)blockIdx.z * gridDim.x + blockIdx.x) * 64 + (slot)] = clock64(); \
  } while (0)

__device__ __forceinline__ float warp_colsum32(float (&v)[32], int lane) {
#pragma unroll
  for (int off = 16; off >= 1; off >>= 1) {
    const bool upper = (lane & off) != 0;
#pragma unroll
    for (int i = 0; i < off; ++i) {
      float send = upper ? v[i] : v[i + off];
      float keep = upper ? v[i + off] : v[i];
      v[i] = keep + __shfl_xor_sync(0xffffffffu, send, off);
    }
  }
  return v[0];  // sum over the 32 lanes of column `lane`
}

__device__ __forceinline__ void consumers_sync() { asm volatile("bar.sync 1, 256;" ::: "memory"); }

// 32 channels of pixel row m of a staging chunk (128B-swizzled, 128 rows x 128 B)
__device__ __forceinline__ void ld_row32(const uint8_t *chunk, int m, float (&v)[32]) {
  const uint8_t *row = chunk + m * 128;
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const float4 t = *reinterpret_cast<const float4 *>(row + ((j ^ (m & 7)) << 4));
    v[4 * j] = t.x; v[4 * j + 1] = t.y; v[4 * j + 2] = t.z; v[4 * j + 3] = t.w;
  }
}
__device__ __forceinline__ void st_row32(uint8_t *chunk, int m, const float (&v)[32]) {
  uint8_t *row = chunk + m * 128;
#pragma unroll
  for (int j = 0; j < 8; ++j)
    *reinterpret_cast<float4 *>(row + ((j ^ (m & 7)) << 4)) = make_float4(v[4 * j], v[4 * j + 1], v[4 * j + 2], v[4 * j + 3]);
}

// bias, activation, Dropout2d scale and TF32 rounding of 32 output channels of one pixel.  Every option is tested ONCE
// per chunk, never per element: a switch inside the unrolled element loop becomes 32 indirect branches.
__device__ __forceinline__ void epilogue_chunk(float (&v)[32], const float *bias, int narrow_k, int act, float slope,
                                               const float *cs, int rtf) {
  if (bias && narrow_k) {
#pragma unroll
    for (int j = 0; j < 32; ++j)
      if (j < narrow_k) v[j] += __ldg(bias + j);
  } else if (bias) {
    const float4 *b4 = reinterpret_cast<const float4 *>(bias);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      float4 b = __ldg(b4 + j);
      v[4 * j] += b.x; v[4 * j + 1] += b.y; v[4 * j + 2] += b.z; v[4 * j + 3] += b.w;
    }
  }
  if (act == B200GAN_ACT_LRELU) {
#pragma unroll
    for (int j = 0; j < 32; ++j) v[j] = v[j] > 0.f ? v[j] : v[j] * slope;
  } else if (act == B200GAN_ACT_RELU) {
#pragma unroll
    for (int j = 0; j < 32; ++j) v[j] = fmaxf(v[j], 0.f);
  } else if (act == B200GAN_ACT_TANH) {
#pragma unroll
    for (int j = 0; j < 32; ++j) v[j] = tanhf(v[j]);
  } else if (act == B200GAN_ACT_SIGMOID) {
#pragma unroll
    for (int j = 0; j < 32; ++j) v[j] = 1.f / (1.f + __expf(-v[j]));
  }
  if (cs) {
    const float4 *s4 = reinterpret_cast<const float4 *>(cs);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      float4 b = __ldg(s4 + j);
      v[4 * j] *= b.x; v[4 * j + 1] *= b.y; v[4 * j + 2] *= b.z; v[4 * j + 3] *= b.w;
    }
  }
  if (rtf) {
#pragma unroll
    for (int j = 0; j < 32; ++j) v[j] = round_tf32(v[j]);
  }
}

// shared-memory budget of conv_tc_kernel: the ring, reused as the staging tile of all BN channels after the last MMA
template <int BN, int STAGES>
struct TcSmem {
  static constexpr int STAGE_BYTES = TC_A_BYTES + BN * TC_BK * 4;
  static constexpr int RING = STAGES * STAGE_BYTES;
  static constexpr int STAGING = (BN / 32) * TC_A_BYTES;
  static constexpr int MAIN = RING > STAGING ? RING : STAGING;
  static constexpr int TOTAL = MAIN + 1024 + 256 + 4 * BN * 2 * 4;  // + alignment slack, barriers, statistics
};

template <int BN, int STAGES>
__global__ void __launch_bounds__(TC_THREADS, 1)
conv_tc_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
               const __grid_constant__ CUtensorMap tmY, const __grid_constant__ TcParams p) {
  using L = TcSmem<BN, STAGES>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t *smem = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint64_t *full = reinterpret_cast<uint64_t *>(smem + L::MAIN);
  uint64_t *empty = full + STAGES;
  float *red = reinterpret_cast<float *>(smem + L::MAIN + 256);  // [4][BN][2]

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int ph = blockIdx.z / p.ksplit, ks = blockIdx.z % p.ksplit;
  const int ntile = blockIdx.y;
  const int BW = 1 << p.bw_log2, BH = 1 << p.bh_log2;
  int t = blockIdx.x;
  const int tw = t % p.tiles_w;
  t /= p.tiles_w;
  const int th = t % p.tiles_h;
  const int tn = t / p.tiles_h;
  const int w0 = tw << p.bw_log2, h0 = th << p.bh_log2;
  const int n0 = tn * (TC_BM >> (p.bw_log2 + p.bh_log2));
  const int tap0 = p.tap_begin[ph];
  const int iters_all = (p.tap_begin[ph + 1] - tap0) * p.kchunks;
  const int it0 = (int)((long long)iters_all * ks / p.ksplit), it1 = (int)((long long)iters_all * (ks + 1) / p.ksplit);
  const int iters = it1 - it0;   // >= 1: the host never asks for more splits than iterations

  if (threadIdx.x == 0) {
    TC_TRACE(0);
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    tma_prefetch_desc(&tmY);
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], 2);  // one arrival per consumer warpgroup
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp == 0) {
    if (lane == 0) {
      // ===== TMA producer =====
      int stage = 0;
      uint32_t phase = 0;
      int tap = it0 / p.kchunks, kc = it0 % p.kchunks;
      for (int it = 0; it < iters; ++it) {
        mbar_wait(&empty[stage], phase ^ 1);
        uint8_t *sa = smem + stage * L::STAGE_BYTES;
        uint8_t *sb = sa + TC_A_BYTES;
        const TcTap tp = p.taps[tap0 + tap];
        if (it < 16) TC_TRACE(2 + it);
        mbar_arrive_expect_tx(&full[stage], L::STAGE_BYTES);
        tma_load_5d(sa, &tmA, &full[stage], tp.dc + kc * TC_BK, w0 + tp.dw, tp.da, h0 + tp.dh, n0);
        tma_load_3d(sb, &tmB, &full[stage], kc * TC_BK, ntile * BN, tp.bt);
        if (++kc == p.kchunks) {
          kc = 0;
          ++tap;
        }
        if (++stage == STAGES) {
          stage = 0;
          phase ^= 1;
        }
      }
    }
  } else if (warp >= 4) {
    const int ct = threadIdx.x - 128;
    const int half = ct >> 7;  // consumer warpgroup: MMA rows [64 * half, +64) of the tile
    {
      // ===== MMA: the previous stage is released once the wgmma group issued after it has been waited for =====
      float acc[BN / 2];  // the first MMA overwrites it (scale_d = 0)
      int stage = 0, prev = 0;
      uint32_t phase = 0;
      for (int it = 0; it < iters; ++it) {
        mbar_wait(&full[stage], phase);
        if (ct == 0 && it < 16) TC_TRACE(20 + it);
        const uint32_t sa = smem_u32(smem + stage * L::STAGE_BYTES) + half * (TC_A_BYTES / 2);
        const uint32_t sb = smem_u32(smem + stage * L::STAGE_BYTES + TC_A_BYTES);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < TC_BK / 8; ++k)
          wgmma_tf32<BN>(acc, gmma_desc_sw128(sa + k * 32), gmma_desc_sw128(sb + k * 32), (it > 0 || k > 0) ? 1u : 0u);
        wgmma_commit();
        wgmma_wait<1>();
        if (it > 0 && (ct & 127) == 0) mbar_arrive(&empty[prev]);
        prev = stage;
        if (++stage == STAGES) {
          stage = 0;
          phase ^= 1;
        }
      }
      wgmma_wait<0>();
      wgmma_fence_regs<BN / 2>(acc);
      consumers_sync();  // every MMA of both halves has retired: the ring is free for the staging tile
      store_acc_sw128<BN>(smem, acc, half * 64);
    }
    consumers_sync();
    // ===== epilogue: thread <-> pixel row m of the tile, the two warpgroups take alternate 32-channel chunks =====
    const int q = (ct >> 5) & 3;
    const int m = ct & 127;
    const int lw = m & (BW - 1);
    const int lh = (m >> p.bw_log2) & (BH - 1);
    const int ln = m >> (p.bw_log2 + p.bh_log2);
    const int ow = w0 + lw, oh = h0 + lh, on = n0 + ln;
    const bool valid = (ow < p.Wo) && (oh < p.Ho) && (on < p.N);
    const float *cs = p.chan_scale && valid ? p.chan_scale + (int64_t)on * p.ldk + ntile * BN : nullptr;
    const bool partial = p.ksplit > 1;  // raw partial sums: no bias / activation / statistics (the host checked)
    if (ct == 0) TC_TRACE(40);
#pragma unroll 1
    for (int c = half * 32; c < BN; c += 64) {
      float v[32];
      uint8_t *chunk = smem + (c >> 5) * TC_A_BYTES;
      ld_row32(chunk, m, v);
      epilogue_chunk(v, p.bias ? p.bias + (p.narrow_k ? 0 : ntile * BN + c) : nullptr, p.narrow_k, p.act, p.slope,
                     cs ? cs + c : nullptr, p.rtf);
      if (p.narrow_k) {
        // fewer than 32 real output channels: one pixel's channels are 4..124 contiguous bytes, written directly
        if (valid) {
          float *dst = p.y + ((int64_t)(on * p.Ho + oh) * p.Wo + ow) * p.narrow_k;
#pragma unroll
          for (int j = 0; j < 32; ++j)
            if (j < p.narrow_k) dst[j] = v[j];
        }
      } else {
        st_row32(chunk, m, v);
      }
      if (p.stats) {
        float s2[32];
#pragma unroll
        for (int j = 0; j < 32; ++j) {
          v[j] = valid ? v[j] : 0.f;
          s2[j] = v[j] * v[j];
        }
        float cs1 = warp_colsum32(v, lane);
        float cs2 = warp_colsum32(s2, lane);
        red[(q * BN + c + lane) * 2 + 0] = cs1;
        red[(q * BN + c + lane) * 2 + 1] = cs2;
      }
    }
    fence_proxy_async();  // generic-proxy smem writes -> visible to the async (TMA) proxy
    consumers_sync();
    if (ct == 0 && !p.narrow_k) {
      TC_TRACE(44);
#pragma unroll 1
      for (int c = 0; c < BN; c += 32) {
        if (partial)
          tma_reduce_add_5d(&tmY, smem + (c >> 5) * TC_A_BYTES, p.out_dc[ph] + ntile * BN + c, w0, p.out_da[ph], h0, n0);
        else
          tma_store_5d(&tmY, smem + (c >> 5) * TC_A_BYTES, p.out_dc[ph] + ntile * BN + c, w0, p.out_da[ph], h0, n0);
      }
      tma_store_commit_and_wait_read();
      TC_TRACE(45);
    }
    if (p.stats) {
      for (int e = ct; e < BN; e += 256) {
        float a = 0.f, b = 0.f;
#pragma unroll
        for (int qq = 0; qq < 4; ++qq) {
          a += red[(qq * BN + e) * 2 + 0];
          b += red[(qq * BN + e) * 2 + 1];
        }
        const int gidx = (p.stats_per_sample ? n0 * p.ldk : 0) + ntile * BN + e;
        atomicAdd(p.stats + gidx, (double)a);
        atomicAdd(p.stats + p.stats_groups + gidx, (double)b);
      }
    }
  }
  if (threadIdx.x == 128) TC_TRACE(42);
}

// ---- all-phase kernel for the folded Upsample(2x)+Conv3x3 forward -------------------------------------------
// The four output phases of the fold read 2x2 windows of the SAME nine shifted input tiles (dh, dw in {-1,0,1}).  The
// per-phase kernel above fetches 16 A boxes per k-chunk; this one fetches the 9 distinct ones once and feeds each to
// every phase that uses it (1, 2 or 4 of the four register accumulators; the centre shift is fetched twice so that a
// stage holds at most two B boxes): operand ingest per MMA drops from 24 KB to 18 KB.  BN = 64: four accumulators of
// 64 x 64 per consumer warpgroup = 128 registers per thread.
constexpr int MP_BN = 64;
constexpr int MP_STAGES = 6;
constexpr int MP_B_BYTES = MP_BN * TC_BK * 4;
constexpr int MP_MAX_USES = 2;  // B boxes per stage; the centre shift (used by all four phases) takes two stages
constexpr int MP_STEPS = 10;
constexpr int MP_STAGE_BYTES = TC_A_BYTES + MP_MAX_USES * MP_B_BYTES;
constexpr int MP_MAIN = MP_STAGES * MP_STAGE_BYTES;  // >= the four 32 KB staging buffers of the epilogue
static_assert(MP_MAIN >= 4 * 2 * TC_A_BYTES, "all-phase staging buffers");

struct MpStep {
  int8_t dw, dh, nb, pad_;
  int8_t acc[MP_MAX_USES];  // accumulator (= output phase) of each use
  int8_t bt[MP_MAX_USES];   // tap block of each use in the packed weight matrix
};

// The fixed step schedule: shifts (dh, dw) in row-major order, one stage per shift (the centre shift, read by all four
// phases, takes two); phase (a,b) reads shift (dh,dw) through its tap (dr,ds) = (dh-a+1, dw-b+1) when both are in {0,1}.
// A compile-time table, so that the consumers pick each MMA's accumulator statically.
struct MpSchedule {
  MpStep s[MP_STEPS];
  int n;
};
__host__ __device__ constexpr MpSchedule mp_schedule() {
  MpSchedule r{};
  for (int dh = -1; dh <= 1; ++dh)
    for (int dw = -1; dw <= 1; ++dw) {
      int cur = -1;
      for (int a = 0; a < 2; ++a)
        for (int b = 0; b < 2; ++b) {
          const int dr = dh - a + 1, ds = dw - b + 1;
          if (dr < 0 || dr > 1 || ds < 0 || ds > 1) continue;
          if (cur < 0 || r.s[cur].nb == MP_MAX_USES) {
            cur = r.n++;
            r.s[cur].dw = (int8_t)dw;
            r.s[cur].dh = (int8_t)dh;
          }
          const int ph = a * 2 + b;
          r.s[cur].acc[r.s[cur].nb] = (int8_t)ph;
          r.s[cur].bt[r.s[cur].nb] = (int8_t)(ph * 4 + dr * 2 + ds);
          ++r.s[cur].nb;
        }
    }
  return r;
}
static_assert(mp_schedule().n == MP_STEPS, "all-phase step schedule");
// true when use U of step S is the first MMA into its accumulator (it overwrites: scale_d = 0 on its first k-chunk)
__host__ __device__ constexpr bool mp_first_use(int S, int U) {
  const MpSchedule r = mp_schedule();
  for (int s = 0; s <= S; ++s)
    for (int u = 0; u < r.s[s].nb && (s < S || u < U); ++u)
      if (r.s[s].acc[u] == r.s[S].acc[U]) return false;
  return true;
}

struct MpParams {
  MpStep steps[MP_STEPS];  // = mp_schedule() (the producer's copy)
  int32_t kout_total, kchunks, bw_log2, bh_log2, tiles_w, tiles_h, N, Ho, Wo;
  int32_t out_dc[4], out_da[4];
  int32_t ldk;
  const float *bias;
  const float *chan_scale;
  double *stats;
  int32_t stats_groups, stats_per_sample, act;
  float slope;
  int32_t rtf;
  long long *trace;  // bring-up: per-CTA clock64 timeline (64 slots per CTA) or nullptr
};

// use U of step S: four K8 slices of one B box into the accumulator of its phase
template <int S, int U>
__device__ __forceinline__ void mp_mma_use(float *acc0, float *acc1, float *acc2, float *acc3, uint32_t sa, uint32_t sb,
                                           bool first_chunk) {
  constexpr int A = mp_schedule().s[S].acc[U];
  constexpr bool fresh = mp_first_use(S, U);
#pragma unroll
  for (int k = 0; k < TC_BK / 8; ++k) {
    const uint64_t da = gmma_desc_sw128(sa + k * 32), db = gmma_desc_sw128(sb + k * 32);
    const uint32_t scale_d = (fresh && first_chunk && k == 0) ? 0u : 1u;
    if constexpr (A == 0) wgmma_tf32<MP_BN>(acc0, da, db, scale_d);
    else if constexpr (A == 1) wgmma_tf32<MP_BN>(acc1, da, db, scale_d);
    else if constexpr (A == 2) wgmma_tf32<MP_BN>(acc2, da, db, scale_d);
    else wgmma_tf32<MP_BN>(acc3, da, db, scale_d);
  }
}

// consumer side of steps S.. : every k-chunk of step S is one stage of the ring; the previous stage is released once the
// wgmma group issued after it has been waited for
template <int S>
__device__ __forceinline__ void mp_consume(float *acc0, float *acc1, float *acc2, float *acc3, uint8_t *smem, uint64_t *full,
                                           uint64_t *empty, int kchunks, int half, bool leader, int &stage, uint32_t &phase,
                                           int &prev, int &it) {
  constexpr int NB = mp_schedule().s[S].nb;
#pragma unroll 1
  for (int kc = 0; kc < kchunks; ++kc, ++it) {
    mbar_wait(&full[stage], phase);
    const uint32_t base = smem_u32(smem + stage * MP_STAGE_BYTES);
    const uint32_t sa = base + half * (TC_A_BYTES / 2);
    wgmma_fence();
    mp_mma_use<S, 0>(acc0, acc1, acc2, acc3, sa, base + TC_A_BYTES, kc == 0);
    if constexpr (NB > 1) mp_mma_use<S, 1>(acc0, acc1, acc2, acc3, sa, base + TC_A_BYTES + MP_B_BYTES, kc == 0);
    wgmma_commit();
    wgmma_wait<1>();
    if (it > 0 && leader) mbar_arrive(&empty[prev]);
    prev = stage;
    if (++stage == MP_STAGES) {
      stage = 0;
      phase ^= 1;
    }
  }
  if constexpr (S + 1 < MP_STEPS)
    mp_consume<S + 1>(acc0, acc1, acc2, acc3, smem, full, empty, kchunks, half, leader, stage, phase, prev, it);
}

__global__ void __launch_bounds__(TC_THREADS, 1)
conv_tc_up2_allphase_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                            const __grid_constant__ CUtensorMap tmY, const __grid_constant__ MpParams p) {
  constexpr int BN = MP_BN;
  extern __shared__ uint8_t smem_raw[];
  uint8_t *smem = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint64_t *full = reinterpret_cast<uint64_t *>(smem + MP_MAIN);
  uint64_t *empty = full + MP_STAGES;
  float *red = reinterpret_cast<float *>(smem + MP_MAIN + 256);  // [4][BN][2]

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int ntile = blockIdx.y;
  const int BW = 1 << p.bw_log2, BH = 1 << p.bh_log2;
  int t = blockIdx.x;
  const int tw = t % p.tiles_w;
  t /= p.tiles_w;
  const int th = t % p.tiles_h;
  const int tn = t / p.tiles_h;
  const int w0 = tw << p.bw_log2, h0 = th << p.bh_log2;
  const int n0 = tn * (TC_BM >> (p.bw_log2 + p.bh_log2));
  const int iters = MP_STEPS * p.kchunks;

  if (threadIdx.x == 0) {
    TC_TRACE(0);
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    tma_prefetch_desc(&tmY);
    for (int s = 0; s < MP_STAGES; ++s) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], 2);
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp == 0) {
    if (lane == 0) {
      // ===== TMA producer: step-major, k-chunk-minor =====
      int stage = 0, step = 0, kc = 0;
      uint32_t phase = 0;
      for (int it = 0; it < iters; ++it) {
        mbar_wait(&empty[stage], phase ^ 1);
        uint8_t *sa = smem + stage * MP_STAGE_BYTES;
        const MpStep sp = p.steps[step];
        if (it < 16) TC_TRACE(2 + it);
        mbar_arrive_expect_tx(&full[stage], TC_A_BYTES + sp.nb * MP_B_BYTES);
        tma_load_5d(sa, &tmA, &full[stage], kc * TC_BK, w0 + sp.dw, 0, h0 + sp.dh, n0);
#pragma unroll 1
        for (int u = 0; u < sp.nb; ++u)
          tma_load_2d(sa + TC_A_BYTES + u * MP_B_BYTES, &tmB, &full[stage], kc * TC_BK,
                      sp.bt[u] * p.kout_total + ntile * BN);
        if (++kc == p.kchunks) {
          kc = 0;
          ++step;
        }
        if (++stage == MP_STAGES) {
          stage = 0;
          phase ^= 1;
        }
      }
    }
  } else if (warp >= 4) {
    const int ct = threadIdx.x - 128;
    const int half = ct >> 7;
    // ===== MMA: one A box feeds every phase that reads this shift =====
    float acc0[BN / 2], acc1[BN / 2], acc2[BN / 2], acc3[BN / 2];  // each phase's first MMA overwrites (scale_d = 0)
    {
      int stage = 0, prev = 0, it = 0;
      uint32_t phase = 0;
      mp_consume<0>(acc0, acc1, acc2, acc3, smem, full, empty, p.kchunks, half, (ct & 127) == 0, stage, phase, prev, it);
      wgmma_wait<0>();
      wgmma_fence_regs<BN / 2>(acc0);
      wgmma_fence_regs<BN / 2>(acc1);
      wgmma_fence_regs<BN / 2>(acc2);
      wgmma_fence_regs<BN / 2>(acc3);
    }
    consumers_sync();  // every MMA has retired: the ring is free for the staging buffers
    // ===== epilogue: all four accumulators (= output phases) go to their own 32 KB staging buffer first, so that no
    // accumulator is live during the element-wise work; then phase by phase, the TMA store of phase j overlapping the
    // epilogue of phase j+1; warpgroup `half` takes channels [32 * half, +32) =====
    store_acc_sw128<BN>(smem + 0 * (2 * TC_A_BYTES), acc0, half * 64);
    store_acc_sw128<BN>(smem + 1 * (2 * TC_A_BYTES), acc1, half * 64);
    store_acc_sw128<BN>(smem + 2 * (2 * TC_A_BYTES), acc2, half * 64);
    store_acc_sw128<BN>(smem + 3 * (2 * TC_A_BYTES), acc3, half * 64);
    consumers_sync();
    const int q = (ct >> 5) & 3;
    const int m = ct & 127;
    const int c = half * 32;
    const int lw = m & (BW - 1);
    const int lh = (m >> p.bw_log2) & (BH - 1);
    const int ln = m >> (p.bw_log2 + p.bh_log2);
    const int ow = w0 + lw, oh = h0 + lh, on = n0 + ln;
    const bool valid = (ow < p.Wo) && (oh < p.Ho) && (on < p.N);
    const float *cs = p.chan_scale && valid ? p.chan_scale + (int64_t)on * p.ldk + ntile * BN + c : nullptr;
    const float *bias = p.bias ? p.bias + ntile * BN + c : nullptr;
    float st1 = 0.f, st2 = 0.f;
    if (ct == 0) TC_TRACE(40);
#pragma unroll 1
    for (int j = 0; j < 4; ++j) {
      uint8_t *buf = smem + j * (2 * TC_A_BYTES);
      float v[32];
      uint8_t *chunk = buf + half * TC_A_BYTES;
      ld_row32(chunk, m, v);
      epilogue_chunk(v, bias, 0, p.act, p.slope, cs, p.rtf);
      st_row32(chunk, m, v);
      if (p.stats) {
        float s2[32];
#pragma unroll
        for (int e = 0; e < 32; ++e) {
          v[e] = valid ? v[e] : 0.f;
          s2[e] = v[e] * v[e];
        }
        st1 += warp_colsum32(v, lane);
        st2 += warp_colsum32(s2, lane);
      }
      fence_proxy_async();
      consumers_sync();
      if (ct == 0) {
        TC_TRACE(50 + 3 * j);
#pragma unroll
        for (int cc = 0; cc < BN; cc += 32)
          tma_store_5d(&tmY, buf + (cc >> 5) * TC_A_BYTES, p.out_dc[j] + ntile * BN + cc, w0, p.out_da[j], h0, n0);
        asm volatile("cp.async.bulk.commit_group;" ::: "memory");
      }
    }
    if (ct == 0) {
      asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
      TC_TRACE(41);
    }
    if (p.stats) {
      red[(q * BN + c + lane) * 2 + 0] = st1;
      red[(q * BN + c + lane) * 2 + 1] = st2;
      consumers_sync();
      if (ct < BN) {
        float a = 0.f, b = 0.f;
#pragma unroll
        for (int qq = 0; qq < 4; ++qq) {
          a += red[(qq * BN + ct) * 2 + 0];
          b += red[(qq * BN + ct) * 2 + 1];
        }
        const int gidx = (p.stats_per_sample ? n0 * p.ldk : 0) + ntile * BN + ct;
        atomicAdd(p.stats + gidx, (double)a);
        atomicAdd(p.stats + p.stats_groups + gidx, (double)b);
      }
    }
  }
  if (threadIdx.x == 128) TC_TRACE(42);
}

// ---- host ----------------------------------------------------------------------------------------
static int ilog2_ceil(int v) {
  int l = 0;
  while ((1 << l) < v) ++l;
  return l;
}

template <int BN, int STAGES>
static int launch_tc(const CUtensorMap &tmA, const CUtensorMap &tmB, const CUtensorMap &tmY, const TcParams &p, dim3 grid,
                     cudaStream_t st) {
  constexpr int SMEM = TcSmem<BN, STAGES>::TOTAL;
  static std::atomic<uint64_t> attr_done{0};
  if (int e = ensure_dynamic_smem(conv_tc_kernel<BN, STAGES>, SMEM, attr_done)) return e;
  conv_tc_kernel<BN, STAGES><<<grid, TC_THREADS, SMEM, st>>>(tmA, tmB, tmY, p);
  B2_LAUNCH_CHECK();
  return B200GAN_OK;
}

int tc_wgrad_supported(const b200gan_conv_geom *g);  // wgrad_tc.cu

// Which passes of which geometries the tensor-core path takes.
//   gather form  (out[p] = sum_t in[stride*p + off_t] B_t): Conv2d fprop, ConvTranspose2d dgrad
//   scatter form (out[h] = sum_{t | stride divides h+pad-t} in[(h+pad-t)/stride] B_t): Conv2d dgrad, ConvTranspose2d fprop
// stride 2 is handled with parity views: the gathered tensor {2C, W/2, 2, H/2, N} for the gather form, the
// produced tensor (four output phases with their own tap subsets) for the scatter form.
static bool tc_is_gather(const b200gan_conv_geom *g, int pass) { return (pass == 0) != (g->transposed != 0); }

int tc_supported(const b200gan_conv_geom *g, int pass) {
  if (g->pad_mode != B200GAN_PAD_ZERO || g->N < 1) return 0;
  if (pass == 2) return tc_wgrad_supported(g);  // weight gradient: wgrad_tc.cu
  if (g->stride != 1 && g->stride != 2) return 0;
  const int cin = pass == 0 ? g->C : g->K;   // contraction channels
  const int cout = pass == 0 ? g->K : g->C;  // produced channels
  // fewer than 32 produced channels: only the plain stride-1 gather form (Conv2d forward), B rows zero-padded by TMA
  const bool narrow = cout < 32 && pass == 0 && !g->transposed && g->up == 1 && g->stride == 1;
  if (cin % 32 != 0 || (cout % 32 != 0 && !narrow) || 2 * cin > 32767) return 0;
  if (g->R * g->S > 49 || g->R > 15 || g->S > 15 || g->pad_t > 15 || g->pad_l > 15) return 0;
  if (g->up == 2) {
    if (g->transposed || g->stride != 1) return 0;
    if (!(g->R == 3 && g->S == 3 && g->pad_t == 1 && g->pad_l == 1 && g->pad_b == 1 && g->pad_r == 1)) return 0;
    return cout % 64 == 0;
  }
  if (g->stride == 2) {
    // the full-resolution side (Conv2d input / ConvTranspose2d output) is the one seen through a parity view
    const int Hf = g->transposed ? g->P : g->H, Wf = g->transposed ? g->Q : g->W;
    if ((Hf & 1) || (Wf & 1)) return 0;
    if (!tc_is_gather(g, pass)) {  // scatter form: 4 phases, each at most 16 taps in total budget
      int taps = 0;
      for (int a = 0; a < 2; ++a)
        for (int b = 0; b < 2; ++b) {
          int nr = 0, ns = 0;
          for (int r = 0; r < g->R; ++r) nr += ((a + g->pad_t - r) % 2 == 0);
          for (int s2 = 0; s2 < g->S; ++s2) ns += ((b + g->pad_l - s2) % 2 == 0);
          taps += nr * ns;
        }
      if (taps > TC_MAX_TAPS) return 0;
    }
  }
  return 1;
}

// Shared by fprop and dgrad.
//  in      : contracted activation tensor [N][Hi][Wi][Cc] (x for fprop, dy for dgrad)
//  phase_in: 1 -> `in` is addressed through the parity view {2Cc, Wi/2, 2, Hi/2, N} (dgrad of UP2; stride-2 gathers)
//  btaps   : number of tap blocks in the packed weight matrix (rows = btaps * Kout)
//  out     : N x Ho x Wo pixels per phase.  phase_out: 1 -> y is the full-resolution tensor [N][2Ho][2Wo][ldk]
//            addressed through the phase view {2*ldk, Wo, 2, Ho, N}; phase z writes (out_dc[z], out_da[z]).
static int run_tc(const float *in, int N, int Hi, int Wi, int Cc, bool phase_in, const float *packedB, int Kout,
                  int btaps, int nphase, const int *tap_begin, const TcTap *taps, int Ho, int Wo, bool phase_out,
                  const int *out_dc, const int *out_da, int ldk, const b200gan_epilogue *ep, float *y,
                  cudaStream_t st) {
  const int narrow_k = Kout < 32 ? Kout : 0;
  const int Kreal = Kout;
  if (narrow_k) Kout = 32;  // MMA N = 32; rows >= Kreal of every B box are TMA out-of-bounds zeros
  int BN = (Kout % 128 == 0) ? 128 : (Kout % 64 == 0 ? 64 : 32);
  TcParams p;
  memset(&p, 0, sizeof(p));
  const int total_taps = tap_begin[nphase];
  for (int i = 0; i <= 4; ++i) p.tap_begin[i] = tap_begin[i < nphase ? i : nphase];
  for (int i = 0; i < total_taps; ++i) p.taps[i] = taps[i];
  p.kout_total = Kout;
  p.kchunks = Cc / TC_BK;
  int bwl = ilog2_ceil(Wo);
  if (bwl > 7) bwl = 7;
  int bhl = ilog2_ceil(Ho);
  if (bhl > 7 - bwl) bhl = 7 - bwl;
  const int BW = 1 << bwl, BH = 1 << bhl, BNn = TC_BM / (BW * BH);
  p.bw_log2 = bwl;
  p.bh_log2 = bhl;
  p.tiles_w = ceil_div(Wo, BW);
  p.tiles_h = ceil_div(Ho, BH);
  {
    // 256-wide tiles (A 16 KB + B 32 KB per stage feed 2 x 4 x M64 N256 K8: the 128-channel A box is fetched half as
    // often per output channel) when the layer still gives every SM a CTA
    const int64_t tiles = (int64_t)p.tiles_w * p.tiles_h * ceil_div(N, BNn) * nphase;
    if (Kout % 256 == 0 && tiles * (Kout / 256) >= num_sms()) BN = 256;
  }
  p.N = N;
  p.Ho = Ho;
  p.Wo = Wo;
  for (int i = 0; i < 4; ++i) {
    p.out_dc[i] = i < nphase ? out_dc[i] : 0;
    p.out_da[i] = i < nphase ? out_da[i] : 0;
  }
  p.ldk = ldk;
  p.bias = ep ? ep->bias : nullptr;
  p.chan_scale = ep ? ep->chan_scale : nullptr;
  p.stats = ep ? ep->stats : nullptr;
  p.stats_per_sample = ep ? ep->stats_per_sample : 0;
  p.stats_groups = p.stats_per_sample ? N * ldk : ldk;
  if (p.stats && p.stats_per_sample && BNn != 1)
    B2_UNSUPPORTED("tensor-core fprop: per-sample statistics need one image per tile (H*W >= 128 per phase)");
  p.act = ep ? ep->act : 0;
  p.slope = ep ? ep->slope : 0.f;
  p.rtf = ep ? ep->round_tf32 : 0;
  p.y = y;
  p.narrow_k = narrow_k;
  if (narrow_k) {
    B2_CHECK_ARG(!phase_in && !phase_out && nphase == 1, "tensor-core conv: narrow output only in the plain gather form");
    B2_CHECK_ARG(!p.chan_scale, "tensor-core conv: Dropout2d scale with fewer than 32 output channels");
  }
  p.ksplit = 1;
  double *deferred_stats = nullptr;
  if (narrow_k && p.stats) {  // statistics of a narrow layer: separate pass
    deferred_stats = p.stats;
    p.stats = nullptr;
  }
  {
    // few output tiles (deep U-Net layers at 1x1 .. 16x16 pixels): split the contraction so that the machine is used
    const bool plain = !p.bias && !p.chan_scale && p.act == B200GAN_ACT_NONE && !p.rtf;
    const int64_t ctas = (int64_t)p.tiles_w * p.tiles_h * ceil_div(N, BNn) * (Kout / BN) * nphase;
    int min_iters = 1 << 30;
    for (int z = 0; z < nphase; ++z) {
      const int it = (tap_begin[z + 1] - tap_begin[z]) * p.kchunks;
      if (it < min_iters) min_iters = it;
    }
    if (plain && !narrow_k && ctas < num_sms() && min_iters >= 16) {
      int ks = (int)((2 * num_sms() + ctas - 1) / ctas);
      if (ks > min_iters / 8) ks = min_iters / 8;
      if (ks > 32) ks = 32;
      if (ks >= 2) {
        p.ksplit = ks;
        if (p.stats) {  // partial tiles cannot carry the norm statistics: one extra pass over the (small) output
          deferred_stats = p.stats;
          p.stats = nullptr;
        }
      }
    }
  }
  p.trace = nullptr;
  if (const char *tv = getenv("B200GAN_TC_TRACE")) p.trace = reinterpret_cast<long long *>(strtoull(tv, nullptr, 0));
  B2_CHECK_ARG(((uintptr_t)in % 16 == 0) && ((uintptr_t)packedB % 16 == 0) && ((uintptr_t)y % 16 == 0),
               "tensor-core conv: pointers must be 16-byte aligned");
  if (p.ksplit > 1) {
    const int64_t out_elems = phase_out ? (int64_t)N * (2 * Ho) * (2 * Wo) * ldk : (int64_t)N * Ho * Wo * ldk;
    B2_CUDA(cudaMemsetAsync(y, 0, (size_t)out_elems * sizeof(float), st));
  }

  CUtensorMap tmA, tmB, tmY;
  if (!narrow_k) {
    // output map: box = one 32-channel chunk of the 128-pixel tile; TMA clips rows outside the tensor
    uint64_t dims[5], strides[4];
    uint32_t box[5] = {TC_BK, (uint32_t)BW, 1, (uint32_t)BH, (uint32_t)BNn};
    const uint64_t L = (uint64_t)ldk;
    if (!phase_out) {
      dims[0] = L; dims[1] = Wo; dims[2] = 1; dims[3] = Ho; dims[4] = N;
      strides[0] = L * 4; strides[1] = (uint64_t)Wo * L * 4; strides[2] = (uint64_t)Wo * L * 4;
      strides[3] = (uint64_t)Ho * Wo * L * 4;
    } else {
      dims[0] = 2 * L; dims[1] = Wo; dims[2] = 2; dims[3] = Ho; dims[4] = N;
      strides[0] = 2 * L * 4; strides[1] = (uint64_t)2 * Wo * L * 4; strides[2] = (uint64_t)4 * Wo * L * 4;
      strides[3] = (uint64_t)4 * Ho * Wo * L * 4;
    }
    if (int e = make_tmap_f32(&tmY, y, 5, dims, strides, box)) return e;
  }
  {
    uint64_t dims[5], strides[4];
    uint32_t box[5] = {TC_BK, (uint32_t)BW, 1, (uint32_t)BH, (uint32_t)BNn};
    if (!phase_in) {
      dims[0] = Cc; dims[1] = Wi; dims[2] = 1; dims[3] = Hi; dims[4] = N;
      strides[0] = (uint64_t)Cc * 4;
      strides[1] = (uint64_t)Wi * Cc * 4;  // size-1 dim: any legal stride
      strides[2] = (uint64_t)Wi * Cc * 4;
      strides[3] = (uint64_t)Hi * Wi * Cc * 4;
    } else {
      dims[0] = 2 * (uint64_t)Cc; dims[1] = Wi / 2; dims[2] = 2; dims[3] = Hi / 2; dims[4] = N;
      strides[0] = (uint64_t)2 * Cc * 4;
      strides[1] = (uint64_t)Wi * Cc * 4;
      strides[2] = (uint64_t)2 * Wi * Cc * 4;
      strides[3] = (uint64_t)Hi * Wi * Cc * 4;
    }
    if (int e = make_tmap_f32(&tmA, in, 5, dims, strides, box)) return e;
  }
  if (narrow_k) tmY = tmA;  // never used for stores (rows of < 32 channels cannot be a TMA box): any valid descriptor
  {
    // weights [tap][Kreal][Cc] as a rank-3 map: a box never runs into the next tap, rows beyond Kreal are zero fill
    uint64_t dims[3] = {(uint64_t)Cc, (uint64_t)Kreal, (uint64_t)btaps};
    uint64_t strides[2] = {(uint64_t)Cc * 4, (uint64_t)Kreal * Cc * 4};
    uint32_t box[3] = {TC_BK, (uint32_t)BN, 1};
    if (int e = make_tmap_f32(&tmB, packedB, 3, dims, strides, box)) return e;
  }
  dim3 grid((unsigned)(p.tiles_w * p.tiles_h * ceil_div(N, BNn)), (unsigned)(Kout / BN), (unsigned)(nphase * p.ksplit));
  int rc;
  if (BN == 256) rc = launch_tc<256, 4>(tmA, tmB, tmY, p, grid, st);
  else if (BN == 128) rc = launch_tc<128, 6>(tmA, tmB, tmY, p, grid, st);
  else if (BN == 64) rc = launch_tc<64, 8>(tmA, tmB, tmY, p, grid, st);
  else rc = launch_tc<32, 8>(tmA, tmB, tmY, p, grid, st);
  if (rc == B200GAN_OK && deferred_stats) {
    b200gan_norm_desc nd;
    memset(&nd, 0, sizeof(nd));
    nd.N = N;
    nd.HW = phase_out ? 4 * Ho * Wo : Ho * Wo;
    nd.C = ldk;
    nd.per_sample = p.stats_per_sample;
    rc = b200gan_norm_stats(&nd, y, deferred_stats, st);
  }
  return rc;
}

// Folded Upsample(2x)+Conv3x3 forward with all four phases in one CTA (conv_tc_up2_allphase_kernel).
// x: [N][H][W][C]; y: [N][2H][2W][K] seen through the phase view; packed: [ph][tp][K][C] (B200GAN_PACK_TC_FPROP_UP2).
static int run_up2_allphase(const float *x, int N, int H, int W, int C, const float *packed, int K,
                            const b200gan_epilogue *ep, float *y, cudaStream_t st) {
  MpParams p;
  memset(&p, 0, sizeof(p));
  constexpr MpSchedule sched = mp_schedule();
  for (int i = 0; i < MP_STEPS; ++i) p.steps[i] = sched.s[i];
  p.kout_total = K;
  p.kchunks = C / TC_BK;
  int bwl = ilog2_ceil(W);
  if (bwl > 7) bwl = 7;
  int bhl = ilog2_ceil(H);
  if (bhl > 7 - bwl) bhl = 7 - bwl;
  const int BW = 1 << bwl, BH = 1 << bhl, BNn = TC_BM / (BW * BH);
  p.bw_log2 = bwl;
  p.bh_log2 = bhl;
  p.tiles_w = ceil_div(W, BW);
  p.tiles_h = ceil_div(H, BH);
  p.N = N;
  p.Ho = H;
  p.Wo = W;
  for (int ph = 0; ph < 4; ++ph) {
    p.out_dc[ph] = (ph & 1) * K;
    p.out_da[ph] = ph >> 1;
  }
  p.ldk = K;
  p.bias = ep ? ep->bias : nullptr;
  p.chan_scale = ep ? ep->chan_scale : nullptr;
  p.stats = ep ? ep->stats : nullptr;
  p.stats_per_sample = ep ? ep->stats_per_sample : 0;
  p.stats_groups = p.stats_per_sample ? N * K : K;
  if (p.stats && p.stats_per_sample && BNn != 1)
    B2_UNSUPPORTED("tensor-core fprop: per-sample statistics need one image per tile (H*W >= 128 per phase)");
  p.act = ep ? ep->act : 0;
  p.slope = ep ? ep->slope : 0.f;
  p.rtf = ep ? ep->round_tf32 : 0;
  p.trace = nullptr;
  if (const char *tv = getenv("B200GAN_TC_TRACE")) p.trace = reinterpret_cast<long long *>(strtoull(tv, nullptr, 0));
  B2_CHECK_ARG(((uintptr_t)x % 16 == 0) && ((uintptr_t)packed % 16 == 0) && ((uintptr_t)y % 16 == 0),
               "tensor-core conv: pointers must be 16-byte aligned");
  CUtensorMap tmA, tmB, tmY;
  uint32_t box[5] = {TC_BK, (uint32_t)BW, 1, (uint32_t)BH, (uint32_t)BNn};
  {
    const uint64_t L = (uint64_t)K;
    uint64_t dims[5] = {2 * L, (uint64_t)W, 2, (uint64_t)H, (uint64_t)N};
    uint64_t strides[4] = {2 * L * 4, (uint64_t)2 * W * L * 4, (uint64_t)4 * W * L * 4, (uint64_t)4 * H * W * L * 4};
    if (int e = make_tmap_f32(&tmY, y, 5, dims, strides, box)) return e;
  }
  {
    uint64_t dims[5] = {(uint64_t)C, (uint64_t)W, 1, (uint64_t)H, (uint64_t)N};
    uint64_t strides[4] = {(uint64_t)C * 4, (uint64_t)W * C * 4, (uint64_t)W * C * 4, (uint64_t)H * W * C * 4};
    if (int e = make_tmap_f32(&tmA, x, 5, dims, strides, box)) return e;
  }
  {
    uint64_t dims[2] = {(uint64_t)C, (uint64_t)16 * K};
    uint64_t strides[1] = {(uint64_t)C * 4};
    uint32_t bbox[2] = {TC_BK, (uint32_t)MP_BN};
    if (int e = make_tmap_f32(&tmB, packed, 2, dims, strides, bbox)) return e;
  }
  constexpr int SMEM = MP_MAIN + 1024 + 256 + 4 * MP_BN * 2 * 4;
  static std::atomic<uint64_t> attr_done{0};
  if (int e = ensure_dynamic_smem(conv_tc_up2_allphase_kernel, SMEM, attr_done)) return e;
  dim3 grid((unsigned)(p.tiles_w * p.tiles_h * ceil_div(N, BNn)), (unsigned)(K / MP_BN), 1);
  conv_tc_up2_allphase_kernel<<<grid, TC_THREADS, SMEM, st>>>(tmA, tmB, tmY, p);
  B2_LAUNCH_CHECK();
  return B200GAN_OK;
}

static inline int floordiv2(int v) { return v >= 0 ? v / 2 : -((-v + 1) / 2); }

// gather form.  in: [N][Hi][Wi][Cc]; out: [N][Po][Qo][Kout]; B: [R*S][Kout][Cc]
static int tc_gather(const float *in, int N, int Hi, int Wi, int Cc, int R, int S, int stride, int pad_t, int pad_l,
                     const float *packedB, int Kout, int Po, int Qo, const b200gan_epilogue *ep, float *out,
                     cudaStream_t st) {
  TcTap taps[TC_MAX_TAPS];
  memset(taps, 0, sizeof(taps));
  int tap_begin[5] = {0, 0, 0, 0, 0};
  int out_dc[4] = {0, 0, 0, 0}, out_da[4] = {0, 0, 0, 0};
  int nt = 0;
  for (int r = 0; r < R; ++r)
    for (int s = 0; s < S; ++s) {
      TcTap &t = taps[nt];
      const int eh = r - pad_t, ew = s - pad_l;
      if (stride == 1) {
        t.dc = 0; t.dw = (int8_t)ew; t.da = 0; t.dh = (int8_t)eh;
      } else {  // in[2p + eh] = parity view [p + floor(eh/2)][eh mod 2]
        t.dh = (int8_t)floordiv2(eh); t.da = (int8_t)(eh & 1);
        t.dw = (int8_t)floordiv2(ew); t.dc = (int16_t)((ew & 1) * Cc);
      }
      t.bt = (int8_t)nt;
      ++nt;
    }
  tap_begin[1] = nt;
  return run_tc(in, N, Hi, Wi, Cc, stride == 2, packedB, Kout, R * S, 1, tap_begin, taps, Po, Qo, false, out_dc, out_da,
                Kout, ep, out, st);
}

// scatter form.  in: [N][Pi][Qi][Cc]; out: [N][Ho][Wo][Kout] (full resolution); B: [R*S][Kout][Cc]
static int tc_scatter(const float *in, int N, int Pi, int Qi, int Cc, int R, int S, int stride, int pad_t, int pad_l,
                      const float *packedB, int Kout, int Ho, int Wo, const b200gan_epilogue *ep, float *out,
                      cudaStream_t st) {
  TcTap taps[TC_MAX_TAPS];
  memset(taps, 0, sizeof(taps));
  int tap_begin[5] = {0, 0, 0, 0, 0};
  int out_dc[4] = {0, 0, 0, 0}, out_da[4] = {0, 0, 0, 0};
  if (stride == 1) {
    int nt = 0;
    for (int r = 0; r < R; ++r)
      for (int s = 0; s < S; ++s) {
        TcTap &t = taps[nt];
        t.dc = 0; t.dw = (int8_t)(pad_l - s); t.da = 0; t.dh = (int8_t)(pad_t - r); t.bt = (int8_t)nt;
        ++nt;
      }
    tap_begin[1] = nt;
    return run_tc(in, N, Pi, Qi, Cc, false, packedB, Kout, R * S, 1, tap_begin, taps, Ho, Wo, false, out_dc, out_da, Kout,
                  ep, out, st);
  }
  int nt = 0;
  for (int ph = 0; ph < 4; ++ph) {
    const int a = ph >> 1, b = ph & 1;
    tap_begin[ph] = nt;
    for (int r = 0; r < R; ++r) {
      if ((a + pad_t - r) % 2 != 0) continue;
      for (int s = 0; s < S; ++s) {
        if ((b + pad_l - s) % 2 != 0) continue;
        TcTap &t = taps[nt++];
        t.dc = 0; t.da = 0;
        t.dh = (int8_t)((a + pad_t - r) / 2);  // exact: numerator is even
        t.dw = (int8_t)((b + pad_l - s) / 2);
        t.bt = (int8_t)(r * S + s);
      }
    }
    out_dc[ph] = b * Kout;
    out_da[ph] = a;
  }
  tap_begin[4] = nt;
  return run_tc(in, N, Pi, Qi, Cc, false, packedB, Kout, R * S, 4, tap_begin, taps, Ho / 2, Wo / 2, true, out_dc, out_da,
                Kout, ep, out, st);
}

int tc_fprop(const b200gan_conv_geom *g, const b200gan_epilogue *ep, const float *x, const float *packed, float *y,
             cudaStream_t st) {
  b200gan_epilogue e2;
  if (ep) e2 = *ep;
  const b200gan_epilogue *e = ep ? &e2 : nullptr;
  if (g->up == 2) {
    // 64-wide output tiles: all four phases in one CTA (9 operand fetches per k-chunk instead of 16)
    if (g->K % 128 != 0 && g->K % 64 == 0)
      return run_up2_allphase(x, g->N, g->H, g->W, g->C, packed, g->K, e, y, st);
    // phase (a,b): out[2i+a][2j+b] = sum_{dr,ds} x[i+a-1+dr][j+b-1+ds] * Wf[a][b][dr][ds]
    TcTap taps[TC_MAX_TAPS];
    memset(taps, 0, sizeof(taps));
    int tap_begin[5] = {0, 4, 8, 12, 16};
    int out_dc[4], out_da[4];
    for (int ph = 0; ph < 4; ++ph) {
      int a = ph >> 1, b = ph & 1;
      for (int tp = 0; tp < 4; ++tp) {
        int dr = tp >> 1, ds = tp & 1;
        TcTap &t = taps[ph * 4 + tp];
        t.dc = 0; t.dw = (int8_t)(b - 1 + ds); t.da = 0; t.dh = (int8_t)(a - 1 + dr); t.bt = (int8_t)(ph * 4 + tp);
      }
      out_dc[ph] = b * g->K;
      out_da[ph] = a;
    }
    return run_tc(x, g->N, g->H, g->W, g->C, false, packed, g->K, 16, 4, tap_begin, taps, g->H, g->W, true, out_dc, out_da,
                  g->K, e, y, st);
  }
  if (g->transposed)  // ConvTranspose2d forward: scatter x into the (stride x larger) output
    return tc_scatter(x, g->N, g->H, g->W, g->C, g->R, g->S, g->stride, g->pad_t, g->pad_l, packed, g->K, g->P, g->Q, e, y,
                      st);
  return tc_gather(x, g->N, g->H, g->W, g->C, g->R, g->S, g->stride, g->pad_t, g->pad_l, packed, g->K, g->P, g->Q, e, y, st);
}

int tc_dgrad(const b200gan_conv_geom *g, const float *dy, const float *packed, float *dx, cudaStream_t st) {
  if (g->up == 2) {
    // dx[i][j] = sum_{a,b,dr,ds} dy[2(i-(a-1+dr))+a][2(j-(b-1+ds))+b] * Wf[a][b][dr][ds]^T
    TcTap taps[TC_MAX_TAPS];
    memset(taps, 0, sizeof(taps));
    int tap_begin[5] = {0, 16, 16, 16, 16};
    int out_dc[4] = {0, 0, 0, 0}, out_da[4] = {0, 0, 0, 0};
    for (int ph = 0; ph < 4; ++ph) {
      int a = ph >> 1, b = ph & 1;
      for (int tp = 0; tp < 4; ++tp) {
        int dr = tp >> 1, ds = tp & 1;
        TcTap &t = taps[ph * 4 + tp];
        t.dc = (int16_t)(b * g->K); t.dw = (int8_t)(-(b - 1 + ds)); t.da = (int8_t)a; t.dh = (int8_t)(-(a - 1 + dr));
        t.bt = (int8_t)(ph * 4 + tp);
      }
    }
    return run_tc(dy, g->N, g->P, g->Q, g->K, true, packed, g->C, 16, 1, tap_begin, taps, g->H, g->W, false, out_dc, out_da,
                  g->C, nullptr, dx, st);
  }
  if (g->transposed)  // dx[ih] = sum dy[stride*ih - pad + r] w: gather over dy
    return tc_gather(dy, g->N, g->P, g->Q, g->K, g->R, g->S, g->stride, g->pad_t, g->pad_l, packed, g->C, g->H, g->W, nullptr,
                     dx, st);
  return tc_scatter(dy, g->N, g->P, g->Q, g->K, g->R, g->S, g->stride, g->pad_t, g->pad_l, packed, g->C, g->H, g->W, nullptr,
                    dx, st);
}

}  // namespace b200gan
