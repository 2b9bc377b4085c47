// narrow_block.cu -- the Discriminator's strided conv blocks as a fused chain of fp32 kernels.
//
// Reference: dcgan.py:77-88
//     block = [nn.Conv2d(in, out, 3, 2, 1), nn.LeakyReLU(0.2, inplace=True), nn.Dropout2d(0.25)] (+ nn.BatchNorm2d(out, 0.8))
//     self.model = nn.Sequential(*block(1, 16, bn=False), *block(16, 32), *block(32, 64), *block(64, 128))
// At the BASELINE size these four layers move 16 MB per pass and execute 0.94 GFLOP: they are launch- and latency-bound,
// and un-fused they cost ~15 launches forward and ~35 backward per discriminator pass (conv, epilogue backward, bias
// gradient, BatchNorm statistics / finalize / apply / backward reduce / backward apply / parameter gradients, ...).
// Here a layer l keeps only a_l = dropout(lrelu(conv_l(x_l) + b_l)) and the batch sums of a_l in memory; the normalised
// tensor x_{l+1} = BN_l(a_l) is never written:
//   nbk_fprop2  x_l = a_{l-1} * scale + shift applied while gathering (BatchNorm "apply" of the producer folded into the
//               consumer's loads; zero padding stays zero), bias + LeakyReLU + Dropout2d scale in registers, the sums
//               / sums of squares the NEXT BatchNorm needs reduced in the epilogue (warp shuffles -> one fp64 atomic per
//               channel and block).  The BatchNorm finalisation (mean, rstd, running statistics) happens in the prologue
//               of the consumer: no finalize / apply kernels at all.
//   nbk_dz      dz_l = BN_l-backward(G_{l+1}) * dropout scale * lrelu'(a_l), element-wise from the sums the upstream
//               dgrad accumulated, + the bias gradient.
//   nbk_wgrad   dW_l from dz_l and x_l (recomputed from a_{l-1} while staging the patch in shared memory); thread =
//               (input channel, 4 output channels) x all taps in registers, pixels streamed through shared memory.
//   nbk_dgrad2  G_l = transposed gather of dz_l by stride-parity class + the sums BN_{l-1}'s backward needs, in the epilogue.
//   nbk_tail_*  BN_4 apply fused with the NHWC -> NCHW layout change the script's .view needs (dcgan.py:96), and back.
// G_l is the gradient w.r.t. the VIRTUAL tensor x_l; the BatchNorm backward is finished by the consumer (nbk_dz of layer
// l-1) once the sums are complete.  See b200gan/functional.py (NbConvFn, NbTailFn) for the autograd wiring.
#include "tc_common.cuh"
#include <string.h>

namespace b200gan {

struct NbBn {
  const double *stats;  // [groups][2][C]: sum, sum of squares over a group's batch (null: no BatchNorm on this edge)
  const float *gamma, *beta;
  float eps;
  double count;         // elements per channel and GROUP
  int groups;           // the batch is `groups` equal runs of images with independent statistics (train.dcgan_step:
                        // the discriminator's real and fake passes of dcgan.py:178-179 in one launch per layer)
};

__device__ __forceinline__ void nb_bn_consts(const NbBn &bn, int C, int c, float &mean, float &rstd, float &sc,
                                             float &sh, double *var_out = nullptr, int grp = 0) {
  const double *st = bn.stats + (size_t)grp * 2 * C;
  const double m = st[c] / bn.count;
  double var = st[C + c] / bn.count - m * m;
  if (var < 0.0) var = 0.0;
  if (var_out) *var_out = var;
  rstd = (float)(1.0 / sqrt(var + (double)bn.eps));
  mean = (float)m;
  const float ga = bn.gamma ? bn.gamma[c] : 1.f, be = bn.beta ? bn.beta[c] : 0.f;
  sc = ga * rstd;
  sh = be - mean * sc;
}

// running statistics: one update per group, in batch order (= the order of the reference's separate forward passes)
__device__ __forceinline__ void nb_update_running(const NbBn &bn, int C, int c, float *rm, float *rv, float momentum) {
  float m_run = rm[c], v_run = rv[c];
  for (int grp = 0; grp < bn.groups; ++grp) {
    float mean, rstd, sc, sh;
    double var;
    nb_bn_consts(bn, C, c, mean, rstd, sc, sh, &var, grp);
    const double unbiased = bn.count > 1.0 ? var * bn.count / (bn.count - 1.0) : var;
    m_run = (1.f - momentum) * m_run + momentum * mean;
    v_run = (1.f - momentum) * v_run + momentum * (float)unbiased;
  }
  rm[c] = m_run;
  rv[c] = v_run;
}

__device__ __forceinline__ float nb_act(float v, int act, float slope) {
  if (act == B200GAN_ACT_LRELU) return v > 0.f ? v : v * slope;
  if (act == B200GAN_ACT_RELU) return fmaxf(v, 0.f);
  return v;
}
__device__ __forceinline__ float nb_act_grad(float a, int act, float slope) {
  if (act == B200GAN_ACT_LRELU) return a > 0.f ? 1.f : slope;
  if (act == B200GAN_ACT_RELU) return a > 0.f ? 1.f : 0.f;
  return 1.f;
}

__device__ __forceinline__ int ceil_div_dev(int a, int b) { return (a + b - 1) / b; }
// sum over the 32 lanes of a warp
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

constexpr int NB_MAXC = 128;
constexpr int NB_MAX_GROUPS = 4;   // statistics groups per batch (NbBn::groups)

// ---- forward: shared-memory staged kernels -------------------------------------------------------------------------
// Copy a [rows][cols][C] window of an NHWC image into shared memory with channel pitch CP, applying v * sc + sh to
// elements inside the image; positions outside are 0 (zero padding comes after the normalisation) or mirrored.
// src_img == nullptr (tile hangs over the batch): all zeros.  Consecutive threads read consecutive channels: coalesced.
__device__ __forceinline__ void nb_stage(float *dst, int CP, const float *src_img, int h0, int w0, int rows, int cols, int C,
                                         int H, int W, const float *sc_s, const float *sh_s, bool reflect, int tid) {
  if ((C & 3) == 0) {
    const int C4 = C >> 2, total = rows * cols * C4;
    for (int i = tid; i < total; i += 256) {
      const int c4 = i % C4, pix = i / C4;
      const int pc = pix % cols, pr = pix / cols;
      int ih = h0 + pr, iw = w0 + pc;
      if (reflect) {
        ih = reflect_idx(ih, H);
        iw = reflect_idx(iw, W);
      }
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (src_img && ih >= 0 && ih < H && iw >= 0 && iw < W) {
        v = __ldg(reinterpret_cast<const float4 *>(src_img + ((int64_t)ih * W + iw) * C) + c4);
        if (sc_s) {
          const float4 a = *reinterpret_cast<const float4 *>(sc_s + 4 * c4), b = *reinterpret_cast<const float4 *>(sh_s + 4 * c4);
          v.x = fmaf(v.x, a.x, b.x); v.y = fmaf(v.y, a.y, b.y); v.z = fmaf(v.z, a.z, b.z); v.w = fmaf(v.w, a.w, b.w);
        }
      }
      *reinterpret_cast<float4 *>(dst + (int64_t)pix * CP + 4 * c4) = v;
    }
  } else {
    const int total = rows * cols * C;
    for (int i = tid; i < total; i += 256) {
      const int cc = i % C, pix = i / C;
      const int pc = pix % cols, pr = pix / cols;
      int ih = h0 + pr, iw = w0 + pc;
      if (reflect) {
        ih = reflect_idx(ih, H);
        iw = reflect_idx(iw, W);
      }
      float v = 0.f;
      if (src_img && ih >= 0 && ih < H && iw >= 0 && iw < W) {
        v = __ldg(src_img + ((int64_t)ih * W + iw) * C + cc);
        if (sc_s) v = fmaf(v, sc_s[cc], sh_s[cc]);
      }
      dst[(int64_t)pix * CP + cc] = v;
    }
  }
}

// tile of TP = TN images x TR x TQ pixels (powers of two); 256 threads = (TP / PT pixel threads) x (KG channel groups),
// a thread computes PT pixels x KT outputs
struct NbTile {
  int TN, TR, TQ, TP, KG, KB;   // KB = KG * KT output channels per block
  int tiles_r, tiles_q;
};

struct NbFprop2 {
  const float *x, *wp, *bias, *cs;
  float *y;
  double *out_stats;
  NbBn in_bn;
  float *rm, *rv;
  long long *nbt;
  float momentum;
  int N, H, W, C, P, Q, K, R, S, stride, pad_t, pad_l;
  float slope;
  int act;
  NbTile t;
  int PR, PC, CP;   // patch rows, columns, channel pitch (C + 4: lanes = pixels 2 * CP floats apart stay 2-way conflicted at worst)
  int reflect;      // reflection padding (stand-alone use: cyclegan/models.py:49-50), chains are zero-padded
  int rtf;          // store y rounded to TF32 (a wgmma conv consumes it next)
  int groups;       // statistics groups of the batch (NbBn::groups of the edges; 1 stand-alone)
};
// Forward: the patch (BatchNorm of the producer applied while staging) and this block's slice of the weights live in
// shared memory.  Thread = PT pixels x KT output channels in registers: lanes of a warp are consecutive pixels (pixel i
// of a thread is lp + i * TPX), the weights are read as broadcasts -- one LDS.128 of weights feeds 4 * PT FMAs, one of
// activations 4 * KT (the first version had PT = 1: 3.8 FMAs per shared-memory load, and stalled on them).
// dynamic smem: w [R*S*C][KB] | patch [TN][PR][PC][CP] | sc, sh [C] | red [8][2*KT]
template <int KT, int PT>
__global__ void __launch_bounds__(256)
nbk_fprop2_kernel(const __grid_constant__ NbFprop2 p) {
  extern __shared__ __align__(16) float nsm[];
  const NbTile &t = p.t;
  const int taps = p.R * p.S;
  float *w_s = nsm;
  float *x_s = w_s + (size_t)taps * p.C * t.KB;
  float *sc_s = x_s + (((size_t)t.TN * p.PR * p.PC * p.CP + 3) & ~(size_t)3);
  float *sh_s = sc_s + ((p.C + 3) & ~3);
  float *red = sh_s + ((p.C + 3) & ~3);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const bool has_in = p.in_bn.stats != nullptr;
  // the tile's images belong to ONE statistics group (the planner keeps TN a divisor of the group size)
  const int grp = (int)((blockIdx.x / (t.tiles_q * t.tiles_r)) * t.TN) / (p.N / p.groups);
  for (int cc = tid; cc < p.C; cc += 256) {
    float mean, rstd, sc = 1.f, sh = 0.f;
    if (has_in) {
      nb_bn_consts(p.in_bn, p.C, cc, mean, rstd, sc, sh, nullptr, grp);
      if (blockIdx.x == 0 && blockIdx.y == 0 && p.rm) nb_update_running(p.in_bn, p.C, cc, p.rm, p.rv, p.momentum);
    }
    sc_s[cc] = sc;
    sh_s[cc] = sh;
  }
  if (has_in && blockIdx.x == 0 && blockIdx.y == 0 && tid == 0 && p.nbt) *p.nbt += p.in_bn.groups;
  // this block's weights: rows (tap, c) of KB consecutive output channels
  const int kbase = blockIdx.y * t.KB;
  {
    const int KB4 = t.KB >> 2, total = taps * p.C * KB4;
#pragma unroll 4
    for (int i = tid; i < total; i += 256) {
      const int col = i % KB4, row = i / KB4;
      reinterpret_cast<float4 *>(w_s)[i] = __ldg(reinterpret_cast<const float4 *>(p.wp + (int64_t)row * p.K + kbase) + col);
    }
  }
  __syncthreads();
  int tile = blockIdx.x;
  const int tq = tile % t.tiles_q;
  tile /= t.tiles_q;
  const int tr = tile % t.tiles_r;
  const int n0 = (tile / t.tiles_r) * t.TN;
  const int p0 = tr * t.TR, q0 = tq * t.TQ;
  for (int li = 0; li < t.TN; ++li) {
    const int n = n0 + li;
    nb_stage(x_s + (size_t)li * p.PR * p.PC * p.CP, p.CP, n < p.N ? p.x + (int64_t)n * p.H * p.W * p.C : nullptr,
             p0 * p.stride - p.pad_t, q0 * p.stride - p.pad_l, p.PR, p.PC, p.C, p.H, p.W, has_in ? sc_s : nullptr, sh_s,
             p.reflect != 0, tid);
  }
  __syncthreads();

  const int TPX = t.TP / PT;                 // pixel threads (a multiple of 32: a warp has one channel group)
  const int lpx = tid % TPX, kgi = tid / TPX;
  int xoff[PT];
  int64_t yoff[PT];                          // < 0: pixel outside the tensor
  int nn[PT];
#pragma unroll
  for (int i = 0; i < PT; ++i) {
    const int lp = lpx + i * TPX;
    const int lq = lp % t.TQ, lr = (lp / t.TQ) % t.TR, li = lp / (t.TQ * t.TR);
    const int n = n0 + li, po = p0 + lr, qo = q0 + lq;
    xoff[i] = ((li * p.PR + lr * p.stride) * p.PC + lq * p.stride) * p.CP;
    nn[i] = n;
    yoff[i] = (n < p.N && po < p.P && qo < p.Q) ? ((int64_t)(n * p.P + po) * p.Q + qo) * p.K : -1;
  }
  float acc[PT][KT];
#pragma unroll
  for (int i = 0; i < PT; ++i)
#pragma unroll
    for (int j = 0; j < KT; ++j) acc[i][j] = 0.f;
  const float *wb = w_s + kgi * KT;
  const int KB = t.KB;
  for (int r = 0; r < p.R; ++r) {
    for (int s = 0; s < p.S; ++s) {
      const float *xt = x_s + (r * p.PC + s) * p.CP;
      const float *wt = wb + (size_t)(r * p.S + s) * p.C * KB;
      if ((p.C & 3) == 0) {
#pragma unroll 2
        for (int c = 0; c < p.C; c += 4) {
          float xs[PT][4];
#pragma unroll
          for (int i = 0; i < PT; ++i) {
            const float4 xv = *reinterpret_cast<const float4 *>(xt + xoff[i] + c);
            xs[i][0] = xv.x; xs[i][1] = xv.y; xs[i][2] = xv.z; xs[i][3] = xv.w;
          }
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            const float *wr = wt + (size_t)(c + j) * KB;
#pragma unroll
            for (int u = 0; u < KT / 4; ++u) {
              const float4 w4 = *reinterpret_cast<const float4 *>(wr + 4 * u);
#pragma unroll
              for (int i = 0; i < PT; ++i) {
                acc[i][4 * u + 0] = fmaf(xs[i][j], w4.x, acc[i][4 * u + 0]);
                acc[i][4 * u + 1] = fmaf(xs[i][j], w4.y, acc[i][4 * u + 1]);
                acc[i][4 * u + 2] = fmaf(xs[i][j], w4.z, acc[i][4 * u + 2]);
                acc[i][4 * u + 3] = fmaf(xs[i][j], w4.w, acc[i][4 * u + 3]);
              }
            }
          }
        }
      } else {
        for (int c = 0; c < p.C; ++c) {
          float xs[PT];
#pragma unroll
          for (int i = 0; i < PT; ++i) xs[i] = xt[xoff[i] + c];
          const float *wr = wt + (size_t)c * KB;
#pragma unroll
          for (int u = 0; u < KT / 4; ++u) {
            const float4 w4 = *reinterpret_cast<const float4 *>(wr + 4 * u);
#pragma unroll
            for (int i = 0; i < PT; ++i) {
              acc[i][4 * u + 0] = fmaf(xs[i], w4.x, acc[i][4 * u + 0]);
              acc[i][4 * u + 1] = fmaf(xs[i], w4.y, acc[i][4 * u + 1]);
              acc[i][4 * u + 2] = fmaf(xs[i], w4.z, acc[i][4 * u + 2]);
              acc[i][4 * u + 3] = fmaf(xs[i], w4.w, acc[i][4 * u + 3]);
            }
          }
        }
      }
    }
  }
  const int k0 = kbase + kgi * KT;
  float s1[KT], s2[KT];
#pragma unroll
  for (int j = 0; j < KT; ++j) s1[j] = s2[j] = 0.f;
#pragma unroll
  for (int i = 0; i < PT; ++i) {
    const bool valid = yoff[i] >= 0;
#pragma unroll
    for (int j = 0; j < KT; ++j) {
      float v = acc[i][j];
      if (p.bias) v += __ldg(p.bias + k0 + j);
      v = nb_act(v, p.act, p.slope);
      if (p.cs && valid) v *= __ldg(p.cs + (int64_t)nn[i] * p.K + k0 + j);
      if (p.rtf) v = round_tf32(v);
      v = valid ? v : 0.f;
      acc[i][j] = v;
      s1[j] += v;
      s2[j] = fmaf(v, v, s2[j]);
    }
    if (valid) {
      float *yo = p.y + yoff[i] + k0;
#pragma unroll
      for (int u = 0; u < KT / 4; ++u)
        *reinterpret_cast<float4 *>(yo + 4 * u) =
            make_float4(acc[i][4 * u], acc[i][4 * u + 1], acc[i][4 * u + 2], acc[i][4 * u + 3]);
    }
  }
  if (p.out_stats) {
#pragma unroll
    for (int j = 0; j < KT; ++j) {
      const float a1 = warp_sum(s1[j]), a2 = warp_sum(s2[j]);
      if (lane == 0) {
        red[warp * 2 * KT + j] = a1;
        red[warp * 2 * KT + KT + j] = a2;
      }
    }
    __syncthreads();
    if (tid < t.KG * 2 * KT) {   // the TPX / 32 warps of a channel group are consecutive
      const int g = tid / (2 * KT), idx = tid % (2 * KT), wpg = TPX >> 5;
      float tsum = 0.f;
      for (int wi = 0; wi < wpg; ++wi) tsum += red[(g * wpg + wi) * 2 * KT + idx];
      atomicAdd(p.out_stats + (size_t)grp * 2 * p.K + (idx < KT ? 0 : p.K) + kbase + g * KT + (idx % KT), (double)tsum);
    }
  }
}

// ---- dz = BatchNorm backward (from complete sums) * Dropout2d scale * act'(a), + bias gradient ---------------------------
struct NbDz {
  const float *g, *a, *cs;
  float *dz, *db;
  NbBn out_bn;
  const double *sums;  // [2][K]: sum G, sum G * ahat (null with out_bn.stats == null)
  int64_t rows;        // N * P * Q
  int64_t PQ;
  int K;
  float slope;
  int act;
};
__global__ void __launch_bounds__(256)
nbk_dz_kernel(const __grid_constant__ NbDz p) {
  __shared__ float red[256][4];
  const int tid = threadIdx.x;
  const int K4 = p.K >> 2;              // 256 % K4 == 0 (checked by the launcher)
  const int kq = tid % K4;
  const int rows_per_block = 256 / K4;
  const bool has_bn = p.out_bn.stats != nullptr;
  const int grp = blockIdx.y;                                  // statistics group = a contiguous run of rows
  const int64_t grows = p.rows / gridDim.y, grow0 = grp * grows;
  float mean[4], rstd[4], sc[4], m1[4], m2[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    mean[j] = 0.f; rstd[j] = 0.f; sc[j] = 1.f; m1[j] = 0.f; m2[j] = 0.f;
    if (has_bn) {
      float sh;
      nb_bn_consts(p.out_bn, p.K, kq * 4 + j, mean[j], rstd[j], sc[j], sh, nullptr, grp);
      m1[j] = (float)(p.sums[(size_t)grp * 2 * p.K + kq * 4 + j] / p.out_bn.count);
      m2[j] = (float)(p.sums[(size_t)grp * 2 * p.K + p.K + kq * 4 + j] / p.out_bn.count);
    }
  }
  float dbs[4] = {0.f, 0.f, 0.f, 0.f};
  const int64_t row_end = grow0 + grows;
  for (int64_t row = grow0 + (int64_t)blockIdx.x * rows_per_block + tid / K4; row < row_end;
       row += (int64_t)gridDim.x * rows_per_block) {
    const int64_t off = row * p.K + kq * 4;
    const float4 gv = __ldg(reinterpret_cast<const float4 *>(p.g + off));
    const float4 av = __ldg(reinterpret_cast<const float4 *>(p.a + off));
    const float G[4] = {gv.x, gv.y, gv.z, gv.w}, A[4] = {av.x, av.y, av.z, av.w};
    float csv[4] = {1.f, 1.f, 1.f, 1.f};
    if (p.cs) {
      const float4 c4 = __ldg(reinterpret_cast<const float4 *>(p.cs + (row / p.PQ) * p.K + kq * 4));
      csv[0] = c4.x; csv[1] = c4.y; csv[2] = c4.z; csv[3] = c4.w;
    }
    float o[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      float dA = G[j];
      if (has_bn) dA = sc[j] * (G[j] - m1[j] - ((A[j] - mean[j]) * rstd[j]) * m2[j]);
      o[j] = dA * csv[j] * nb_act_grad(A[j], p.act, p.slope);
      dbs[j] += o[j];
    }
    *reinterpret_cast<float4 *>(p.dz + off) = make_float4(o[0], o[1], o[2], o[3]);
  }
  if (p.db) {
#pragma unroll
    for (int j = 0; j < 4; ++j) red[tid][j] = dbs[j];
    __syncthreads();
    if (tid < K4) {
      float t4[4] = {0.f, 0.f, 0.f, 0.f};
      for (int r = 0; r < rows_per_block; ++r)
#pragma unroll
        for (int j = 0; j < 4; ++j) t4[j] += red[r * K4 + tid][j];
#pragma unroll
      for (int j = 0; j < 4; ++j) atomicAdd(p.db + tid * 4 + j, t4[j]);
    }
  }
}

// ---- weight gradient ---------------------------------------------------------------------------------------------------
struct NbWgrad {
  const float *x, *dz;
  float *dw;
  float *ws;       // per-block partial slabs [gridDim.x][dw_elems] (null: atomics straight into dw)
  int dw_elems;
  NbBn in_bn;
  int N, H, W, C, P, Q, K, R, S, stride, pad_t, pad_l;
  int TN, TR, TQ, tiles_r, tiles_q;  // tile = TN images x TR x TQ output pixels (TN > 1 only for whole small images)
  int PR, PC;                    // patch rows / columns = (TR-1)*stride + R, (TQ-1)*stride + S
  int SPB, PS;                   // sets per block (<= 256, a power of two), pixel split = 256 / SPB
  int nsets;                     // C * K/4 (* R in row mode)
  int row_mode;                  // 1: a set owns ONE filter row (TAPS = S): 7x7 filters (cyclegan/models.py:50)
  int reflect;                   // 1: the virtual input is reflection-padded (cyclegan/models.py:49) instead of zero-padded
};
// thread = set (c, kg: 4 output channels) x all TAPS taps in registers, and one of PS pixel phases.
// grid = (persistent blocks over tiles, set chunks).
// dynamic smem: patch [TN][PR][PC][C] | dz tile [TN*TR*TQ][K4*4] | sc, sh [C] | pixel offsets [TN*TR*TQ] | set bases [SPB]
template <int TAPS>
__global__ void __launch_bounds__(256, 2)   // two blocks per SM: 148 registers (one block per SM) cost 40 % on the 4x4 layers
nbk_wgrad_kernel(const __grid_constant__ NbWgrad p) {
  extern __shared__ __align__(16) float nsm[];
  const int tile_px = p.TN * p.TR * p.TQ;
  const int K4 = (p.K + 3) >> 2, KP = K4 * 4;   // output channels padded to a multiple of 4 inside the dz tile
  const int patch_img = p.PR * p.PC * p.C;
  int *sbase_s = reinterpret_cast<int *>(nsm);   // tables first: the phase reduction reuses everything behind them
  int *sk_s = sbase_s + p.SPB;
  int *poff_s = sk_s + p.SPB;
  float *x_s = nsm + ((2 * p.SPB + tile_px + 3) & ~3);
  float *dz_s = x_s + (((size_t)p.TN * patch_img + 3) & ~(size_t)3);
  const int Cr = (p.C + 3) & ~3;
  const int groups = p.in_bn.groups, img_per_group = p.N / groups;
  float *sc_s = dz_s + (size_t)tile_px * KP;    // [groups][Cr]
  float *sh_s = sc_s + (size_t)groups * Cr;     // [groups][Cr]
  const int tid = threadIdx.x;
  const bool has_in = p.in_bn.stats != nullptr;
  for (int i = tid; i < groups * p.C; i += 256) {
    const int gq = i / p.C, cc = i - gq * p.C;
    float mean, rstd, sc = 1.f, sh = 0.f;
    if (has_in) nb_bn_consts(p.in_bn, p.C, cc, mean, rstd, sc, sh, nullptr, gq);
    sc_s[gq * Cr + cc] = sc;
    sh_s[gq * Cr + cc] = sh;
  }
  // the integer divisions happen once per block, not once per pixel / output value
  for (int pix = tid; pix < tile_px; pix += 256) {
    const int lq = pix % p.TQ, lr = (pix / p.TQ) % p.TR, li = pix / (p.TQ * p.TR);
    poff_s[pix] = li * patch_img + ((lr * p.stride) * p.PC + lq * p.stride) * p.C;
  }
  const int RS = p.R * p.S;
  for (int sl = tid; sl < p.SPB; sl += 256) {
    const int set_o = blockIdx.y * p.SPB + sl;
    int base = -1, k0 = 0;
    if (set_o < p.nsets) {
      const int co = set_o % p.C, kgo = (set_o / p.C) % K4;
      const int ro = p.row_mode ? set_o / (p.C * K4) : 0;
      k0 = kgo * 4;
      base = (k0 * p.C + co) * RS + ro * p.S;             // dw index of (k = 4 kg, c, r, s = 0)
    }
    sbase_s[sl] = base;
    sk_s[sl] = k0;
  }
  const int set_local = tid & (p.SPB - 1), psplit = tid / p.SPB;
  const int set = blockIdx.y * p.SPB + set_local;
  const bool set_ok = set < p.nsets;
  const int c = set_ok ? set % p.C : 0, kg = set_ok ? (set / p.C) % K4 : 0;
  const int r_own = (set_ok && p.row_mode) ? set / (p.C * K4) : 0;   // filter row of this set (row mode)
  float acc[TAPS][4];
#pragma unroll
  for (int t = 0; t < TAPS; ++t)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[t][j] = 0.f;
  const int ntiles = ceil_div_dev(p.N, p.TN) * p.tiles_r * p.tiles_q;
  int toff[TAPS];  // offset of tap t inside the patch, relative to the pixel's top-left element
#pragma unroll
  for (int t = 0; t < TAPS; ++t) toff[t] = p.row_mode ? (r_own * p.PC + t) * p.C : ((t / p.S) * p.PC + (t % p.S)) * p.C;
  __syncthreads();
  for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const int tq = tile % p.tiles_q;
    const int tr = (tile / p.tiles_q) % p.tiles_r;
    const int n0 = (tile / (p.tiles_q * p.tiles_r)) * p.TN;
    const int p0 = tr * p.TR, q0 = tq * p.TQ;
    // patch of x_l = a_{l-1} * scale + shift (zero outside the image: the conv's zero padding comes after the norm)
    const int h0 = p0 * p.stride - p.pad_t, w0 = q0 * p.stride - p.pad_l;
    for (int li = 0; li < p.TN; ++li) {
      const int n = n0 + li;
      const int gq = n < p.N ? n / img_per_group : 0;
      nb_stage(x_s + (size_t)li * patch_img, p.C, n < p.N ? p.x + (int64_t)n * p.H * p.W * p.C : nullptr, h0, w0, p.PR, p.PC,
               p.C, p.H, p.W, has_in ? sc_s + gq * Cr : nullptr, sh_s + gq * Cr, p.reflect != 0, tid);
    }
    const int img_px = p.TR * p.TQ;
    if ((p.K & 3) == 0) {
      for (int i = tid; i < tile_px * K4; i += 256) {
        const int k4 = i % K4, pix = i / K4;
        const int li = pix / img_px, rem = pix - li * img_px;
        const int lr = rem / p.TQ, lq = rem - lr * p.TQ;
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (n0 + li < p.N && p0 + lr < p.P && q0 + lq < p.Q)
          v = __ldg(reinterpret_cast<const float4 *>(p.dz + ((int64_t)((n0 + li) * p.P + p0 + lr) * p.Q + q0 + lq) * p.K) + k4);
        reinterpret_cast<float4 *>(dz_s)[i] = v;
      }
    } else {
      for (int i = tid; i < tile_px * KP; i += 256) {
        const int k = i % KP, pix = i / KP;
        const int li = pix / img_px, rem = pix - li * img_px;
        const int lr = rem / p.TQ, lq = rem - lr * p.TQ;
        float v = 0.f;
        if (k < p.K && n0 + li < p.N && p0 + lr < p.P && q0 + lq < p.Q)
          v = __ldg(p.dz + ((int64_t)((n0 + li) * p.P + p0 + lr) * p.Q + q0 + lq) * p.K + k);
        dz_s[i] = v;
      }
    }
    __syncthreads();
    if (set_ok) {
      const float *xc = x_s + c;
      const float *dk = dz_s + kg * 4;
#pragma unroll 2
      for (int pix = psplit; pix < tile_px; pix += p.PS) {
        const float4 d4 = *reinterpret_cast<const float4 *>(dk + pix * KP);
        const float *xb = xc + poff_s[pix];
#pragma unroll
        for (int t = 0; t < TAPS; ++t) {
          const float xv = xb[toff[t]];
          acc[t][0] = fmaf(xv, d4.x, acc[t][0]);
          acc[t][1] = fmaf(xv, d4.y, acc[t][1]);
          acc[t][2] = fmaf(xv, d4.z, acc[t][2]);
          acc[t][3] = fmaf(xv, d4.w, acc[t][3]);
        }
      }
    }
    __syncthreads();
  }
  // Reduce the PS pixel phases of every set through shared memory (the tile loop ended with a barrier), then ONE value per
  // (set, tap, k) and block goes out: a plain store into this block's slab of the workspace (summed by
  // nbk_wgrad_reduce_kernel, deterministic), or an atomic into dw when the layer has few weights.  Same-address fp32
  // atomics run at ~28 G/s on this part: one per thread and tap (the first version) cost 0.1 - 1.2 ms per layer.
  constexpr int TPAD = TAPS | 1;   // odd pitch: lanes = consecutive sets write conflict-free
  float *red = x_s;                // [PS][4][SPB][TPAD]
#pragma unroll
  for (int j = 0; j < 4; ++j)
#pragma unroll
    for (int t = 0; t < TAPS; ++t) red[((size_t)(psplit * 4 + j) * p.SPB + set_local) * TPAD + t] = acc[t][j];
  __syncthreads();
  const int nout = 4 * p.SPB * TAPS;
  const int kstride = p.C * RS;
  float *slab = p.ws ? p.ws + (size_t)blockIdx.x * p.dw_elems : nullptr;
  for (int o = tid; o < nout; o += 256) {
    const int t = o % TAPS, rest = o / TAPS;          // TAPS is a compile-time constant, SPB a power of two
    const int sl = rest & (p.SPB - 1), j = rest / p.SPB;
    const int base = sbase_s[sl];
    if (base < 0) continue;
    if (sk_s[sl] + j >= p.K) continue;
    float sum = 0.f;
    for (int ps = 0; ps < p.PS; ++ps) sum += red[((size_t)(ps * 4 + j) * p.SPB + sl) * TPAD + t];
    const int idx = base + j * kstride + t;           // dw[k][c][r][s] (parameter layout)
    if (slab) slab[idx] = sum;
    else atomicAdd(p.dw + idx, sum);
  }
}

// dw[e] = sum over the slabs; block = 32 consecutive elements x 8 slab phases
__global__ void __launch_bounds__(256)
nbk_wgrad_reduce_kernel(const float *__restrict__ ws, float *__restrict__ dw, int elems, int nslabs) {
  __shared__ float part[8][32];
  const int e = blockIdx.x * 32 + (threadIdx.x & 31), ph = threadIdx.x >> 5;
  float a = 0.f;
  if (e < elems) {
#pragma unroll 4
    for (int sl = ph; sl < nslabs; sl += 8) a += __ldg(ws + (size_t)sl * elems + e);
  }
  part[ph][threadIdx.x & 31] = a;
  __syncthreads();
  if (ph == 0 && e < elems) {
    float t = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) t += part[i][threadIdx.x];
    dw[e] = t;
  }
}

// ---- data gradient + the sums of the upstream BatchNorm's backward ----------------------------------------------------------
struct NbDgrad2 {
  const float *dz, *wp, *a_prev;
  float *g_out;
  double *sums;
  NbBn in_bn;
  int N, H, W, C, P, Q, K, R, S, stride, pad_t, pad_l;
  NbTile t;         // tile of class pixels; KB = input channels (outputs of this pass) per block
  int KP;           // channel pitch of the staged dz window (K + 4)
  int PRm, PCm;     // window rows / columns of the class with the most taps (shared-memory carve-up)
  int tapsm;        // most taps of a class
};
// Data gradient: blockIdx.z = stride-parity class (all its pixels use the same Rc x Sc taps), the dz window of the
// tile and the class's slice of the weights staged in shared memory; lanes = consecutive class pixels (consecutive dz
// pixels: conflict-free float4 reads with pitch K + 4), the KT input channels of a thread read weights as broadcasts.
// dynamic smem: w [tapsm*K][KB] | window [TN][PRm][PCm][KP] | mean, rstd [C] | red [8][2*KT]
template <int KT, int PT>
__global__ void __launch_bounds__(256)
nbk_dgrad2_kernel(const __grid_constant__ NbDgrad2 p) {
  extern __shared__ __align__(16) float nsm[];
  const NbTile &t = p.t;
  float *w_s = nsm;
  float *d_s = w_s + (((size_t)p.tapsm * p.K * t.KB + 3) & ~(size_t)3);
  float *mean_s = d_s + (((size_t)t.TN * p.PRm * p.PCm * p.KP + 3) & ~(size_t)3);
  float *rstd_s = mean_s + ((p.C + 3) & ~3);
  float *red = rstd_s + ((p.C + 3) & ~3);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const bool has_in = p.sums != nullptr;
  // one statistics group per tile (the planner keeps TN a divisor of the group size)
  const int grp = (int)((blockIdx.x / (t.tiles_q * t.tiles_r)) * t.TN) / (p.N / p.in_bn.groups);
  if (has_in) {
    for (int cc = tid; cc < p.C; cc += 256) {
      float sc, sh;
      nb_bn_consts(p.in_bn, p.C, cc, mean_s[cc], rstd_s[cc], sc, sh, nullptr, grp);
    }
  }
  const int st = p.stride;
  const int cls = blockIdx.z;
  const int pa = cls / st, pb = cls % st;               // first row / column of the class
  const int r0 = (pa + p.pad_t) % st, s0 = (pb + p.pad_l) % st;
  const int Rc = r0 < p.R ? (p.R - r0 + st - 1) / st : 0, Sc = s0 < p.S ? (p.S - s0 + st - 1) / st : 0;
  const int Hc = pa < p.H ? (p.H - pa + st - 1) / st : 0, Wc = pb < p.W ? (p.W - pb + st - 1) / st : 0;
  const int oh = (pa + p.pad_t - r0) / st, ow = (pb + p.pad_l - s0) / st;   // dz row of class row i, tap ir: i + oh - ir
  const int cbase = blockIdx.y * t.KB;
  const int KB = t.KB;
  // weights of the class: w_s[(ti * K + k) * KB + cc] = wp[((r * S + s) * K + k) * C + cbase + cc]
  if ((KB & 3) == 0) {
    const int KB4 = KB >> 2, total = Rc * Sc * p.K * KB4;
#pragma unroll 4
    for (int i = tid; i < total; i += 256) {
      const int col = i % KB4, row = i / KB4;
      const int k = row % p.K, ti = row / p.K;
      const int r = r0 + st * (ti / Sc), s_ = s0 + st * (ti % Sc);
      reinterpret_cast<float4 *>(w_s)[i] =
          __ldg(reinterpret_cast<const float4 *>(p.wp + ((int64_t)(r * p.S + s_) * p.K + k) * p.C + cbase) + col);
    }
  } else {
    const int total = Rc * Sc * p.K * KB;
    for (int i = tid; i < total; i += 256) {
      const int col = i % KB, row = i / KB;
      const int k = row % p.K, ti = row / p.K;
      const int r = r0 + st * (ti / Sc), s_ = s0 + st * (ti % Sc);
      w_s[i] = __ldg(p.wp + ((int64_t)(r * p.S + s_) * p.K + k) * p.C + cbase + col);
    }
  }
  int tile = blockIdx.x;
  const int tq = tile % t.tiles_q;
  tile /= t.tiles_q;
  const int tr = tile % t.tiles_r;
  const int n0 = (tile / t.tiles_r) * t.TN;
  const int i0 = tr * t.TR, j0 = tq * t.TQ;
  const int PRc = t.TR + (Rc > 0 ? Rc - 1 : 0), PCc = t.TQ + (Sc > 0 ? Sc - 1 : 0);
  for (int li = 0; li < t.TN; ++li) {
    const int n = n0 + li;
    nb_stage(d_s + (size_t)li * PRc * PCc * p.KP, p.KP, n < p.N ? p.dz + (int64_t)n * p.P * p.Q * p.K : nullptr,
             i0 + oh - (Rc - 1), j0 + ow - (Sc - 1), PRc, PCc, p.K, p.P, p.Q, nullptr, nullptr, false, tid);
  }
  __syncthreads();

  const int TPX = t.TP / PT;
  const int lpx = tid % TPX, cgi = tid / TPX;
  int doff[PT];
  int64_t opix[PT];   // < 0: class pixel outside the tensor
#pragma unroll
  for (int i = 0; i < PT; ++i) {
    const int lp = lpx + i * TPX;
    const int lq = lp % t.TQ, lr = (lp / t.TQ) % t.TR, li = lp / (t.TQ * t.TR);
    const int n = n0 + li, ci = i0 + lr, cj = j0 + lq;
    doff[i] = ((li * PRc + lr) * PCc + lq) * p.KP;
    opix[i] = (n < p.N && ci < Hc && cj < Wc) ? (int64_t)(n * p.H + pa + st * ci) * p.W + pb + st * cj : -1;
  }
  float acc[PT][KT];
#pragma unroll
  for (int i = 0; i < PT; ++i)
#pragma unroll
    for (int j = 0; j < KT; ++j) acc[i][j] = 0.f;
  const float *wb = w_s + cgi * KT;
  for (int ir = 0; ir < Rc; ++ir) {
    for (int is = 0; is < Sc; ++is) {
      const float *dt = d_s + ((Rc - 1 - ir) * PCc + (Sc - 1 - is)) * p.KP;
      const float *wt = wb + (size_t)(ir * Sc + is) * p.K * KB;
#pragma unroll 2
      for (int k = 0; k < p.K; k += 4) {
        float ds[PT][4];
#pragma unroll
        for (int i = 0; i < PT; ++i) {
          const float4 dv = *reinterpret_cast<const float4 *>(dt + doff[i] + k);
          ds[i][0] = dv.x; ds[i][1] = dv.y; ds[i][2] = dv.z; ds[i][3] = dv.w;
        }
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const float *wr = wt + (size_t)(k + j) * KB;
          if (KT % 4 == 0) {
#pragma unroll
            for (int u = 0; u < KT / 4; ++u) {
              const float4 w4 = *reinterpret_cast<const float4 *>(wr + 4 * u);
#pragma unroll
              for (int i = 0; i < PT; ++i) {
                acc[i][4 * u + 0] = fmaf(ds[i][j], w4.x, acc[i][4 * u + 0]);
                acc[i][4 * u + 1] = fmaf(ds[i][j], w4.y, acc[i][4 * u + 1]);
                acc[i][4 * u + 2] = fmaf(ds[i][j], w4.z, acc[i][4 * u + 2]);
                acc[i][4 * u + 3] = fmaf(ds[i][j], w4.w, acc[i][4 * u + 3]);
              }
            }
          } else {
#pragma unroll
            for (int u = 0; u < KT; ++u) {
              const float wv = wr[u];
#pragma unroll
              for (int i = 0; i < PT; ++i) acc[i][u] = fmaf(ds[i][j], wv, acc[i][u]);
            }
          }
        }
      }
    }
  }
  const int c0 = cbase + cgi * KT;
  float s1[KT], s2[KT];
#pragma unroll
  for (int j = 0; j < KT; ++j) s1[j] = s2[j] = 0.f;
#pragma unroll
  for (int i = 0; i < PT; ++i) {
    if (opix[i] < 0) continue;
    float *go = p.g_out + opix[i] * p.C + c0;
    if (KT % 4 == 0) {
#pragma unroll
      for (int u = 0; u < KT / 4; ++u)
        *reinterpret_cast<float4 *>(go + 4 * u) =
            make_float4(acc[i][4 * u], acc[i][4 * u + 1], acc[i][4 * u + 2], acc[i][4 * u + 3]);
    } else {
#pragma unroll
      for (int j = 0; j < KT; ++j) go[j] = acc[i][j];
    }
    if (has_in) {
      float ah[KT];
      if (KT % 4 == 0) {
#pragma unroll
        for (int u = 0; u < KT / 4; ++u) {
          const float4 a4 = __ldg(reinterpret_cast<const float4 *>(p.a_prev + opix[i] * p.C + c0) + u);
          ah[4 * u] = a4.x; ah[4 * u + 1] = a4.y; ah[4 * u + 2] = a4.z; ah[4 * u + 3] = a4.w;
        }
      } else {
#pragma unroll
        for (int j = 0; j < KT; ++j) ah[j] = __ldg(p.a_prev + opix[i] * p.C + c0 + j);
      }
#pragma unroll
      for (int j = 0; j < KT; ++j) {
        s1[j] += acc[i][j];
        s2[j] = fmaf(acc[i][j], (ah[j] - mean_s[c0 + j]) * rstd_s[c0 + j], s2[j]);
      }
    }
  }
  if (has_in) {
#pragma unroll
    for (int j = 0; j < KT; ++j) {
      const float a1 = warp_sum(s1[j]), a2 = warp_sum(s2[j]);
      if (lane == 0) {
        red[warp * 2 * KT + j] = a1;
        red[warp * 2 * KT + KT + j] = a2;
      }
    }
    __syncthreads();
    if (tid < t.KG * 2 * KT) {
      const int g = tid / (2 * KT), idx = tid % (2 * KT), wpg = TPX >> 5;
      float tsum = 0.f;
      for (int wi = 0; wi < wpg; ++wi) tsum += red[(g * wpg + wi) * 2 * KT + idx];
      atomicAdd(p.sums + (size_t)grp * 2 * p.C + (idx < KT ? 0 : p.C) + cbase + g * KT + (idx % KT), (double)tsum);
    }
  }
}

// ---- tail: BatchNorm apply (+ layout) forward, layout + sums backward ----------------------------------------------------------
struct NbTail {
  const float *a;      // [N][HW][C]
  const float *dout;   // backward: gradient of the output (layout `nchw`)
  float *out;          // forward: [N][C][HW] (nchw) or [N][HW][C]
  float *g;            // backward: [N][HW][C]
  double *sums;        // backward: [2][C]
  NbBn bn;
  float *rm, *rv;
  long long *nbt;
  float momentum;
  int N, HW, C, nchw;
};
__global__ void __launch_bounds__(256)
nbk_tail_fwd_kernel(const __grid_constant__ NbTail p) {
  __shared__ float sc_s[NB_MAXC], sh_s[NB_MAXC];
  const int tid = threadIdx.x;
  const int grp = blockIdx.y;   // statistics group = a contiguous run of images
  if (tid < p.C) {
    float mean, rstd;
    nb_bn_consts(p.bn, p.C, tid, mean, rstd, sc_s[tid], sh_s[tid], nullptr, grp);
    if (blockIdx.x == 0 && grp == 0 && p.rm) nb_update_running(p.bn, p.C, tid, p.rm, p.rv, p.momentum);
  }
  if (blockIdx.x == 0 && grp == 0 && tid == 0 && p.nbt) *p.nbt += p.bn.groups;
  __syncthreads();
  const int64_t gtotal = (int64_t)(p.N / gridDim.y) * p.HW * p.C, total = (grp + 1) * gtotal;
  for (int64_t i = grp * gtotal + (int64_t)blockIdx.x * 256 + tid; i < total; i += (int64_t)gridDim.x * 256) {
    int c;
    int64_t src;
    if (p.nchw) {  // i enumerates the OUTPUT [n][c][hw]
      const int hw = (int)(i % p.HW);
      c = (int)((i / p.HW) % p.C);
      const int64_t n = i / ((int64_t)p.HW * p.C);
      src = (n * p.HW + hw) * p.C + c;
    } else {
      c = (int)(i % p.C);
      src = i;
    }
    p.out[i] = fmaf(__ldg(p.a + src), sc_s[c], sh_s[c]);
  }
}
// total threads of the grid are a multiple of C, so a thread keeps ONE channel over its grid-stride loop
__global__ void __launch_bounds__(256)
nbk_tail_bwd_kernel(const __grid_constant__ NbTail p) {
  __shared__ float mean_s[NB_MAXC], rstd_s[NB_MAXC];
  __shared__ float red[256][2];
  const int tid = threadIdx.x;
  const int grp = blockIdx.y;
  if (tid < p.C) {
    float sc, sh;
    nb_bn_consts(p.bn, p.C, tid, mean_s[tid], rstd_s[tid], sc, sh, nullptr, grp);
  }
  __syncthreads();
  // a group's elements start at a multiple of C, so the channel of a thread is the same in every group
  const int64_t gtotal = (int64_t)(p.N / gridDim.y) * p.HW * p.C, total = (grp + 1) * gtotal;
  const int c = (int)(((int64_t)blockIdx.x * 256 + tid) % p.C);
  float s1 = 0.f, s2 = 0.f;
  for (int64_t i = grp * gtotal + (int64_t)blockIdx.x * 256 + tid; i < total; i += (int64_t)gridDim.x * 256) {
    int64_t src = i;   // i enumerates g [n][hw][c]
    if (p.nchw) {
      const int64_t row = i / p.C;
      const int hw = (int)(row % p.HW);
      const int64_t n = row / p.HW;
      src = (n * p.C + c) * p.HW + hw;
    }
    const float gv = __ldg(p.dout + src);
    p.g[i] = gv;
    const float ah = (__ldg(p.a + i) - mean_s[c]) * rstd_s[c];
    s1 += gv;
    s2 = fmaf(gv, ah, s2);
  }
  red[tid][0] = s1;
  red[tid][1] = s2;
  __syncthreads();
  if (tid < p.C && tid < 256) {   // 256 % C == 0 or C % 256 == 0 (C <= 128 here): thread `tid` owns channel (block offset + tid) % C
    float t1 = 0.f, t2 = 0.f;
    for (int j = tid; j < 256; j += p.C) {
      t1 += red[j][0];
      t2 += red[j][1];
    }
    const int ch = (int)(((int64_t)blockIdx.x * 256 + tid) % p.C);
    atomicAdd(p.sums + (size_t)grp * 2 * p.C + ch, (double)t1);
    atomicAdd(p.sums + (size_t)grp * 2 * p.C + p.C + ch, (double)t2);
  }
}

static NbBn to_bn(const b200gan_nb_bn *b) {
  NbBn r;
  r.stats = b ? b->stats : nullptr;
  r.gamma = b ? b->gamma : nullptr;
  r.beta = b ? b->beta : nullptr;
  r.eps = b ? b->eps : 0.f;
  r.count = b ? b->count : 1.0;
  r.groups = (b && b->groups > 1) ? b->groups : 1;
  return r;
}

static bool is_pow2(int v) { return v > 0 && (v & (v - 1)) == 0; }

}  // namespace b200gan

using namespace b200gan;

namespace b200gan {
static int pow2ceil(int v) {
  int r = 1;
  while (r < v) r *= 2;
  return r;
}
constexpr size_t NB_SMEM_MAX = 200 * 1024;

struct NbPlan {
  NbTile t;
  int KT, PT;
  size_t smem;
  bool ok;
};
// Tile / register-tile choice of the staged kernels.  nout: channels this pass produces; wrow: weight floats per produced
// channel held in shared memory; (Ho, Wo): pixel grid the tiles cover; patch(TN, TR, TQ): floats of the staged window.
// Cost model (per FMA, relative): a thread's PT x KT tile needs PT + KT shared-memory float4 loads (4 wavefronts each)
// per 4 * PT * KT FMAs, against 4 FMA issue slots per cycle: max(1/4, (PT + KT) / (PT * KT)); divided by the SMs the
// grid can fill.
template <class F>
static NbPlan nb_plan(int nout, int64_t wrow, int cin, int N, int Ho, int Wo, int nclasses, bool allow_pt, int groups,
                      bool nclasses_is_dgrad, F patch) {
  NbPlan best;
  memset(&best, 0, sizeof(best));
  double best_cost = 1e30;
  int kts[3] = {0, 0, 0};
  if (nout % 16 == 0) { kts[0] = 16; kts[1] = 8; kts[2] = 4; }
  else if (nout % 8 == 0) { kts[0] = 8; kts[1] = 4; }
  else if (nout % 4 == 0) kts[0] = 4;
  else if (nout == 3 || nout == 6) kts[0] = nout;   // image-side data gradients: all channels of a pixel in one thread
  else kts[0] = 1;
  // tuning hook (tools/nb_sweep.py): B200GAN_NB_FORCE_{FPROP,DGRAD}="KT:PT:KG" restricts the search to one candidate
  int fkt = 0, fpt = 0, fkg = 0;
  if (const char *f = getenv(nclasses_is_dgrad ? "B200GAN_NB_FORCE_DGRAD" : "B200GAN_NB_FORCE_FPROP"))
    if (sscanf(f, "%d:%d:%d", &fkt, &fpt, &fkg) != 3) fkt = fpt = fkg = 0;
  for (int ki = 0; ki < 3 && kts[ki]; ++ki) {
    const int KT = kts[ki];
    for (int PT = (allow_pt || fpt > 1) ? 4 : 1; PT >= 1; PT /= 2) {
      for (int KG = 8; KG >= 1; KG /= 2) {
        const int KB = KG * KT;
        if (KB > nout || nout % KB != 0) continue;
        if (fkt && (KT != fkt || PT != fpt || KG != fkg)) continue;
        NbTile t;
        t.KG = KG; t.KB = KB; t.TP = PT * (256 / KG);
        t.TQ = pow2ceil(Wo) < 32 ? pow2ceil(Wo) : 32;
        if (t.TQ > t.TP) t.TQ = t.TP;
        t.TR = pow2ceil(Ho) < t.TP / t.TQ ? pow2ceil(Ho) : t.TP / t.TQ;
        t.TN = t.TP / (t.TQ * t.TR);
        if (t.TN > 1 && t.TN / 2 >= N) continue;           // tile mostly empty: a smaller PT / larger KG fits better
        if (groups > 1 && (N / groups) % t.TN != 0) continue;   // a tile must not straddle two statistics groups
        t.tiles_r = ceil_div(Ho, t.TR);
        t.tiles_q = ceil_div(Wo, t.TQ);
        const size_t floats = (size_t)((wrow * KB + 3) & ~(int64_t)3) + ((patch(t.TN, t.TR, t.TQ) + 3) & ~(size_t)3) +
                              2 * (size_t)((cin + 3) & ~3) + 8 * 2 * 16;
        const size_t smem = floats * sizeof(float);
        if (smem > NB_SMEM_MAX) continue;
        const int64_t blocks = (int64_t)ceil_div(N, t.TN) * t.tiles_r * t.tiles_q * (nout / KB) * nclasses;
        double cost = (double)(PT + KT) / (double)(PT * KT);
        if (cost < 0.25) cost = 0.25;
        cost /= (double)(blocks < num_sms() ? blocks : num_sms());
        // staging (a third of a block's life, latency-bound) only overlaps with another block's FMAs when two blocks
        // are resident per SM and the grid is large enough to put two on every SM
        if (smem > 110 * 1024 || blocks < 256) cost *= 1.4;
        if (cost < best_cost) {
          best_cost = cost;
          best.t = t; best.KT = KT; best.PT = PT; best.smem = smem; best.ok = true;
        }
      }
    }
  }
  return best;
}
static NbPlan nb_plan_fprop(const b200gan_conv_geom *g, int groups = 1) {
  const int CP = (g->C % 4 == 0) ? g->C + 4 : g->C;
  return nb_plan(g->K, (int64_t)g->R * g->S * g->C, g->C, g->N, g->P, g->Q, 1, g->R * g->S * g->C >= 16, groups, false,
                 [&](int TN, int TR, int TQ) {
    return (size_t)TN * ((TR - 1) * g->stride + g->R) * ((TQ - 1) * g->stride + g->S) * CP;
  });
}
static NbPlan nb_plan_dgrad(const b200gan_conv_geom *g, int groups = 1) {
  const int st = g->stride;
  const int Rm = ceil_div(g->R, st), Sm = ceil_div(g->S, st);
  return nb_plan(g->C, (int64_t)Rm * Sm * g->K, g->C, g->N, ceil_div(g->H, st), ceil_div(g->W, st), st * st, g->C >= 4,
                 groups, true, [&](int TN, int TR, int TQ) { return (size_t)TN * (TR + Rm - 1) * (TQ + Sm - 1) * (g->K + 4); });
}
}  // namespace b200gan

// geometry the fused chain takes: Conv2d, zero padding, no folded upsample, stride 1 or 2, <= 128 channels either side,
// K a power of two >= 4 (the channel-group mappings above), fp32 SIMT, and a tile plan that fits in shared memory.
extern "C" int b200gan_nb_supported(const b200gan_conv_geom *g);
// the chain layer can run with `groups` statistics groups: a tile plan exists whose tiles stay inside one group
extern "C" int b200gan_nb_groups_supported(const b200gan_conv_geom *g, int32_t groups) {
  if (!b200gan_nb_supported(g)) return 0;
  if (groups <= 1) return 1;
  if (groups > NB_MAX_GROUPS || g->N % groups != 0) return 0;
  return nb_plan_fprop(g, groups).ok && nb_plan_dgrad(g, groups).ok ? 1 : 0;
}

extern "C" int b200gan_nb_supported(const b200gan_conv_geom *g) {
  if (!g || validate_geom(g) != B200GAN_OK) return 0;
  if (g->transposed || g->up != 1 || g->pad_mode != B200GAN_PAD_ZERO) return 0;
  if (g->stride != 1 && g->stride != 2) return 0;
  if (g->pad_t != g->pad_b || g->pad_l != g->pad_r) return 0;
  if (g->C < 1 || g->C > NB_MAXC || g->K < 4 || g->K > NB_MAXC || !is_pow2(g->K)) return 0;
  if (g->C > 1 && (g->C % 4 != 0)) return 0;
  if (g->R * g->S != 9 && g->R * g->S != 16) return 0;
  if ((int64_t)g->R * g->S * g->C * g->K * 4 > (int64_t)512 * 1024) return 0;
  if (!nb_plan_fprop(g).ok || !nb_plan_dgrad(g).ok) return 0;
  return 1;
}

namespace b200gan {
static int nb_fprop2_launch(const b200gan_conv_geom *g, const NbBn &in_bn, float *rm, float *rv, long long *nbt,
                            float momentum, const float *x, const float *packed, const float *bias, int act, float slope,
                            const float *chan_scale, float *y, double *out_stats, int reflect, int rtf, int groups,
                            cudaStream_t st) {
  B2_CHECK_ARG(groups >= 1 && groups <= NB_MAX_GROUPS && g->N % groups == 0, "nb_fprop: bad statistics group count");
  const NbPlan pl = nb_plan_fprop(g, groups);
  B2_CHECK_ARG(pl.ok, "nb_fprop: no tile plan fits in shared memory");
  NbFprop2 q;
  q.x = x; q.wp = packed; q.bias = bias; q.cs = chan_scale; q.y = y; q.out_stats = out_stats;
  q.in_bn = in_bn; q.rm = rm; q.rv = rv; q.nbt = nbt; q.momentum = momentum;
  q.N = g->N; q.H = g->H; q.W = g->W; q.C = g->C; q.P = g->P; q.Q = g->Q; q.K = g->K; q.R = g->R; q.S = g->S;
  q.stride = g->stride; q.pad_t = g->pad_t; q.pad_l = g->pad_l; q.slope = slope; q.act = act;
  q.t = pl.t;
  q.PR = (pl.t.TR - 1) * g->stride + g->R;
  q.PC = (pl.t.TQ - 1) * g->stride + g->S;
  q.CP = (g->C % 4 == 0) ? g->C + 4 : g->C;
  q.reflect = reflect;
  q.rtf = rtf;
  q.groups = groups;
  dim3 grid((unsigned)(ceil_div(g->N, pl.t.TN) * pl.t.tiles_r * pl.t.tiles_q), (unsigned)(g->K / pl.t.KB));
#define NB_FPROP_CASE(KT_, PT_)                                                                              \
  if (pl.KT == KT_ && pl.PT == PT_) {                                                                        \
    static std::atomic<uint64_t> done{0};                                                                    \
    if (int e = ensure_dynamic_smem(nbk_fprop2_kernel<KT_, PT_>, (int)NB_SMEM_MAX, done)) return e;          \
    nbk_fprop2_kernel<KT_, PT_><<<grid, 256, pl.smem, st>>>(q);                                              \
  }
  NB_FPROP_CASE(16, 1) NB_FPROP_CASE(16, 2) NB_FPROP_CASE(16, 4)
  NB_FPROP_CASE(8, 1) NB_FPROP_CASE(8, 2) NB_FPROP_CASE(8, 4)
  NB_FPROP_CASE(4, 1) NB_FPROP_CASE(4, 2) NB_FPROP_CASE(4, 4)
#undef NB_FPROP_CASE
  B2_LAUNCH_CHECK();
  return B200GAN_OK;
}

// Stand-alone use of the staged forward kernel: layers with a handful of INPUT channels (the image side of every
// network: pix2pix/models.py:76,118  Conv2d(3 | 6, 64, 4, 2, 1); cyclegan/models.py:49-50  ReflectionPad2d(3) +
// Conv2d(3, 64, 7)), where a tensor-core tile has no K dimension to speak of.
bool nb_plain_fprop_ok(const b200gan_conv_geom *g) {
  if (!g || g->transposed || g->up != 1) return false;
  if (g->pad_mode != B200GAN_PAD_ZERO && g->pad_mode != B200GAN_PAD_REFLECT) return false;
  if (g->stride != 1 && g->stride != 2) return false;
  if (g->C < 1 || g->C > 8 || g->K < 16 || g->K > NB_MAXC || g->K % 16 != 0) return false;
  if (g->R != g->S || (g->R != 3 && g->R != 4 && g->R != 7)) return false;
  return nb_plan_fprop(g).ok;
}
int nb_plain_fprop(const b200gan_conv_geom *g, const b200gan_epilogue *ep, const float *x, const float *packed, float *y,
                   cudaStream_t st) {
  if ((int64_t)g->N * g->P * g->Q == 0) return B200GAN_OK;
  NbBn none = to_bn(nullptr);
  return nb_fprop2_launch(g, none, nullptr, nullptr, nullptr, 0.f, x, packed, ep ? ep->bias : nullptr,
                          ep ? ep->act : B200GAN_ACT_NONE, ep ? ep->slope : 0.f, ep ? ep->chan_scale : nullptr, y, nullptr,
                          g->pad_mode == B200GAN_PAD_REFLECT ? 1 : 0, ep ? ep->round_tf32 : 0, 1, st);
}
}  // namespace b200gan

extern "C" int b200gan_nb_fprop(const b200gan_conv_geom *g, const b200gan_nb_bn *in_bn, float *running_mean,
                                float *running_var, int64_t *num_batches_tracked, float momentum, const float *x,
                                const float *packed, const float *bias, int32_t act, float slope, const float *chan_scale,
                                float *y, double *out_stats, int32_t groups, void *stream) {
  B2_CHECK_ARG(b200gan_nb_supported(g), "nb_fprop: unsupported geometry");
  if (groups < 1) groups = 1;
  B2_CHECK_ARG(!(in_bn && in_bn->stats) || (in_bn->groups > 1 ? in_bn->groups : 1) == groups,
               "nb_fprop: the input edge and the call disagree on the statistics group count");
  B2_CHECK_ARG(x && packed && y, "nb_fprop: null pointer");
  B2_CHECK_ARG((((uintptr_t)x | (uintptr_t)packed | (uintptr_t)y) & 15) == 0, "nb_fprop: pointers must be 16-byte aligned");
  cudaStream_t st = as_stream(stream);
  if (out_stats) B2_CUDA(cudaMemsetAsync(out_stats, 0, (size_t)groups * 2 * g->K * sizeof(double), st));
  if ((int64_t)g->N * g->P * g->Q == 0) return B200GAN_OK;
  return nb_fprop2_launch(g, to_bn(in_bn), running_mean, running_var, reinterpret_cast<long long *>(num_batches_tracked),
                          momentum, x, packed, bias, act, slope, chan_scale, y, out_stats, 0, 0, groups, st);
}

extern "C" int b200gan_nb_dz(int32_t N, int64_t PQ, int32_t K, const float *g, const float *a, const float *chan_scale,
                             int32_t act, float slope, const b200gan_nb_bn *out_bn, const double *sums, float *dz, float *db,
                             void *stream) {
  B2_CHECK_ARG(g && a && dz && N > 0 && PQ > 0, "nb_dz: bad arguments");
  B2_CHECK_ARG(K >= 4 && K <= NB_MAXC && is_pow2(K), "nb_dz: K must be a power of two in [4, 128]");
  B2_CHECK_ARG(!(out_bn && out_bn->stats) || sums, "nb_dz: BatchNorm backward needs the sums");
  cudaStream_t st = as_stream(stream);
  if (db) B2_CUDA(cudaMemsetAsync(db, 0, (size_t)K * sizeof(float), st));
  NbDz p;
  p.g = g; p.a = a; p.cs = chan_scale; p.dz = dz; p.db = db; p.out_bn = to_bn(out_bn); p.sums = sums;
  p.rows = (int64_t)N * PQ; p.PQ = PQ; p.K = K; p.slope = slope; p.act = act;
  const int rows_per_block = 256 / (K / 4);
  const int groups = p.out_bn.stats ? p.out_bn.groups : 1;
  B2_CHECK_ARG(N % groups == 0, "nb_dz: the batch must split evenly into the statistics groups");
  int64_t blocks = ceil_div64(p.rows / groups, rows_per_block * 4);
  if (blocks > num_sms() * 4 / groups) blocks = num_sms() * 4 / groups;
  if (blocks < 1) blocks = 1;
  nbk_dz_kernel<<<dim3((unsigned)blocks, (unsigned)groups), 256, 0, st>>>(p);
  B2_LAUNCH_CHECK();
  return B200GAN_OK;
}

namespace b200gan {
// The weight-gradient kernel alone takes more geometries than the chain: any C <= 128, K a multiple of 4 up to 128.
bool nb_wgrad_ok(const b200gan_conv_geom *g) {
  if (!g || g->transposed || g->up != 1) return false;
  if (g->pad_mode != B200GAN_PAD_ZERO && g->pad_mode != B200GAN_PAD_REFLECT) return false;
  if (g->stride != 1 && g->stride != 2) return false;
  if (g->pad_t != g->pad_b || g->pad_l != g->pad_r) return false;
  if (g->C < 1 || g->C > 512 || g->K < 1 || g->K > NB_MAXC) return false;
  if (g->C > NB_MAXC && g->K > 8) return false;   // wide inputs only for the few-output-channel layers
  if (g->R * g->S != 9 && g->R * g->S != 16 && !(g->R == 7 && g->S == 7)) return false;
  const int PR = g->R, PC = g->S;  // smallest tile (one pixel) must fit
  return (size_t)(PR * PC * g->C + g->K + 2 * g->C + 8 + 2 * 256 + 8) * sizeof(float) <= 96 * 1024;
}
int nb_wgrad_run(const b200gan_conv_geom *g, const b200gan_nb_bn *in_bn, const float *x, const float *dz, float *dw,
                 float *workspace, cudaStream_t st);
size_t nb_wgrad_workspace_floats(const b200gan_conv_geom *g);
int nb_wgrad_reduce(const float *ws, float *dw, int elems, int nslabs, cudaStream_t st);

struct NbWgPlan {
  int TN, TR, TQ, SPB, PS, nsets, nchunks, gx, row_mode;
  size_t smem;
  bool use_ws;
};
static NbWgPlan nb_wgrad_plan(const b200gan_conv_geom *g) {
  NbWgPlan w;
  // room for the scale / shift tables of up to NB_MAX_GROUPS statistics groups, whatever the call uses: the plan (and
  // with it the workspace size) must not depend on the group count
  const int groups = g->C <= NB_MAXC ? NB_MAX_GROUPS : 1;
  w.row_mode = (g->R * g->S > 16) ? 1 : 0;
  w.nsets = g->C * ((g->K + 3) / 4) * (w.row_mode ? g->R : 1);
  int spb = 256;
  if (w.nsets < 256) {  // fewer sets than threads: several threads share a set and split the pixels of a tile
    spb = 1;
    while (spb < w.nsets) spb *= 2;     // smallest power of two >= nsets (256 % spb == 0)
  }
  w.SPB = spb;
  w.PS = 256 / spb;
  w.nchunks = ceil_div(w.nsets, spb);
  // output tile: up to 128 pixels, whole rows when the map is narrow, several whole images when they are small; the
  // patch must fit in shared memory
  w.TQ = g->Q < 32 ? g->Q : 32;
  w.TR = 128 / w.TQ;
  if (w.TR > g->P) w.TR = g->P;
  w.TN = 1;
  if (w.TR == g->P && w.TQ == g->Q) {
    w.TN = 128 / (g->P * g->Q);
    if (w.TN > g->N) w.TN = g->N;
    if (w.TN < 1) w.TN = 1;
  }
  auto tile_bytes = [&](int TN, int TR, int TQ) {
    const int PR = (TR - 1) * g->stride + g->R, PC = (TQ - 1) * g->stride + g->S;
    const size_t tables = (size_t)((2 * spb + TN * TR * TQ + 3) & ~3);
    return (tables + (((size_t)TN * PR * PC * g->C + 3) & ~(size_t)3) + (size_t)TN * TR * TQ * ((g->K + 3) / 4 * 4) +
            2 * (size_t)groups * ((g->C + 3) & ~3)) * sizeof(float);
  };
  while (w.TN > 1 && tile_bytes(w.TN, w.TR, w.TQ) > 96 * 1024) w.TN = (w.TN + 1) / 2;
  while (w.TR > 1 && tile_bytes(w.TN, w.TR, w.TQ) > 96 * 1024) w.TR = (w.TR + 1) / 2;
  while (w.TQ > 1 && tile_bytes(w.TN, w.TR, w.TQ) > 96 * 1024) w.TQ = (w.TQ + 1) / 2;
  w.smem = tile_bytes(w.TN, w.TR, w.TQ);
  const int ntiles = ceil_div(g->N, w.TN) * ceil_div(g->P, w.TR) * ceil_div(g->Q, w.TQ);
  w.gx = (2 * num_sms()) / w.nchunks;
  if (w.gx < 8) w.gx = 8;
  if (w.gx > ntiles) w.gx = ntiles;
  if (w.gx < 1) w.gx = 1;
  const int taps = w.row_mode ? g->S : g->R * g->S;
  // phase reduction buffer, reuses the tile memory behind the tables
  const size_t red = ((size_t)((2 * spb + w.TN * w.TR * w.TQ + 3) & ~3) + (size_t)256 * 4 * (taps | 1)) * sizeof(float);
  if (w.smem < red) w.smem = red;
  // one value per weight and block: beyond ~1e5 same-address atomics per launch the slabs + reduce kernel are faster
  w.use_ws = (int64_t)w.gx * g->K * g->C * g->R * g->S > 100000;
  return w;
}
size_t nb_wgrad_workspace_floats(const b200gan_conv_geom *g) {
  if (!nb_wgrad_ok(g) || (int64_t)g->N * g->P * g->Q == 0) return 0;
  const NbWgPlan w = nb_wgrad_plan(g);
  return w.use_ws ? (size_t)w.gx * g->K * g->C * g->R * g->S : 0;
}
}  // namespace b200gan

extern "C" size_t b200gan_nb_wgrad_workspace_floats(const b200gan_conv_geom *g) {
  if (!g || validate_geom(g) != B200GAN_OK) return 0;
  return nb_wgrad_workspace_floats(g);
}

extern "C" int b200gan_nb_wgrad(const b200gan_conv_geom *g, const b200gan_nb_bn *in_bn, const float *x, const float *dz,
                                float *dw, float *workspace, void *stream) {
  B2_CHECK_ARG(validate_geom(g) == B200GAN_OK && nb_wgrad_ok(g), "nb_wgrad: unsupported geometry");
  B2_CHECK_ARG(x && dz && dw, "nb_wgrad: null pointer");
  return nb_wgrad_run(g, in_bn, x, dz, dw, workspace, as_stream(stream));
}

int b200gan::nb_wgrad_run(const b200gan_conv_geom *g, const b200gan_nb_bn *in_bn, const float *x, const float *dz,
                          float *dw, float *workspace, cudaStream_t st) {
  const int dw_elems = g->K * g->C * g->R * g->S;
  if ((int64_t)g->N * g->P * g->Q == 0) {
    B2_CUDA(cudaMemsetAsync(dw, 0, (size_t)dw_elems * sizeof(float), st));
    return B200GAN_OK;
  }
  const int groups = (in_bn && in_bn->stats && in_bn->groups > 1) ? in_bn->groups : 1;
  B2_CHECK_ARG(g->N % groups == 0, "nb_wgrad: the batch must split evenly into the statistics groups");
  B2_CHECK_ARG(groups == 1 || (groups <= NB_MAX_GROUPS && g->C <= NB_MAXC), "nb_wgrad: too many statistics groups");
  const NbWgPlan w = nb_wgrad_plan(g);
  B2_CHECK_ARG(w.smem <= 96 * 1024, "nb_wgrad: tile does not fit in shared memory");
  const bool use_ws = w.use_ws && workspace != nullptr;
  if (!use_ws) B2_CUDA(cudaMemsetAsync(dw, 0, (size_t)dw_elems * sizeof(float), st));
  NbWgrad p;
  p.x = x; p.dz = dz; p.dw = dw; p.ws = use_ws ? workspace : nullptr; p.dw_elems = dw_elems; p.in_bn = to_bn(in_bn);
  p.N = g->N; p.H = g->H; p.W = g->W; p.C = g->C; p.P = g->P; p.Q = g->Q; p.K = g->K; p.R = g->R; p.S = g->S;
  p.stride = g->stride; p.pad_t = g->pad_t; p.pad_l = g->pad_l;
  p.TN = w.TN; p.TR = w.TR; p.TQ = w.TQ;
  p.tiles_r = ceil_div(g->P, p.TR);
  p.tiles_q = ceil_div(g->Q, p.TQ);
  p.PR = (p.TR - 1) * g->stride + g->R;
  p.PC = (p.TQ - 1) * g->stride + g->S;
  p.row_mode = w.row_mode;
  p.reflect = g->pad_mode == B200GAN_PAD_REFLECT ? 1 : 0;
  p.nsets = w.nsets;
  p.SPB = w.SPB;
  p.PS = w.PS;
  const int taps = g->R * g->S;
  static std::atomic<uint64_t> done9{0}, done16{0}, done7{0};
  dim3 grid((unsigned)w.gx, (unsigned)w.nchunks);
  if (p.row_mode) {
    if (int e = ensure_dynamic_smem(nbk_wgrad_kernel<7>, 96 * 1024, done7)) return e;
    nbk_wgrad_kernel<7><<<grid, 256, w.smem, st>>>(p);
  } else if (taps == 9) {
    if (int e = ensure_dynamic_smem(nbk_wgrad_kernel<9>, 96 * 1024, done9)) return e;
    nbk_wgrad_kernel<9><<<grid, 256, w.smem, st>>>(p);
  } else {
    if (int e = ensure_dynamic_smem(nbk_wgrad_kernel<16>, 96 * 1024, done16)) return e;
    nbk_wgrad_kernel<16><<<grid, 256, w.smem, st>>>(p);
  }
  B2_LAUNCH_CHECK();
  if (use_ws) return nb_wgrad_reduce(workspace, dw, dw_elems, w.gx, st);
  return B200GAN_OK;
}

int b200gan::nb_wgrad_reduce(const float *ws, float *dw, int elems, int nslabs, cudaStream_t st) {
  nbk_wgrad_reduce_kernel<<<(unsigned)ceil_div(elems, 32), 256, 0, st>>>(ws, dw, elems, nslabs);
  B2_LAUNCH_CHECK();
  return B200GAN_OK;
}

namespace b200gan {
static int nb_dgrad2_launch(const b200gan_conv_geom *g, const float *dz, const float *packed, const NbBn &in_bn,
                            const float *a_prev, float *g_out, double *sums, cudaStream_t st) {
  const int st_ = g->stride;
  const int groups = in_bn.stats ? in_bn.groups : 1;
  B2_CHECK_ARG(groups <= NB_MAX_GROUPS && g->N % groups == 0, "nb_dgrad: bad statistics group count");
  const NbPlan pl = nb_plan_dgrad(g, groups);
  B2_CHECK_ARG(pl.ok, "nb_dgrad: no tile plan fits in shared memory");
  NbDgrad2 q;
  q.dz = dz; q.wp = packed; q.a_prev = a_prev; q.g_out = g_out; q.sums = sums; q.in_bn = in_bn;
  q.N = g->N; q.H = g->H; q.W = g->W; q.C = g->C; q.P = g->P; q.Q = g->Q; q.K = g->K; q.R = g->R; q.S = g->S;
  q.stride = g->stride; q.pad_t = g->pad_t; q.pad_l = g->pad_l;
  q.t = pl.t;
  q.KP = g->K + 4;
  const int Rm = ceil_div(g->R, st_), Sm = ceil_div(g->S, st_);
  q.PRm = pl.t.TR + Rm - 1;
  q.PCm = pl.t.TQ + Sm - 1;
  q.tapsm = Rm * Sm;
  dim3 grid((unsigned)(ceil_div(g->N, pl.t.TN) * pl.t.tiles_r * pl.t.tiles_q), (unsigned)(g->C / pl.t.KB),
            (unsigned)(st_ * st_));
#define NB_DGRAD_CASE(KT_, PT_)                                                                              \
  if (pl.KT == KT_ && pl.PT == PT_) {                                                                        \
    static std::atomic<uint64_t> done{0};                                                                    \
    if (int e = ensure_dynamic_smem(nbk_dgrad2_kernel<KT_, PT_>, (int)NB_SMEM_MAX, done)) return e;          \
    nbk_dgrad2_kernel<KT_, PT_><<<grid, 256, pl.smem, st>>>(q);                                              \
  }
  NB_DGRAD_CASE(16, 1) NB_DGRAD_CASE(16, 2) NB_DGRAD_CASE(16, 4)
  NB_DGRAD_CASE(8, 1) NB_DGRAD_CASE(8, 2) NB_DGRAD_CASE(8, 4)
  NB_DGRAD_CASE(4, 1) NB_DGRAD_CASE(4, 2) NB_DGRAD_CASE(4, 4)
  NB_DGRAD_CASE(6, 1) NB_DGRAD_CASE(6, 2) NB_DGRAD_CASE(6, 4)
  NB_DGRAD_CASE(3, 1) NB_DGRAD_CASE(3, 2) NB_DGRAD_CASE(3, 4)
  NB_DGRAD_CASE(1, 1)
#undef NB_DGRAD_CASE
  B2_LAUNCH_CHECK();
  return B200GAN_OK;
}

// Stand-alone data gradient of a layer with a handful of INPUT channels (the discriminators' first conv, whose input
// gradient flows back into the generator: pix2pix/models.py:118 Conv2d(6, 64, 4, 2, 1); cyclegan/models.py:116).
bool nb_plain_dgrad_ok(const b200gan_conv_geom *g) {
  if (!g || g->transposed || g->up != 1 || g->pad_mode != B200GAN_PAD_ZERO) return false;
  if (g->stride != 1 && g->stride != 2) return false;
  if (g->pad_t != g->pad_b || g->pad_l != g->pad_r) return false;
  if (g->C < 1 || g->C > 8 || (g->C != 1 && g->C != 3 && g->C != 6 && g->C % 4 != 0)) return false;
  if (g->K < 4 || g->K > NB_MAXC || g->K % 4 != 0) return false;
  if (g->R * g->S != 9 && g->R * g->S != 16 && !(g->R == 7 && g->S == 7 && g->stride == 1)) return false;
  return nb_plan_dgrad(g).ok;
}
int nb_plain_dgrad(const b200gan_conv_geom *g, const float *dy, const float *packed, float *dx, cudaStream_t st) {
  if ((int64_t)g->N * g->H * g->W == 0) return B200GAN_OK;
  NbBn none = to_bn(nullptr);
  return nb_dgrad2_launch(g, dy, packed, none, nullptr, dx, nullptr, st);
}
}  // namespace b200gan

extern "C" int b200gan_nb_dgrad(const b200gan_conv_geom *g, const float *dz, const float *packed,
                                const b200gan_nb_bn *in_bn, const float *a_prev, float *g_out, double *sums,
                                void *stream) {
  B2_CHECK_ARG(b200gan_nb_supported(g), "nb_dgrad: unsupported geometry");
  B2_CHECK_ARG(dz && packed && g_out, "nb_dgrad: null pointer");
  B2_CHECK_ARG(!sums || (in_bn && in_bn->stats && a_prev), "nb_dgrad: sums need the upstream BatchNorm and its input");
  cudaStream_t st = as_stream(stream);
  const int dgroups = (in_bn && in_bn->stats && in_bn->groups > 1) ? in_bn->groups : 1;
  if (sums) B2_CUDA(cudaMemsetAsync(sums, 0, (size_t)dgroups * 2 * g->C * sizeof(double), st));
  if ((int64_t)g->N * g->H * g->W == 0) return B200GAN_OK;
  return nb_dgrad2_launch(g, dz, packed, to_bn(in_bn), a_prev, g_out, sums, st);
}

static int tail_grid(int64_t total, int C) {
  int64_t blocks = ceil_div64(total, 256 * 4);
  if (blocks > num_sms() * 4) blocks = num_sms() * 4;
  if (blocks < 1) blocks = 1;
  // total threads a multiple of C (C <= 128 divides 256 when it is a power of two; otherwise round the block count)
  while ((blocks * 256) % C != 0) ++blocks;
  return (int)blocks;
}

extern "C" int b200gan_nb_tail_fwd(int32_t N, int32_t HW, int32_t C, const b200gan_nb_bn *bn, float *running_mean,
                                   float *running_var, int64_t *num_batches_tracked, float momentum, const float *a,
                                   float *out, int32_t nchw, void *stream) {
  B2_CHECK_ARG(bn && bn->stats && a && out && N > 0 && HW > 0 && C > 0 && C <= NB_MAXC, "nb_tail_fwd: bad arguments");
  NbTail p;
  memset(&p, 0, sizeof(p));
  p.a = a; p.out = out; p.bn = to_bn(bn); p.rm = running_mean; p.rv = running_var;
  p.nbt = reinterpret_cast<long long *>(num_batches_tracked); p.momentum = momentum;
  p.N = N; p.HW = HW; p.C = C; p.nchw = nchw;
  const int groups = p.bn.groups;
  B2_CHECK_ARG(groups <= NB_MAX_GROUPS && N % groups == 0, "nb_tail_fwd: bad statistics group count");
  nbk_tail_fwd_kernel<<<dim3((unsigned)tail_grid((int64_t)(N / groups) * HW * C, C), (unsigned)groups), 256, 0,
                        as_stream(stream)>>>(p);
  B2_LAUNCH_CHECK();
  return B200GAN_OK;
}

extern "C" int b200gan_nb_tail_bwd(int32_t N, int32_t HW, int32_t C, const b200gan_nb_bn *bn, const float *a,
                                   const float *dout, int32_t nchw, float *g, double *sums, void *stream) {
  B2_CHECK_ARG(bn && bn->stats && a && dout && g && sums && N > 0 && HW > 0 && C > 0 && C <= NB_MAXC,
               "nb_tail_bwd: bad arguments");
  B2_CHECK_ARG(256 % C == 0, "nb_tail_bwd: C must divide 256");
  cudaStream_t st = as_stream(stream);
  const int groups = (bn->groups > 1) ? bn->groups : 1;
  B2_CHECK_ARG(groups <= NB_MAX_GROUPS && N % groups == 0, "nb_tail_bwd: bad statistics group count");
  B2_CUDA(cudaMemsetAsync(sums, 0, (size_t)groups * 2 * C * sizeof(double), st));
  NbTail p;
  memset(&p, 0, sizeof(p));
  p.a = a; p.dout = dout; p.g = g; p.sums = sums; p.bn = to_bn(bn);
  p.N = N; p.HW = HW; p.C = C; p.nchw = nchw;
  nbk_tail_bwd_kernel<<<dim3((unsigned)tail_grid((int64_t)(N / groups) * HW * C, C), (unsigned)groups), 256, 0, st>>>(p);
  B2_LAUNCH_CHECK();
  return B200GAN_OK;
}
