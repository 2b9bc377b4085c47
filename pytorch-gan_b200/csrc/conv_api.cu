// conv_api.cu -- C-ABI entry points for convolution: validation, weight packing, and the
// choice between the wgmma TF32 kernels (conv_tc.cu / wgrad_tc.cu) and the fp32 SIMT kernels
// (conv_simt.cu).  See include/b200gan.h for the contract and the reference call sites.
#include "common.cuh"
#include <atomic>
#include <mutex>
#include <string.h>
#include <stdlib.h>

namespace b200gan {

// conv_simt.cu
int simt_gather_gemm(int N, int H, int W, int C, int P, int Q, int K, int R, int S, int stride,
                     int pad_t, int pad_l, int pad_mode, int up, int mode,
                     const b200gan_epilogue *ep, const float *x, const float *wp, float *y,
                     cudaStream_t st);
int simt_wgrad(int N, int H, int W, int Cg, int P, int Q, int Cd, int R, int S, int stride,
               int pad_t, int pad_l, int pad_mode, int up, const float *xg, const float *dn,
               float *dw, cudaStream_t st);
int simt_colsum(const float *x, float *out, int64_t M, int C, cudaStream_t st);
// narrow_block.cu: shared-memory staged weight gradient of the narrow layers
bool nb_wgrad_ok(const b200gan_conv_geom *g);
int nb_wgrad_run(const b200gan_conv_geom *g, const b200gan_nb_bn *in_bn, const float *x, const float *dz, float *dw,
                 float *workspace, cudaStream_t st);
size_t nb_wgrad_workspace_floats(const b200gan_conv_geom *g);
// narrow_block.cu: the staged SIMT kernels on their own, for layers with <= 8 input channels
bool nb_plain_fprop_ok(const b200gan_conv_geom *g);
int nb_plain_fprop(const b200gan_conv_geom *g, const b200gan_epilogue *ep, const float *x, const float *packed, float *y,
                   cudaStream_t st);
bool nb_plain_dgrad_ok(const b200gan_conv_geom *g);
int nb_plain_dgrad(const b200gan_conv_geom *g, const float *dy, const float *packed, float *dx, cudaStream_t st);
// fewk.cu: stride-1 convs with K <= 4 output channels (lanes = input channels)
bool fewk_ok(const b200gan_conv_geom *g, int pas);
int fewk_fprop(const b200gan_conv_geom *g, const b200gan_epilogue *ep, const float *x, const float *packed, float *y,
               cudaStream_t st);
int fewk_dgrad(const b200gan_conv_geom *g, const float *dy, const float *packed, float *dx, cudaStream_t st);
int fewk_wgrad(const b200gan_conv_geom *g, const float *x, const float *dy, float *dw, float *workspace, cudaStream_t st);
size_t fewk_wgrad_workspace_floats(const b200gan_conv_geom *g);
// conv_tc.cu / wgrad_tc.cu
int tc_supported(const b200gan_conv_geom *g, int pass);
int tc_fprop(const b200gan_conv_geom *g, const b200gan_epilogue *ep, const float *x,
             const float *packed, float *y, cudaStream_t st);
int tc_dgrad(const b200gan_conv_geom *g, const float *dy, const float *packed, float *dx,
             cudaStream_t st);
size_t tc_wgrad_workspace_floats(const b200gan_conv_geom *g);
int tc_wgrad(const b200gan_conv_geom *g, const float *x, const float *dy, float *dw, float *ws,
             cudaStream_t st);

static thread_local char g_err[512] = "";
void set_error(const char *fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

int num_sms() {
  static std::atomic<int> cache[64];
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) {
    cudaGetLastError();
    return 132;
  }
  int v = cache[dev].load(std::memory_order_relaxed);
  if (v > 0) return v;
  if (cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || v <= 0) {
    cudaGetLastError();
    return 132;
  }
  cache[dev].store(v, std::memory_order_relaxed);
  return v;
}

int validate_geom(const b200gan_conv_geom *g) {
  B2_CHECK_ARG(g != nullptr, "conv: null geometry");
  B2_CHECK_ARG(g->N >= 0 && g->H > 0 && g->W > 0 && g->C > 0 && g->K > 0 && g->R > 0 && g->S > 0,
               "conv: bad dims N=%d H=%d W=%d C=%d K=%d R=%d S=%d", g->N, g->H, g->W, g->C, g->K,
               g->R, g->S);
  B2_CHECK_ARG(g->stride >= 1, "conv: stride must be >= 1");
  B2_CHECK_ARG(g->up == 1 || g->up == 2, "conv: up must be 1 or 2");
  B2_CHECK_ARG(g->pad_t >= 0 && g->pad_l >= 0 && g->pad_b >= 0 && g->pad_r >= 0, "conv: negative padding");
  int P, Q;
  if (g->transposed) {
    B2_CHECK_ARG(g->up == 1 && g->pad_mode == B200GAN_PAD_ZERO,
                 "conv: ConvTranspose2d cannot fold upsample / reflection padding");
    B2_CHECK_ARG(g->pad_t == g->pad_b && g->pad_l == g->pad_r, "conv: ConvTranspose2d padding must be symmetric");
    P = (g->H - 1) * g->stride - 2 * g->pad_t + g->R;
    Q = (g->W - 1) * g->stride - 2 * g->pad_l + g->S;
  } else {
    int Hv = g->H * g->up, Wv = g->W * g->up;
    if (g->pad_mode == B200GAN_PAD_REFLECT)
      B2_CHECK_ARG(g->pad_t < Hv && g->pad_b < Hv && g->pad_l < Wv && g->pad_r < Wv,
                   "conv: reflection padding must be smaller than the input");
    int Hp = Hv + g->pad_t + g->pad_b, Wp = Wv + g->pad_l + g->pad_r;
    B2_CHECK_ARG(Hp >= g->R && Wp >= g->S, "conv: filter larger than padded input");
    P = (Hp - g->R) / g->stride + 1;
    Q = (Wp - g->S) / g->stride + 1;
  }
  B2_CHECK_ARG(P == g->P && Q == g->Q, "conv: output size mismatch: expected %dx%d, got %dx%d", P, Q,
               g->P, g->Q);
  B2_CHECK_ARG((int64_t)g->N * g->H * g->W * g->C < (1LL << 40) && (int64_t)g->N * P * Q * g->K < (1LL << 40),
               "conv: tensor too large");
  return B200GAN_OK;
}

// ---- weight packing ---------------------------------------------------------------------------
// 3x3 s1 p1 conv behind a nearest x2 upsample == four 2x2 "phase" filters on the low-res input:
// out[2i+a][2j+b] = sum_{dr,ds in {0,1}} x[i+a-1+dr][j+b-1+ds] * Wf[a][b][dr][ds]
// Wf[a][b][dr][ds] = sum_{r in Rset(a,dr)} sum_{s in Rset(b,ds)} W[r][s],
// Rset(0,0)={0} Rset(0,1)={1,2} Rset(1,0)={0,1} Rset(1,1)={2}.
__device__ __forceinline__ void up2_rset(int a, int d, int &lo, int &hi) {
  if (a == 0) { lo = d == 0 ? 0 : 1; hi = d == 0 ? 0 : 2; }
  else        { lo = d == 0 ? 0 : 2; hi = d == 0 ? 1 : 2; }
}

// ---- every packed copy of an optimizer's weights in ONE launch ---------------------------------------------------
// The weights change once per optimizer step, and every conv keeps 1-2 packed copies (fprop / dgrad layouts): per-copy
// pack launches were 21 of the DCGAN step's launches.  The job table travels as a kernel argument; a single copy
// (b200gan_pack_weights) is a table of one job.
constexpr int PACK_MAX_JOBS = 24;
constexpr int PACK_CHUNK = 256 * 8;  // packed elements per block
struct PackJob {
  const float *src;
  float *dst;
  int R, S, Cin, Cout, transposed, kind;
  int tiles_ci;     // > 0: tile mode, a block transposes a 32 (Cout) x 8 (Cin) x taps tile through shared memory
  long long total;
};
constexpr int PACK_CO_T = 32, PACK_CI_T = 8, PACK_RS_MAX = 16;
struct PackTable {
  PackJob job[PACK_MAX_JOBS];
  int block_begin[PACK_MAX_JOBS + 1];
  int count;
};
__device__ __forceinline__ float pack_element(const PackJob &j, long long i) {
  const bool up2 = j.kind == B200GAN_PACK_TC_FPROP_UP2 || j.kind == B200GAN_PACK_TC_DGRAD_UP2;
  // order 0: dst[t][ci][co], order 1: dst[t][co][ci]
  const int order = (j.kind == B200GAN_PACK_SIMT_DGRAD || j.kind == B200GAN_PACK_TC_FPROP || j.kind == B200GAN_PACK_TC_FPROP_UP2) ? 1 : 0;
  int ci, co;
  long long t;
  if (order == 0) { co = (int)(i % j.Cout); t = i / j.Cout; ci = (int)(t % j.Cin); t /= j.Cin; }
  else            { ci = (int)(i % j.Cin);  t = i / j.Cin;  co = (int)(t % j.Cout); t /= j.Cout; }
  if (!up2) {
    const int s = (int)(t % j.S), r = (int)(t / j.S);
    const long long si = j.transposed ? (((long long)ci * j.Cout + co) * j.R + r) * j.S + s
                                      : (((long long)co * j.Cin + ci) * j.R + r) * j.S + s;
    const float v = j.src[si];
    return (j.kind == B200GAN_PACK_TC_FPROP || j.kind == B200GAN_PACK_TC_DGRAD) ? round_tf32(v) : v;
  }
  const int tap = (int)(t % 4), ph = (int)(t / 4);
  const int a = ph >> 1, b = ph & 1, dr = tap >> 1, ds = tap & 1;
  int rlo, rhi, slo, shi;
  up2_rset(a, dr, rlo, rhi);
  up2_rset(b, ds, slo, shi);
  float v = 0.f;
  for (int r = rlo; r <= rhi; ++r)
    for (int s = slo; s <= shi; ++s) v += j.src[(((long long)co * j.Cin + ci) * 3 + r) * 3 + s];
  return round_tf32(v);
}
// Tile mode.  The parameter layout keeps the taps innermost ([Cout][Cin][R][S]) and every packed layout keeps them
// outermost, so a thread-per-destination-element gather reads 4 bytes out of every 32-byte sector it touches and the
// rest of the sector is needed by blocks far away (measured: 557 us for the 54 M U-Net weights, 1.5 TB/s of useful
// traffic).  Here a block loads whole contiguous runs (8 input channels x all taps of one output channel = 512 B for a
// 4x4 filter) into shared memory and writes 128-byte (order 0) / 32-byte (order 1) segments per tap.
// RS_ = R * S as a compile-time constant (16: 4x4, 9: 3x3; 0: run time): every index decomposition below divides by it, and
// with run-time divisors the kernel was bound by integer division (no faster than the element-wise gather)
template <int RS_>
__device__ __forceinline__ void pack_tile(const PackJob &j, int tile, float (*s)[PACK_CI_T * PACK_RS_MAX + 1]) {
  const int RS = RS_ ? RS_ : j.R * j.S;
  const int tci = tile % j.tiles_ci, tco = tile / j.tiles_ci;
  const int co0 = tco * PACK_CO_T, ci0 = tci * PACK_CI_T;
  const int tid = threadIdx.x;
  const int run = PACK_CI_T * RS;
  if (!j.transposed) {
    for (int e = tid; e < PACK_CO_T * run; e += 256) {
      const int co_l = e / run, rem = e - co_l * run;
      const int ci_l = rem / RS;
      float v = 0.f;
      if (co0 + co_l < j.Cout && ci0 + ci_l < j.Cin) v = j.src[((long long)(co0 + co_l) * j.Cin + ci0) * RS + rem];
      s[co_l][rem] = v;
    }
  } else {  // ConvTranspose2d parameter: [Cin][Cout][R][S]
    const int crun = PACK_CO_T * RS;
    for (int e = tid; e < PACK_CI_T * crun; e += 256) {
      const int ci_l = e / crun, rem = e - ci_l * crun;
      const int co_l = rem / RS, t = rem - co_l * RS;
      float v = 0.f;
      if (co0 + co_l < j.Cout && ci0 + ci_l < j.Cin) v = j.src[((long long)(ci0 + ci_l) * j.Cout + co0) * RS + rem];
      s[co_l][ci_l * RS + t] = v;
    }
  }
  __syncthreads();
  const bool up2 = j.kind == B200GAN_PACK_TC_FPROP_UP2 || j.kind == B200GAN_PACK_TC_DGRAD_UP2;
  const bool rtf = up2 || j.kind == B200GAN_PACK_TC_FPROP || j.kind == B200GAN_PACK_TC_DGRAD;
  const int order = (j.kind == B200GAN_PACK_SIMT_DGRAD || j.kind == B200GAN_PACK_TC_FPROP || j.kind == B200GAN_PACK_TC_FPROP_UP2) ? 1 : 0;
  const int taps_out = up2 ? 16 : RS;
  for (int e = tid; e < PACK_CO_T * PACK_CI_T * taps_out; e += 256) {
    int co_l, ci_l, t;
    if (order == 0) { co_l = e % PACK_CO_T; ci_l = (e / PACK_CO_T) % PACK_CI_T; t = e / (PACK_CO_T * PACK_CI_T); }
    else            { ci_l = e % PACK_CI_T; co_l = (e / PACK_CI_T) % PACK_CO_T; t = e / (PACK_CO_T * PACK_CI_T); }
    const int co = co0 + co_l, ci = ci0 + ci_l;
    if (co >= j.Cout || ci >= j.Cin) continue;
    float v;
    if (!up2) {
      v = s[co_l][ci_l * RS + t];
    } else {
      const int tap = t % 4, ph = t / 4;
      const int a = ph >> 1, b = ph & 1, dr = tap >> 1, ds = tap & 1;
      int rlo, rhi, slo, shi;
      up2_rset(a, dr, rlo, rhi);
      up2_rset(b, ds, slo, shi);
      v = 0.f;
      for (int r = rlo; r <= rhi; ++r)
        for (int q = slo; q <= shi; ++q) v += s[co_l][ci_l * 9 + r * 3 + q];
    }
    const long long di = order == 0 ? ((long long)t * j.Cin + ci) * j.Cout + co : ((long long)t * j.Cout + co) * j.Cin + ci;
    j.dst[di] = rtf ? round_tf32(v) : v;
  }
}

__global__ void __launch_bounds__(256) pack_multi_kernel(const __grid_constant__ PackTable tb) {
  int lo = 0, hi = tb.count;
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (tb.block_begin[mid] <= (int)blockIdx.x) lo = mid; else hi = mid;
  }
  const PackJob &j = tb.job[lo];
  if (j.tiles_ci > 0) {
    __shared__ float s[PACK_CO_T][PACK_CI_T * PACK_RS_MAX + 1];
    const int tile = (int)blockIdx.x - tb.block_begin[lo];
    const int rs = j.R * j.S;
    if (rs == 16) pack_tile<16>(j, tile, s);
    else if (rs == 9) pack_tile<9>(j, tile, s);
    else pack_tile<0>(j, tile, s);
    return;
  }
  const long long i0 = (long long)((int)blockIdx.x - tb.block_begin[lo]) * PACK_CHUNK;
  long long i1 = i0 + PACK_CHUNK;
  if (i1 > j.total) i1 = j.total;
  for (long long i = i0 + threadIdx.x; i < i1; i += 256) j.dst[i] = pack_element(j, i);
}

}  // namespace b200gan

using namespace b200gan;

// Validate one packing job and append it to the table (tb.count < PACK_MAX_JOBS; tb.block_begin[tb.count] holds the
// blocks of the jobs before it).
static int pack_table_add(PackTable &tb, const b200gan_conv_geom *g, int pack, const float *w, float *packed) {
  if (int e = validate_geom(g)) return e;
  B2_CHECK_ARG(w && packed, "pack_weights: null pointer");
  B2_CHECK_ARG(pack >= B200GAN_PACK_SIMT_FPROP && pack <= B200GAN_PACK_TC_DGRAD_UP2, "pack_weights: unknown pack id %d", pack);
  if (pack == B200GAN_PACK_TC_FPROP_UP2 || pack == B200GAN_PACK_TC_DGRAD_UP2)
    B2_CHECK_ARG(!g->transposed && g->up == 2 && g->R == 3 && g->S == 3 && g->stride == 1 && g->pad_t == 1 &&
                     g->pad_l == 1 && g->pad_b == 1 && g->pad_r == 1 && g->pad_mode == B200GAN_PAD_ZERO,
                 "pack_weights: UP2 fold needs a 3x3 s1 p1 zero-padded conv behind a x2 upsample");
  PackJob &j = tb.job[tb.count];
  j.src = w; j.dst = packed;
  j.R = g->R; j.S = g->S; j.Cin = g->C; j.Cout = g->K; j.transposed = g->transposed;
  j.kind = pack;
  j.total = (long long)b200gan_packed_weight_floats(g, pack);
  int blocks = tb.block_begin[tb.count];
  j.tiles_ci = 0;
  if (j.R * j.S <= PACK_RS_MAX && j.Cin >= PACK_CI_T && j.Cout >= PACK_CO_T) {
    j.tiles_ci = ceil_div(j.Cin, PACK_CI_T);
    blocks += j.tiles_ci * ceil_div(j.Cout, PACK_CO_T);
  } else {
    blocks += (int)ceil_div64(j.total, PACK_CHUNK);
  }
  tb.block_begin[++tb.count] = blocks;
  return B200GAN_OK;
}

static int pack_table_launch(const PackTable &tb, cudaStream_t st) {
  const int blocks = tb.block_begin[tb.count];
  if (blocks > 0) {
    pack_multi_kernel<<<(unsigned)blocks, 256, 0, st>>>(tb);
    B2_LAUNCH_CHECK();
  }
  return B200GAN_OK;
}

extern "C" int b200gan_pack_weights_multi(const b200gan_pack_job *jobs, int32_t count, void *stream) {
  B2_CHECK_ARG(count >= 0 && (count == 0 || jobs != nullptr), "pack_weights_multi: bad arguments");
  cudaStream_t st = as_stream(stream);
  for (int base = 0; base < count; base += PACK_MAX_JOBS) {
    PackTable tb;
    tb.count = 0;
    tb.block_begin[0] = 0;
    for (int i = base; i < count && tb.count < PACK_MAX_JOBS; ++i)
      if (int e = pack_table_add(tb, &jobs[i].geom, jobs[i].pack, jobs[i].w, jobs[i].packed)) return e;
    if (int e = pack_table_launch(tb, st)) return e;
  }
  return B200GAN_OK;
}

extern "C" int b200gan_version(void) { return B200GAN_VERSION; }
extern "C" const char *b200gan_last_error(void) { return g_err; }

extern "C" int b200gan_check_device(void) {
  int dev = 0;
  B2_CUDA(cudaGetDevice(&dev));
  cudaDeviceProp p;
  B2_CUDA(cudaGetDeviceProperties(&p, dev));
  if (p.major != 9 || p.minor != 0) {
    set_error("device %s is sm_%d%d; libb200gan is built for sm_90a only", p.name, p.major, p.minor);
    return B200GAN_E_ARCH;
  }
  return B200GAN_OK;
}

extern "C" size_t b200gan_packed_weight_floats(const b200gan_conv_geom *g, int pack) {
  if (!g) return 0;
  size_t base = (size_t)g->R * g->S * g->C * g->K;
  if (pack == B200GAN_PACK_TC_FPROP_UP2 || pack == B200GAN_PACK_TC_DGRAD_UP2)
    return (size_t)16 * g->C * g->K;
  return base;
}

extern "C" int b200gan_pack_weights(const b200gan_conv_geom *g, int pack, const float *w, float *packed,
                                    void *stream) {
  PackTable tb;
  tb.count = 0;
  tb.block_begin[0] = 0;
  if (int e = pack_table_add(tb, g, pack, w, packed)) return e;
  return pack_table_launch(tb, as_stream(stream));
}

extern "C" int b200gan_conv2d_supported(const b200gan_conv_geom *g, int pass, int algo) {
  if (validate_geom(g) != B200GAN_OK) return 0;
  if (algo == B200GAN_ALGO_SIMT) return 1;
  return tc_supported(g, pass);
}

static int resolve_algo(const b200gan_conv_geom *g, int pass, int algo) {
  if (algo == B200GAN_ALGO_AUTO) return tc_supported(g, pass) ? B200GAN_ALGO_TC : B200GAN_ALGO_SIMT;
  return algo;
}

extern "C" int b200gan_conv2d_fprop(const b200gan_conv_geom *g, const b200gan_epilogue *ep, const float *x,
                                    const float *packed, float *y, int algo, void *stream) {
  if (int e = validate_geom(g)) return e;
  B2_CHECK_ARG(x && packed && y, "conv2d_fprop: null pointer");
  B2_CHECK_ARG(algo != B200GAN_ALGO_AUTO, "conv2d_fprop: the packed layout fixes the algorithm; pass SIMT or TC");
  cudaStream_t st = as_stream(stream);
  if (algo == B200GAN_ALGO_TC) {
    if (!tc_supported(g, 0)) B2_UNSUPPORTED("conv2d_fprop: geometry not supported by the tensor-core path");
    return tc_fprop(g, ep, x, packed, y, st);
  }
  int rc;
  if (fewk_ok(g, 0) && !(ep && (ep->chan_scale || ep->round_tf32))) {
    b200gan_epilogue e2;
    if (ep) { e2 = *ep; e2.stats = nullptr; }
    rc = fewk_fprop(g, ep ? &e2 : nullptr, x, packed, y, st);
  } else if (nb_plain_fprop_ok(g)) {
    rc = nb_plain_fprop(g, ep, x, packed, y, st);
  } else {
    rc = simt_gather_gemm(g->N, g->H, g->W, g->C, g->P, g->Q, g->K, g->R, g->S, g->stride, g->pad_t, g->pad_l,
                          g->pad_mode, g->up, g->transposed ? 1 : 0, ep, x, packed, y, st);
  }
  if (rc) return rc;
  if (ep && ep->stats) {
    b200gan_norm_desc nd;
    memset(&nd, 0, sizeof(nd));
    nd.N = g->N; nd.HW = g->P * g->Q; nd.C = g->K; nd.per_sample = ep->stats_per_sample;
    return b200gan_norm_stats(&nd, y, ep->stats, stream);
  }
  return B200GAN_OK;
}

extern "C" size_t b200gan_conv2d_dgrad_workspace_floats(const b200gan_conv_geom *g, int algo) {
  if (!g || g->transposed) return 0;
  if (resolve_algo(g, 1, algo) == B200GAN_ALGO_TC) return 0;
  if (fewk_ok(g, 1) || nb_plain_dgrad_ok(g)) return 0;
  size_t n = 0;
  int Hv = g->H * g->up, Wv = g->W * g->up;
  if (g->pad_mode == B200GAN_PAD_REFLECT)
    n += (size_t)g->N * (Hv + g->pad_t + g->pad_b) * (Wv + g->pad_l + g->pad_r) * g->C;
  if (g->up == 2) n += (size_t)g->N * Hv * Wv * g->C;
  return n;
}

extern "C" int b200gan_conv2d_dgrad(const b200gan_conv_geom *g, const float *dy, const float *packed, float *dx,
                                    float *workspace, int algo, void *stream) {
  if (int e = validate_geom(g)) return e;
  B2_CHECK_ARG(dy && packed && dx, "conv2d_dgrad: null pointer");
  B2_CHECK_ARG(algo != B200GAN_ALGO_AUTO, "conv2d_dgrad: pass SIMT or TC explicitly");
  cudaStream_t st = as_stream(stream);
  if (algo == B200GAN_ALGO_TC) {
    if (!tc_supported(g, 1)) B2_UNSUPPORTED("conv2d_dgrad: geometry not supported by the tensor-core path");
    return tc_dgrad(g, dy, packed, dx, st);
  }
  if (g->transposed) {
    // dx[n,ih,iw,c] = sum_{r,s,k} dy[n, ih*stride - pad + r, iw*stride - pad + s, k] * w[c,k,r,s]
    return simt_gather_gemm(g->N, g->P, g->Q, g->K, g->H, g->W, g->C, g->R, g->S, g->stride, g->pad_t, g->pad_l,
                            B200GAN_PAD_ZERO, 1, 0, nullptr, dy, packed, dx, st);
  }
  if (fewk_ok(g, 1)) return fewk_dgrad(g, dy, packed, dx, st);
  if (nb_plain_dgrad_ok(g)) return nb_plain_dgrad(g, dy, packed, dx, st);
  int Hv = g->H * g->up, Wv = g->W * g->up;
  bool reflect = g->pad_mode == B200GAN_PAD_REFLECT;
  B2_CHECK_ARG(!(reflect || g->up == 2) || workspace, "conv2d_dgrad: workspace required for reflect / upsample");
  float *ws_pad = nullptr, *ws_up = nullptr;
  if (reflect) {
    ws_pad = workspace;
    workspace += (size_t)g->N * (Hv + g->pad_t + g->pad_b) * (Wv + g->pad_l + g->pad_r) * g->C;
  }
  if (g->up == 2) ws_up = workspace;
  // gradient w.r.t. the virtual (upsampled, possibly explicitly padded) input
  float *dvirt = reflect ? ws_pad : (g->up == 2 ? ws_up : dx);
  int oh = reflect ? Hv + g->pad_t + g->pad_b : Hv;
  int ow = reflect ? Wv + g->pad_l + g->pad_r : Wv;
  int rc;
  b200gan_conv_geom gv = *g;   // the same convolution seen from the explicitly padded virtual input: no padding left
  gv.H = oh; gv.W = ow; gv.up = 1; gv.pad_mode = B200GAN_PAD_ZERO;
  if (reflect) gv.pad_t = gv.pad_l = gv.pad_b = gv.pad_r = 0;
  if (reflect && g->up == 1 && fewk_ok(&gv, 1)) {
    // few output channels (cyclegan/models.py:88-90: ReflectionPad2d(3) + Conv2d(64, 3, 7)): the channel-lane kernel
    // writes the gradient of the padded tensor, pad2d_bwd folds the mirrored border back
    rc = fewk_dgrad(&gv, dy, packed, dvirt, st);
  } else if (reflect && g->up == 1 && nb_plain_dgrad_ok(&gv)) {
    // few input channels behind a reflection pad (cyclegan/models.py:49-50: the stem, when its input is a generated image)
    rc = nb_plain_dgrad(&gv, dy, packed, dvirt, st);
  } else {
    rc = simt_gather_gemm(g->N, g->P, g->Q, g->K, oh, ow, g->C, g->R, g->S, g->stride, reflect ? 0 : g->pad_t,
                          reflect ? 0 : g->pad_l, B200GAN_PAD_ZERO, 1, 1, nullptr, dy, packed, dvirt, st);
  }
  if (rc) return rc;
  if (reflect) {
    float *dst = g->up == 2 ? ws_up : dx;
    rc = b200gan_pad2d_bwd(ws_pad, dst, g->N, Hv, Wv, g->C, g->pad_t, g->pad_l, g->pad_b, g->pad_r,
                           B200GAN_PAD_REFLECT, stream);
    if (rc) return rc;
  }
  if (g->up == 2) return b200gan_upsample2x_bwd(ws_up, dx, g->N, g->H, g->W, g->C, stream);
  return B200GAN_OK;
}

static bool nb_wgrad_routed(const b200gan_conv_geom *g) {
  // narrow layers only: beyond ~2e10 MACs (wide layers that are not tensor-core shaped) the generic kernel's larger
  // tiles win
  return nb_wgrad_ok(g) && (int64_t)g->N * g->P * g->Q * g->K * g->C * g->R * g->S <= (int64_t)2e10;
}

extern "C" size_t b200gan_conv2d_wgrad_workspace_floats(const b200gan_conv_geom *g, int algo) {
  if (!g) return 0;
  if (resolve_algo(g, 2, algo) == B200GAN_ALGO_TC) return tc_wgrad_workspace_floats(g);
  if (fewk_ok(g, 2)) return fewk_wgrad_workspace_floats(g);
  if (nb_wgrad_routed(g)) return nb_wgrad_workspace_floats(g);
  return 0;
}

extern "C" int b200gan_conv2d_wgrad(const b200gan_conv_geom *g, const float *x, const float *dy, float *dw,
                                    float *db, float *workspace, int algo, void *stream) {
  if (int e = validate_geom(g)) return e;
  B2_CHECK_ARG(x && dy && dw, "conv2d_wgrad: null pointer");
  cudaStream_t st = as_stream(stream);
  int a = resolve_algo(g, 2, algo);
  int rc;
  if (a == B200GAN_ALGO_TC) {
    if (!tc_supported(g, 2)) B2_UNSUPPORTED("conv2d_wgrad: geometry not supported by the tensor-core path");
    rc = tc_wgrad(g, x, dy, dw, workspace, st);
  } else if (fewk_ok(g, 2)) {
    // K <= 4 output channels, stride 1 (the image / patch output layers): lanes = input channels
    rc = fewk_wgrad(g, x, dy, dw, workspace, st);
  } else if (nb_wgrad_routed(g)) {
    // narrow layers (C or K small): patch + dy tile staged in shared memory, all taps of a (c, 4k) set in registers
    rc = nb_wgrad_run(g, nullptr, x, dy, dw, workspace, st);
  } else if (g->transposed) {
    rc = simt_wgrad(g->N, g->P, g->Q, g->K, g->H, g->W, g->C, g->R, g->S, g->stride, g->pad_t, g->pad_l,
                    B200GAN_PAD_ZERO, 1, dy, x, dw, st);
  } else {
    rc = simt_wgrad(g->N, g->H, g->W, g->C, g->P, g->Q, g->K, g->R, g->S, g->stride, g->pad_t, g->pad_l,
                    g->pad_mode, g->up, x, dy, dw, st);
  }
  if (rc) return rc;
  if (db) return simt_colsum(dy, db, (int64_t)g->N * g->P * g->Q, g->K, st);
  return B200GAN_OK;
}
