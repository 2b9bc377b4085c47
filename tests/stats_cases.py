"""Case table of the BatchNorm2d / InstanceNorm2d statistics: every kernel that produces the [sum x, sum x^2] of a
normalisation group, at the reduction sizes the models run, on data whose channels sit at R = |mean| / std of 0, 1,
10^2, 10^3 and 10^4, plus exactly constant channels at a value that is not a short binary fraction.

The variance is formed as E[x^2] - E[x]^2 from those sums (norm_finalize_kernel, nb_bn_consts).  Every producer sums in
fp32 first: per thread (norm_stats_kernel), per warp (the wgmma conv epilogues) or per thread and warp (the chain's
epilogue), then in fp64.  fp32 partial sums of x and x^2 round relative to mean^2 + var, and the subtraction divides
that by var: without a pivot the variance loses accuracy in proportion to R^2.  The bounds here are what a correct fp32
implementation achieves, with no R^2 term: each one follows from the length K of the fp32 chain an element passes
through, mirrored from the launchers (reduce_grid for norm_stats) or read off the epilogues, and from P, a bound on the
fp64 additions into a group.

Paths (one per row): "norm" the stand-alone b200gan_norm_stats -> finalize (and the apply / backward of
norm_cases.Run on the same data); "conv" b200gan_conv2d_fprop on the wgmma path with its fused statistics, or the
deferred norm_stats pass after split-K or after a tile that spans images; "chain" the discriminator chain's out_stats
(b200gan_nb_fprop).  The family owns no entry point: norm, conv and chain do.

tests/test_gpu_norm_statistics.py runs the table against fp64; tests/test_cpu_norm_statistics.py emulates the chains
in numpy, with and without a pivot, to show that the bounds separate the two.
"""
from dataclasses import dataclass, field

import numpy as np

import chain_cases as ch
import norm_cases as nc

NUM_SMS = 132                  # H100 SXM
U = 2.0 ** -23
U64 = 2.0 ** -50               # per fp64 addition, with room
MOMENTUM = 0.1
# (location, spread) of channel c: LADDER[c % 6].  R = 0, 1, 1e2, 1e3, 1e4, and a constant channel
LADDER = ((0.0, 1.0), (1.0, 1.0), (100.0, 1.0), (1000.0, 1.0), (100.0, 0.01), (100.1, 0.0))
BN_EPS, IN_EPS = 0.8, 1e-5     # nn.BatchNorm2d(C, 0.8) of dcgan.py, nn.InstanceNorm2d(C) of cyclegan / pix2pix
TC_BM = 128


@dataclass(frozen=True)
class Case:
    name: str
    path: str                  # "norm", "conv", "chain"
    N: int
    C: int                     # input channels (norm: the normalised channels)
    K: int                     # normalised channels (norm: = C)
    H: int                     # input map (conv / chain) or the normalised map (norm)
    W: int
    per_sample: bool = False   # InstanceNorm groups (n, c), else BatchNorm groups c
    up: int = 1                # conv: folded Upsample(2x) + Conv3x3
    R: int = 3
    stride: int = 1
    drop: bool = False         # conv: a Dropout2d chan_scale in the epilogue (InstanceNorm rows only: per image and
                               # channel it scales a whole group, where in a batch group it would mix the ladder)
    splitk: bool = False       # conv: no bias / activation, so that the contraction may be split
    groups: int = 1            # chain: statistics groups of the batch
    offset: int = 0            # norm: x one float past 16-byte alignment (VEC 1)
    act: str = "lrelu"
    kernels: tuple = ()
    grid: tuple = None
    why: str = ""

    @property
    def id(self):
        return f"{self.path}-{self.name}"

    @property
    def eps(self):
        return IN_EPS if self.per_sample else BN_EPS

    @property
    def P_(self):
        if self.path == "norm":
            return self.H
        if self.up == 2:
            return 2 * self.H
        return (self.H + 2 * (self.R // 2 if self.stride == 1 else 1) - self.R) // self.stride + 1

    @property
    def Q_(self):
        if self.path == "norm":
            return self.W
        if self.up == 2:
            return 2 * self.W
        return (self.W + 2 * (self.R // 2 if self.stride == 1 else 1) - self.R) // self.stride + 1

    @property
    def pad(self):
        return self.R // 2 if self.stride == 1 else 1

    @property
    def m(self):
        """elements of a group"""
        hw = self.P_ * self.Q_
        return hw if self.per_sample else hw * self.N // self.groups

    @property
    def deferred(self):
        """conv: the statistics come from a norm_stats pass over y"""
        return "norm_stats_kernel" in self.kernels


# ---- the conv launcher, mirrored (csrc/conv_tc.cu: tc_tile_shape, tc_block_n, the deferral rules) -----------------------
def _ilog2c(v):
    return max(0, (v - 1).bit_length())


def tc_tile(Ho, Wo):
    """(bwl, bhl, images per 128-pixel tile)"""
    bwl = min(_ilog2c(Wo), 7)
    bhl = min(_ilog2c(Ho), 7 - bwl)
    return bwl, bhl, TC_BM >> (bwl + bhl)


def conv_kernels(N, K, Ho, Wo, up, per_sample, splitk):
    """what b200gan_conv2d_fprop launches for a conv with statistics, Ho x Wo per phase"""
    bwl, bhl, bnn = tc_tile(Ho, Wo)
    deferred = splitk or (per_sample and bnn != 1)
    if up == 2 and K % 128 != 0:
        ks = ("conv_tc_up2_allphase_kernel",)
    else:   # up == 2: four phases of conv_tc_kernel
        tiles = -(-Wo // (1 << bwl)) * -(-Ho // (1 << bhl)) * -(-N // bnn) * (4 if up == 2 else 1)
        bn = 256 if K % 256 == 0 and tiles * (K // 256) >= NUM_SMS else 128 if K % 128 == 0 else \
            64 if K % 64 == 0 else 32
        ks = (f"conv_tc_kernel<{bn}, {dict([(256, 4), (128, 6), (64, 8), (32, 8)])[bn]}>",)
    return ks + (("norm_stats_kernel",) if deferred else ())


def _conv(name, N, C, K, H, W, up=1, per_sample=False, drop=False, splitk=False, R=3, stride=1, why=""):
    Ho, Wo = (H, W) if up == 2 else ((H + 2 * (R // 2 if stride == 1 else 1) - R) // stride + 1,) * 2
    return Case(name, "conv", N, C, K, H, W, per_sample=per_sample, up=up, R=R, stride=stride, drop=drop,
                splitk=splitk, act="none" if splitk else "lrelu",
                kernels=conv_kernels(N, K, Ho, Wo, up, per_sample, splitk), why=why)


def _norm(name, N, C, H, W, per_sample, vec, offset=0, act="none", why=""):
    v = vec
    return Case(name, "norm", N, C, C, H, W, per_sample=per_sample, offset=offset, act=act,
                kernels=("norm_stats_kernel", "norm_stats_kernel", "norm_finalize_kernel", f"norm_apply_kernel<{v}>",
                         f"norm_bwd_reduce_kernel<{v}>", f"norm_bwd_apply_kernel<{v}>", "norm_bwd_params_kernel"),
                why=why)


def _chain(layer, groups):
    row = next(c for c in ch.FPROP if c.name == (layer if groups == 1 else f"{layer}_g{groups}"))
    return Case(row.name, "chain", row.N, row.C, row.K, row.H, row.W, R=row.R, stride=row.stride,
                groups=groups, kernels=row.kernels, grid=row.grid,
                why=f"DCGAN discriminator {layer} at batch 128" + (", real + fake as two groups" if groups > 1 else ""))


CASES = (
    # stand-alone norm_stats -> finalize (and apply / backward), DCGAN generator and CycleGAN / Pix2Pix sizes
    _norm("bn128_16x16", 128, 128, 16, 16, False, 4, why="DCGAN generator BatchNorm(128, 0.8) at batch 128, 16x16"),
    _norm("bn64_64x64", 128, 64, 64, 64, False, 4, act="lrelu",
          why="DCGAN generator BatchNorm(64, 0.8) at batch 128, 64x64: 2^19 elements per group"),
    _norm("in64_256x256", 1, 64, 256, 256, True, 4, act="relu", why="InstanceNorm(64) at 256x256 (CycleGAN, Pix2Pix)"),
    _norm("in64_vec1", 2, 64, 128, 128, True, 1, offset=1, why="InstanceNorm at VEC 1: x one float past alignment"),
    _norm("bn128_vec1", 128, 128, 8, 8, False, 1, offset=1, act="lrelu", why="BatchNorm(128, 0.8) at VEC 1"),
    # the wgmma epilogues: stats_c (BatchNorm) on a ragged map, stats_s (InstanceNorm) one image per tile, the all-phase
    # Upsample(2x) kernel with both, and the deferred passes
    _conv("batchnorm_ragged", 64, 64, 128, 20, 20,
          why="20x20 map in 32x4 tiles: 12 of every 32 columns are outside the output"),
    _conv("instancenorm_one_image_per_tile", 128, 64, 64, 16, 16, per_sample=True,
          why="16x16 map: two tiles per image, per-sample sums change group at every image"),
    _conv("batchnorm_bn256", 96, 64, 256, 16, 16, why="256 output channels and enough tiles for the 256-wide tile"),
    _conv("allphase_instancenorm", 128, 128, 64, 16, 16, up=2, per_sample=True, drop=True,
          why="the all-phase kernel, per-sample sums over four phases"),
    _conv("allphase_batchnorm", 128, 128, 64, 32, 32, up=2, why="the all-phase kernel, batch sums"),
    _conv("dcgan_g_bn128", 128, 128, 128, 16, 16, up=2,
          why="DCGAN generator Upsample + Conv(128, 128) into BatchNorm(128, 0.8), batch 128: four phases of "
              "conv_tc_kernel"),
    _conv("instancenorm_tile_spans_images", 512, 64, 64, 8, 8, per_sample=True,
          why="8x8 map: a tile holds two images, the deferred norm_stats pass"),
    _conv("allphase_instancenorm_tile_spans_images", 2048, 128, 64, 4, 4, up=2, per_sample=True, drop=True,
          why="all-phase kernel at 4x4 per phase: eight images per tile, deferred"),
    _conv("splitk", 1, 256, 256, 4, 4, R=4, stride=2, splitk=True,
          why="split-K: partial tiles cannot carry the sums, the deferred norm_stats pass"),
    # the discriminator chain's epilogue
    _chain("d2", 1), _chain("d3", 1), _chain("d4", 1), _chain("d2", 2), _chain("d4", 2),
)

# the large and offset geometries live here, not in norm_cases.GEOMS (whose bounds the norm-conv suite shares)
NORM_GEOMS = tuple(nc.Geom(c.name, c.N, c.C, c.H, c.W, c.per_sample, not c.per_sample,
                           vec=int(c.kernels[3][-2]), offset=c.offset, why=c.why) for c in CASES if c.path == "norm")


# ---- data --------------------------------------------------------------------------------------------------------------
def ladder(K):
    """(location, spread) per channel, float64 arrays of K"""
    loc = np.array([LADDER[k % len(LADDER)][0] for k in range(K)])
    sd = np.array([LADDER[k % len(LADDER)][1] for k in range(K)])
    return loc, sd


# ---- the summation chains -------------------------------------------------------------------------------------------
def reduce_grid(N, HW, C, per_sample, num_sms=NUM_SMS):
    """(blocks per group, rows per block) of b200gan_norm_stats, as reduce_grid in csrc/norm.cu plans them"""
    rows = HW if per_sample else N * HW
    xb, zb = -(-C // 32), N if per_sample else 1
    want = max(num_sms * 8 // (xb * zb), 1)
    rpb = max(-(-rows // want), 32)
    return -(-rows // rpb), rpb


@dataclass(frozen=True)
class Chain:
    K: int      # fp32 roundings an element's contribution goes through (the unpivoted chain: the longer one)
    P: int      # bound on the fp64 additions into a group
    shape: tuple = field(default=())  # the emulation's layout: see tests/test_cpu_norm_statistics.py


def chain(c, num_sms=NUM_SMS):
    """the fp32 chain of the kernel that sums a group of case c"""
    if c.path == "norm" or c.deferred:
        N, HW, C = (c.N, c.H * c.W, c.C) if c.path == "norm" else (c.N, c.P_ * c.Q_, c.K)
        yb, rpb = reduce_grid(N, HW, C, c.per_sample, num_sms)
        n = -(-rpb // 8)
        # per thread: n serial adds (a) / fmaf (b); 8 threads and yb blocks in fp64
        return Chain(n + 1, 9 * yb + 8, ("norm_stats", yb, rpb))
    if c.path == "conv":
        # a warp's 32 pixels: 5 shuffle levels; the all-phase kernel adds four phases per lane; then 4 warps (quarters)
        phases = 4 if c.kernels[0] == "conv_tc_up2_allphase_kernel" else 1
        return Chain(1 + 5 + (phases - 1) + 3, 2 * -(-c.m // 32) + 8, ("conv", phases))
    # chain: PT pixels per thread, 5 shuffle levels, up to 8 warps of a channel group
    pt = int(c.kernels[0].rstrip(">").split(",")[1])
    return Chain(pt + 5 + 7 + 1, 2 * -(-c.m // 32) + 8, ("chain", pt))


# ---- bounds ---------------------------------------------------------------------------------------------------------
def bounds(K, P, mean, var, dev):
    """(|d mean|, |d var|) bounds of the mean and biased variance implied by [sum x, sum x^2], for fp32 chains of K
    roundings, then P fp64 additions.  dev = max |x - mean| over the group.  A block (a thread's, warp's or tile's
    share of the group) adds either its sums around a pivot inside the group (|x - pivot| <= 2 dev: 2 K u dev and
    8 K u dev^2), or, where its own mean is within 4 of its own standard deviations s of zero (stats_plain_ok in
    csrc/common.cuh), its plain sums from zero (|x| <= |block mean| + s <= 5 dev and x^2 <= 17 s^2 <= 17 dev^2 on
    average): the larger of the two holds."""
    mb = 5 * K * U * dev + U * abs(mean) + U64 * P * abs(mean)
    vb = 17 * K * U * dev * dev + U64 * (P + 4) * (mean * mean + var)
    return mb, vb
