"""Case table of the fused discriminator chain (pytorch-gan_b200/csrc/narrow_block.cu).

One row per call of a chain entry point (b200gan_nb_fprop / nb_dz / nb_wgrad / nb_dgrad / nb_tail_fwd / nb_tail_bwd),
plus the few staged data-gradient instances that only the plain convolution entry reaches (op "plain_dgrad":
b200gan_conv2d_dgrad with ALGO_SIMT on a layer with 3 or 6 input channels).  Each row gives the geometry, the number
of statistics groups the batch is split into, the BatchNorm edge of the call (none; "stats": batch sums only, gamma
and beta NULL; "affine": sums, gamma and beta), whether it takes a Dropout2d chan_scale, the activation, and what the
library must do with it: the kernel instances a trace of the call shows, the grid of the first one (132 SMs), whether
repeating the call gives the same bits, the partial sums `s` added outside one accumulation chain, or a refusal.

The instances and grids are written from the planners (nb_plan, nb_wgrad_plan, tail_grid and b200gan_nb_dz) for a
132-SM H100 SXM, not from a run; tests/test_gpu_fused_conformance.py checks them on such a device.
tests/test_cpu_fused_case_table.py holds the table to the sources and to the library's eligibility predicates.
"""
from dataclasses import dataclass

import torch
import torch.nn.functional as F

from b200gan import _lib

NUM_SMS = 132
OPS = ("fprop", "dz", "wgrad", "dgrad", "plain_dgrad", "tail_fwd", "tail_bwd")
EDGES = ("none", "stats", "affine")


@dataclass(frozen=True)
class Case:
    name: str
    op: str
    N: int
    C: int                      # input channels (dz: unused; tail_*: the channels of a)
    K: int                      # output channels (dz: the channels of a and g)
    H: int                      # input map (dz: the output map P x Q; tail_*: H * W = HW)
    W: int
    R: int = 3                  # square filter, zero padding 1
    stride: int = 2
    groups: int = 1
    edge: str = "none"          # the BatchNorm of the call: in_bn (fprop, wgrad, dgrad), out_bn (dz), bn (tail_*)
    cs: bool = False            # Dropout2d scale [N][K], zeros and negatives included
    act: str = "lrelu"
    out_stats: bool = False     # fprop: out_stats given
    running: bool = False       # fprop / tail_fwd: running_mean, running_var, num_batches_tracked given
    sums: bool = False          # dgrad: sums (and a_prev) given
    ws: bool = False            # wgrad: workspace of b200gan_nb_wgrad_workspace_floats() given (else NULL)
    db: bool = True             # dz: db given
    nchw: int = 0               # tail_*: layout of out / dout
    misalign: bool = False      # x (fprop) one float past 16-byte alignment
    call_groups: int = 0        # fprop: `groups` argument when it differs from the edge's (a refusal)
    kernels: tuple = ()
    grid: tuple = None
    deterministic: bool = True  # the outputs that are not fp64 sums or fp32 atomics repeat bit for bit
    s: int = 0
    error: bool = False
    why: str = ""

    @property
    def P(self):
        if self.op in ("dz", "tail_fwd", "tail_bwd"):
            return self.H
        return (self.H + 2 - self.R) // self.stride + 1

    @property
    def Q(self):
        if self.op in ("dz", "tail_fwd", "tail_bwd"):
            return self.W
        return (self.W + 2 - self.R) // self.stride + 1

    @property
    def id(self):
        return f"{self.name}-{self.op}"


def fp(KT, PT):
    return f"nbk_fprop2_kernel<{KT}, {PT}>"


def dg(KT, PT):
    return f"nbk_dgrad2_kernel<{KT}, {PT}>"


WG9, WG16, WG_RED = "nbk_wgrad_kernel<9>", "nbk_wgrad_kernel<16>", "nbk_wgrad_reduce_kernel"
DZ, TF, TB = "nbk_dz_kernel", "nbk_tail_fwd_kernel", "nbk_tail_bwd_kernel"

_c = Case
# the four discriminator layers of the DCGAN step at 64x64, batch 128 (dcgan.py:77-88), and the real + fake pass of
# train.dcgan_step as two statistics groups of 128
_D = {"d1": (1, 16, 64), "d2": (16, 32, 32), "d3": (32, 64, 16), "d4": (64, 128, 8)}


def _d(layer, groups, suffix="", **kw):
    C, K, H = _D[layer]
    name = (layer if groups == 1 else f"{layer}_g{groups}") + suffix
    return Case(name, N=128 * groups, C=C, K=K, H=H, W=H, groups=groups, **kw)


FPROP = [
    _d("d1", 1, op="fprop", cs=True, out_stats=True, kernels=(fp(16, 1),), grid=(512, 1, 1),
       why="DCGAN layer 1: C = 1 staging, no BatchNorm in front"),
    _d("d1", 2, op="fprop", cs=True, out_stats=True, kernels=(fp(16, 1),), grid=(1024, 1, 1),
       why="layer 1, real + fake: out_stats of two groups without an input edge"),
    _d("d2", 1, op="fprop", edge="affine", cs=True, out_stats=True, running=True, kernels=(fp(4, 4),),
       grid=(256, 1, 1), why="DCGAN layer 2: BatchNorm of layer 1 applied while staging, running statistics"),
    _d("d2", 2, op="fprop", edge="affine", cs=True, out_stats=True, running=True, kernels=(fp(8, 4),),
       grid=(256, 1, 1), why="layer 2 grouped: two running-statistics updates in batch order"),
    _d("d3", 1, op="fprop", edge="affine", cs=True, out_stats=True, running=True, kernels=(fp(4, 4),),
       grid=(64, 2, 1), why="DCGAN layer 3: two images per tile, two channel blocks"),
    _d("d3", 2, op="fprop", edge="affine", cs=True, out_stats=True, running=True, kernels=(fp(8, 4),),
       grid=(128, 1, 1), why="layer 3 grouped"),
    _d("d4", 1, op="fprop", edge="affine", cs=True, out_stats=True, running=True, kernels=(fp(4, 2),),
       grid=(32, 4, 1), why="DCGAN layer 4: four 4x4 output images per tile"),
    _d("d4", 2, op="fprop", edge="affine", cs=True, out_stats=True, running=True, kernels=(fp(4, 2),),
       grid=(64, 4, 1), why="layer 4 grouped: the last tile of the last group"),
    _c("r13", "fprop", 5, 16, 32, 13, 13, edge="stats", act="relu", out_stats=True, running=True,
       kernels=(fp(4, 1),), grid=(2, 8, 1), why="13x13 -> 7x7 clipped by 8x8 tiles; 4-image tiles over N = 5"),
    _c("r9", "fprop", 3, 4, 8, 9, 9, edge="affine", act="none", cs=True, out_stats=True, kernels=(fp(4, 1),),
       grid=(2, 1, 1), why="C = 4 float4 staging, 9x9 map, a 2-image tile hanging over N = 3"),
    _c("r31", "fprop", 7, 1, 4, 31, 31, edge="stats", cs=True, out_stats=True, running=True, kernels=(fp(4, 1),),
       grid=(7, 1, 1), why="C = 1 scalar staging behind a BatchNorm, 31x31 -> 16x16"),
    _c("s1", "fprop", 2, 32, 64, 9, 9, stride=1, edge="affine", cs=True, out_stats=True, kernels=(fp(4, 1),),
       grid=(4, 8, 1), why="stride 1, ragged 9x9 map"),
    _c("k4", "fprop", 6, 8, 16, 24, 24, R=4, edge="affine", cs=True, out_stats=True, kernels=(fp(4, 1),),
       grid=(12, 2, 1), why="4x4 filter, stride 2"),
    _c("g3", "fprop", 3, 16, 32, 32, 32, groups=3, edge="affine", out_stats=True, running=True,
       kernels=(fp(4, 1),), grid=(24, 1, 1), why="three groups of one image: the smallest N the planner allows"),
    _c("g4", "fprop", 4, 16, 32, 32, 32, groups=4, edge="affine", cs=True, out_stats=True, running=True,
       kernels=(fp(4, 1),), grid=(32, 1, 1), why="four groups of one image"),
    _c("kt8", "fprop", 1, 1, 128, 64, 64, stride=1, cs=True, out_stats=True, kernels=(fp(8, 1),), grid=(128, 2, 1),
       why="the only planner choice of <8, 1>: C = 1, stride 1, 128 outputs"),
    _c("kt16pt4", "fprop", 4, 32, 128, 64, 64, R=4, stride=1, edge="affine", out_stats=True,
       kernels=(fp(16, 4),), grid=(64, 2, 1), why="<16, 4>: 4x4 stride 1, 63x63 output clipped by 8x32 tiles"),
    _c("g2_odd", "fprop", 58, 16, 128, 5, 5, stride=1, groups=2, edge="affine", cs=True, out_stats=True,
       running=True, kernels=(fp(8, 2),), grid=(58, 2, 1),
       why="29 images per group: tiles of one image, and <8, 2> wins once the PT = 4 tiles are gone"),
    _c("bad_groups", "fprop", 4, 16, 32, 32, 32, groups=2, call_groups=1, edge="affine", error=True,
       why="the input edge has two groups, the call one"),
    _c("misaligned", "fprop", 4, 16, 32, 32, 32, edge="affine", misalign=True, error=True,
       why="x one float past 16-byte alignment"),
]

DGRAD = [
    _d("d1", 1, op="dgrad", kernels=(dg(1, 1),), grid=(512, 1, 4),
       why="layer 1 data gradient (into the generator): C = 1, no BatchNorm in front"),
    _d("d2", 1, op="dgrad", edge="affine", sums=True, kernels=(dg(8, 4),), grid=(64, 1, 4),
       why="layer 2: the sums of layer 1's BatchNorm backward"),
    _d("d2", 2, op="dgrad", edge="affine", sums=True, kernels=(dg(8, 4),), grid=(128, 1, 4),
       why="layer 2 grouped: sums per group"),
    _d("d3", 1, op="dgrad", edge="affine", sums=True, kernels=(dg(4, 4),), grid=(64, 1, 4), why="layer 3"),
    _d("d3", 2, op="dgrad", edge="affine", sums=True, kernels=(dg(4, 4),), grid=(128, 1, 4), why="layer 3 grouped"),
    _d("d4", 1, op="dgrad", edge="affine", sums=True, kernels=(dg(4, 4),), grid=(16, 2, 4),
       why="layer 4: eight 4x4 class maps per tile"),
    _d("d4", 2, op="dgrad", edge="affine", sums=True, kernels=(dg(4, 4),), grid=(32, 2, 4), why="layer 4 grouped"),
    _c("r13", "dgrad", 5, 16, 32, 13, 13, edge="stats", sums=True, kernels=(dg(4, 1),), grid=(2, 4, 4),
       why="odd map: parity classes of 7 and 6 rows, 4-image tiles over N = 5"),
    _c("r9", "dgrad", 3, 4, 8, 9, 9, edge="affine", sums=True, kernels=(dg(4, 1),), grid=(1, 1, 4),
       why="C = 4, a 4-image tile over N = 3"),
    _c("r31", "dgrad", 7, 1, 4, 31, 31, edge="stats", sums=True, kernels=(dg(1, 1),), grid=(7, 1, 4),
       why="C = 1 behind a BatchNorm: scalar stores and sums"),
    _c("s1", "dgrad", 2, 32, 64, 9, 9, stride=1, edge="affine", sums=True, kernels=(dg(4, 1),), grid=(4, 4, 1),
       why="stride 1: one class"),
    _c("k4", "dgrad", 6, 8, 16, 24, 24, R=4, edge="affine", sums=True, kernels=(dg(4, 1),), grid=(12, 1, 4),
       why="4x4 stride 2: four taps per class"),
    _c("g3", "dgrad", 3, 16, 32, 32, 32, groups=3, edge="affine", sums=True, kernels=(dg(4, 1),), grid=(12, 1, 4),
       why="three groups of one image"),
    _c("g4", "dgrad", 4, 16, 32, 32, 32, groups=4, edge="stats", sums=True, kernels=(dg(4, 1),), grid=(16, 1, 4),
       why="four groups of one image"),
    _c("pt2", "dgrad", 1, 64, 4, 64, 64, stride=1, edge="affine", sums=True, kernels=(dg(4, 2),), grid=(64, 2, 1),
       why="the planner's <4, 2>: K = 4, stride 1"),
    _c("kt16pt4", "dgrad", 4, 128, 32, 64, 64, R=4, stride=1, edge="affine", sums=True, kernels=(dg(16, 4),),
       grid=(64, 2, 1), why="<16, 4>: C = 128, 4x4 stride 1"),
    _c("g2_odd9", "dgrad", 30, 64, 16, 9, 9, groups=2, edge="affine", sums=True, kernels=(dg(8, 2),),
       grid=(30, 1, 4), why="15 images per group, 9x9: one-image tiles, <8, 2>"),
    _c("g2_odd5", "dgrad", 60, 64, 32, 5, 5, groups=2, edge="affine", sums=True, kernels=(dg(8, 1),),
       grid=(30, 1, 4), why="30 images per group, 5x5: two-image tiles, <8, 1>"),
    _c("c3", "plain_dgrad", 4, 3, 64, 16, 16, R=4, kernels=(dg(3, 1),), grid=(1, 1, 4),
       why="Conv2d(3, 64, 4, 2, 1) data gradient through the conv entry: <3, 1>"),
    _c("c6", "plain_dgrad", 4, 6, 64, 16, 16, R=4, kernels=(dg(6, 1),), grid=(1, 1, 4),
       why="Conv2d(6, 64, 4, 2, 1) (pix2pix discriminator) at 16x16: <6, 1>"),
    _c("c6_256", "plain_dgrad", 1, 6, 64, 256, 256, R=4, kernels=(dg(6, 2),), grid=(32, 1, 4),
       why="the pix2pix discriminator's first layer at 256x256, batch 1: <6, 2>"),
    _c("c6_256n2", "plain_dgrad", 2, 6, 16, 256, 256, R=4, kernels=(dg(6, 4),), grid=(32, 1, 4),
       why="6 -> 16 channels at 256x256, batch 2: <6, 4>"),
]

WGRAD = [
    _d("d2", 1, op="wgrad", edge="affine", ws=True, kernels=(WG9, WG_RED), s=258, grid=(256, 1, 1),
       why="layer 2 with per-block slabs: fixed-order reduce"),
    _d("d2", 1, "_atomics", op="wgrad", edge="affine", ws=False, kernels=(WG9,), deterministic=False, s=258, grid=(256, 1, 1),
       why="the same geometry with a NULL workspace: fp32 atomics into a zeroed dw"),
    _d("d3", 2, op="wgrad", edge="affine", ws=True, kernels=(WG9, WG_RED), s=133, grid=(132, 2, 1),
       why="layer 3 grouped: scale / shift per group, two set chunks"),
    _d("d4", 1, op="wgrad", edge="affine", ws=True, kernels=(WG9, WG_RED), s=34, grid=(33, 8, 1), why="layer 4: eight set chunks"),
    _d("d1", 1, op="wgrad", ws=True, kernels=(WG9,), deterministic=False, s=328, grid=(264, 1, 1),
       why="layer 1 (C = 1): too few weights for slabs (workspace size 0); a buffer passed anyway stays untouched"),
    _c("k4", "wgrad", 6, 8, 16, 24, 24, R=4, edge="affine", kernels=(WG16,), deterministic=False, s=20, grid=(12, 1, 1),
       why="4x4 filter: the <16> instance"),
    _c("r13", "wgrad", 5, 16, 32, 13, 13, edge="stats", kernels=(WG9,), deterministic=False, s=5, grid=(3, 1, 1),
       why="ragged 7x7 output, stats-only edge"),
    _c("g3", "wgrad", 3, 16, 32, 32, 32, groups=3, edge="affine", kernels=(WG9,), deterministic=False, s=8, grid=(6, 1, 1),
       why="three groups: per-image scale / shift"),
]


def _dz(name, N, P, K, **kw):
    return Case(name, "dz", N, K, K, P, P, **kw)


DZ_CASES = [
    _dz("k4", 7, 9, 4, edge="affine", cs=True, kernels=(DZ,), grid=(1, 1, 1), deterministic=True,
        why="K = 4: one float4 per row, 256 rows per block"),
    _dz("k128_g2", 256, 4, 128, groups=2, edge="affine", cs=True, kernels=(DZ,), grid=(64, 2, 1),
        why="layer 4's dz at K = 128, two groups: 8 rows per block"),
    _dz("k128_nobn", 128, 4, 128, cs=True, db=False, kernels=(DZ,), grid=(64, 1, 1),
        why="no BatchNorm after the layer, db NULL"),
    _dz("k16_g4", 8, 8, 16, groups=4, edge="stats", act="none", kernels=(DZ,), grid=(1, 4, 1),
        why="four groups, stats-only edge, no activation"),
    _dz("d1", 128, 32, 16, edge="affine", cs=True, kernels=(DZ,), grid=(512, 1, 1), why="DCGAN layer 1's dz"),
    _dz("d1_g2", 256, 32, 16, groups=2, edge="affine", cs=True, kernels=(DZ,), grid=(264, 2, 1),
        why="layer 1 grouped: the block cap num_sms * 4 / groups"),
    _dz("k12", 4, 4, 12, error=True, why="K not a power of two"),
]


def _tail(name, op, N, HW, C, **kw):
    return Case(name, op, N, C, C, HW, 1, **kw)


TAIL = [
    _tail("d4", "tail_fwd", 128, 16, 128, edge="affine", running=True, nchw=1, kernels=(TF,), grid=(256, 1, 1),
          why="end of the DCGAN chain: BatchNorm 4 into NCHW for the .view"),
    _tail("d4_g2", "tail_fwd", 256, 16, 128, groups=2, edge="affine", running=True, nchw=1, kernels=(TF,),
          grid=(256, 2, 1), why="grouped: one running-statistics update per group"),
    _tail("g3", "tail_fwd", 6, 16, 128, groups=3, edge="affine", running=True, kernels=(TF,), grid=(4, 3, 1),
          why="three groups, NHWC"),
    _tail("g4", "tail_fwd", 8, 9, 64, groups=4, edge="stats", running=True, nchw=1, kernels=(TF,), grid=(2, 4, 1),
          why="four groups, 3x3 map, stats-only edge"),
    _tail("c100", "tail_fwd", 4, 25, 100, groups=2, edge="affine", nchw=1, kernels=(TF,), grid=(25, 2, 1),
          why="C = 100: tail_grid rounds the block count up to a multiple of 25"),
    _tail("d4", "tail_bwd", 128, 16, 128, edge="affine", nchw=1, kernels=(TB,), grid=(256, 1, 1),
          why="backward of the chain end from NCHW"),
    _tail("d4_g2", "tail_bwd", 256, 16, 128, groups=2, edge="affine", nchw=1, kernels=(TB,), grid=(256, 2, 1),
          why="grouped sums"),
    _tail("g3", "tail_bwd", 6, 16, 64, groups=3, edge="affine", kernels=(TB,), grid=(2, 3, 1),
          why="three groups, NHWC"),
    _tail("g4", "tail_bwd", 8, 9, 8, groups=4, edge="stats", nchw=1, kernels=(TB,), grid=(1, 4, 1),
          why="four groups, C = 8: 32 threads per channel in a block"),
    _tail("c96", "tail_bwd", 4, 16, 96, edge="affine", error=True, why="256 % C != 0"),
]

CASES = FPROP + DGRAD + WGRAD + DZ_CASES + TAIL

# instances of the two planned kernels that no legal call reaches without the tuning hook B200GAN_NB_FORCE_{FPROP,DGRAD}.
# tests/test_cpu_fused_case_table.py restates nb_plan, sweeps it over legal chain and staged-conv geometries (groups
# 1 - 4 included) and requires this set to be exactly the launched instances the sweep never picks.
HOOK_ONLY = {
    fp(16, 2): "<8, 4> at twice the channel groups has the same tile, grid and shared memory at a lower cost per FMA "
               "(0.375 vs 0.5625) whenever KG <= 4; at KG = 8 the sweep never picks it",
    dg(16, 1): "<8, 2> at twice the channel groups has the same tile at a lower cost per FMA (0.625 vs 1.0625) "
               "whenever KG <= 4; at KG = 8 the sweep never picks it",
    dg(16, 2): "<8, 4> at twice the channel groups has the same tile at a lower cost per FMA (0.375 vs 0.5625) "
               "whenever KG <= 4; at KG = 8 the sweep never picks it",
    dg(3, 2): "C = 3 is the only width that plans KT = 3, and allow_pt needs C >= 4: PT is always 1",
    dg(3, 4): "C = 3 is the only width that plans KT = 3, and allow_pt needs C >= 4: PT is always 1",
}


# ---- fp64 references (device-agnostic: tests/test_cpu_fused_case_table.py holds them to stock torch) -----------------
U = 2.0 ** -23
SLOPE = 0.2
MOMENTUM = 0.1
BN_EPS = 0.8          # nn.BatchNorm2d(out, 0.8) of dcgan.py:82
NBT0 = 7
BLOCK_PARTIAL = 1032  # values a chain kernel sums in fp32 before its fp64 atomic: at most a tile's 1024 pixels
ACT_CODE = {"none": _lib.ACT_NONE, "lrelu": _lib.ACT_LRELU, "relu": _lib.ACT_RELU, "tanh": _lib.ACT_TANH,
            "sigmoid": _lib.ACT_SIGMOID}
NEG_SLOPE = {"none": 1.0, "lrelu": SLOPE, "relu": 0.0}


def group_sums(t, G):
    """[G][2][C] fp64 sum and sum of squares of t [N, ..., C] over each of G equal runs of images"""
    t = t.double().reshape(G, -1, t.shape[-1])
    return torch.stack([t.sum(1), (t * t).sum(1)], 1)


def bn_consts(stats, gamma, beta, count, G, C, eps=BN_EPS):
    """mean, biased var, rstd, scale, shift [G][C] from the batch sums, as nb_bn_consts forms them (in fp64)"""
    st = stats.double().reshape(G, 2, C)
    mean = st[:, 0] / count
    var = (st[:, 1] / count - mean * mean).clamp_min(0)
    rstd = 1 / torch.sqrt(var + eps)
    ga = gamma.double() if gamma is not None else torch.ones_like(mean[0])
    be = beta.double() if beta is not None else torch.zeros_like(mean[0])
    sc = ga * rstd
    return mean, var, rstd, sc, be - mean * sc


def per_image(t, N):
    """[G][C] -> [N][1][1][C]: the group's row for every image of the group"""
    return t.repeat_interleave(N // t.shape[0], 0)[:, None, None, :]


def running_ref(rm, rv, mean, var, count, momentum=MOMENTUM):
    """one torch running-statistics update per group, in batch order"""
    rm, rv = rm.double(), rv.double()
    unb = var * count / (count - 1) if count > 1 else var
    for g in range(mean.shape[0]):
        rm = (1 - momentum) * rm + momentum * mean[g]
        rv = (1 - momentum) * rv + momentum * unb[g]
    return rm, rv


def nchw(t):
    return t.permute(0, 3, 1, 2)


def nhwc(t):
    return t.permute(0, 2, 3, 1)


def conv_fwd(x, w, stride, pad):
    return nhwc(F.conv2d(nchw(x), w, stride=stride, padding=pad))


def conv_dgrad(dz, w, xshape, stride, pad):
    N, H, W, C = xshape
    return nhwc(torch.nn.grad.conv2d_input((N, C, H, W), w, nchw(dz), stride, pad))


def conv_wgrad(x, dz, wshape, stride, pad):
    return torch.nn.grad.conv2d_weight(nchw(x), wshape, nchw(dz), stride, pad)


def bn_bwd_ref(G_, a, mean, rstd, sc, sums, count, cs, act):
    """nb_dz: dz = scale * (G - sum G / count - ahat * sum G ahat / count) * chan_scale * act'(a), groups per image"""
    N = a.shape[0]
    m1, m2 = sums[:, 0] / count, sums[:, 1] / count
    xh = (a - per_image(mean, N)) * per_image(rstd, N)
    dA = per_image(sc, N) * (G_ - per_image(m1, N) - xh * per_image(m2, N))
    return dA * cs * act_grad(act, a)


def act_grad(act, a):
    if act == "lrelu":
        return torch.where(a > 0, 1.0, SLOPE).double()
    if act == "relu":
        return (a > 0).double()
    return torch.ones_like(a, dtype=torch.float64)



def act_out64(act, v):
    return {"none": lambda: v, "tanh": lambda: torch.tanh(v), "sigmoid": lambda: torch.sigmoid(v),
            "lrelu": lambda: torch.where(v > 0, v, v * SLOPE), "relu": lambda: v.clamp_min(0)}[act]()


def act_bound(act, pre, y, bound):
    """carry an input bound through the activation and its fp32 evaluation (the conv suite's epilogue terms)"""
    lip = {"none": 1.0, "lrelu": 1.0, "relu": 1.0, "tanh": 1.0, "sigmoid": 0.25}[act]
    bound = lip * bound + U * y.abs()
    if act == "tanh":
        bound = bound + 4 * U * y.abs() + 2.0 ** -126
    if act == "sigmoid":
        bound = bound + U * (2 + 2 * pre.abs()) / 4 + 2 * U * y.abs()
    return bound




def chain_geom(c):
    return _lib.ConvGeom(c.N, c.H, c.W, c.C, c.K, c.R, c.R, c.stride, 1, 1, 1, 1, _lib.PAD_ZERO, 1, 0, c.P, c.Q)
