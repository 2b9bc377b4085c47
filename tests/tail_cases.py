"""Case table of the generator tail (pytorch-gan_b200/csrc/tail.cu): b200gan_tail_fprop and b200gan_tail_bwd.

Every (C, K) pair the ABI accepts, so that each of the 6 forward instances tail_fprop_tc_kernel<C/4, NB> (NB = 16 at
K = 1, else 32) and each of the 9 backward pairs tail_bwd_reduce_kernel<C/4, K> / tail_bwd_apply_kernel<C/4, K> runs,
across the map widths, activations, range splits and optional outputs where the kernels go wrong.  Each case runs the
forward and then the backward; an `error` case must be refused by both.

tests/test_cpu_fused_case_table.py holds the table to b200gan_tail_supported and to the instances tail.cu launches;
tests/test_gpu_fused_conformance.py runs every case against torch float64.
"""
from dataclasses import dataclass

import torch

from chain_cases import NEG_SLOPE, SLOPE, act_out64, conv_dgrad, conv_fwd, conv_wgrad
from conformance import tf32_rna

ACT_MID = ("none", "lrelu", "relu")
ACT_OUT = ("none", "tanh", "sigmoid")


@dataclass(frozen=True)
class Case:
    name: str
    N: int
    C: int
    K: int
    H: int
    W: int
    act_mid: str = "lrelu"
    act_out: str = "tanh"
    rtf: bool = False            # backward: da rounded to TF32
    bias: bool = True
    dgb: bool = True             # backward: dgamma_dbeta given (else NULL)
    db: bool = True              # backward: db given (else NULL)
    error: bool = False
    why: str = ""

    @property
    def kernels(self):
        c4, nb = self.C // 4, 16 if self.K == 1 else 32
        return (f"tail_fprop_tc_kernel<{c4}, {nb}>", f"tail_bwd_reduce_kernel<{c4}, {self.K}>",
                f"tail_bwd_apply_kernel<{c4}, {self.K}>")

    @property
    def id(self):
        return self.name


_c = Case
CASES = [
    _c("c32k1_w16", 2, 32, 1, 16, 16, why="smallest width: 8 image rows per 128-pixel tile"),
    _c("c32k2_tiny", 1, 32, 2, 3, 16, act_mid="relu", dgb=False,
       why="48 pixels: fewer than one ring chunk (128 at C = 32), one block"),
    _c("c32k3_w32", 2, 32, 3, 30, 32, act_out="none", rtf=True, why="K = 3, 30 rows: ragged tiles"),
    _c("c64k1_dcgan", 4, 64, 1, 64, 64, rtf=True,
       why="the DCGAN generator's tail (dcgan.py:60-63) with the batch reduced"),
    _c("c64k2_row", 5, 64, 2, 1, 64, act_mid="none", act_out="sigmoid",
       why="one-row images: the staged g has a zero row after every row"),
    _c("c64k3_w16", 3, 64, 3, 20, 16, act_mid="relu", db=False, bias=False, why="ragged bands, db and bias NULL"),
    _c("c128k1_mid", 7, 128, 1, 37, 32, why="ranges that start mid-image, 37 rows"),
    _c("c128k2_w128", 1, 128, 2, 5, 128, act_mid="none", act_out="sigmoid", dgb=False, why="W = 128: one row per tile"),
    _c("c128k3_w64", 2, 128, 3, 17, 64, rtf=True, why="K = 3 at C = 128: the largest filter matrix"),
    _c("slab_cap", 8000, 32, 1, 1, 128, why="the staged g caps the range length: more blocks than resident slots"),
    _c("c96", 2, 96, 1, 8, 16, error=True, why="C = 96 is not one of 32, 64, 128"),
    _c("w48", 2, 64, 1, 8, 48, error=True, why="W = 48 is not a power of two"),
    _c("k4", 2, 64, 4, 8, 16, error=True, why="K = 4 > 3"),
    _c("mid_tanh", 2, 64, 1, 8, 16, act_mid="tanh", error=True, why="act_mid must be none, LeakyReLU or ReLU"),
]


# ---- fp64 references (device-agnostic: tests/test_cpu_fused_case_table.py holds them to stock torch) -----------------
def act_mid32(act, v):
    """the tail's LeakyReLU / ReLU in fp32, as the kernel computes it"""
    if act == "lrelu":
        return torch.where(v > 0, v, v * SLOPE)
    if act == "relu":
        return v.clamp_min(0)
    return v

def tail_fwd_ref(a, ss, w, bias, act_mid, act_out):
    """tail.cu forward: operands as the kernel feeds wgmma (RNA TF32); returns out, the linear part and A"""
    C = a.shape[-1]
    pre = (a.double() * ss[:C].double() + ss[C:].double()).float()     # fmaf(a, sc, sh)
    x = tf32_rna(act_mid32(act_mid, pre)).double()
    wr = tf32_rna(w).double()
    conv = conv_fwd(x, wr, 1, 1)
    A = conv_fwd(x.abs(), wr.abs(), 1, 1)
    b = bias.double() if bias is not None else torch.zeros(w.shape[0], dtype=torch.float64, device=a.device)
    return act_out64(act_out, conv + b), conv + b, A, b


def tail_bwd_ref(a, mr, ss, w, g, act_mid, neg_branch):
    """tail.cu backward with the activation's derivative on `neg_branch` (bool mask: take the negative side)"""
    C, K = a.shape[-1], w.shape[0]
    a64 = a.double()
    sc, sh, mean, rstd = ss[:C].double(), ss[C:].double(), mr[:C].double(), mr[C:].double()
    pre = a64 * sc + sh
    neg = NEG_SLOPE[act_mid]
    y = torch.where(neg_branch, pre * neg, pre)
    dy = conv_dgrad(g.double(), w.double(), a.shape, 1, 1)
    dz = torch.where(neg_branch, dy * neg, dy)
    xh = (a64 - mean) * rstd
    total = a.numel() // C
    s1, s2 = dz.sum((0, 1, 2)), (dz * xh).sum((0, 1, 2))
    da = sc * (dz - s1 / total - xh * (s2 / total))
    dw = conv_wgrad(y, g.double(), (K, C, 3, 3), 1, 1)
    return dict(da=da, s1=s1, s2=s2, dw=dw, db=g.double().sum((0, 1, 2)), y=y, dz=dz, xh=xh, pre=pre, dy=dy)


# ---- the modules of the GPU parity tests (test_gpu_tail.py, test_gpu_tail_ranges.py) --------------------------------
def mods(ns, c, k, mid, out):
    """Conv2d(8, c) -> BatchNorm2d(c, 0.8) [-> LeakyReLU / ReLU] -> Conv2d(c, k, 3, 1, 1) [-> Tanh / Sigmoid] from the
    namespace ns"""
    layers = [ns.Conv2d(8, c, 3, 1, 1), ns.BatchNorm2d(c, 0.8)]
    if mid == "lrelu":
        layers.append(ns.LeakyReLU(0.2, inplace=True))
    elif mid == "relu":
        layers.append(ns.ReLU(inplace=True))
    layers.append(ns.Conv2d(c, k, 3, stride=1, padding=1))
    if out == "tanh":
        layers.append(ns.Tanh())
    elif out == "sigmoid":
        layers.append(ns.Sigmoid())
    return ns.Sequential(*layers)
