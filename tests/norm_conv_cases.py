"""Case table of the fused BatchNorm2d [-> LeakyReLU / ReLU] [-> Upsample x2] -> Conv2d backward
(b200gan_conv2d_dgrad_norm, then b200gan_norm_bwd_from_sums), and of the apply-from-sums entry point on its own.

A fused case is one geometry (N, C = norm channels = conv input channels, K = conv output channels, H x W = the norm's
map = the conv's input grid, the filter, up) with the norm's activation, run as functional.NormConvFn runs it: the conv's
data gradient `da` with the norm sums in its epilogue, then dx and dgamma / dbeta from those sums.  It names the kernel
instances of that sequence: conv_tc_kernel<BN, STAGES> with gridDim = (pixel tiles, C / BN, 1), then
norm_bwd_apply_kernel<4> and norm_bwd_params_kernel.  BN follows tc_block_n, the acceptance tc_dgrad_norm_supported
(pytorch-gan_b200/csrc/conv_tc.cu): a Conv2d of stride 1 with zero padding, up 1 or 2, BN <= 128, and a contraction
tc_ksplit does not split (it splits when there are fewer CTAs than SMs and at least 16 (tap, 32-channel) iterations).
A refused case names the code the call returns; it writes nothing.  Tile counts and BN assume a 132-SM H100 SXM.

The from-sums cases run b200gan_norm_bwd_from_sums alone over every geometry of tests/norm_cases.py, the fp64 sums
given: VEC 1 and 4, channel slices, InstanceNorm, non-affine, round_tf32 on and off.

tests/test_cpu_norm_conv_case_table.py checks the table against the library's predicate; tests/
test_gpu_norm_conv_conformance.py runs every case against fp64.
"""
from dataclasses import dataclass

import norm_cases as nc

NUM_SMS = 132
STAGES = {128: 6, 64: 8, 32: 8}
ENTRY_POINTS = ("b200gan_conv2d_dgrad_norm", "b200gan_norm_bwd_from_sums")


@dataclass(frozen=True)
class Case:
    name: str
    N: int
    C: int
    K: int
    H: int
    W: int
    R: int = 3
    S: int = 3
    pads: tuple = (1, 1, 1, 1)  # t, l, b, r
    up: int = 1
    stride: int = 1
    pad_mode: int = 0           # 1: reflection padding
    transposed: bool = False
    act: str = "none"           # the norm's activation: none, lrelu, relu (tanh / sigmoid: refused)
    slope: float = 0.2
    beta0: bool = False         # beta = 0: x * scale + shift > 0 for about half of the pixels
    rtf: bool = False           # round_tf32 on dx
    bn: int = 0                 # expected BN of conv_tc_kernel (0: refused)
    tiles: int = 0              # expected gridDim.x
    refuse: str = ""            # how the call is refused: geometry, per_sample, act, desc_N, desc_C, desc_HW, x_offset
    code: int = 0               # the refusal's return code
    why: str = ""

    @property
    def P(self):
        t, l, b, r = self.pads
        if self.transposed:
            return (self.H - 1) * self.stride - 2 * t + self.R
        return (self.H * self.up + t + b - self.R) // self.stride + 1

    @property
    def Q(self):
        t, l, b, r = self.pads
        if self.transposed:
            return (self.W - 1) * self.stride - 2 * l + self.S
        return (self.W * self.up + l + r - self.S) // self.stride + 1

    @property
    def kernels(self):
        if self.code:
            return ()
        return (f"conv_tc_kernel<{self.bn}, {STAGES[self.bn]}>", "norm_bwd_apply_kernel<4>", "norm_bwd_params_kernel")

    @property
    def grid(self):
        return (self.tiles, self.C // self.bn, 1) if self.bn else None

    @property
    def id(self):
        return self.name


def _a(name, N, C, K, H, W, bn, tiles, why, **kw):
    return Case(name, N, C, K, H, W, bn=bn, tiles=tiles, why=why, **kw)


def _r(name, N, C, K, H, W, why, code=-1, refuse="geometry", **kw):
    return Case(name, N, C, K, H, W, refuse=refuse, code=code, why=why, **kw)


P0 = (0, 0, 0, 0)
ASYM = (2, 2, 1, 1)  # ZeroPad2d((1, 0, 1, 0)) + Conv2d(4, padding=1)

# tiles: 128-pixel boxes of 2^ceil(log2 W) (at most 128) x 2^ceil(log2 H) (the rest of 128) pixels of 128 / box images
ACCEPTED = [
    _a("dcgan_bn128_up_conv128", 128, 128, 128, 16, 16, 128, 256, up=2,
       why="DCGAN block 1 (dcgan.py:53-55) at batch 128: BN = 128, 16x8 tiles"),
    _a("dcgan_bn128_lrelu_up_conv64", 128, 128, 64, 32, 32, 128, 1024, up=2, act="lrelu", slope=0.2,
       why="DCGAN block 2 (dcgan.py:56-59): LeakyReLU(0.2), 32x4 tiles"),
    _a("c256_two_ntiles", 64, 256, 64, 16, 16, 128, 128, act="relu", beta0=True,
       why="128 tiles keep BN = 128 for C = 256: two n-tiles; ReLU masks about half the pixels"),
    _a("c96_three_ntiles", 64, 96, 64, 16, 16, 32, 128, act="lrelu", slope=0.01,
       why="C = 96: BN = 32, three n-tiles; LeakyReLU(0.01)"),
    _a("c192_three_ntiles", 64, 192, 128, 16, 16, 64, 128, act="relu", rtf=True,
       why="C = 192: BN = 64, three n-tiles; dx rounded to TF32"),
    _a("c384_three_ntiles", 64, 384, 64, 16, 16, 128, 128, act="lrelu", slope=0.2,
       why="C = 384: BN = 128, three n-tiles"),
    _a("splitk_edge_in", 8, 64, 32, 16, 16, 64, 16,
       why="16 CTAs but 9 (tap, k-chunk) iterations: just inside the no-split rule"),
    _a("imgs8_per_tile", 33, 64, 32, 4, 4, 64, 5, act="lrelu", slope=0.2,
       why="4x4 maps: 8 images per tile, the last tile runs 7 images past N = 33"),
    _a("imgs32_per_tile", 5, 64, 32, 2, 2, 64, 1, act="relu",
       why="2x2 maps: one tile of 32 image slots holds all 5 images"),
    _a("imgs128_per_tile", 7, 64, 32, 1, 1, 64, 1,
       why="1x1 maps: every tap but the centre reads zero fill; 121 empty image slots"),
    _a("f1x1", 64, 64, 64, 16, 16, 64, 128, R=1, S=1, pads=P0, act="lrelu", slope=0.01, why="1x1 filter: one tap"),
    _a("f3x3_p0", 64, 64, 32, 16, 16, 64, 128, pads=P0, act="relu",
       why="3x3 without padding (14x14 dy): the only accepted non-p1 filter at batch 64, 9 iterations"),
    _a("f5x5", 20, 64, 32, 32, 32, 64, 160, R=5, S=5, pads=(2, 2, 2, 2), act="relu",
       why="5x5: 25 iterations, not split with 160 tiles"),
    _a("f7x7", 20, 64, 32, 32, 32, 64, 160, R=7, S=7, pads=(3, 3, 3, 3), act="lrelu", slope=0.2, rtf=True,
       why="7x7: 49 taps, not split with 160 tiles"),
    _a("f4x4_asym", 20, 64, 32, 32, 32, 64, 160, R=4, S=4, pads=ASYM,
       why="4x4 behind ZeroPad2d((1, 0, 1, 0)): asymmetric padding"),
    _a("relu_up1_3x3", 96, 64, 64, 16, 16, 64, 192, act="relu", why="ReLU, up 1"),
    _a("lrelu_up1_ragged_12x12", 96, 64, 32, 12, 12, 64, 192, act="lrelu", slope=0.1,
       why="16x8 tiles over 12x12 maps: rows and columns outside the map in every tile"),
    _a("none_up2_ragged_10x10", 80, 64, 64, 10, 10, 64, 160, up=2,
       why="up 2 over 10x10 maps: 16x8 tiles with pixels outside the map"),
    _a("relu_up2_k32", 128, 64, 32, 16, 16, 64, 256, up=2, act="relu", why="up 2 with 32 conv output channels"),
]

REFUSED = [
    _r("c256_bn256", 66, 256, 64, 16, 16, "132 tiles with C = 256: BN = 256, which has no norm epilogue"),
    _r("splitk_edge_out", 8, 64, 64, 16, 16, "18 iterations on 16 CTAs: split-K"),
    _r("splitk_5x5", 64, 64, 32, 16, 16, "5x5 at 128 tiles: 25 iterations, split", R=5, S=5, pads=(2, 2, 2, 2)),
    _r("splitk_3x3_p0_k64", 64, 64, 64, 16, 16, "3x3 p0 with K = 64: 18 iterations, split", pads=P0),
    _r("splitk_4x4_asym", 64, 64, 32, 16, 16, "4x4 at 128 tiles: 16 iterations, split", R=4, S=4, pads=ASYM),
    _r("splitk_7x7", 64, 64, 32, 16, 16, "7x7 at 128 tiles: 49 iterations, split", R=7, S=7, pads=(3, 3, 3, 3)),
    _r("reflect", 64, 64, 64, 16, 16, "reflection padding", pad_mode=1),
    _r("stride2", 64, 64, 64, 16, 16, "stride 2 writes its gradient through a phase view", stride=2),
    _r("conv_transpose", 64, 64, 64, 16, 16, "ConvTranspose2d(64, 64, 4, 2, 1)", R=4, S=4, stride=2, transposed=True),
    _r("per_sample", 128, 128, 128, 16, 16, "InstanceNorm statistics", refuse="per_sample", up=2),
    _r("act_tanh", 128, 128, 128, 16, 16, "Tanh after the norm", code=-2, refuse="act", act="tanh", up=2),
    _r("act_sigmoid", 128, 128, 128, 16, 16, "Sigmoid after the norm", code=-2, refuse="act", act="sigmoid", up=2),
    _r("desc_N", 128, 128, 128, 16, 16, "norm N differs from the conv's", code=-2, refuse="desc_N", up=2),
    _r("desc_C", 128, 128, 128, 16, 16, "norm C differs from the conv's", code=-2, refuse="desc_C", up=2),
    _r("desc_HW", 128, 128, 128, 16, 16, "norm HW differs from the conv's", code=-2, refuse="desc_HW", up=2),
    _r("x_offset", 96, 64, 64, 16, 16, "x one float past 16-byte alignment", code=-2, refuse="x_offset"),
]

FUSED = ACCEPTED + REFUSED


# ---- b200gan_norm_bwd_from_sums alone ---------------------------------------------------------------------------------
@dataclass(frozen=True)
class SumsCase:
    geom: nc.Geom
    act: str
    rtf: bool

    @property
    def code(self):
        return -2 if self.act in ("tanh", "sigmoid") else 0

    @property
    def kernels(self):
        if self.code:
            return ()
        return (f"norm_bwd_apply_kernel<{self.geom.vec}>", "norm_bwd_params_kernel")

    @property
    def why(self):
        return f"{self.geom.why}; {self.act}" + (" is refused" if self.code else "")

    @property
    def id(self):
        return f"sums-{self.geom.name}-{self.act}{'-rtf' if self.rtf else ''}"


FROM_SUMS = tuple(SumsCase(g, a, (i + j) % 2 == 1) for i, g in enumerate(nc.GEOMS) for j, a in enumerate(nc.ACTS))

CASES = tuple(FUSED) + FROM_SUMS
