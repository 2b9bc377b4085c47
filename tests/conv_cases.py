"""Route table of the convolution entry points (b200gan_conv2d_fprop / dgrad / wgrad).

One entry per (geometry, pass, algorithm, epilogue) together with what the library must do with it: the kernels that
appear in a trace of the call, the grid of the main kernel where the planner's choice shows there (split-K:
gridDim.z = phases x ksplit; weight gradient: gridDim.x = pixel splits), whether repeating the call must give the
same bits, and the partial sums `s` that are added outside one accumulation chain (k-splits, pixel splits, folded
jobs).  Each case names the edge it exists for.

The table is written from the eligibility predicates (tc_supported, wg_plan, fewk_ok, nb_plain_*_ok, nb_wgrad_ok),
not from a run.  Tile widths and split counts assume a 132-SM H100 SXM; tests/test_gpu_conv_conformance.py checks the
grids only on such a device.

tests/test_cpu_conv_case_table.py checks it against b200gan_conv2d_supported and against the kernels declared in the
sources; tests/test_gpu_conv_conformance.py runs every case.  The fp64 references, their bounds and the bias-gradient
chain of the weight-gradient kernel sit at the end of this module, where the fused norm-conv suite shares them.
"""
import math
from dataclasses import dataclass, replace

import torch
import torch.nn.functional as F

FPROP, DGRAD, WGRAD = 0, 1, 2
PASS_NAMES = {FPROP: "fprop", DGRAD: "dgrad", WGRAD: "wgrad"}
ZERO, REFLECT = 0, 1
NUM_SMS = 132  # the tile widths and split counts below are those of a 132-SM H100 SXM

# epilogue options of an fprop case
EPI_OPTIONS = ("bias", "lrelu", "relu", "tanh", "sigmoid", "chan_scale", "round_tf32", "stats_c", "stats_s")

# every kernel a convolution call can launch besides the convolution kernels themselves
HELPER_KERNELS = {"norm_stats_kernel", "pad2d_bwd_kernel", "pad2d_bwd_v4_kernel", "upsample2x_bwd_kernel"}


@dataclass(frozen=True)
class Case:
    name: str
    N: int
    C: int
    K: int
    H: int
    W: int
    R: int
    S: int
    stride: int = 1
    pads: tuple = (0, 0, 0, 0)  # t, l, b, r of the virtual input (ConvTranspose2d: its `padding`, symmetric)
    pad_mode: int = ZERO
    up: int = 1
    transposed: bool = False
    pas: int = FPROP
    algo: str = "AUTO"          # AUTO: the tensor-core path when b200gan_conv2d_supported says so; SIMT: forced
    epi: tuple = ()             # subset of EPI_OPTIONS (fprop only)
    kernels: tuple = ()         # kernel names expected in the trace ("name" matches any instantiation, "name<a, b>" one)
    grid: tuple = None          # (x, y, z) of kernels[0], or None when it says nothing about the plan
    deterministic: bool = True  # repeating the call gives the same bits (dy / dw / dx; never the fp64 statistics)
    s: int = 0                  # partial sums added outside one accumulation chain
    error: bool = False         # the call must be refused (B200GAN_E_BAD_ARG)
    fused_bias: bool = False    # wgrad through b200gan_conv2d_wgrad_fused_bias (db summed inside wgrad_tc_kernel)
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
    def tc(self):
        """the table expects a wgmma kernel"""
        return any(k.startswith(("conv_tc_", "wgrad_tc_")) for k in self.kernels)

    @property
    def id(self):
        return f"{self.name}-{PASS_NAMES[self.pas]}"


def _c(name, N, C, K, H, W, R, S, **kw):
    return Case(name, N, C, K, H, W, R, S, **kw)


P1 = (1, 1, 1, 1)
P2 = (2, 2, 2, 2)
P3 = (3, 3, 3, 3)

# ---- wgmma forward / data gradient (conv_tc.cu) ------------------------------------------------------------------
TC = [
    # BN = 256 needs K % 256 == 0 and tiles * K / 256 >= NUM_SMS: 32x32 maps are 8 tiles of 32x4 pixels per image
    _c("bn256_on", 17, 32, 256, 32, 32, 3, 3, pads=P1, epi=("bias",), kernels=("conv_tc_kernel<256, 4>",),
       grid=(136, 1, 1), why="BN = 256 just inside tiles * K/256 >= num_sms (136 tiles)"),
    _c("bn256_off", 16, 32, 256, 32, 32, 3, 3, pads=P1, epi=("bias",), kernels=("conv_tc_kernel<128, 6>",),
       grid=(128, 2, 1), why="BN = 256 just outside its rule (128 tiles): BN = 128"),
    _c("bn64_bnn2", 2, 32, 64, 8, 8, 3, 3, pads=P1, epi=("bias", "lrelu"), kernels=("conv_tc_kernel<64, 8>",),
       grid=(1, 1, 1), why="BN = 64; one tile holds two 8x8 images (BNn = 2)"),
    _c("bn32_ragged", 1, 32, 96, 12, 12, 3, 3, pads=P1, epi=("bias",), kernels=("conv_tc_kernel<32, 8>",),
       grid=(2, 3, 1), why="BN = 32 (K = 96); 12x12 map clipped by 16x8 tiles"),
    _c("bnn2_stats", 4, 32, 64, 8, 8, 3, 3, pads=P1, epi=("bias", "stats_c"), kernels=("conv_tc_kernel<64, 8>",),
       grid=(2, 1, 1), why="fused per-channel statistics of tiles that each hold two whole images"),
    _c("bnn_gt_n", 3, 32, 64, 4, 4, 3, 3, pads=P1, epi=("bias", "relu"), kernels=("conv_tc_kernel<64, 8>",),
       grid=(1, 1, 1), why="BNn = 8 images per tile with N = 3"),
    _c("map1x1", 4, 64, 128, 1, 1, 3, 3, pads=P1, epi=("bias", "relu"), kernels=("conv_tc_kernel<128, 6>",),
       grid=(1, 1, 1), why="1x1 map: every tap but the centre reads TMA zero fill; BNn = 128"),
    _c("wide160", 1, 32, 64, 2, 160, 3, 3, pads=P1, epi=("bias",), kernels=("conv_tc_kernel<64, 8>",),
       grid=(4, 1, 1), why="map wider than 128: two tiles across, the second one clipped"),
    _c("f7x7", 1, 32, 64, 16, 16, 7, 7, pads=P3, epi=("bias",), kernels=("conv_tc_kernel<64, 8>",),
       grid=(2, 1, 1), why="7x7 filter, 49 taps"),
    _c("f1x1", 2, 64, 64, 8, 8, 1, 1, epi=("bias",), kernels=("conv_tc_kernel<64, 8>",), grid=(1, 1, 1),
       why="1x1 filter"),
    _c("s2_gather", 2, 32, 64, 16, 16, 4, 4, stride=2, pads=P1, epi=("bias", "lrelu"),
       kernels=("conv_tc_kernel<64, 8>",), grid=(1, 1, 1), why="stride-2 gather through the parity view"),
    _c("narrow3", 2, 32, 3, 8, 8, 3, 3, pads=P1, epi=("bias", "tanh"), kernels=("conv_tc_kernel<32, 8>",),
       grid=(1, 1, 1), why="narrow-K: 3 output channels, direct stores"),
    _c("narrow5", 2, 32, 5, 8, 8, 3, 3, pads=P1, epi=("bias",), kernels=("conv_tc_kernel<32, 8>",), grid=(1, 1, 1),
       why="narrow-K with 5 output channels"),
    _c("narrow31", 1, 64, 31, 8, 8, 3, 3, pads=P1, epi=("bias",), kernels=("conv_tc_kernel<32, 8>",),
       grid=(1, 1, 1), why="narrow-K just inside (31 output channels)"),
    _c("k32_not_narrow", 1, 64, 32, 8, 8, 3, 3, pads=P1, epi=("bias",), kernels=("conv_tc_kernel<32, 8>",),
       grid=(1, 1, 1), why="32 output channels: just outside narrow-K, TMA stores"),
    # split-K: plain epilogue, fewer CTAs than SMs, >= 16 (tap, k-chunk) iterations per phase
    _c("splitk_plain", 1, 256, 256, 4, 4, 4, 4, stride=2, pads=P1, kernels=("conv_tc_kernel<128, 6>",),
       grid=(1, 2, 16), deterministic=False, s=16, why="deep U-Net layer: 2 CTAs, 128 iterations -> 16 k-splits"),
    _c("splitk_bias", 1, 256, 256, 4, 4, 4, 4, stride=2, pads=P1, epi=("bias",), kernels=("conv_tc_kernel<128, 6>",),
       grid=(1, 2, 1), why="the same layer with a bias must not split"),
    _c("splitk_stats", 1, 256, 256, 4, 4, 4, 4, stride=2, pads=P1, epi=("stats_c",),
       kernels=("conv_tc_kernel<128, 6>", "norm_stats_kernel"), grid=(1, 2, 16), deterministic=False, s=16,
       why="split-K with statistics: a deferred norm_stats pass"),
    _c("splitk_short", 1, 32, 64, 4, 4, 3, 3, pads=P1, kernels=("conv_tc_kernel<64, 8>",), grid=(1, 1, 1),
       why="plain epilogue but only 9 iterations: no split"),
    # folded x2 upsample
    _c("up2_allphase_1x1", 2, 32, 64, 1, 1, 3, 3, pads=P1, up=2, epi=("bias", "lrelu"),
       kernels=("conv_tc_up2_allphase_kernel",), grid=(1, 1, 1), why="all-phase kernel at 1x1 per phase"),
    _c("up2_allphase_3x5", 2, 32, 64, 3, 5, 3, 3, pads=P1, up=2, epi=("bias",),
       kernels=("conv_tc_up2_allphase_kernel",), grid=(1, 1, 1), why="all-phase kernel at 3x5 per phase"),
    _c("up2_phases", 2, 32, 128, 4, 4, 3, 3, pads=P1, up=2, epi=("bias",), kernels=("conv_tc_kernel<128, 6>",),
       grid=(1, 1, 4), why="K % 128 == 0: one phase per blockIdx.z"),
    # scatter form (ConvTranspose2d forward)
    _c("tr_s2_4x4", 2, 32, 64, 4, 4, 4, 4, stride=2, pads=(1, 1, 1, 1), transposed=True, epi=("bias",),
       kernels=("conv_tc_kernel<64, 8>",), grid=(1, 1, 4), why="transposed stride 2: four scatter phases"),
]

TC_DGRAD = [
    _c("d_s1", 2, 64, 64, 8, 8, 3, 3, pads=P1, pas=DGRAD, kernels=("conv_tc_kernel<64, 8>",), grid=(1, 1, 2),
       deterministic=False, s=2, why="dgrad is always plain: 1 CTA, 18 iterations -> 2 k-splits"),
    _c("d_bn256_on", 17, 256, 32, 32, 32, 3, 3, pads=P1, pas=DGRAD, kernels=("conv_tc_kernel<256, 4>",),
       grid=(136, 1, 1), why="BN = 256 in dgrad (C = 256, 136 tiles)"),
    _c("d_bn256_off", 16, 256, 32, 32, 32, 3, 3, pads=P1, pas=DGRAD, kernels=("conv_tc_kernel<128, 6>",),
       grid=(128, 2, 1), why="dgrad just outside the BN = 256 rule"),
    _c("d_s2_3x3", 2, 64, 32, 8, 8, 3, 3, stride=2, pads=P1, pas=DGRAD, kernels=("conv_tc_kernel<64, 8>",),
       grid=(1, 1, 4), why="stride-2 scatter, 3x3: phases with 1, 2, 2 and 4 taps"),
    _c("d_s2_4x4", 2, 32, 64, 16, 16, 4, 4, stride=2, pads=P1, pas=DGRAD, kernels=("conv_tc_kernel<32, 8>",),
       grid=(1, 1, 4), why="stride-2 scatter, 4x4: four taps per phase"),
    _c("d_tr_s2", 2, 32, 64, 4, 4, 4, 4, stride=2, pads=P1, transposed=True, pas=DGRAD,
       kernels=("conv_tc_kernel<32, 8>",), grid=(1, 1, 4), deterministic=False, s=4,
       why="transposed stride-2 dgrad: gather over dy, 32 iterations -> 4 k-splits"),
    _c("d_up2", 2, 64, 64, 4, 4, 3, 3, pads=P1, up=2, pas=DGRAD, kernels=("conv_tc_kernel<64, 8>",),
       grid=(1, 1, 4), deterministic=False, s=4, why="up2 dgrad through the phase view of dy, 4 k-splits"),
    _c("d_7x7", 1, 32, 32, 8, 8, 7, 7, pads=P3, pas=DGRAD, kernels=("conv_tc_kernel<32, 8>",), grid=(1, 1, 6),
       deterministic=False, s=6, why="7x7 dgrad, 49 iterations -> 6 k-splits"),
    _c("d_1x1", 2, 64, 64, 8, 8, 1, 1, pas=DGRAD, kernels=("conv_tc_kernel<64, 8>",), grid=(1, 1, 1),
       why="1x1 filter dgrad"),
]

# ---- wgmma weight gradient (wgrad_tc.cu) --------------------------------------------------------------------------
_WG_TILE = ("wgrad_reduce_tile_kernel", "colsum_kernel")
TC_WGRAD = [
    _c("w_nb32", 2, 32, 128, 8, 8, 3, 3, pads=P1, pas=WGRAD, kernels=("wgrad_tc_kernel<32, 8>",) + _WG_TILE,
       grid=(1, 9, 1), why="NB = 32, A = dy"),
    _c("w_nb64", 2, 64, 128, 8, 8, 3, 3, pads=P1, pas=WGRAD, kernels=("wgrad_tc_kernel<64, 8>",) + _WG_TILE,
       grid=(1, 9, 1), why="NB = 64"),
    _c("w_nb128_sisa", 2, 128, 32, 8, 8, 3, 3, pads=P1, pas=WGRAD,
       kernels=("wgrad_tc_kernel<32, 8>",) + _WG_TILE, grid=(1, 9, 1), why="x is A (K = 32 is not a multiple of 128)"),
    _c("w_nb128", 2, 128, 128, 8, 8, 3, 3, pads=P1, pas=WGRAD, kernels=("wgrad_tc_kernel<128, 6>",) + _WG_TILE,
       grid=(1, 9, 1), why="NB = 128"),
    _c("w_nb256", 2, 256, 128, 8, 8, 3, 3, pads=P1, pas=WGRAD, kernels=("wgrad_tc_kernel<256, 3>",) + _WG_TILE,
       grid=(1, 9, 1), why="NB = 256"),
    _c("w_ipb2", 3, 32, 128, 4, 4, 3, 3, pads=P1, pas=WGRAD, kernels=("wgrad_tc_kernel<32, 8>",) + _WG_TILE,
       grid=(1, 9, 1), why="4x4 maps: two images per 32-pixel box, the last box half past N"),
    _c("w_splits", 4, 32, 128, 32, 32, 3, 3, pads=P1, pas=WGRAD, kernels=("wgrad_tc_kernel<32, 8>",) + _WG_TILE,
       grid=(13, 9, 1), deterministic=False, s=13, why="128 pixel tiles -> 13 pixel splits reduce-added at L2"),
    _c("w_7x7", 1, 32, 128, 8, 8, 7, 7, pads=P3, pas=WGRAD,
       kernels=("wgrad_tc_kernel<32, 8>", "wgrad_reduce_kernel", "colsum_kernel"), grid=(1, 49, 1),
       why="R*S = 49 > 16: the generic wgrad_reduce_kernel"),
    _c("w_s2", 2, 32, 128, 16, 16, 4, 4, stride=2, pads=P1, pas=WGRAD,
       kernels=("wgrad_tc_kernel<32, 8>",) + _WG_TILE, grid=(1, 16, 1), why="stride 2: x through the parity view"),
    _c("w_tr_s2", 2, 128, 32, 4, 4, 4, 4, stride=2, pads=P1, transposed=True, pas=WGRAD,
       kernels=("wgrad_tc_kernel<32, 8>",) + _WG_TILE, grid=(1, 16, 1), why="transposed stride-2 wgrad: dy shifted"),
    _c("w_up2", 2, 32, 128, 4, 4, 3, 3, pads=P1, up=2, pas=WGRAD, kernels=("wgrad_tc_kernel<32, 8>",) + _WG_TILE,
       grid=(1, 16, 1), s=4, why="up2: 16 (phase, tap) jobs folded into 9 taps by the reduce"),
]

# ---- fp32 SIMT (conv_simt.cu) ---------------------------------------------------------------------------------------
SIMT = [
    _c("simt_gemm", 2, 32, 64, 8, 8, 3, 3, pads=P1, algo="SIMT", epi=("bias", "lrelu"),
       kernels=("conv_gather_gemm_kernel",), grid=(2, 1, 1), why="SIMT forced on a TC-eligible fprop"),
    _c("simt_gemm", 2, 32, 64, 8, 8, 3, 3, pads=P1, algo="SIMT", pas=DGRAD, kernels=("conv_gather_gemm_kernel",),
       why="SIMT forced on a TC-eligible dgrad: virtual-input gather, stride 1"),
    _c("simt_s2", 2, 32, 64, 8, 8, 3, 3, stride=2, pads=P1, algo="SIMT", pas=DGRAD,
       kernels=("conv_gather_gemm_kernel",), grid=(1, 1, 4), why="stride-2 transposed gather in parity classes"),
    _c("simt_wg_staged", 2, 32, 128, 8, 8, 3, 3, pads=P1, algo="SIMT", pas=WGRAD,
       kernels=("nbk_wgrad_kernel<9>", "colsum_kernel"), deterministic=False,
       why="SIMT forced on a TC-eligible wgrad: the staged kernel with fp32 atomics"),
    _c("simt_5x5", 2, 32, 64, 8, 8, 5, 5, pads=P2, pas=WGRAD, kernels=("conv_wgrad_kernel", "colsum_kernel"),
       deterministic=False, s=528, why="5x5: neither TC (no 128-channel operand) nor staged: conv_wgrad_kernel"),
    _c("simt_5x5", 2, 32, 64, 8, 8, 5, 5, pads=P2, algo="SIMT", epi=("bias",), kernels=("conv_gather_gemm_kernel",),
       why="5x5 forward forced onto the generic gather GEMM"),
    _c("smallk_gather", 2, 33, 3, 8, 8, 3, 3, pads=P1, epi=("bias",), kernels=("conv_gather_gemm_kernel",),
       why="K = 3 with C = 33 (not fewk): 3 of the tile's 64 output columns, a reduction that is not a multiple of 16"),
    _c("smallk_vec", 2, 64, 1, 8, 8, 4, 4, stride=2, pads=P1, epi=("bias", "sigmoid"),
       kernels=("conv_gather_gemm_kernel",), why="K = 1, stride 2 (not fewk): one output column of the tile"),
    _c("smallc", 2, 3, 12, 8, 8, 4, 4, stride=2, pads=P1, epi=("bias",), kernels=("conv_gather_gemm_kernel",),
       why="C = 3, K = 12 (not a multiple of 16, so not staged): 12 of the tile's 64 output columns"),
    _c("s3_smallc", 2, 3, 8, 8, 8, 3, 3, pads=P1, epi=("bias", "lrelu"), kernels=("conv_gather_gemm_kernel",),
       why="3x3 s1 p1 with C = 3, K = 8: a 27-long reduction, its second 16-wide slice partly empty"),
    _c("s3_smallk", 2, 16, 2, 8, 8, 3, 3, pads=P1, epi=("bias",), kernels=("conv_gather_gemm_kernel",),
       why="3x3 s1 p1 with K = 2, C = 16 (too few channels for fewk)"),
    _c("smallcd", 2, 64, 2, 8, 8, 5, 5, stride=2, pads=P2, pas=WGRAD,
       kernels=("conv_wgrad_kernel", "colsum_kernel"), deterministic=False, s=528,
       why="wgrad with 2 output channels, 5x5 s2: 2 of the tile's 64 dense columns"),
    _c("tr_cd1", 2, 1, 16, 8, 8, 3, 3, pads=P1, transposed=True, pas=WGRAD,
       kernels=("conv_wgrad_kernel", "colsum_kernel"), deterministic=False, s=528,
       why="ConvTranspose2d(1, 16, 3, 1, 1) wgrad: one dense channel, gathered over dy"),
    _c("tr_simt_s2", 2, 32, 64, 4, 4, 4, 4, stride=2, pads=P1, transposed=True, algo="SIMT",
       epi=("bias",), kernels=("conv_gather_gemm_kernel",), grid=(1, 1, 4),
       why="transposed stride-2 fprop forced onto SIMT: parity classes"),
    _c("tr_simt_s2", 2, 64, 3, 4, 4, 4, 4, stride=2, pads=P1, transposed=True, pas=DGRAD,
       kernels=("conv_gather_gemm_kernel",), why="transposed dgrad with 3 output channels: SIMT gather over dy"),
    _c("tr_simt_s2", 2, 64, 3, 4, 4, 4, 4, stride=2, pads=P1, transposed=True, pas=WGRAD,
       kernels=("conv_wgrad_kernel", "colsum_kernel"), deterministic=False, s=528, why="transposed SIMT wgrad"),
    _c("virt_up2_reflect", 2, 32, 16, 4, 4, 3, 3, pads=P1, pad_mode=REFLECT, up=2, pas=DGRAD,
       kernels=("conv_gather_gemm_kernel", "pad2d_bwd_v4_kernel", "upsample2x_bwd_kernel"), s=8,
       why="virtual dgrad: reflection fold then upsample fold, both through the workspace"),
    _c("virt_up2_reflect", 2, 32, 16, 4, 4, 3, 3, pads=P1, pad_mode=REFLECT, up=2, epi=("bias",),
       kernels=("conv_gather_gemm_kernel",), why="reflect + up2 forward gather"),
    _c("virt_up2_reflect", 2, 32, 16, 4, 4, 3, 3, pads=P1, pad_mode=REFLECT, up=2, pas=WGRAD,
       kernels=("conv_wgrad_kernel", "colsum_kernel"), deterministic=False, s=528, why="reflect + up2 wgrad"),
    _c("simt_up2", 2, 32, 48, 4, 4, 3, 3, pads=P1, up=2, pas=DGRAD,
       kernels=("conv_gather_gemm_kernel", "upsample2x_bwd_kernel"), s=4,
       why="up2 dgrad off the TC path (K = 48 is not a multiple of 32): gather, then the upsample fold"),
]

# ---- fewk.cu: K <= 4 output channels, stride 1 -----------------------------------------------------------------------
FEWK = [
    _c("fewk7_reflect", 2, 64, 3, 16, 16, 7, 7, pads=P3, pad_mode=REFLECT, epi=("bias", "tanh"),
       kernels=("fewk_fprop_kernel<7, 3>",), why="ReflectionPad2d(3) + Conv2d(64, 3, 7)"),
    _c("fewk7_reflect", 2, 64, 3, 16, 16, 7, 7, pads=P3, pad_mode=REFLECT, pas=DGRAD,
       kernels=("fewk_dgrad_kernel<7, 3>", "pad2d_bwd_v4_kernel"), s=4,
       why="reflection through the fewk dgrad and the pad fold"),
    _c("fewk7_reflect", 2, 64, 3, 16, 16, 7, 7, pads=P3, pad_mode=REFLECT, pas=WGRAD,
       kernels=("fewk_wgrad_kernel<7, 3>", "nbk_wgrad_reduce_kernel", "colsum_kernel"), s=264,
       why="fewk wgrad: per-block slabs + fixed-order reduce"),
    _c("fewk3", 2, 32, 4, 8, 8, 3, 3, pads=P1, algo="SIMT", epi=("bias",), kernels=("fewk_fprop_kernel<3, 4>",),
       why="3x3 fewk forward (AUTO would take the narrow-K wgmma kernel)"),
    _c("fewk3", 2, 32, 4, 8, 8, 3, 3, pads=P1, pas=DGRAD, kernels=("fewk_dgrad_kernel<3, 4>",), why="3x3 fewk dgrad"),
    _c("fewk3", 2, 32, 4, 8, 8, 3, 3, pads=P1, pas=WGRAD,
       kernels=("fewk_wgrad_kernel<3, 4>", "nbk_wgrad_reduce_kernel", "colsum_kernel"), s=264,
       why="3x3 fewk wgrad"),
    _c("fewk4_up2", 2, 32, 3, 4, 4, 4, 4, pads=(2, 2, 1, 1), up=2, epi=("bias", "tanh"),
       kernels=("fewk_fprop_up2_kernel<4, 3, 0>",),
       why="Upsample + ZeroPad2d((1,0,1,0)) + Conv2d(C, 3, 4, padding=1): folded, even pad_l"),
    _c("fewk4_up2", 2, 32, 3, 4, 4, 4, 4, pads=(2, 2, 1, 1), up=2, pas=DGRAD,
       kernels=("fewk_dgrad_up2_kernel<4, 3>",), s=8, why="fewk up2 dgrad"),
    _c("fewk4_up2", 2, 32, 3, 4, 4, 4, 4, pads=(2, 2, 1, 1), up=2, pas=WGRAD,
       kernels=("fewk_wgrad_up2_kernel<4, 3, 0>", "nbk_wgrad_reduce_kernel", "colsum_kernel"), s=272,
       why="fewk up2 wgrad"),
    _c("fewk3_up2", 2, 64, 1, 4, 4, 3, 3, pads=P1, up=2, epi=("bias",), kernels=("fewk_fprop_up2_kernel<3, 1, 1>",),
       why="Upsample + Conv2d(C, 1, 3, 1, 1): folded, odd pad_l"),
    _c("fewk3_up2", 2, 64, 1, 4, 4, 3, 3, pads=P1, up=2, pas=DGRAD, kernels=("fewk_dgrad_up2_kernel<3, 1>",), s=8,
       why="fewk 3x3 up2 dgrad"),
    _c("fewk3_up2", 2, 64, 1, 4, 4, 3, 3, pads=P1, up=2, pas=WGRAD,
       kernels=("fewk_wgrad_up2_kernel<3, 1, 1>", "nbk_wgrad_reduce_kernel", "colsum_kernel"), s=272,
       why="fewk 3x3 up2 wgrad"),
]

# ---- narrow_block.cu: the staged kernels on their own (few input channels) -------------------------------------------
STAGED = [
    _c("nb4_s2", 4, 3, 64, 16, 16, 4, 4, stride=2, pads=P1, epi=("bias", "lrelu"), kernels=("nbk_fprop2_kernel",),
       why="Conv2d(3, 64, 4, 2, 1): staged forward (at N = 2 the dgrad plan's tiles would be mostly empty)"),
    _c("nb4_s2", 4, 3, 64, 16, 16, 4, 4, stride=2, pads=P1, pas=DGRAD, kernels=("nbk_dgrad2_kernel",),
       grid=(None, None, 4), why="staged dgrad, four parity classes"),
    _c("nb4_s2", 4, 3, 64, 16, 16, 4, 4, stride=2, pads=P1, pas=WGRAD,
       kernels=("nbk_wgrad_kernel<16>", "colsum_kernel"), deterministic=False, why="staged wgrad with atomics"),
    _c("nb_asym", 2, 3, 64, 16, 16, 4, 4, stride=2, pads=(2, 2, 1, 1), epi=("bias",), kernels=("nbk_fprop2_kernel",),
       why="ZeroPad2d((1,0,1,0)) + Conv2d(3, 64, 4, 2, 1): asymmetric padding, allowed by nb_plain_fprop_ok"),
    _c("nb_asym", 2, 3, 64, 16, 16, 4, 4, stride=2, pads=(2, 2, 1, 1), pas=DGRAD,
       kernels=("conv_gather_gemm_kernel",), why="asymmetric padding is not staged in dgrad: SIMT gather"),
    _c("nb_asym", 2, 3, 64, 16, 16, 4, 4, stride=2, pads=(2, 2, 1, 1), pas=WGRAD,
       kernels=("conv_wgrad_kernel", "colsum_kernel"), deterministic=False, s=528,
       why="asymmetric padding is not staged in wgrad: SIMT"),
    _c("nb7_reflect", 2, 3, 64, 16, 16, 7, 7, pads=P3, pad_mode=REFLECT, epi=("bias", "relu"),
       kernels=("nbk_fprop2_kernel",), why="ReflectionPad2d(3) + Conv2d(3, 64, 7): staged forward, reflected"),
    _c("nb7_reflect", 2, 3, 64, 16, 16, 7, 7, pads=P3, pad_mode=REFLECT, pas=DGRAD,
       kernels=("nbk_dgrad2_kernel", "pad2d_bwd_kernel"), s=4,
       why="reflection through the staged dgrad and the pad fold (C = 3: scalar pad kernel)"),
    _c("nb7_reflect", 2, 3, 64, 16, 16, 7, 7, pads=P3, pad_mode=REFLECT, pas=WGRAD,
       kernels=("nbk_wgrad_kernel<7>", "colsum_kernel"), deterministic=False, why="staged 7x7 wgrad, row mode"),
    _c("nb_ws", 4, 8, 128, 32, 32, 3, 3, pads=P1, pas=WGRAD,
       kernels=("nbk_wgrad_kernel<9>", "nbk_wgrad_reduce_kernel", "colsum_kernel"), s=32,
       why="staged wgrad with per-block slabs: deterministic"),
]

GEOMETRY_CASES = TC + TC_DGRAD + TC_WGRAD + SIMT + FEWK + STAGED


# ---- the bias gradient summed inside the tensor-core weight gradient (b200gan_conv2d_wgrad_fused_bias) ---------------
def _fused(c, why):
    """c through the fused-bias entry point: a Conv2d on the tensor-core route launches no colsum_kernel; a
    ConvTranspose2d and every other route still sum db with it"""
    tc_conv2d = c.tc and not c.transposed
    return replace(c, name=c.name + "_fb", fused_bias=True, why=why,
                   kernels=tuple(k for k in c.kernels if not (tc_conv2d and k == "colsum_kernel")))


def _wg(name, N, C, K, H, W, kernel, grid, s=0, **kw):
    """a 3x3 tensor-core wgrad case; grid = (pixel splits, jobs, M-tiles x N-tiles) from wg_plan at 132 SMs"""
    return _c(name, N, C, K, H, W, 3, 3, pads=P1, pas=WGRAD, kernels=(kernel,) + _WG_TILE, grid=grid, s=s,
              deterministic=grid[0] == 1, **kw)


_BY_NAME = {(c.name, c.pas): c for c in GEOMETRY_CASES}
FUSED_BIAS = [_fused(c, f"fused db on {c.why}") for c in TC_WGRAD] + [
    _fused(_wg("w_k256", 2, 32, 256, 8, 8, "wgrad_tc_kernel<32, 8>", (1, 9, 2)), "dy is A over two M-tiles: channels 128.. come from M-tile 1"),
    _fused(_wg("w_k384", 2, 32, 384, 8, 8, "wgrad_tc_kernel<32, 8>", (1, 9, 3)), "dy is A over three M-tiles"),
    _fused(_wg("w_c256_k64", 2, 256, 64, 8, 8, "wgrad_tc_kernel<64, 8>", (1, 9, 2)), "C = 256, K = 64: dy is B, x spans two M-tiles"),
    _fused(_wg("w_dcgan_up2_k128", 128, 128, 128, 16, 16, "wgrad_tc_kernel<128, 6>", (8, 16, 1), s=32, up=2),
           "DCGAN conv1 (dcgan.py:54-55): dy is A, four phase jobs x 8 pixel splits add to each channel"),
    _fused(_wg("w_dcgan_up2_k64", 32, 128, 64, 32, 32, "wgrad_tc_kernel<64, 8>", (8, 16, 1), s=32, up=2),
           "DCGAN conv2 (dcgan.py:58-59) at batch 32: dy is B (NB = 64); at batch 128 one image's share of dw lies "
           "below the dw bound of a 512-stage split"),
    _fused(_wg("w_k128_many_splits", 256, 64, 128, 16, 16, "wgrad_tc_kernel<64, 8>", (14, 9, 1), s=14), "dy is A, 14 pixel splits"),
    _fused(_wg("w_k32_b_operand", 64, 128, 32, 20, 20, "wgrad_tc_kernel<32, 8>", (14, 9, 1), s=14),
           "K = 32: dy is B (NB = 32); 20x20 maps clipped by 32x1 boxes"),
    _fused(_wg("w_s2_k128", 64, 64, 128, 32, 32, "wgrad_tc_kernel<64, 8>", (14, 9, 1), s=14, stride=2),
           "stride 2: x through the parity view, dy summed at the output grid"),
] + [_fused(_BY_NAME[(n, WGRAD)], f"fused-bias entry point off the tensor-core route: {w}") for n, w in (
    ("simt_wg_staged", "SIMT forced, the staged kernel"), ("simt_5x5", "5x5, conv_wgrad_kernel"),
    ("fewk3", "few output channels"), ("nb4_s2", "few input channels, staged"))]
GEOMETRY_CASES = GEOMETRY_CASES + FUSED_BIAS

# ---- epilogue matrix: one case per option and one with all of them, for every fprop family ---------------------------
# (family, base case, main kernels, tile images BNn (per-sample statistics fuse only at 1), fuses statistics at all)
_FAMILIES = [
    (_c("ep_tc", 2, 32, 64, 16, 16, 3, 3, pads=P1), ("conv_tc_kernel<64, 8>",), True, True),
    (_c("ep_tc_bnn", 8, 32, 64, 4, 4, 3, 3, pads=P1), ("conv_tc_kernel<64, 8>",), False, True),
    (_c("ep_narrow", 2, 32, 5, 8, 8, 3, 3, pads=P1), ("conv_tc_kernel<32, 8>",), False, False),
    (_c("ep_allphase", 2, 32, 64, 3, 3, 3, 3, pads=P1, up=2), ("conv_tc_up2_allphase_kernel",), False, True),
    (_c("ep_phases", 2, 32, 128, 4, 4, 3, 3, pads=P1, up=2), ("conv_tc_kernel<128, 6>",), False, True),
    (_c("ep_scatter", 2, 32, 64, 4, 4, 4, 4, stride=2, pads=P1, transposed=True), ("conv_tc_kernel<64, 8>",), False,
     True),
    (_c("ep_simt", 2, 32, 64, 8, 8, 3, 3, pads=P1, algo="SIMT"), ("conv_gather_gemm_kernel",), False, False),
    (_c("ep_staged", 2, 3, 64, 16, 16, 4, 4, stride=2, pads=P1), ("nbk_fprop2_kernel",), False, False),
    (_c("ep_fewk", 2, 32, 3, 8, 8, 3, 3, pads=P1, algo="SIMT"), ("fewk_fprop_kernel<3, 3>",), False, False),
]
_SINGLE = [("none",), ("bias",), ("lrelu",), ("relu",), ("tanh",), ("sigmoid",), ("chan_scale",), ("round_tf32",),
           ("stats_c",), ("stats_s",)]
_ALL = ("bias", "lrelu", "chan_scale", "round_tf32", "stats_s")


def _epilogue_cases():
    out = []
    for base, kern, per_sample_fused, fuses in _FAMILIES:
        narrow = base.name == "ep_narrow"
        fewk = base.name == "ep_fewk"
        for opts in _SINGLE + [_ALL]:
            epi = tuple(o for o in opts if o != "none")
            name = base.name + "-" + ("all" if opts == _ALL else opts[0])
            ks = kern
            if fewk and ("chan_scale" in epi or "round_tf32" in epi):
                ks = ("conv_gather_gemm_kernel",)  # fewk takes neither option: the SIMT gather GEMM does
            stats = [o for o in epi if o.startswith("stats")]
            deferred = stats and not (fuses and (stats[0] == "stats_c" or per_sample_fused))
            if deferred:
                ks = ks + ("norm_stats_kernel",)
            error = narrow and "chan_scale" in epi
            if error:
                ks = ()
            out.append(replace(base, name=name, epi=epi, kernels=ks, error=error,
                               why="narrow-K must refuse a Dropout2d scale" if error else
                               f"epilogue {'+'.join(epi) or 'none'} on the {base.name[3:]} family"))
    return out


EPILOGUE_CASES = _epilogue_cases()
CASES = GEOMETRY_CASES + EPILOGUE_CASES

# sources whose __global__ convolution kernels the table must cover; narrow_block.cu only for the kernels the
# convolution entry points reach (the staged forward, data and weight gradient and the slab reduce)
COVERED_SOURCES = ("conv_tc.cu", "wgrad_tc.cu", "conv_simt.cu", "fewk.cu")
NARROW_BLOCK_KERNELS = ("nbk_fprop2_kernel", "nbk_dgrad2_kernel", "nbk_wgrad_kernel", "nbk_wgrad_reduce_kernel")


def base_name(kernel):
    return kernel.split("<", 1)[0]


# ---- the weight-gradient plan (a mirror of wg_plan in csrc/wgrad_tc.cu) -----------------------------------------------
@dataclass(frozen=True)
class WgPlan:
    s_is_a: int      # 1: x is the A operand and dy (the dense operand D) is B
    NB: int          # output channels of a CTA's B side
    njobs: int       # filter taps, or 16 (phase, tap) jobs of the x2 upsample fold
    mtiles: int
    ntiles: int
    Ho: int          # pixel grid of D the contraction runs over
    Wo: int
    bwl: int         # the 32-pixel box is 2^bwl x 2^bhl pixels of ipb images
    bhl: int
    ipb: int
    tiles_w: int
    tiles_h: int
    tiles_total: int
    tps: int         # tiles per pixel split
    nsplits: int

    @property
    def grid(self):
        return (self.nsplits, self.njobs, self.mtiles * self.ntiles)


def _ilog2c(v):
    return max(0, (v - 1).bit_length())


def wg_plan(c, num_sms=NUM_SMS):
    """the tensor-core weight gradient's plan of a geometry it accepts, as wg_plan computes it"""
    up2 = c.up == 2
    sch, dch = (c.K, c.C) if c.transposed else (c.C, c.K)
    s_is_a = 0 if dch % 128 == 0 else 1
    mch, nch = (sch, dch) if s_is_a else (dch, sch)
    NB = 256 if nch % 256 == 0 else 128 if nch % 128 == 0 else 64 if nch % 64 == 0 else 32
    njobs = 16 if up2 else c.R * c.S
    Ho = c.H if up2 or c.transposed else c.P
    Wo = c.W if up2 or c.transposed else c.Q
    bwl = min(_ilog2c(Wo), 5)
    bhl = min(_ilog2c(Ho), 5 - bwl)
    tiles_w, tiles_h, ipb = -(-Wo // (1 << bwl)), -(-Ho // (1 << bhl)), 32 >> (bwl + bhl)
    total = -(-c.N // ipb) * tiles_w * tiles_h
    per_split = njobs * (mch // 128) * (nch // NB)
    max_ns = min(max(total // 8, 1), 4 * num_sms)
    ns, best = 1, -1
    for s in range(1, max_ns + 1):
        cost = -(-s * per_split // num_sms) * (-(-total // s) + 8)
        if best < 0 or cost < best:
            best, ns = cost, s
    tps = -(-total // ns)
    return WgPlan(s_is_a, NB, njobs, mch // 128, nch // NB, Ho, Wo, bwl, bhl, ipb, tiles_w, tiles_h, total, tps,
                  -(-total // tps))


# ---- fp64 references and their bounds ---------------------------------------------------------------------------------
U = 2.0 ** -23
EPS_UP2_FOLD = 2.0 ** -11 + 3 * 2.0 ** -24


def geom(c):
    from b200gan import _lib
    t, l, b, r = c.pads
    return _lib.ConvGeom(c.N, c.H, c.W, c.C, c.K, c.R, c.S, c.stride, t, l, b, r, c.pad_mode, c.up, int(c.transposed),
                         c.P, c.Q)


def wshape(c):
    return (c.C, c.K, c.R, c.S) if c.transposed else (c.K, c.C, c.R, c.S)


def conv_ref(c, x_nchw, w):
    t, l, b, r = c.pads
    if c.transposed:
        return F.conv_transpose2d(x_nchw, w, stride=c.stride, padding=(t, l))
    if c.up == 2:
        x_nchw = x_nchw.repeat_interleave(2, 2).repeat_interleave(2, 3)
    x_nchw = F.pad(x_nchw, (l, r, t, b), mode="reflect" if c.pad_mode == REFLECT else "constant")
    return F.conv2d(x_nchw, w, stride=c.stride)


def nchw(t_nhwc):
    return t_nhwc.permute(0, 3, 1, 2)


def operands(c, x, dy, w):
    """x, dy, w in fp64 as the kernel's arithmetic sees them (wgmma truncates raw activations to TF32, the packed
    weights are RNA-rounded); and eps_op, the operand rounding the reference does not reproduce"""
    from conformance import tf32_rna, tf32_trunc
    eps_op = 0.0
    if c.tc:
        x, dy = tf32_trunc(x), tf32_trunc(dy)
        if c.pas != WGRAD:
            if c.up == 2:
                eps_op = EPS_UP2_FOLD  # the fold's fp32 sums and their RNA are not reproduced
            else:
                w = tf32_rna(w)
    return x.double(), dy.double(), w.double(), eps_op


def conv_pass_ref(c, x, dy, w):
    """the pass's linear result in fp64 (NHWC for activations, parameter layout for dw)"""
    if c.pas == FPROP:
        return conv_ref(c, nchw(x), w).permute(0, 2, 3, 1)
    if c.pas == DGRAD:
        xv = torch.zeros(c.N, c.C, c.H, c.W, dtype=torch.float64, device="cuda", requires_grad=True)
        y = conv_ref(c, xv, w)
        (g,) = torch.autograd.grad(y, xv, nchw(dy))
        return g.permute(0, 2, 3, 1)
    wv = torch.zeros_like(w, requires_grad=True)
    y = conv_ref(c, nchw(x), wv)
    (g,) = torch.autograd.grad(y, wv, nchw(dy))
    return g


def contraction(c):
    if c.pas == FPROP:
        return c.R * c.S * c.C
    if c.pas == DGRAD:
        return c.R * c.S * c.K * c.up * c.up
    return c.N * (c.H * c.W if c.transposed else c.P * c.Q)


def conv_bound(c, A, eps_op, num_sms=NUM_SMS):
    """wgmma: eps_op A + 2^-22 (ceil(n / 8) + s + 4) A;  fp32: 2^-23 (n + s + 4) A.  A tensor-core weight gradient
    accumulates in one chain only the pixels of its split (at most 32 per tile), and the s splits are added after"""
    n = contraction(c)
    if c.tc and c.pas == WGRAD:
        n = min(n, 32 * wg_plan(c, num_sms).tps)
    if c.tc:
        return eps_op * A + 2.0 ** -22 * (math.ceil(n / 8) + c.s + 4) * A
    return U * (n + c.s + 4) * A


def one_tap(c, w):
    m = torch.zeros_like(w)
    m[:, :, c.R // 2, c.S // 2] = 1
    return w * m


def fused_db_bound(c, dy, num_sms):
    """The bound on db of b200gan_conv2d_wgrad_fused_bias on the tensor-core route, per channel, from the sums the
    kernel actually forms.  Every fp32 addition rounds once, by at most 2^-24 of its result, and the result is
    replaced here by its exact value (the difference is second order and covered by the last factor):
      dy = A (K % 128 == 0): a thread sums, stage after stage of its split's 32-pixel boxes, the pairs of pixel rows
                             8k + 2j, 8k + 2j + 1 (k < 4) that its fragment holds; two shuffles add the four threads j;
      dy = B:                a thread adds pixel row j of every stage; five shuffles add the 32 threads;
      then one fp32 atomic per CTA and channel onto zero, in any order: each result is at most the sum of the
    CTAs' |partial|.  CTAs of a channel: pixel splits x the jobs that read dy (one; four phases of the upsample fold)."""
    u = 2.0 ** -24
    pl = wg_plan(c, num_sms)
    ns, tps, BW, BH, ipb = pl.nsplits, pl.tps, 1 << pl.bwl, 1 << pl.bhl, pl.ipb
    views = [dy[:, a::2, b::2] for a in (0, 1) for b in (0, 1)] if c.up == 2 else [dy]
    chain = torch.zeros(c.K, dtype=torch.float64, device=dy.device)
    parts = []
    for d in views:
        N, Ho, Wo, K = d.shape
        nimg = -(-N // ipb) * ipb
        t = torch.zeros(nimg, pl.tiles_h * BH, pl.tiles_w * BW, K, dtype=torch.float64, device=dy.device)
        t[:N, :Ho, :Wo] = d.double()
        t = t.view(nimg // ipb, ipb, pl.tiles_h, BH, pl.tiles_w, BW, K).permute(0, 2, 4, 1, 3, 5, 6)
        t = t.reshape(pl.tiles_total, 32, K)  # box row = w + BW (h + BH image), TMA zero fill past the map and N
        t = torch.cat([t, t.new_zeros(ns * tps - pl.tiles_total, 32, K)]).view(ns, tps, 32, K)
        if not pl.s_is_a:
            r = t.view(ns, tps, 4, 8, K)
            pairs = r[:, :, :, 0::2] + r[:, :, :, 1::2]          # [split, stage, k, j, K]
            acc = pairs.reshape(ns, tps * 4, 4, K).cumsum(1)
            chain += pairs.abs().sum((0, 1, 2, 3)) + acc.abs().sum((0, 1, 2))
            a = acc[:, -1]
            s01, s23 = a[:, 0] + a[:, 1], a[:, 2] + a[:, 3]
            p = s01 + s23
            chain += (s01.abs() + s23.abs() + p.abs()).sum(0)
        else:
            acc = t.cumsum(1)                                     # [split, stage, lane, K]
            chain += acc.abs().sum((0, 1, 2))
            v = acc[:, -1]
            for lvl, o in enumerate((16, 8, 4, 2, 1), 1):
                v = v + v[:, torch.arange(32, device=dy.device) ^ o]
                chain += v.abs().sum((0, 1)) / 2 ** lvl           # 2^lvl lanes hold each sum
            p = v[:, 0]
        parts.append(p)
    P = torch.cat(parts)
    depth = 4 * tps + 5 + P.shape[0]
    return u * (chain + (P.shape[0] - 1) * P.abs().sum(0)) * (1 + 2 * depth * u)
