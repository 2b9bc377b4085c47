"""The phase-major mode of the tensor-core weight gradient, element by element against fp64.

A Conv2d after Upsample(x2) whose input x has a multiple of 128 channels (and dy does not) on maps at least 8 pixels
wide runs wgrad_tc_kernel phase-major: the CTA at blockIdx.y = 4 phase + q computes all four taps of its output phase
over quarter q of its pixel split, from one transpose of dy and one halo box of x per stage.  The grid and the kernel
instance are those of the per-job form.  Each case states the instance and grid it runs on a 132-SM H100, whether the
plan is phase-major (b200gan_conv2d_wgrad_phase_major), and goes through conformance.run_case: guards, the route, a
CUDA-graph replay, and dw against the fp64 reference under conv_bound.  With the fused-bias entry point db is held to
conv_cases.fused_db_bound.

s, the partial sums added outside one accumulation chain: the 4 (phase, tap) jobs the reduce folds into a weight, times
the pixel splits, times 4 quarters in phase-major mode.
"""
import ctypes
from dataclasses import replace

import pytest
import torch

import conv_cases as cc
from b200gan import _lib, ops
from conformance import Arena, check_elementwise, first_grid, not_vacuous, run_case
from conv_cases import P1, WGRAD, conv_bound, conv_pass_ref, fused_db_bound, geom, operands, wg_plan, wshape

pytestmark = pytest.mark.gpu

_TILE = ("wgrad_reduce_tile_kernel",)


def _case(name, N, C, K, H, W, kernel, grid, phase_major, fused=False, why=""):
    c = cc.Case(name, N, C, K, H, W, 3, 3, pads=P1, up=2, pas=WGRAD, fused_bias=fused, why=why,
                kernels=(kernel,) + _TILE + (() if fused else ("colsum_kernel",)), grid=grid)
    pl = wg_plan(c)
    s = 4 * pl.nsplits * (4 if phase_major else 1)
    return replace(c, s=s, deterministic=False), phase_major


CASES = [
    _case("dcgan_conv2_b128", 128, 128, 64, 32, 32, "wgrad_tc_kernel<64, 8>", (8, 16, 1), True,
          why="DCGAN conv2 (dcgan.py:58-59) at the benchmark's batch: 32x1 boxes, 8 splits"),
    _case("dcgan_conv2_b128_fb", 128, 128, 64, 32, 32, "wgrad_tc_kernel<64, 8>", (8, 16, 1), True, fused=True,
          why="the same through b200gan_conv2d_wgrad_fused_bias: db from every phase-major CTA of M-tile 0"),
    _case("nb32", 4, 128, 32, 16, 16, "wgrad_tc_kernel<32, 8>", (4, 16, 1), True, fused=True,
          why="K = 32: NB = 32, the four-stage ring fills the per-job ring exactly; 16x2 boxes"),
    _case("cyclegan_128_64", 1, 128, 64, 64, 64, "wgrad_tc_kernel<64, 8>", (8, 16, 1), True, fused=True,
          why="CycleGAN's Upsample -> Conv2d(128, 64) (cyclegan/models.py) at batch 1"),
    _case("ragged_quarters", 5, 128, 64, 8, 8, "wgrad_tc_kernel<64, 8>", (1, 16, 1), True, fused=True,
          why="8x4 boxes: 10 tiles in one split, quarters of 3, 3, 3, 1"),
    _case("empty_quarter", 1, 128, 64, 8, 8, "wgrad_tc_kernel<64, 8>", (1, 16, 1), True, fused=True,
          why="2 tiles in one split: quarters of 1, 1, 0, 0; the empty ones add nothing"),
    _case("ipb4", 3, 128, 64, 1, 8, "wgrad_tc_kernel<64, 8>", (1, 16, 1), True, fused=True,
          why="1x8 maps: 8x1 boxes of 4 images, 72-row halo chunks, the last box past N"),
    _case("bw4_per_job", 2, 128, 64, 4, 4, "wgrad_tc_kernel<64, 8>", (1, 16, 1), False, fused=True,
          why="4x4 maps: 4-pixel boxes split a k slice over box rows, so the per-job form runs"),
    _case("c256_mt1", 2, 256, 64, 16, 16, "wgrad_tc_kernel<64, 8>", (2, 16, 2), True, fused=True,
          why="C = 256: x spans two M-tiles; db from M-tile 0 only"),
]


class Run:
    """One weight-gradient call on the guarded buffers of conformance.Arena."""

    def __init__(self, c, seed=0):
        self.c = c
        lib = self.lib = _lib.load()
        self.g = geom(c)
        gen = torch.Generator(device="cpu").manual_seed(seed)
        x = torch.randn(c.N, c.H, c.W, c.C, generator=gen)
        dy = torch.randn(c.N, c.P, c.Q, c.K, generator=gen)
        self.inp = {"x": x.cuda(), "dy": dy.cuda(), "w": torch.zeros(wshape(c), device="cuda")}
        nws = lib.b200gan_conv2d_wgrad_workspace_floats(ctypes.byref(self.g), _lib.ALGO_AUTO)
        self.arena = Arena([("x", x.numel(), torch.float32, "in"), ("dy", dy.numel(), torch.float32, "in"),
                            ("dw", c.K * c.C * 9, torch.float32, "out"), ("db", c.K, torch.float32, "out"),
                            ("ws", nws, torch.float32, "ws")])

    def prepare(self):
        self.arena.prepare(self.inp)

    def call(self, stream_handle):
        a = self.arena
        wgrad = self.lib.b200gan_conv2d_wgrad_fused_bias if self.c.fused_bias else self.lib.b200gan_conv2d_wgrad
        return wgrad(ctypes.byref(self.g), a.ptr("x"), a.ptr("dy"), a.ptr("dw"), a.ptr("db"), a.ptr("ws"),
                     _lib.ALGO_AUTO, stream_handle)

    def outputs(self):
        return self.arena.outputs()

    def check(self, what):
        c, outs = self.c, self.outputs()
        sms = torch.cuda.get_device_properties(0).multi_processor_count
        x, dy, w, eps_op = operands(c, self.inp["x"], self.inp["dy"], self.inp["w"])
        ref = conv_pass_ref(c, x, dy, w)
        bound = conv_bound(c, conv_pass_ref(c, x.abs(), dy.abs(), w), eps_op, sms)
        worst = check_elementwise(what, outs["dw"], ref, bound, "(param index)")
        if c.N > 1 and c.N <= 32:  # at batch 128 one image's share of dw is below the bound of a 512-stage split
            not_vacuous(what, bound, conv_pass_ref(replace(c, N=1), x[:1], dy[:1], w).abs())
        dyf = self.inp["dy"]
        db_ref = dyf.double().sum((0, 1, 2))
        if c.fused_bias:
            db_bound = fused_db_bound(c, dyf, sms)
        else:
            db_bound = cc.U * (c.N * c.P * c.Q + 1100) * dyf.double().abs().sum((0, 1, 2))
        return max(worst, check_elementwise(what + " db", outs["db"], db_ref, db_bound, "(k,)"))


@pytest.mark.parametrize("case", CASES, ids=lambda cp: cp[0].name)
def test_wgrad_phase_case(case):
    c, phase_major = case
    g = geom(c)
    assert ops.conv_wgrad_phase_major(g) == phase_major, f"{c.name}: phase-major plan is not {phase_major}"
    assert wg_plan(c).s_is_a == 1 and wg_plan(c).grid == c.grid, f"{c.name}: {wg_plan(c)} is not the stated plan"
    run_case(Run(c), c.name, first_grid(c.kernels, c.grid), varies=("dw", "db", "ws"), ordered=False,
             num_sms=cc.NUM_SMS)


def test_wgrad_phase_major_query():
    """the plan query answers for the tensor-core route only, and no phase-major plan without the x2 upsample"""
    def g_of(**kw):
        base = dict(N=2, C=128, K=64, H=16, W=16)
        base.update(kw)
        c = cc.Case("q", base["N"], base["C"], base["K"], base["H"], base["W"], 3, 3, pads=P1,
                    up=kw.get("up", 2), pas=WGRAD)
        return geom(c)
    assert ops.conv_wgrad_phase_major(g_of())
    assert not ops.conv_wgrad_phase_major(g_of(up=1)), "no upsample: the per-tap jobs"
    assert not ops.conv_wgrad_phase_major(g_of(C=64, K=128)), "dy is A (DCGAN conv1 form): the per-job path"
    assert not ops.conv_wgrad_phase_major(g_of(C=48)), "not on the tensor-core route at all"
