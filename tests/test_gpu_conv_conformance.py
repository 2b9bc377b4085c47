"""Every convolution route of tests/conv_cases.py, element by element against an fp64 reference.

Each case calls the C ABI directly on the guarded buffers of tests/conformance.py (Arena) and runs its protocol; the
statistics start at known non-zero values, since the header promises accumulation, not overwrite.  The route is a set:
every traced kernel is one the table names, and every kernel it names is traced.
The reference is torch float64 on the GPU, fed the operands the kernel feeds its arithmetic (packed wgmma weights
rounded to TF32 with RNA, raw activations truncated to TF32 by wgmma; SIMT kernels use fp32 as is).  A, the same
operation on absolute values, scales an error bound that follows from the arithmetic, not from a fit:
  wgmma   |y - ref| <= eps_op * A + 2^-22 * (ceil(n / 8) + s + 4) * A
  fp32    |y - ref| <= 2^-23 * (n + s + 4) * A
with n the contraction length (a tensor-core weight gradient: the pixels of one split) and s the partial sums added
outside one accumulation chain; eps_op is the operand rounding the reference does not reproduce (the x2 upsample fold's
fp32 tap sums before RNA).  The bound is carried through the epilogue with its Lipschitz constants.  The bias gradient that b200gan_conv2d_wgrad_fused_bias sums inside
the tensor-core weight gradient is held to the bound of its actual summation chain (conv_cases.fused_db_bound).
"""
import ctypes
import math

import numpy as np
import pytest
import torch

import conv_cases as cc
from b200gan import _lib
from conformance import STATS_FILL, Arena, check_elementwise, first_grid, not_vacuous, np_rna, run_case, tf32_rna, \
    tf32_trunc
from conv_cases import U, conv_bound, conv_pass_ref, fused_db_bound, geom, one_tap, operands, wshape

pytestmark = pytest.mark.gpu

SLOPE = 0.2


# ---- the case as tensors -----------------------------------------------------------------------------------------
def resolve_algo(c, lib, g):
    if c.pas == cc.WGRAD and c.algo == "AUTO":
        return _lib.ALGO_AUTO
    if c.algo == "SIMT":
        return _lib.ALGO_SIMT
    return _lib.ALGO_TC if lib.b200gan_conv2d_supported(ctypes.byref(g), c.pas, _lib.ALGO_TC) else _lib.ALGO_SIMT


def pack_kind(c, algo):
    if algo == _lib.ALGO_TC:
        if c.pas == cc.FPROP:
            return _lib.PACK_TC_FPROP_UP2 if c.up == 2 else _lib.PACK_TC_FPROP
        return _lib.PACK_TC_DGRAD_UP2 if c.up == 2 else _lib.PACK_TC_DGRAD
    return _lib.PACK_SIMT_FPROP if c.pas == cc.FPROP else _lib.PACK_SIMT_DGRAD


def make_inputs(c, seed):
    g = torch.Generator(device="cpu").manual_seed(seed)
    x = torch.randn(c.N, c.H, c.W, c.C, generator=g)
    dy = torch.randn(c.N, c.P, c.Q, c.K, generator=g)
    fan = c.C * c.R * c.S
    w = torch.randn(*wshape(c), generator=g) / math.sqrt(fan)
    bias = torch.randn(c.K, generator=g) * 0.5
    cs = torch.where(torch.rand(c.N, c.K, generator=g) < 0.25, torch.zeros(()), 0.5 + 1.5 * torch.rand(c.N, c.K,
                                                                                                     generator=g))
    cs = cs * torch.where(torch.rand(c.N, c.K, generator=g) < 0.5, -1.0, 1.0)
    return {k: v.float().cuda() for k, v in dict(x=x, dy=dy, w=w, bias=bias, cs=cs).items()}


def act_of(epi):
    for a, code in (("lrelu", _lib.ACT_LRELU), ("relu", _lib.ACT_RELU), ("tanh", _lib.ACT_TANH),
                    ("sigmoid", _lib.ACT_SIGMOID)):
        if a in epi:
            return a, code
    return None, _lib.ACT_NONE


class Run:
    """One case: arena, packed weights, the call as a closure over a stream."""

    def __init__(self, c, seed=0):
        self.c = c
        lib = self.lib = _lib.load()
        self.g = geom(c)
        self.algo = resolve_algo(c, lib, self.g)
        self.inp = make_inputs(c, seed)
        N, C, K, P, Q, H, W = c.N, c.C, c.K, c.P, c.Q, c.H, c.W
        specs = []
        if c.pas in (cc.FPROP, cc.DGRAD):
            self.kind = pack_kind(c, self.algo)
            nw = lib.b200gan_packed_weight_floats(ctypes.byref(self.g), self.kind)
            self.packed = torch.empty(nw, device="cuda")
            _lib.check(lib.b200gan_pack_weights(ctypes.byref(self.g), self.kind, self.inp["w"].data_ptr(),
                                                self.packed.data_ptr(), None), "pack")
        if c.pas == cc.FPROP:
            specs += [("x", N * H * W * C, torch.float32, "in"), ("w", self.packed.numel(), torch.float32, "in"),
                      ("y", N * P * Q * K, torch.float32, "out")]
            if "bias" in c.epi:
                specs.append(("bias", K, torch.float32, "in"))
            if "chan_scale" in c.epi:
                specs.append(("cs", N * K, torch.float32, "in"))
            self.per_sample = "stats_s" in c.epi
            if self.per_sample or "stats_c" in c.epi:
                specs.append(("stats", 2 * (N * K if self.per_sample else K), torch.float64, "stats"))
        elif c.pas == cc.DGRAD:
            nws = lib.b200gan_conv2d_dgrad_workspace_floats(ctypes.byref(self.g), self.algo)
            specs += [("dy", N * P * Q * K, torch.float32, "in"), ("w", self.packed.numel(), torch.float32, "in"),
                      ("dx", N * H * W * C, torch.float32, "out")]
            if nws:
                specs.append(("ws", nws, torch.float32, "ws"))
        else:
            nws = lib.b200gan_conv2d_wgrad_workspace_floats(ctypes.byref(self.g), self.algo)
            specs += [("x", N * H * W * C, torch.float32, "in"), ("dy", N * P * Q * K, torch.float32, "in"),
                      ("dw", K * C * c.R * c.S, torch.float32, "out"), ("db", K, torch.float32, "out")]
            if nws:
                specs.append(("ws", nws, torch.float32, "ws"))
        self.arena = Arena(specs)
        self.data = dict(x=self.inp["x"], dy=self.inp["dy"], bias=self.inp["bias"], cs=self.inp["cs"])
        if c.pas != cc.WGRAD:
            self.data["w"] = self.packed

    def prepare(self):
        self.arena.prepare(self.data)

    def call(self, stream_handle):
        c, lib, a = self.c, self.lib, self.arena
        if c.pas == cc.FPROP:
            name, code = act_of(c.epi)
            ep = _lib.Epilogue(a.ptr("bias"), code, SLOPE, a.ptr("cs"), a.ptr("stats"), int("stats_s" in c.epi),
                               int("round_tf32" in c.epi))
            return lib.b200gan_conv2d_fprop(ctypes.byref(self.g), ctypes.byref(ep), a.ptr("x"), a.ptr("w"), a.ptr("y"),
                                            self.algo, stream_handle)
        if c.pas == cc.DGRAD:
            return lib.b200gan_conv2d_dgrad(ctypes.byref(self.g), a.ptr("dy"), a.ptr("w"), a.ptr("dx"), a.ptr("ws"),
                                            self.algo, stream_handle)
        wgrad = lib.b200gan_conv2d_wgrad_fused_bias if c.fused_bias else lib.b200gan_conv2d_wgrad
        return wgrad(ctypes.byref(self.g), a.ptr("x"), a.ptr("dy"), a.ptr("dw"), a.ptr("db"), a.ptr("ws"), self.algo,
                     stream_handle)

    def outputs(self):
        return self.arena.outputs()

    def check(self, what):
        return check_outputs(self, self.outputs(), what)


# ---- fp64 reference: conv_cases holds the linear part and its bound; the epilogue is here ------------------------
def apply_act(name, v):
    if name == "lrelu":
        return torch.where(v > 0, v, v * SLOPE)
    if name == "relu":
        return v.clamp_min(0)
    if name == "tanh":
        return torch.tanh(v)
    if name == "sigmoid":
        return torch.sigmoid(v)
    return v


LIPSCHITZ = {None: 1.0, "lrelu": max(1.0, SLOPE), "relu": 1.0, "tanh": 1.0, "sigmoid": 0.25}


def epilogue_ref(run, conv, bound):
    """y_ref and its bound after bias, activation, chan_scale and TF32 rounding"""
    c, inp = run.c, run.inp
    pre = conv
    b = torch.zeros_like(conv)
    if "bias" in c.epi:
        b = inp["bias"].double().expand_as(conv)
        pre = conv + b
    bound = bound + U * (pre.abs() + b.abs())  # the fp32 bias add
    name, _ = act_of(c.epi)
    y = apply_act(name, pre)
    bound = LIPSCHITZ[name] * bound + U * y.abs()
    if name == "tanh":
        bound = bound + 4 * U * y.abs() + 2.0 ** -126
    if name == "sigmoid":  # __expf: 2 + 1.16 |v| ulps of exp(-v), times y (1 - y) <= 1/4, and the reciprocal
        bound = bound + U * (2 + 2 * pre.abs()) / 4 + 2 * U * y.abs()
    if "chan_scale" in c.epi:
        s = inp["cs"].double().view(c.N, 1, 1, c.K)
        y = y * s
        bound = bound * s.abs() + U * y.abs()
    if "round_tf32" in c.epi:
        bound = bound + 2.0 ** -11 * (y.abs() + bound)
    return y, bound


# ---- the per-case test ---------------------------------------------------------------------------------------------
def check_outputs(run, outs, what):
    """every output of the call against the fp64 reference; returns the worst |err|/bound"""
    c = run.c
    x, dy, w, eps_op = operands(c, run.inp["x"], run.inp["dy"], run.inp["w"])
    ref = conv_pass_ref(c, x, dy, w)
    A = conv_pass_ref(c, x.abs(), dy.abs(), w.abs())
    bound = conv_bound(c, A, eps_op, torch.cuda.get_device_properties(0).multi_processor_count)
    worst = 0.0
    if c.pas == cc.FPROP:
        y_ref, b = epilogue_ref(run, ref, bound)
        y = outs["y"]
        worst = check_elementwise(what, y, y_ref, b, "(n, p, q, k)")
        if "round_tf32" in c.epi:
            assert ((y.view(torch.int32) & 0x1FFF) == 0).all(), f"{what}: round_tf32 output not TF32-representable"
        if "stats" in outs:
            check_stats(run, y, outs["stats"], what)
        not_vacuous(what, bound, conv_pass_ref(c, x, dy, one_tap(c, w)).abs())
    elif c.pas == cc.DGRAD:
        worst = check_elementwise(what, outs["dx"], ref, bound, "(n, h, w, c)")
        not_vacuous(what, bound, conv_pass_ref(c, x, dy, one_tap(c, w)).abs())
    else:
        worst = check_elementwise(what, outs["dw"], ref, bound, "(param index)")
        db_ref = run.inp["dy"].double().sum((0, 1, 2))
        db_A = run.inp["dy"].double().abs().sum((0, 1, 2))
        if c.fused_bias and c.tc and not c.transposed:
            db_bound = fused_db_bound(c, run.inp["dy"], torch.cuda.get_device_properties(0).multi_processor_count)
            not_vacuous(what + " db", db_bound, run.inp["dy"].double().abs().reshape(-1))
        else:
            db_bound = U * (c.N * c.P * c.Q + 1100) * db_A
        worst = max(worst, check_elementwise(what + " db", outs["db"], db_ref, db_bound, "(k,)"))
        if c.N > 1:
            not_vacuous(what, bound, conv_pass_ref(replace_n(c), x[:1], dy[:1], w).abs())
    return worst


def replace_n(c):
    from dataclasses import replace
    return replace(c, N=1)


def check_stats(run, y, stats, what):
    c = run.c
    G = stats.numel() // 2
    y64 = y.double().view(c.N, c.P * c.Q, c.K)
    if "stats_s" in c.epi:
        s1, s2 = y64.sum(1).reshape(-1), (y64 * y64).sum(1).reshape(-1)
        a1, m = y64.abs().sum(1).reshape(-1), c.P * c.Q
    else:
        s1, s2 = y64.sum((0, 1)), (y64 * y64).sum((0, 1))
        a1, m = y64.abs().sum((0, 1)), c.N * c.P * c.Q
    # m: values a kernel sums in fp32 before its fp64 atomic (at most all of the group's)
    got1, got2 = stats[:G] - STATS_FILL[0], stats[G:] - STATS_FILL[1]
    b1, b2 = U * (m + 8) * a1, U * (m + 8) * s2
    for nm, got, want, b in (("sum", got1, s1, b1), ("sum of squares", got2, s2, b2)):
        err = (got - want).abs()
        bad = (err > b + 1e-300).nonzero()
        assert bad.numel() == 0, f"{what}: stats {nm} group {bad[0].item()}: {got[bad[0]].item():.9g} vs fp64 sum of " \
                                 f"the kernel's output {want[bad[0]].item():.9g} (bound {b[bad[0]].item():.3e}; " \
                                 "statistics must accumulate onto the caller's values)"


@pytest.mark.parametrize("case", cc.CASES, ids=lambda c: c.id)
def test_conv_case(case):
    run = Run(case)
    # fp64 statistics and db are summed atomically; a route not marked deterministic repeats nothing bit for bit
    varies = ("stats", "db", "ws") if case.deterministic else tuple(run.arena.t)
    run_case(run, case.id, first_grid(case.kernels, case.grid), refuse=(-2,) if case.error else (), varies=varies,
             ordered=False, num_sms=cc.NUM_SMS)


# ---- rounding probe --------------------------------------------------------------------------------------------------
LOW_BITS = (0x0000, 0x0001, 0x0FFF, 0x1000, 0x1001, 0x1FFF, 0x0800, 0x1800)


def probe_values(n, gen):
    """fp32 values with chosen low 13 mantissa bits, both signs, moderate exponents"""
    base = (torch.randint(0x3E800000, 0x40800000, (n,), generator=gen, dtype=torch.int64) & ~0x1FFF)
    low = torch.tensor(LOW_BITS, dtype=torch.int64)[torch.arange(n) % len(LOW_BITS)]
    sign = (torch.arange(n) // len(LOW_BITS) % 2) << 31
    return ((base | low | sign) & 0xFFFFFFFF).to(torch.int64).to(torch.int32).view(torch.float32)


def _probe_geom(N, C, K, H, W):
    c = cc.Case("probe", N, C, K, H, W, 1, 1, why="rounding probe")
    return c, geom(c)


def _one_hot_weights(K, C):
    w = torch.zeros(K, C, 1, 1)
    for k in range(K):
        w[k, k % C, 0, 0] = 1.0
    return w


def test_rounding_probe_fprop():
    """1x1 wgmma fprop: y = the operand's value after what the tensor cores do to it, bit for bit"""
    lib = _lib.load()
    gen = torch.Generator().manual_seed(5)
    c, g = _probe_geom(2, 32, 32, 4, 4)
    # (a) raw activations through one-hot weights: y[k] = trunc(x[k])
    x = probe_values(c.N * c.H * c.W * c.C, gen).view(c.N, c.H, c.W, c.C).cuda()
    w = _one_hot_weights(c.K, c.C).cuda()
    packed = torch.empty(lib.b200gan_packed_weight_floats(ctypes.byref(g), _lib.PACK_TC_FPROP), device="cuda")
    _lib.check(lib.b200gan_pack_weights(ctypes.byref(g), _lib.PACK_TC_FPROP, w.data_ptr(), packed.data_ptr(), None))
    y = torch.full((c.N, c.H, c.W, c.K), float("nan"), device="cuda")
    ep = _lib.Epilogue(None, 0, 0.0, None, None, 0, 0)
    _lib.check(lib.b200gan_conv2d_fprop(ctypes.byref(g), ctypes.byref(ep), x.data_ptr(), packed.data_ptr(), y.data_ptr(),
                                        _lib.ALGO_TC, None))
    torch.cuda.synchronize()
    want = tf32_trunc(x)
    assert torch.equal(y.view(torch.int32), want.view(torch.int32)), \
        f"activations: wgmma does not truncate to TF32: x {x.flatten()[:8].tolist()} y {y.flatten()[:8].tolist()}"
    # (b) raw weights through one-hot activations: y = RNA(w) from the packing
    wr = probe_values(c.K * c.C, gen).view(c.K, c.C, 1, 1).cuda()
    xo = torch.zeros(c.N, c.H, c.W, c.C, device="cuda")
    pix = torch.arange(c.N * c.H * c.W) % c.C
    xo.view(-1, c.C)[torch.arange(c.N * c.H * c.W), pix] = 1.0
    _lib.check(lib.b200gan_pack_weights(ctypes.byref(g), _lib.PACK_TC_FPROP, wr.data_ptr(), packed.data_ptr(), None))
    _lib.check(lib.b200gan_conv2d_fprop(ctypes.byref(g), ctypes.byref(ep), xo.data_ptr(), packed.data_ptr(),
                                        y.data_ptr(), _lib.ALGO_TC, None))
    torch.cuda.synchronize()
    want = tf32_rna(wr.view(c.K, c.C))[:, pix.cuda()].t().reshape(c.N, c.H, c.W, c.K)
    assert torch.equal(y.view(torch.int32), want.view(torch.int32)), "packed weights are not RNA-rounded TF32"


def test_rounding_probe_dgrad():
    lib = _lib.load()
    gen = torch.Generator().manual_seed(6)
    c, g = _probe_geom(2, 32, 32, 4, 4)
    dy = probe_values(c.N * c.P * c.Q * c.K, gen).view(c.N, c.P, c.Q, c.K).cuda()
    w = _one_hot_weights(c.K, c.C).cuda()
    packed = torch.empty(lib.b200gan_packed_weight_floats(ctypes.byref(g), _lib.PACK_TC_DGRAD), device="cuda")
    _lib.check(lib.b200gan_pack_weights(ctypes.byref(g), _lib.PACK_TC_DGRAD, w.data_ptr(), packed.data_ptr(), None))
    dx = torch.full((c.N, c.H, c.W, c.C), float("nan"), device="cuda")
    _lib.check(lib.b200gan_conv2d_dgrad(ctypes.byref(g), dy.data_ptr(), packed.data_ptr(), dx.data_ptr(), None,
                                        _lib.ALGO_TC, None))
    torch.cuda.synchronize()
    assert torch.equal(dx.view(torch.int32), tf32_trunc(dy).view(torch.int32)), "dgrad: dy is not truncated to TF32"


@pytest.mark.parametrize("raw", ["x", "dy"])
def test_rounding_probe_wgrad(raw):
    """one pixel: dw[k][c] = dy[k] * x[c] with the other operand exactly 1"""
    lib = _lib.load()
    gen = torch.Generator().manual_seed(7)
    c, g = _probe_geom(1, 128, 128, 1, 1)
    x = torch.ones(1, 1, 1, c.C)
    dy = torch.ones(1, 1, 1, c.K)
    if raw == "x":
        x = probe_values(c.C, gen).view(1, 1, 1, c.C)
    else:
        dy = probe_values(c.K, gen).view(1, 1, 1, c.K)
    x, dy = x.cuda(), dy.cuda()
    ws = torch.full((lib.b200gan_conv2d_wgrad_workspace_floats(ctypes.byref(g), _lib.ALGO_TC),), float("nan"),
                    device="cuda")
    dw = torch.full((c.K, c.C, 1, 1), float("nan"), device="cuda")
    _lib.check(lib.b200gan_conv2d_wgrad(ctypes.byref(g), x.data_ptr(), dy.data_ptr(), dw.data_ptr(), None,
                                        ws.data_ptr(), _lib.ALGO_TC, None))
    torch.cuda.synchronize()
    want = (tf32_trunc(dy).view(c.K, 1) * tf32_trunc(x).view(1, c.C)).view(c.K, c.C, 1, 1)
    assert torch.equal(dw.view(torch.int32), want.view(torch.int32)), f"wgrad: {raw} is not truncated to TF32"


# ---- packing ---------------------------------------------------------------------------------------------------------
def np_pack(c, kind, w):
    """numpy emulation of b200gan_pack_weights: order, RNA, and the up2 fold's fp32 sum order"""
    w = np.asarray(w, dtype=np.float32)
    kcrs = w.transpose(1, 0, 2, 3) if c.transposed else w  # [Cout][Cin][R][S]
    if kind in (_lib.PACK_TC_FPROP_UP2, _lib.PACK_TC_DGRAD_UP2):
        rset = {(0, 0): (0, 0), (0, 1): (1, 2), (1, 0): (0, 1), (1, 1): (2, 2)}
        out = np.zeros((16, c.K, c.C), np.float32)
        for ph in range(4):
            a, b = ph >> 1, ph & 1
            for tap in range(4):
                dr, ds = tap >> 1, tap & 1
                v = np.zeros((c.K, c.C), np.float32)
                for r in range(rset[a, dr][0], rset[a, dr][1] + 1):
                    for s in range(rset[b, ds][0], rset[b, ds][1] + 1):
                        v = (v + kcrs[:, :, r, s]).astype(np.float32)
                out[ph * 4 + tap] = v
        out = np_rna(out)
        return (out if kind == _lib.PACK_TC_FPROP_UP2 else out.transpose(0, 2, 1)).reshape(-1)
    t = kcrs.reshape(c.K, c.C, c.R * c.S).transpose(2, 0, 1)  # [tap][Cout][Cin], taps unflipped
    if kind in (_lib.PACK_TC_FPROP, _lib.PACK_TC_DGRAD):
        t = np_rna(t)
    if kind in (_lib.PACK_SIMT_FPROP, _lib.PACK_TC_DGRAD):
        t = t.transpose(0, 2, 1)  # [tap][Cin][Cout]
    return np.ascontiguousarray(t).reshape(-1)


_PACK_GEOMS = [
    cc.Case("tile9", 1, 16, 64, 4, 4, 3, 3, pads=cc.P1, why="tile mode, R*S = 9"),
    cc.Case("tile16", 1, 8, 32, 8, 8, 4, 4, stride=2, pads=cc.P1, why="tile mode, R*S = 16"),
    cc.Case("tile4", 1, 8, 40, 4, 4, 2, 2, why="pack_tile<0>: 2x2 taps, Cout not a multiple of 32"),
    cc.Case("elem7", 1, 16, 32, 8, 8, 7, 7, pads=cc.P3, why="element mode: 49 taps"),
    cc.Case("elem_cin3", 1, 3, 64, 8, 8, 4, 4, stride=2, pads=cc.P1, why="element mode: Cin < 8"),
    cc.Case("elem_cout3", 1, 64, 3, 8, 8, 3, 3, pads=cc.P1, why="element mode: Cout < 32"),
    cc.Case("tr_tile", 1, 32, 64, 4, 4, 4, 4, stride=2, pads=cc.P1, transposed=True, why="ConvTranspose2d, tile"),
    cc.Case("tr_elem", 1, 64, 3, 4, 4, 4, 4, stride=2, pads=cc.P1, transposed=True, why="ConvTranspose2d, element"),
    cc.Case("up2_tile", 1, 16, 64, 4, 4, 3, 3, pads=cc.P1, up=2, why="up2 fold, tile mode"),
    cc.Case("up2_elem", 1, 3, 16, 4, 4, 3, 3, pads=cc.P1, up=2, why="up2 fold, element mode"),
]


def _pack_jobs():
    jobs = []
    for c in _PACK_GEOMS:
        kinds = [_lib.PACK_SIMT_FPROP, _lib.PACK_SIMT_DGRAD, _lib.PACK_TC_FPROP, _lib.PACK_TC_DGRAD]
        if c.up == 2:
            kinds += [_lib.PACK_TC_FPROP_UP2, _lib.PACK_TC_DGRAD_UP2]
        jobs += [(c, k) for k in kinds]
    return jobs


def _weights(c, seed):
    gen = torch.Generator().manual_seed(seed)
    # values with random low mantissa bits (RNA ties included) so that rounding and sum order show
    w = torch.randn(*wshape(c), generator=gen)
    ties = torch.rand(*wshape(c), generator=gen) < 0.2
    bits = w.view(torch.int32)
    bits = torch.where(ties, (bits & ~0x1FFF) | 0x1000, bits)
    return bits.view(torch.float32)


@pytest.mark.parametrize("job", _pack_jobs(), ids=lambda j: f"{j[0].name}-{j[1]}")
def test_pack_weights_bit_exact(job):
    c, kind = job
    lib = _lib.load()
    g = geom(c)
    w = _weights(c, 11)
    n = lib.b200gan_packed_weight_floats(ctypes.byref(g), kind)
    out = torch.full((n + 2048,), float("nan"), device="cuda")
    _lib.check(lib.b200gan_pack_weights(ctypes.byref(g), kind, w.cuda().data_ptr(), out[1024:].data_ptr(), None))
    torch.cuda.synchronize()
    assert torch.isnan(out[:1024]).all() and torch.isnan(out[1024 + n:]).all(), "pack wrote outside its output"
    want = np_pack(c, kind, w.numpy())
    got = out[1024:1024 + n].cpu().numpy()
    diff = np.nonzero(got.view(np.int32) != want.view(np.int32))[0]
    assert diff.size == 0, f"{c.name} pack {kind}: first mismatch at {diff[0]}: {got[diff[0]]!r} vs {want[diff[0]]!r}"


def test_pack_weights_multi_30_jobs():
    """a 30-job table: two launches (24 + 6), every copy equal to the emulation"""
    lib = _lib.load()
    jobs = (_pack_jobs() * 2)[:30]
    assert len(jobs) == 30
    table = (_lib.PackJob * len(jobs))()
    keep = []
    for i, (c, kind) in enumerate(jobs):
        w = _weights(c, 100 + i).cuda()
        g = geom(c)
        out = torch.full((lib.b200gan_packed_weight_floats(ctypes.byref(g), kind),), float("nan"), device="cuda")
        table[i].w, table[i].packed, table[i].geom, table[i].pack = w.data_ptr(), out.data_ptr(), g, kind
        keep.append((c, kind, w, out))
    _lib.check(lib.b200gan_pack_weights_multi(table, len(jobs), None))
    torch.cuda.synchronize()
    for i, (c, kind, w, out) in enumerate(keep):
        want = np_pack(c, kind, w.cpu().numpy())
        got = out.cpu().numpy()
        assert np.array_equal(got.view(np.int32), want.view(np.int32)), f"job {i} ({c.name}, pack {kind})"
