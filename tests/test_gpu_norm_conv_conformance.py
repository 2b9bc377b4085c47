"""Every case of tests/norm_conv_cases.py, element by element against fp64, through the conformance protocol.

A fused case runs b200gan_conv2d_dgrad_norm and then b200gan_norm_bwd_from_sums on the guarded buffers of
tests/conformance.py, with fixed fp32 norm state built on the host: mean_rstd from x's fp64 batch statistics,
scale = gamma * rstd and shift = beta - mean * scale in fp32.  Checked:
  - da is b200gan_conv2d_dgrad's output on the same inputs, bit for bit, and within the conv suite's bound of the fp64
    data gradient of the TF32-modelled operands (conv_cases.conv_bound);
  - dgb = (S2, S1) cast to fp32, against fp64 sums over the kernel's own da: dy' = da * act'(x * scale + shift) (the
    fp64 sign of x * scale + shift is that of the kernel's fmaf: the product of two fp32 values is exact) and
    xhat = (x - mean) * rstd.  Bound: each term carries r roundings (dy' * slope; x - mean, * rstd, dy' * xhat), then
    8 fp32 additions (a 32-row warp column sum of depth 5, four warps in order), then one fp64 atomic per tile;
  - dx against gamma rstd (dy' - S1/m - xhat S2/m) from the same fp64 sums: 10 roundings of the magnitudes that enter
    (dy' * slope, the sums' cast and the 1/m scaling, xhat, the two subtractions and gamma * rstd), plus what the sums'
    own bound moves;
  - sums come back zeroed.
A from-sums case gives the fp64 sums as an input: dgb is their fp32 cast bit for bit, and dx has the same bound
without the sums' error.  Refused calls write nothing.
"""
import ctypes
import math

import pytest
import torch

import conv_cases as cc
import norm_conv_cases as ncc
from b200gan import _lib
from conformance import Arena, bits_equal, check_elementwise, not_vacuous, run_case
from norm_cases import SLOPE

pytestmark = pytest.mark.gpu

u = 2.0 ** -24
ACT = {"none": _lib.ACT_NONE, "lrelu": _lib.ACT_LRELU, "relu": _lib.ACT_RELU, "tanh": _lib.ACT_TANH,
       "sigmoid": _lib.ACT_SIGMOID}
F32, F64 = torch.float32, torch.float64


def gamma_rn(k):
    """gamma_k = k u / (1 - k u): the relative bound of k roundings"""
    return k * u / (1 - k * u)


# ---- norm state and fp64 references ---------------------------------------------------------------------------------
def norm_state(x, gamma, beta, per_sample, eps):
    """x [N][HW][C] -> fp32 mean_rstd [2][G] and scale_shift [2][G] as b200gan_norm_finalize defines them"""
    dims = (1,) if per_sample else (0, 1)
    x64 = x.double()
    mean = x64.mean(dims)
    rstd = 1 / torch.sqrt(((x64 - x64.mean(dims, keepdim=True)) ** 2).mean(dims) + eps)
    mean, rstd = mean.float().reshape(-1), rstd.float().reshape(-1)
    G, C = mean.numel(), x.shape[2]
    ga = (gamma if gamma is not None else torch.ones(C, device=x.device)).repeat(G // C)
    be = (beta if beta is not None else torch.zeros(C, device=x.device)).repeat(G // C)
    scale = ga * rstd
    return torch.cat([mean, rstd]), torch.cat([scale, be - mean * scale])


def groups(t, N, C, per_sample):
    """[2][G] -> two fp64 tensors that broadcast against [N][HW][C]"""
    t = t.double().view(2, N if per_sample else 1, 1, C)
    return t[0], t[1]


def terms(x, dy, mean_rstd, scale_shift, act, slope, per_sample):
    """fp64 dy' = dy * act'(x * scale + shift) and xhat = (x - mean) * rstd from the fp32 operands the kernels read"""
    N, HW, C = x.shape
    x = x.double()
    mean, rstd = groups(mean_rstd, N, C, per_sample)
    sc, sh = groups(scale_shift, N, C, per_sample)
    pre = x * sc + sh
    lo = float(torch.tensor(slope, dtype=F32)) if act == "lrelu" else 0.0
    mask = torch.where(pre > 0, 1.0, lo) if act in ("lrelu", "relu") else torch.ones_like(pre)
    return dy.double().view(N, HW, C) * mask, (x - mean) * rstd, rstd


def dx_check(what, dx, dz, xh, rstd, gamma, S1, S2, m, rtf, bS1=0.0, bS2=0.0):
    """dx against gamma rstd (dz - S1/m - xhat S2/m)"""
    gr = (gamma.double() if gamma is not None else 1.0) * rstd
    m1, m2 = S1 / m, S2 / m
    ref = gr * (dz - m1 - xh * m2)
    b = gr.abs() * (gamma_rn(10) * (dz.abs() + m1.abs() + (xh * m2).abs()) + (bS1 + xh.abs() * bS2) / m)
    if rtf:
        b = b + 2.0 ** -11 * (ref.abs() + b)
        assert ((dx.view(torch.int32) & 0x1FFF) == 0).all(), f"{what}: round_tf32 dx not TF32-representable"
    worst = check_elementwise(what + " dx", dx, ref, b, "(n, hw, c)")
    not_vacuous(what + " dx", b, (gr * dz).abs().expand_as(b))
    return worst


# ---- the fused data gradient and apply-from-sums -----------------------------------------------------------------
def conv_case(c):
    """the case's data gradient as a conv table case: the conv suite's reference and bound take it"""
    kernels = (c.kernels[0],) if c.kernels else ("conv_tc_kernel",)
    return cc.Case(c.name, c.N, c.C, c.K, c.H, c.W, c.R, c.S, stride=c.stride, pads=c.pads, pad_mode=c.pad_mode,
                   up=c.up, transposed=c.transposed, pas=cc.DGRAD, kernels=kernels)


class FusedRun:
    def __init__(self, c, seed=0):
        self.c, lib = c, _lib.load()
        self.lib = lib
        N, C, K, HW = c.N, c.C, c.K, c.H * c.W
        gen = torch.Generator().manual_seed(seed)
        self.cg = conv_case(c)
        self.g = cc.geom(self.cg)
        self.x = (torch.randn(N, HW, C, generator=gen) * 1.5 + 0.3).cuda()
        self.dy = torch.randn(N, c.P, c.Q, K, generator=gen).cuda()
        self.w = (torch.randn(*cc.wshape(self.cg), generator=gen) / math.sqrt(C * c.R * c.S)).cuda()
        self.gamma = (0.5 + torch.rand(C, generator=gen)).cuda()
        beta = torch.zeros(C) if c.beta0 else 0.3 * torch.randn(C, generator=gen)
        self.eps = 0.8 if C == 128 else 1e-5
        self.mean_rstd, self.scale_shift = norm_state(self.x, self.gamma, beta.cuda(), False, self.eps)
        if not c.code:
            kind = _lib.PACK_TC_DGRAD_UP2 if c.up == 2 else _lib.PACK_TC_DGRAD
            self.packed = torch.empty(lib.b200gan_packed_weight_floats(ctypes.byref(self.g), kind), device="cuda")
            _lib.check(lib.b200gan_pack_weights(ctypes.byref(self.g), kind, self.w.data_ptr(), self.packed.data_ptr(),
                                                None), "pack")
        else:  # never read: the call refuses first
            self.packed = torch.zeros(K * C * c.R * c.S * (16 if c.up == 2 else 1), device="cuda")
        self.off = 1 if c.refuse == "x_offset" else 0
        n = N * HW * C
        self.arena = Arena([("dy", self.dy.numel(), F32, "in"), ("w", self.packed.numel(), F32, "in"),
                            ("x", n + self.off, F32, "in"), ("mean_rstd", 2 * C, F32, "in"),
                            ("scale_shift", 2 * C, F32, "in"), ("gamma", C, F32, "in"), ("da", n, F32, "out"),
                            ("sums", 2 * C, F64, "ws"), ("dx", n, F32, "out"), ("dgb", 2 * C, F32, "out")])
        lead = torch.full((self.off,), float("nan"), device="cuda")
        self.data = dict(dy=self.dy, w=self.packed, x=torch.cat([lead, self.x.reshape(-1)]), mean_rstd=self.mean_rstd,
                         scale_shift=self.scale_shift, gamma=self.gamma)
        dN, dC, dHW = N + (c.refuse == "desc_N"), C - 32 * (c.refuse == "desc_C"), HW + (c.refuse == "desc_HW")
        self.d = _lib.NormDesc(dN, dHW, dC, int(c.refuse == "per_sample"), self.eps, 0.0, ACT[c.act], c.slope,
                               int(c.rtf))

    def prepare(self):
        self.arena.prepare(self.data)
        self.arena.t["sums"].zero_()  # "zero on entry": the call must not depend on a prefill

    def ptr(self, name):
        return self.arena.ptr(name) + (4 * self.off if name == "x" else 0)

    def call(self, st):
        lib, p, d = self.lib, self.ptr, ctypes.byref(self.d)
        rc = lib.b200gan_conv2d_dgrad_norm(ctypes.byref(self.g), d, p("dy"), p("w"), p("x"), p("mean_rstd"),
                                           p("scale_shift"), p("sums"), p("da"), st)
        if rc:
            return rc
        return lib.b200gan_norm_bwd_from_sums(d, p("da"), p("x"), p("mean_rstd"), p("scale_shift"), p("gamma"),
                                              p("sums"), p("dx"), p("dgb"), st)

    def outputs(self):
        return self.arena.outputs()

    def check(self, what):
        c, t, lib = self.c, self.arena.t, self.lib
        N, C, HW = c.N, c.C, c.H * c.W
        da = t["da"]
        plain = torch.full_like(da, float("nan"))
        assert lib.b200gan_conv2d_dgrad(ctypes.byref(self.g), self.ptr("dy"), self.ptr("w"), plain.data_ptr(), None,
                                        _lib.ALGO_TC, torch.cuda.current_stream().cuda_stream) == 0
        torch.cuda.synchronize()
        bits_equal(what + ": da against b200gan_conv2d_dgrad", da, plain)
        x, dy, w, eps_op = cc.operands(self.cg, self.x.view(N, c.H, c.W, C), self.dy, self.w)
        ref = cc.conv_pass_ref(self.cg, x, dy, w)
        A = cc.conv_pass_ref(self.cg, x.abs(), dy.abs(), w.abs())
        b = cc.conv_bound(self.cg, A, eps_op)
        worst = check_elementwise(what + " da", da, ref, b, "(n, h, w, c)")
        not_vacuous(what + " da", b, cc.conv_pass_ref(self.cg, x, dy, cc.one_tap(self.cg, w)).abs())

        dz, xh, rstd = terms(self.x, da, self.mean_rstd, self.scale_shift, c.act, c.slope, False)
        p = dz * xh
        r = 1 if c.act == "lrelu" else 0   # dy' * slope
        S1, S2 = dz.sum((0, 1)), p.sum((0, 1))
        a1, a2 = dz.abs().sum((0, 1)), p.abs().sum((0, 1))
        atomics = c.tiles * 2.0 ** -52
        bS1 = (gamma_rn(r + 8) + atomics) * a1
        bS2 = (gamma_rn(r + 3 + 8) + atomics) * a2
        dgb = t["dgb"].double()
        worst = max(worst, check_elementwise(what + " dgamma", dgb[:C], S2, bS2 + u * (S2.abs() + bS2), "(c,)"),
                    check_elementwise(what + " dbeta", dgb[C:], S1, bS1 + u * (S1.abs() + bS1), "(c,)"))
        not_vacuous(what + " dgamma", bS2, p.abs().reshape(-1))
        not_vacuous(what + " dbeta", bS1, dz.abs().reshape(-1))
        worst = max(worst, dx_check(what, t["dx"].view(N, HW, C), dz, xh, rstd, self.gamma, S1, S2, N * HW, c.rtf,
                                    bS1, bS2))
        assert (t["sums"] == 0).all(), f"{what}: the sums are not handed back zeroed"
        return worst


def fused_launches(c):
    return [(c.kernels[0], c.grid), (c.kernels[1], (None, 1, 1)), (c.kernels[2], None)] if c.kernels else []


@pytest.mark.parametrize("case", ncc.FUSED, ids=lambda c: c.id)
def test_fused_case(case):
    # the sums are fp64 atomics in no fixed order: dx and dgamma / dbeta may differ in their last bits; da may not
    run_case(FusedRun(case), case.id, fused_launches(case), refuse=(case.code,) if case.code else (),
             varies=("sums", "dx", "dgb"), family=("conv_tc_", "norm_bwd_"), num_sms=ncc.NUM_SMS)


# ---- apply-from-sums on every norm geometry -------------------------------------------------------------------------
class SumsRun:
    def __init__(self, case, seed=0):
        self.c, g = case, case.geom
        self.lib = _lib.load()
        self.G = g.N * g.C if g.per_sample else g.C
        n = g.N * g.H * g.W * g.C
        gen = torch.Generator().manual_seed(seed)
        self.x = (torch.randn(g.N, g.H * g.W, g.C, generator=gen) * 2 + 0.5).cuda()
        self.dy = torch.randn(g.N, g.H * g.W, g.C, generator=gen).cuda()
        self.gamma = (1 + 0.5 * torch.randn(g.C, generator=gen)).cuda() if g.affine else None
        beta = (0.3 * torch.randn(g.C, generator=gen)).cuda() if g.affine else None
        self.eps = 1e-5 if g.per_sample else 0.8
        self.mean_rstd, self.scale_shift = norm_state(self.x, self.gamma, beta, g.per_sample, self.eps)
        dims = (1,) if g.per_sample else (0, 1)
        dz, xh, _ = terms(self.x, self.dy, self.mean_rstd, self.scale_shift, case.act, SLOPE, g.per_sample)
        self.S1, self.S2 = dz.sum(dims).reshape(-1), (dz * xh).sum(dims).reshape(-1)
        specs = [("dy", n, F32, "in"), ("x", n + g.offset, F32, "in"), ("mean_rstd", 2 * self.G, F32, "in"),
                 ("scale_shift", 2 * self.G, F32, "in"), ("sums", 2 * self.G, F64, "io"), ("dx", n, F32, "out")]
        if g.affine:
            specs += [("gamma", g.C, F32, "in"), ("dgb", 2 * self.G, F32, "out")]
        self.arena = Arena(specs)
        lead = torch.full((g.offset,), float("nan"), device="cuda")
        self.data = dict(dy=self.dy, x=torch.cat([lead, self.x.reshape(-1)]), mean_rstd=self.mean_rstd,
                         scale_shift=self.scale_shift, sums=torch.cat([self.S1, self.S2]), gamma=self.gamma)
        self.d = _lib.NormDesc(g.N, g.H * g.W, g.C, int(g.per_sample), self.eps, 0.0, ACT[case.act], SLOPE,
                               int(case.rtf))

    def prepare(self):
        self.arena.prepare(self.data)

    def ptr(self, name):
        p = self.arena.ptr(name)
        return p + 4 * self.c.geom.offset if name == "x" else p

    def call(self, st):
        p = self.ptr
        return self.lib.b200gan_norm_bwd_from_sums(ctypes.byref(self.d), p("dy"), p("x"), p("mean_rstd"),
                                                   p("scale_shift"), p("gamma"), p("sums"), p("dx"), p("dgb"), st)

    def outputs(self):
        return self.arena.outputs()

    def check(self, what):
        c, g, t = self.c, self.c.geom, self.arena.t
        dz, xh, rstd = terms(self.x, self.dy, self.mean_rstd, self.scale_shift, c.act, SLOPE, g.per_sample)
        shape = (g.N if g.per_sample else 1, 1, g.C)
        m = g.H * g.W * (1 if g.per_sample else g.N)
        worst = dx_check(what, t["dx"].view(g.N, g.H * g.W, g.C), dz, xh, rstd, self.gamma, self.S1.view(shape),
                         self.S2.view(shape), m, c.rtf)
        if g.affine:
            bits_equal(what + " dgamma", t["dgb"][:self.G], self.S2.float())
            bits_equal(what + " dbeta", t["dgb"][self.G:], self.S1.float())
        assert (t["sums"] == 0).all(), f"{what}: the sums are not handed back zeroed"
        return worst


def sums_launches(c):
    g = c.geom
    return [(c.kernels[0], (None, g.N if g.per_sample else 1, g.slices)), (c.kernels[1], None)] if c.kernels else []


@pytest.mark.parametrize("case", ncc.FROM_SUMS, ids=lambda c: c.id)
def test_from_sums_case(case):
    run_case(SumsRun(case), case.id, sums_launches(case), refuse=(case.code,) if case.code else (),
             family=("norm_bwd_",))
