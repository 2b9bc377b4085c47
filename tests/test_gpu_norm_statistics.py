"""Every row of tests/stats_cases.py against fp64: the BatchNorm / InstanceNorm statistics each kernel produces, at the
models' reduction sizes, on channels far from zero and exactly constant ones.

The data is what the kernel itself wrote (y of a conv or chain call, x of a stand-alone run), grouped as the
normalisation groups it: fp64 mean, biased variance and max |x - mean| per group.  Checked element by element:
  - the mean and variance implied by the kernel's [sum x, sum x^2], formed as norm_finalize_kernel forms them;
  - mean_rstd, scale_shift, running_mean and running_var (unbiased) of a b200gan_norm_finalize call on those sums;
  - for the stand-alone path, y, dx and the rest of norm_cases.check_outputs on the same data;
  - the route each row names, eagerly and replayed from a CUDA graph (tests/conformance.py).
The bounds follow from each kernel's fp32 summation chain (stats_cases.chain, stats_cases.bounds) and carry no term in
(mean / std)^2: an implementation whose fp32 partial sums are taken around zero fails them on the far channels.
"""
import ctypes
import math

import numpy as np
import pytest
import torch

import norm_cases as nc
import stats_cases as sc
from b200gan import _lib
from conformance import Arena, check_elementwise, first_grid, not_vacuous, run_case

pytestmark = pytest.mark.gpu

U = sc.U
SLOPE = 0.2


def grouped(t, c):
    """[G, m] float64 of an NHWC tensor: InstanceNorm groups (n, k), or BatchNorm groups (statistics group, k)"""
    t = t.double().reshape(c.N, -1, c.K)
    if c.per_sample:
        return t.permute(0, 2, 1).reshape(c.N * c.K, -1)
    return t.reshape(c.groups, -1, c.K).permute(0, 2, 1).reshape(c.groups * c.K, -1)


def split_sums(raw, c):
    """(sum x, sum x^2) per group of the kernel's statistics buffer ([groups][2][K] for the chain, [2][G] otherwise)"""
    if c.path == "chain":
        s = raw.view(c.groups, 2, c.K)
        return s[:, 0].reshape(-1), s[:, 1].reshape(-1)
    G = raw.numel() // 2
    return raw[:G], raw[G:]


def check_statistics(what, c, data, raw, gamma, beta, rm0, rv0):
    """the statistics of case c from its sums `raw` against fp64 statistics of `data`; the worst |err|/bound"""
    lib = _lib.load()
    ch = sc.chain(c, torch.cuda.get_device_properties(0).multi_processor_count)
    m = data.shape[1]
    mean = data.mean(1)
    var = ((data - mean[:, None]) ** 2).mean(1)
    dev = (data - mean[:, None]).abs().amax(1)
    mb, vb = sc.bounds(ch.K, ch.P, mean, var, dev)
    s1, s2 = split_sums(raw, c)
    mean_k = s1 / m
    var_k = (s2 / m - mean_k * mean_k).clamp_min(0)
    worst = check_elementwise(f"{what} mean from the sums", mean_k, mean, mb)
    worst = max(worst, check_elementwise(f"{what} variance from the sums", var_k, var, vb))
    not_vacuous(f"{what} mean", mb, var.sqrt())
    not_vacuous(f"{what} variance", vb, var)

    # finalize on the kernel's sums, one call per statistics group of the batch
    eps = float(np.float32(c.eps))
    rstd = 1 / torch.sqrt(var + eps)
    rb = rstd * (0.5 * vb / (var + eps) + 2 * U)
    G = mean.numel() // c.groups
    HW = m if c.per_sample else m * c.groups // c.N
    ch_idx = torch.arange(mean.numel(), device="cuda") % c.K
    ga, be = gamma.double()[ch_idx], beta.double()[ch_idx]
    for gi in range(c.groups):
        at = slice(gi * G, (gi + 1) * G)
        d = _lib.NormDesc(c.N // c.groups, HW, c.K, int(c.per_sample), c.eps, sc.MOMENTUM, 0, 0.0, 0)
        sums = torch.cat([s1[at], s2[at]]).contiguous()
        mr = torch.full((2 * G,), float("nan"), device="cuda")
        ss = torch.full((2 * G,), float("nan"), device="cuda")
        rm, rv = rm0.clone(), rv0.clone()
        nbt = torch.zeros(1, dtype=torch.int64, device="cuda")
        run = not c.per_sample
        rc = lib.b200gan_norm_finalize(ctypes.byref(d), sums.data_ptr(), gamma.data_ptr(), beta.data_ptr(),
                                       mr.data_ptr(), ss.data_ptr(), rm.data_ptr() if run else None,
                                       rv.data_ptr() if run else None, nbt.data_ptr(), None)
        assert rc == 0, lib.b200gan_last_error().decode()
        torch.cuda.synchronize()
        mu, r, mbg, rbg, g_, b_ = mean[at], rstd[at], mb[at], rb[at], ga[at], be[at]
        w = f"{what} group set {gi}"
        worst = max(worst, check_elementwise(f"{w} mean_rstd mean", mr[:G], mu, mbg + U * mu.abs()))
        worst = max(worst, check_elementwise(f"{w} mean_rstd rstd", mr[G:], r, rbg))
        not_vacuous(f"{w} rstd", rbg, r)
        scale = g_ * r
        scb = g_.abs() * rbg + U * scale.abs()
        shift = b_ - mu * scale
        shb = mu.abs() * scb + scale.abs() * (mbg + U * mu.abs()) + 3 * U * ((mu * scale).abs() + b_.abs())
        worst = max(worst, check_elementwise(f"{w} scale", ss[:G], scale, scb))
        worst = max(worst, check_elementwise(f"{w} shift", ss[G:], shift, shb))
        if run:
            mom = sc.MOMENTUM
            unb = var[at] * m / (m - 1)
            rm_ref = (1 - mom) * rm0.double() + mom * mu
            rv_ref = (1 - mom) * rv0.double() + mom * unb
            worst = max(worst, check_elementwise(f"{w} running_mean", rm, rm_ref,
                                                 mom * mbg + 4 * U * (rm0.double().abs() + mu.abs())))
            worst = max(worst, check_elementwise(f"{w} running_var", rv, rv_ref,
                                                 mom * vb[at] * m / (m - 1) + 4 * U * (rv0.double().abs() + unb)))
    return worst


def params(K, gen):
    gamma = (1 + 0.5 * torch.randn(K, generator=gen)).cuda()
    beta = (0.3 * torch.randn(K, generator=gen)).cuda()
    rm0 = (0.1 * torch.randn(K, generator=gen)).cuda()
    rv0 = (1 + torch.rand(K, generator=gen)).cuda()
    return gamma, beta, rm0, rv0


# ---- the stand-alone path: norm_cases.Run on ladder data, with one more norm_stats into `raw` ---------------------------
class NormRun(nc.Run):
    def __init__(self, c, geom, seed=0):
        super().__init__(nc.Case(geom, c.act, False), seed)
        self.sc = c
        gen = torch.Generator().manual_seed(seed + 1)
        loc, sd = (torch.from_numpy(a).float() for a in sc.ladder(c.C))
        self.x = (loc + sd * torch.randn(c.N, c.H * c.W, c.C, generator=gen)).cuda()
        self.data["x"] = torch.cat([torch.full((c.offset,), float("nan"), device="cuda"), self.x.reshape(-1)])
        self.arena = Arena(self.arena.specs + [("raw", 2 * self.G, torch.float64, "ws")])
        if c.per_sample:
            self.gamma, self.beta = params(c.C, gen)[:2]

    def prepare(self):
        super().prepare()
        self.arena.t["raw"].zero_()

    def call(self, st):
        rc = self.lib.b200gan_norm_stats(ctypes.byref(self.d), self.ptr("x"), self.ptr("raw"), st)
        return rc or super().call(st)

    def check(self, what):
        c = self.sc
        worst = check_statistics(what, c, grouped(self.x, c), self.arena.t["raw"], self.gamma, self.beta, self.rm0,
                                 self.rv0)
        return max(worst, nc.check_outputs(self, what))


# ---- conv and chain: a bias ladder with small weights (a zero-weight channel is constant) -------------------------------
def ladder_weights(c, gen):
    loc, sd = (torch.from_numpy(a).float() for a in sc.ladder(c.K))
    w = torch.randn(c.K, c.C, c.R, c.R, generator=gen) * (sd / math.sqrt(c.C * c.R * c.R))[:, None, None, None]
    return w, loc


class ConvRun:
    """b200gan_conv2d_fprop on the wgmma path with its statistics in `raw`"""

    def __init__(self, c, seed=0):
        from b200gan import ops
        self.c, lib = c, _lib.load()
        self.lib = lib
        gen = torch.Generator().manual_seed(seed)
        x = torch.randn(c.N, c.H, c.W, c.C, generator=gen)
        w, loc = ladder_weights(c, gen)
        if c.splitk:   # no bias: the location rides on input channel 0 = 1 through a tap that never meets the padding
            x[..., 0] = 1
            w[:, 0] = 0
            w[:, 0, c.pad, c.pad] = loc
        self.g, out = ops.make_geom((c.N, c.C, c.H, c.W), tuple(w.shape), c.stride, (c.pad,) * 4, _lib.PAD_ZERO, c.up,
                                    False)
        assert ops.tc_supported(self.g, 0), c.id
        kind = _lib.PACK_TC_FPROP_UP2 if c.up == 2 else _lib.PACK_TC_FPROP
        self.packed = torch.empty(lib.b200gan_packed_weight_floats(ctypes.byref(self.g), kind), device="cuda")
        w = w.cuda()
        _lib.check(lib.b200gan_pack_weights(ctypes.byref(self.g), kind, w.data_ptr(), self.packed.data_ptr(), None))
        torch.cuda.synchronize()
        self.gamma, self.beta, self.rm0, self.rv0 = params(c.K, gen)
        G = c.N * c.K if c.per_sample else c.K
        specs = [("x", x.numel(), torch.float32, "in"), ("w", self.packed.numel(), torch.float32, "in"),
                 ("y", c.N * c.P_ * c.Q_ * c.K, torch.float32, "out"), ("raw", 2 * G, torch.float64, "ws")]
        self.data = dict(x=x.cuda(), w=self.packed)
        if not c.splitk:
            specs.append(("bias", c.K, torch.float32, "in"))
            self.data["bias"] = loc.cuda()
        if c.drop:
            specs.append(("cs", c.N * c.K, torch.float32, "in"))
            self.data["cs"] = ((torch.rand(c.N, c.K, generator=gen) < 0.8).float() * 1.25).cuda()
        self.arena = Arena(specs)

    def prepare(self):
        self.arena.prepare(self.data)
        self.arena.t["raw"].zero_()

    def outputs(self):
        return self.arena.outputs()

    def call(self, st):
        a, c = self.arena, self.c
        act = _lib.ACT_NONE if c.act == "none" else _lib.ACT_LRELU
        self.ep = _lib.Epilogue(a.ptr("bias"), act, SLOPE, a.ptr("cs"), a.ptr("raw"), int(c.per_sample), 0)
        return self.lib.b200gan_conv2d_fprop(ctypes.byref(self.g), ctypes.byref(self.ep), a.ptr("x"), a.ptr("w"),
                                             a.ptr("y"), _lib.ALGO_TC, st)

    def check(self, what):
        y = self.arena.t["y"]
        assert not torch.isnan(y).any(), f"{what}: y has elements the conv never wrote"
        return check_statistics(what, self.c, grouped(y, self.c), self.arena.t["raw"], self.gamma, self.beta,
                                self.rm0, self.rv0)


class ChainRun(ConvRun):
    """b200gan_nb_fprop without an input BatchNorm or a Dropout2d scale, with out_stats in `raw`"""

    def __init__(self, c, seed=0):
        self.c, lib = c, _lib.load()
        self.lib = lib
        gen = torch.Generator().manual_seed(seed)
        x = torch.randn(c.N, c.H, c.W, c.C, generator=gen)
        w, loc = ladder_weights(c, gen)
        self.g = _lib.ConvGeom(c.N, c.H, c.W, c.C, c.K, c.R, c.R, c.stride, 1, 1, 1, 1, _lib.PAD_ZERO, 1, 0, c.P_, c.Q_)
        self.packed = torch.empty(lib.b200gan_packed_weight_floats(ctypes.byref(self.g), _lib.PACK_SIMT_FPROP),
                                  device="cuda")
        w = w.cuda()
        _lib.check(lib.b200gan_pack_weights(ctypes.byref(self.g), _lib.PACK_SIMT_FPROP, w.data_ptr(),
                                            self.packed.data_ptr(), None))
        torch.cuda.synchronize()
        self.gamma, self.beta, self.rm0, self.rv0 = params(c.K, gen)
        self.arena = Arena([("x", x.numel(), torch.float32, "in"), ("w", self.packed.numel(), torch.float32, "in"),
                            ("bias", c.K, torch.float32, "in"), ("y", c.N * c.P_ * c.Q_ * c.K, torch.float32, "out"),
                            ("raw", c.groups * 2 * c.K, torch.float64, "ws")])
        self.data = dict(x=x.cuda(), w=self.packed, bias=loc.cuda())

    def call(self, st):
        a, c = self.arena, self.c
        return self.lib.b200gan_nb_fprop(ctypes.byref(self.g), None, None, None, None, sc.MOMENTUM, a.ptr("x"),
                                         a.ptr("w"), a.ptr("bias"), _lib.ACT_LRELU, SLOPE, a.ptr("cs"), a.ptr("y"),
                                         a.ptr("raw"), c.groups, st)


GEOMS = {g.name: g for g in sc.NORM_GEOMS}


@pytest.mark.parametrize("case", sc.CASES, ids=lambda c: c.id)
def test_norm_statistics(case):
    c = case
    if c.path == "norm":
        run = NormRun(c, GEOMS[c.name])
        varies = ("y", "mean_rstd", "scale_shift", "dx", "dgb", "running_mean", "running_var", "raw")
        run_case(run, c.id, [(k, None) for k in c.kernels], varies=varies, family=("norm_",))
    elif c.path == "conv":
        run_case(ConvRun(c), c.id, [(k, None) for k in c.kernels], varies=("raw", "y") if c.splitk else ("raw",),
                 family=("conv_tc", "norm_"))
    else:
        run_case(ChainRun(c), c.id, first_grid(c.kernels, c.grid), varies=("raw",), family=("nbk_",),
                 num_sms=sc.NUM_SMS)
