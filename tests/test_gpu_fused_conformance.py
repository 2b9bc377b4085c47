"""Every case of tests/chain_cases.py and tests/tail_cases.py, element by element against torch float64.

Each case calls the C ABI directly on the guarded buffers of the convolution conformance test (Arena): inputs
between NaN guards, outputs started as NaN, sentinels around everything the library writes.  The fp64 statistics
and sums buffers start at non-zero values, so a kernel that accumulates into them instead of overwriting them (the
header's "OVERWRITTEN" contracts) fails; num_batches_tracked starts at 7.

The reference feeds the operands the kernel feeds:
  - chain: the BatchNorm constants from the same fp64 batch sums the call receives; the bound carries the fp32
    rounding of scale / shift (nb_bn_consts) and of the staged x = fmaf(a, scale, shift) through |w|;
  - generator tail forward: the normalised, activated operand and the weights rounded to TF32 with RNA, as the
    kernel rounds both before wgmma;
  - generator tail backward: the recomputed pre-activation fmaf(a, scale, shift); an element whose fp64
    pre-activation lies within a few ulps of 0 may take either branch of the activation's derivative.
Bounds follow the conv suite: 2^-23 (n + s + 4) A for fp32 chains of length n with s partial sums added outside
them, 2^-22 (ceil(n / 8) + s + 4) A for wgmma, carried through the epilogue with Lipschitz constants; an fp64 sum
of fp32 block partials is bounded by the partial length times the sum of |term|.
"""
import ctypes
import math

import pytest
import torch
import torch.nn.functional as F

import chain_cases as ch
import tail_cases as tl
from b200gan import _lib
from test_gpu_conv_conformance import Arena, tf32_rna, traced_kernels

pytestmark = pytest.mark.gpu

U = 2.0 ** -23
SLOPE = 0.2
MOMENTUM = 0.1
BN_EPS = 0.8          # nn.BatchNorm2d(out, 0.8) of dcgan.py:82
NBT0 = 7
BLOCK_PARTIAL = 1032  # values a chain kernel sums in fp32 before its fp64 atomic: at most a tile's 1024 pixels
ACT_CODE = {"none": _lib.ACT_NONE, "lrelu": _lib.ACT_LRELU, "relu": _lib.ACT_RELU, "tanh": _lib.ACT_TANH,
            "sigmoid": _lib.ACT_SIGMOID}
NEG_SLOPE = {"none": 1.0, "lrelu": SLOPE, "relu": 0.0}


# ---- fp64 references (device-agnostic: tests/test_cpu_fused_case_table.py holds them to stock torch) -----------------
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


def act_mid32(act, v):
    """the tail's LeakyReLU / ReLU in fp32, as the kernel computes it"""
    if act == "lrelu":
        return torch.where(v > 0, v, v * SLOPE)
    if act == "relu":
        return v.clamp_min(0)
    return v


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


# ---- checks ---------------------------------------------------------------------------------------------------------
def check(what, got, ref, bound, alt=None):
    """|got - ref| <= bound element by element; where `alt` is not NaN, matching alt instead is accepted"""
    got = got.double().reshape(ref.shape)
    assert not torch.isnan(got).any(), f"{what}: NaN at {tuple(torch.isnan(got).nonzero()[0].tolist())} " \
                                       "(an element never written, or a guard read)"
    err = (got - ref).abs()
    if alt is not None:
        err = torch.where(torch.isnan(alt), err, torch.minimum(err, (got - alt).abs()))
    bad = (err > bound).nonzero()
    if bad.numel():
        at = tuple(bad[0].tolist())
        raise AssertionError(f"{what}: |err| {err[at].item():.3e} > bound {bound[at].item():.3e} at {at}; got "
                             f"{got[at].item():.9g}, fp64 {ref[at].item():.9g}")
    ratio = err / bound.clamp_min(1e-300)
    return ratio.max().item() if ratio.numel() else 0.0


def check_sums(what, got, ref, bound):
    return check(what + " (an OVERWRITTEN buffer: accumulating onto its old contents fails)", got, ref, bound)


# ---- chain runs ------------------------------------------------------------------------------------------------------
def chain_geom(c):
    return _lib.ConvGeom(c.N, c.H, c.W, c.C, c.K, c.R, c.R, c.stride, 1, 1, 1, 1, _lib.PAD_ZERO, 1, 0, c.P, c.Q)


class ChainRun:
    def __init__(self, c, seed=0):
        self.c = c
        lib = self.lib = _lib.load()
        gen = torch.Generator().manual_seed(seed)
        G, N, C, K = c.groups, c.N, c.C, c.K
        f32, f64 = torch.float32, torch.float64
        self.G = G
        self.has_bn = c.edge != "none"
        self.affine = c.edge == "affine"
        specs, data = [], {}

        def inp(name, t, dtype=f32):
            specs.append((name, t.numel(), dtype, "in"))
            data[name] = t.to(dtype).cuda()

        # the BatchNorm of the edge: channels Cb of the tensor `ab` it normalises
        self.op = c.op
        if c.op in ("fprop", "wgrad", "dgrad", "plain_dgrad"):
            self.g = chain_geom(c)
            ab_shape, Cb = (N, c.H, c.W, C), C
        elif c.op == "dz":
            ab_shape, Cb = (N, c.H, c.W, K), K
        else:
            ab_shape, Cb = (N, c.H * c.W, C), C
        self.Cb = Cb
        self.count = float(N // G * math.prod(ab_shape[1:-1]))
        # stored activations: mean away from 0 and a share of negatives (the LeakyReLU mask of nb_dz)
        self.a = torch.randn(*ab_shape, generator=gen) * 1.5 + 0.3
        self.gamma = 1 + 0.5 * torch.randn(Cb, generator=gen)
        self.beta = 0.3 * torch.randn(Cb, generator=gen)
        self.rm0 = 0.1 * torch.randn(Cb, generator=gen)
        self.rv0 = 1 + torch.rand(Cb, generator=gen)
        w = torch.randn(K, C, c.R, c.R, generator=gen) / math.sqrt(C * c.R * c.R)
        self.w = w.cuda()
        self.bias = (0.5 * torch.randn(K, generator=gen)).cuda()
        cs = torch.where(torch.rand(N, K, generator=gen) < 0.25, torch.zeros(()),
                         0.5 + 1.5 * torch.rand(N, K, generator=gen))
        self.cs = (cs * torch.where(torch.rand(N, K, generator=gen) < 0.5, -1.0, 1.0)).cuda()
        self.dz_in = torch.randn(N, c.P, c.Q, K, generator=gen).cuda()      # dgrad / wgrad: gradient at the output
        self.grad_in = torch.randn(*ab_shape, generator=gen).cuda()         # dz: G; tail_bwd: dout (NHWC order)
        self.stats = group_sums(self.a, G)
        if self.has_bn:
            inp("stats_in", self.stats, f64)
            if self.affine:
                inp("gamma", self.gamma)
                inp("beta", self.beta)
        self.a = self.a.cuda()
        if c.op == "fprop":
            self.kind = _lib.PACK_SIMT_FPROP
            self._pack()
            inp("x", torch.cat([torch.full((1,), float("nan"), device="cuda"), self.a.reshape(-1)]) if c.misalign
                else self.a)
            inp("w", self.packed)
            inp("bias", self.bias)
            if c.cs:
                inp("cs", self.cs)
            specs.append(("y", N * c.P * c.Q * K, f32, "out"))
            if c.out_stats:
                specs.append(("out_stats", G * 2 * K, f64, "stats"))
        elif c.op in ("dgrad", "plain_dgrad"):
            self.kind = _lib.PACK_SIMT_DGRAD
            self._pack()
            inp("dz", self.dz_in)
            inp("w", self.packed)
            specs.append(("g_out", N * c.H * c.W * C, f32, "out"))
            if c.op == "dgrad":
                inp("a_prev", self.a)
                if c.sums:
                    specs.append(("sums", G * 2 * C, f64, "stats"))
            else:
                nws = lib.b200gan_conv2d_dgrad_workspace_floats(ctypes.byref(self.g), _lib.ALGO_SIMT)
                if nws:
                    specs.append(("ws", nws, f32, "ws"))
        elif c.op == "wgrad":
            inp("x", self.a)
            inp("dz", self.dz_in)
            specs.append(("dw", K * C * c.R * c.R, f32, "out"))
            nws = lib.b200gan_nb_wgrad_workspace_floats(ctypes.byref(self.g)) if c.ws else 0
            # a plan without slabs takes the atomics; a buffer passed anyway must stay untouched (checked below)
            self.unused_ws = c.ws and nws == 0
            if c.ws:
                specs.append(("ws", nws or 1024, f32, "ws"))
        elif c.op == "dz":
            inp("g", self.grad_in)
            inp("a", self.a)
            if c.cs:
                inp("cs", self.cs)
            if self.has_bn:
                mean, var, rstd, sc, sh = bn_consts(self.stats, self.gamma if self.affine else None,
                                                    self.beta if self.affine else None, self.count, G, K)
                a64, g64 = self.a.double().cpu(), self.grad_in.double().cpu()
                xh = (a64 - per_image(mean, N)) * per_image(rstd, N)
                self.sums_in = torch.stack([g64.reshape(G, -1, K).sum(1), (g64 * xh).reshape(G, -1, K).sum(1)], 1)
                inp("sums", self.sums_in, f64)
            specs.append(("dz", N * c.H * c.W * K, f32, "out"))
            if c.db:
                specs.append(("db", K, f32, "out"))
        elif c.op == "tail_fwd":
            inp("a", self.a)
            specs.append(("out", self.a.numel(), f32, "out"))
        else:
            inp("a", self.a)
            dout = self.grad_in.permute(0, 2, 1) if c.nchw else self.grad_in
            inp("dout", dout.contiguous())
            specs += [("g", self.a.numel(), f32, "out"), ("sums", G * 2 * C, f64, "stats")]
        self.running = c.running and self.has_bn
        if self.running:
            specs += [("running_mean", Cb, f32, "ws"), ("running_var", Cb, f32, "ws")]
            inp("nbt", torch.tensor([NBT0]), torch.int64)
        self.arena = Arena(specs)
        self.data = data

    def _pack(self):
        lib = self.lib
        n = lib.b200gan_packed_weight_floats(ctypes.byref(self.g), self.kind)
        self.packed = torch.empty(n, device="cuda")
        _lib.check(lib.b200gan_pack_weights(ctypes.byref(self.g), self.kind, self.w.data_ptr(),
                                            self.packed.data_ptr(), None), "pack")

    def prepare(self):
        self.arena.prepare(self.data)
        if self.running:
            self.arena.t["running_mean"].copy_(self.rm0)
            self.arena.t["running_var"].copy_(self.rv0)

    def ptr(self, name):
        p = self.arena.ptr(name)
        return p + 4 if (name == "x" and self.c.misalign) else p

    def bn(self, groups=None):
        if not self.has_bn:
            return None
        p = self.ptr
        self._bn = _lib.NbBn(p("stats_in"), p("gamma"), p("beta"), BN_EPS, self.count, groups or self.G, 0)
        return ctypes.byref(self._bn)

    def call(self, st):
        c, lib, p = self.c, self.lib, self.ptr
        g = ctypes.byref(self.g) if hasattr(self, "g") else None
        if c.op == "fprop":
            return lib.b200gan_nb_fprop(g, self.bn(), p("running_mean"), p("running_var"), p("nbt"), MOMENTUM, p("x"),
                                        p("w"), p("bias"), ACT_CODE[c.act], SLOPE, p("cs"), p("y"), p("out_stats"),
                                        c.call_groups or c.groups, st)
        if c.op == "dgrad":
            return lib.b200gan_nb_dgrad(g, p("dz"), p("w"), self.bn(), p("a_prev"), p("g_out"), p("sums"), st)
        if c.op == "plain_dgrad":
            return lib.b200gan_conv2d_dgrad(g, p("dz"), p("w"), p("g_out"), p("ws"), _lib.ALGO_SIMT, st)
        if c.op == "wgrad":
            return lib.b200gan_nb_wgrad(g, self.bn(), p("x"), p("dz"), p("dw"), p("ws"), st)
        if c.op == "dz":
            return lib.b200gan_nb_dz(c.N, c.H * c.W, c.K, p("g"), p("a"), p("cs"), ACT_CODE[c.act], SLOPE, self.bn(),
                                     p("sums"), p("dz"), p("db"), st)
        if c.op == "tail_fwd":
            return lib.b200gan_nb_tail_fwd(c.N, c.H * c.W, c.C, self.bn(), p("running_mean"), p("running_var"),
                                           p("nbt"), MOMENTUM, p("a"), p("out"), c.nchw, st)
        return lib.b200gan_nb_tail_bwd(c.N, c.H * c.W, c.C, self.bn(), p("a"), p("dout"), c.nchw, p("g"), p("sums"), st)

    def outputs(self):
        return {k: v.clone() for k, v in self.arena.t.items() if self.arena.layout[k][3] != "in" or k == "nbt"}

    # -- reference -----------------------------------------------------------------------------------------------
    def consts(self):
        """fp64 BatchNorm constants [G][C] and the bound of the fp32 scale / shift the kernel forms from them"""
        c, C = self.c, self.Cb
        if not self.has_bn:
            one = torch.ones(self.G, C, dtype=torch.float64, device="cuda")
            return None, None, None, one, one * 0, one * 0, one * 0
        mean, var, rstd, sc, sh = bn_consts(self.stats.cuda(), self.gamma.cuda() if self.affine else None,
                                            self.beta.cuda() if self.affine else None, self.count, self.G, C)
        be = self.beta.cuda().double() if self.affine else torch.zeros_like(sc[0])
        esc = 3 * U * sc.abs()
        esh = 2 * U * be.abs() + 6 * U * (mean * sc).abs()
        return mean, var, rstd, sc, sh, esc, esh

    def staged_x(self):
        """x = BN(a) in fp64 and the bound of the staged fp32 fmaf(a, scale, shift)"""
        mean, var, rstd, sc, sh, esc, esh = self.consts()
        N, C = self.c.N, self.Cb
        a = self.a.double().reshape(N, -1, 1, C)   # tail_*: [N][HW][C]
        x = a * per_image(sc, N) + per_image(sh, N)
        e = a.abs() * per_image(esc, N) + per_image(esh, N) + U * x.abs() if self.has_bn else torch.zeros_like(x)
        return x.reshape(self.a.shape), e.reshape(self.a.shape)

    def check(self, outs, what):
        return getattr(self, "_check_" + self.c.op)(outs, what)

    def _check_running(self, outs, what):
        """running statistics and num_batches_tracked; the worst |err|/bound"""
        if not self.running:
            return 0.0
        mean, var, rstd, *_ = self.consts()
        rm, rv = running_ref(self.rm0.cuda(), self.rv0.cuda(), mean, var, self.count)
        unb = var * self.count / (self.count - 1)
        worst = check(what + " running_mean", outs["running_mean"], rm,
                      8 * U * (self.rm0.cuda().double().abs() + mean.abs().sum(0)) + 1e-30)
        worst = max(worst, check(what + " running_var", outs["running_var"], rv,
                                 8 * U * (self.rv0.cuda().double().abs() + unb.abs().sum(0)) + 1e-30))
        assert outs["nbt"].item() == NBT0 + self.G, f"{what}: num_batches_tracked {outs['nbt'].item()}"
        return worst

    def _check_fprop(self, outs, what):
        c = self.c
        x, e = self.staged_x()
        w = self.w.double()
        n = c.R * c.R * c.C
        conv = conv_fwd(x, w, c.stride, 1)
        bound = U * (n + 4) * conv_fwd(x.abs(), w.abs(), c.stride, 1) + conv_fwd(e, w.abs(), c.stride, 1)
        b = self.bias.double()
        pre = conv + b
        bound = bound + U * (pre.abs() + b.abs())
        y = act_out64(c.act, pre)
        bound = act_bound(c.act, pre, y, bound)
        if c.cs:
            s = self.cs.double().view(c.N, 1, 1, c.K)
            y = y * s
            bound = bound * s.abs() + U * y.abs()
        worst = check(what + " y", outs["y"], y, bound)
        if c.out_stats:
            yk = outs["y"].double().view(self.G, -1, c.K)
            ref = torch.stack([yk.sum(1), (yk * yk).sum(1)], 1)
            bnd = U * (BLOCK_PARTIAL + 8) * torch.stack([yk.abs().sum(1), (yk * yk).sum(1)], 1)
            worst = max(worst, check_sums(what + " out_stats", outs["out_stats"], ref, bnd + 1e-300))
        return max(worst, self._check_running(outs, what))

    def _check_dgrad(self, outs, what):
        c = self.c
        w, dz = self.w.double(), self.dz_in.double()
        shape = (c.N, c.H, c.W, c.C)
        ref = conv_dgrad(dz, w, shape, c.stride, 1)
        bound = U * (c.R * c.R * c.K + 4) * conv_dgrad(dz.abs(), w.abs(), shape, c.stride, 1)
        worst = check(what + " g_out", outs["g_out"], ref, bound)
        if c.op == "dgrad" and c.sums:
            mean, var, rstd, *_ = self.consts()
            a = self.a.double()
            gk = outs["g_out"].double().reshape(a.shape)
            ah = (a - per_image(mean, c.N)) * per_image(rstd, c.N)
            eah = 3 * U * (a.abs() + per_image(mean.abs(), c.N)) * per_image(rstd, c.N) + 2 * U * ah.abs()
            G, C = self.G, c.C
            grp = lambda t: t.reshape(G, -1, C).sum(1)
            ref = torch.stack([grp(gk), grp(gk * ah)], 1)
            bnd = torch.stack([U * (BLOCK_PARTIAL + 8) * grp(gk.abs()),
                               U * (BLOCK_PARTIAL + 8) * grp((gk * ah).abs()) + grp(gk.abs() * eah)], 1)
            worst = max(worst, check_sums(what + " sums", outs["sums"], ref, bnd + 1e-300))
        return worst

    _check_plain_dgrad = _check_dgrad

    def _check_wgrad(self, outs, what):
        c = self.c
        x, e = self.staged_x()
        dz = self.dz_in.double()
        shape = (c.K, c.C, c.R, c.R)
        ref = conv_wgrad(x, dz, shape, c.stride, 1)
        n = c.N * c.P * c.Q
        bound = U * (n + c.s + 4) * conv_wgrad(x.abs(), dz.abs(), shape, c.stride, 1) + \
            conv_wgrad(e, dz.abs(), shape, c.stride, 1)
        if self.unused_ws:
            assert torch.isnan(outs["ws"]).all(), f"{what}: a workspace the plan does not use was written"
        return check(what + " dw", outs["dw"], ref, bound)

    def _check_dz(self, outs, what):
        c = self.c
        N, K = c.N, c.K
        a, G_ = self.a.double(), self.grad_in.double()
        cs = self.cs.double().view(N, 1, 1, K) if c.cs else torch.ones(N, 1, 1, K, dtype=torch.float64, device="cuda")
        if self.has_bn:
            mean, var, rstd, sc, sh, esc, esh = self.consts()
            sums = self.sums_in.cuda()
            ref = bn_bwd_ref(G_, a, mean, rstd, sc, sums, self.count, cs, c.act)
            m1, m2 = sums[:, 0] / self.count, sums[:, 1] / self.count
            T = G_.abs() + per_image(m1.abs(), N) + \
                (a.abs() + per_image(mean.abs(), N)) * per_image(rstd, N) * per_image(m2.abs(), N)
            bound = 8 * U * per_image(sc.abs(), N) * T * cs.abs() * act_grad(c.act, a) + 2 * U * ref.abs()
        else:
            ref = G_ * cs * act_grad(c.act, a)
            bound = 2 * U * ref.abs()
        worst = check(what + " dz", outs["dz"], ref, bound)
        if c.db:
            rows = N * c.H * c.W
            worst = max(worst, check(what + " db", outs["db"], ref.sum((0, 1, 2)),
                                     bound.sum((0, 1, 2)) + U * (rows + 16) * ref.abs().sum((0, 1, 2))))
        return worst

    def _check_tail_fwd(self, outs, what):
        c = self.c
        x, e = self.staged_x()
        out = x.permute(0, 2, 1) if c.nchw else x
        bnd = e.permute(0, 2, 1) if c.nchw else e
        worst = check(what + " out", outs["out"], out, bnd)
        return max(worst, self._check_running(outs, what))

    def _check_tail_bwd(self, outs, what):
        c = self.c
        got, want = outs["g"].view(torch.int32), self.grad_in.contiguous().view(-1).view(torch.int32)
        bad = (got != want).nonzero()
        assert bad.numel() == 0, f"{what}: g is not dout re-laid out bit for bit (first difference at {bad[0].item()})"
        mean, var, rstd, *_ = self.consts()
        a, g = self.a.double(), self.grad_in.double()
        N, G, C = c.N, self.G, c.C
        ah = (a - mean.repeat_interleave(N // G, 0)[:, None, :]) * rstd.repeat_interleave(N // G, 0)[:, None, :]
        eah = 3 * U * (a.abs() + mean.abs().repeat_interleave(N // G, 0)[:, None, :]) * \
            rstd.repeat_interleave(N // G, 0)[:, None, :] + 2 * U * ah.abs()
        grp = lambda t: t.reshape(G, -1, C).sum(1)
        m = math.ceil(N // G * c.H * c.W * C / 256) + 256
        ref = torch.stack([grp(g), grp(g * ah)], 1)
        bnd = torch.stack([U * m * grp(g.abs()), U * m * grp((g * ah).abs()) + grp(g.abs() * eah)], 1)
        # g is compared bit for bit above: the sums are the only bounded output
        return check_sums(what + " sums", outs["sums"], ref, bnd + 1e-300)


# ---- generator tail runs -------------------------------------------------------------------------------------------
class TailRun:
    def __init__(self, c, seed=0):
        self.c = c
        lib = self.lib = _lib.load()
        gen = torch.Generator().manual_seed(seed)
        N, H, W, C, K = c.N, c.H, c.W, c.C, c.K
        self.d = _lib.TailDesc(N, H, W, C, K, ACT_CODE[c.act_mid], SLOPE, ACT_CODE[c.act_out])
        a = torch.randn(N, H, W, C, generator=gen) * 1.5 + 0.3
        a64 = a.double().reshape(-1, C)
        mean, var = a64.mean(0), a64.var(0, unbiased=False)
        rstd = 1 / torch.sqrt(var + 1e-5)
        gamma, beta = 1 + 0.3 * torch.randn(C, generator=gen).double(), 0.3 * torch.randn(C, generator=gen).double()
        sc = gamma * rstd
        self.a = a.cuda()
        self.mr = torch.cat([mean, rstd]).float().cuda()
        self.ss = torch.cat([sc, beta - mean * sc]).float().cuda()
        self.w = (torch.randn(K, C, 3, 3, generator=gen) / math.sqrt(9 * C)).cuda()
        self.bias = (0.5 * torch.randn(K, generator=gen)).cuda() if c.bias else None
        self.g = torch.randn(N, H, W, K, generator=gen).cuda()
        f32 = torch.float32
        specs = [("a", a.numel(), f32, "in"), ("mr", 2 * C, f32, "in"), ("ss", 2 * C, f32, "in"),
                 ("w", self.w.numel(), f32, "in"), ("g", self.g.numel(), f32, "in"),
                 ("out", N * H * W * K, f32, "out"), ("da", a.numel(), f32, "out"), ("dw", K * C * 9, f32, "out")]
        if c.bias:
            specs.append(("bias", K, f32, "in"))
        if c.dgb:
            specs.append(("dgb", 2 * C, f32, "out"))
        if c.db:
            specs.append(("db", K, f32, "out"))
        nws = lib.b200gan_tail_bwd_workspace_bytes(ctypes.byref(self.d))
        specs.append(("ws", -(-nws // 4), f32, "ws"))
        self.arena = Arena(specs)
        self.data = dict(a=self.a, mr=self.mr, ss=self.ss, w=self.w, g=self.g, bias=self.bias)

    def prepare(self):
        self.arena.prepare(self.data)

    def call(self, st):
        lib, p, d, c = self.lib, self.arena.ptr, ctypes.byref(self.d), self.c
        rc = lib.b200gan_tail_fprop(d, p("a"), p("ss"), p("w"), p("bias"), p("out"), st)
        if rc and not c.error:
            return rc
        rb = lib.b200gan_tail_bwd(d, p("a"), p("mr"), p("ss"), p("w"), p("g"), p("ws"), p("da"), p("dgb"), p("dw"),
                                  p("db"), int(c.rtf), st)
        if c.error:   # a refusal case: both entry points must refuse (the backward's code if both do, else 0)
            return rb if rc and rb else 0
        return rb

    def outputs(self):
        return {k: v.clone() for k, v in self.arena.t.items() if self.arena.layout[k][3] != "in"}

    def check(self, outs, what):
        c = self.c
        C, K = c.C, c.K
        # forward
        out, pre, A, b = tail_fwd_ref(self.a, self.ss, self.w, self.bias, c.act_mid, c.act_out)
        bound = 2.0 ** -22 * (math.ceil(9 * C / 8) + 9 + 4) * A
        bound = bound + U * (pre.abs() + b.abs())
        worst = check(what + " out", outs["out"], out, act_bound(c.act_out, pre, out, bound))
        # backward: both branches of the activation's derivative where the pre-activation is within ulps of 0
        a64 = self.a.double()
        pre64 = a64 * self.ss[:C].double() + self.ss[C:].double()
        near0 = pre64.abs() <= 4 * U * ((a64 * self.ss[:C].double()).abs() + self.ss[C:].double().abs())
        r = tail_bwd_ref(self.a, self.mr, self.ss, self.w, self.g, c.act_mid, pre64 <= 0)
        ra = tail_bwd_ref(self.a, self.mr, self.ss, self.w, self.g, c.act_mid, pre64 > 0) if near0.any() else None
        total = c.N * c.H * c.W
        m = math.ceil(total / 100) + 300      # pixels of one block's range (>= 100 SMs) + the in-block reductions
        neg = NEG_SLOPE[c.act_mid]
        gk = self.g.double()
        A_dy = conv_dgrad(gk.abs(), self.w.double().abs(), self.a.shape, 1, 1)
        bdz = U * (9 * K + 4) * A_dy * torch.where(pre64 > 0, 1.0, neg).double()
        dz, xh = r["dz"], r["xh"]
        mean, rstd = self.mr[:C].double(), self.mr[C:].double()
        exh = 2 * U * (a64.abs() + mean.abs()) * rstd
        flip = (ra["dz"] - dz).abs() * near0 if ra is not None else torch.zeros_like(dz)
        S = lambda t: t.sum((0, 1, 2))
        bs1 = U * m * S(dz.abs()) + S(bdz) + S(flip)
        bs2 = U * m * S((dz * xh).abs()) + S(bdz * xh.abs() + dz.abs() * exh) + S(flip * xh.abs())
        if c.dgb:
            worst = max(worst, check(what + " dgamma", outs["dgb"][:C], r["s2"], bs2 + U * r["s2"].abs()))
            worst = max(worst, check(what + " dbeta", outs["dgb"][C:], r["s1"], bs1 + U * r["s1"].abs()))
        sc = self.ss[:C].double()
        m1, m2 = r["s1"] / total, r["s2"] / total
        bda = sc.abs() * (bdz + bs1 / total + exh * m2.abs() + xh.abs() * bs2 / total +
                          4 * U * (dz.abs() + m1.abs() + (xh * m2).abs())) + U * r["da"].abs()
        if c.rtf:
            bda = bda + 2.0 ** -11 * (r["da"].abs() + bda)
        alt = torch.where(near0, ra["da"], torch.full_like(r["da"], float("nan"))) if ra is not None else None
        worst = max(worst, check(what + " da", outs["da"], r["da"], bda, alt))
        if c.rtf:
            assert ((outs["da"].view(torch.int32) & 0x1FFF) == 0).all(), f"{what}: round_tf32 da not TF32-representable"
        shape = (K, C, 3, 3)
        y_flip = (ra["y"] - r["y"]).abs() * near0 if ra is not None else torch.zeros_like(r["y"])
        bdw = U * (m + 4) * conv_wgrad(r["y"].abs(), gk.abs(), shape, 1, 1) + \
            conv_wgrad(U * r["pre"].abs() + y_flip, gk.abs(), shape, 1, 1)
        worst = max(worst, check(what + " dw", outs["dw"], r["dw"], bdw))
        if c.db:
            worst = max(worst, check(what + " db", outs["db"], r["db"], U * (m + 4) * S(gk.abs())))
        return worst


# ---- the per-case test ---------------------------------------------------------------------------------------------
def check_route(run, kernels, grid):
    """the family's kernels of one call, in launch order, and the first one's grid on a 132-SM device"""
    c = run.c
    marker = torch.zeros(1, device="cuda")
    names, seen = [], []
    # the first launch of a profiler session can lose its kernel record (see test_gpu_norm_conformance.check_route):
    # a marker goes first; a record lost anyway does not repeat, a route that differs from the table does
    for _ in range(3):
        run.prepare()
        seen = [(n, g) for n, g in traced_kernels(lambda: (marker.zero_(), run.call(
            torch.cuda.current_stream().cuda_stream))) if n.startswith(("nbk_", "tail_"))]
        names = [n for n, _ in seen]
        if names == list(kernels):
            break
    if not seen:
        return "the profiler recorded no CUDA kernel activity on this machine"
    assert names == list(kernels), f"{c.id}: trace {names}, table {list(kernels)}"
    if grid is not None and torch.cuda.get_device_properties(0).multi_processor_count == ch.NUM_SMS:
        assert tuple(seen[0][1]) == tuple(grid), f"{c.id}: {names[0]} grid {seen[0][1]}, table {grid}"
    return None


# fp64 sums and fp32 atomics (tail.cu's backward: sums -> da, dgamma_dbeta; dw, db), running statistics from them;
# a chain wgrad's dw repeats only with the slab workspace
ALWAYS_VARIES = {"out_stats", "sums", "db", "ws", "dgb", "running_mean", "running_var", "nbt"}
MAY_VARY = {"dw", "da"}


def run_case(run, kernels, grid, deterministic, bad_rc):
    c = run.c
    lib = run.lib
    run.prepare()
    before = run.outputs()
    rc = run.call(torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    if c.error:
        assert rc in bad_rc, f"{c.id}: expected a refusal, rc = {rc}"
        run.arena.check_guards(c.id)
        after = run.outputs()
        for k, v in before.items():
            same = (v.view(torch.uint8) == after[k].view(torch.uint8)).all()
            assert same, f"{c.id}: refused call wrote {k}"
        return
    assert rc == 0, f"{c.id}: rc {rc}: {lib.b200gan_last_error().decode()}"
    run.arena.check_guards(c.id)
    eager = run.outputs()
    worst = run.check(eager, c.id + " eager")

    skip_reason = check_route(run, kernels, grid)

    # CUDA graph on a side stream, replayed once
    side = torch.cuda.Stream()
    run.prepare()
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=side):
        rc = run.call(side.cuda_stream)
    assert rc == 0, f"{c.id}: rc {rc} under capture: {lib.b200gan_last_error().decode()}"
    run.prepare()
    torch.cuda.synchronize()
    graph.replay()
    torch.cuda.synchronize()
    run.arena.check_guards(c.id + " graph")
    replay = run.outputs()
    for k, v in replay.items():
        if k in ALWAYS_VARIES or (k in MAY_VARY and not deterministic):
            continue
        same = v.view(torch.uint8) == eager[k].view(torch.uint8)
        assert same.all(), f"{c.id}: graph replay differs from the eager call in {k} (marked deterministic)"
    worst = max(worst, run.check(replay, c.id + " graph"))
    print(f"\n{c.id}: worst |err|/bound {worst:.3g}, kernels {list(kernels)}")
    if skip_reason:
        pytest.skip(skip_reason)


@pytest.mark.parametrize("case", ch.CASES, ids=lambda c: c.id)
def test_chain_case(case):
    run_case(ChainRun(case), case.kernels, case.grid, case.deterministic, (-2,))


@pytest.mark.parametrize("case", tl.CASES, ids=lambda c: c.id)
def test_tail_case(case):
    run_case(TailRun(case), case.kernels, None, False, (-1, -2))
