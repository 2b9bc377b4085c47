"""Every case of tests/chain_cases.py and tests/tail_cases.py, element by element against torch float64.

Each case calls the C ABI directly on the guarded buffers of tests/conformance.py (Arena) and runs its protocol: inputs
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

import chain_cases as ch
import tail_cases as tl
from b200gan import _lib
from chain_cases import (ACT_CODE, BLOCK_PARTIAL, BN_EPS, MOMENTUM, NBT0, NEG_SLOPE, SLOPE, U, act_bound, act_grad,
                         act_out64, bn_bwd_ref, bn_consts, chain_geom, conv_dgrad, conv_fwd, conv_wgrad, group_sums,
                         per_image, running_ref)
from conformance import Arena, check_elementwise, first_grid, run_case
from tail_cases import tail_bwd_ref, tail_fwd_ref

pytestmark = pytest.mark.gpu


# ---- checks ---------------------------------------------------------------------------------------------------------
def check_sums(what, got, ref, bound):
    return check_elementwise(what + " (an OVERWRITTEN buffer: accumulating onto its old contents fails)", got, ref, bound)


# ---- chain runs ------------------------------------------------------------------------------------------------------
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

    def check(self, what):
        return getattr(self, "_check_" + self.c.op)(self.outputs(), what)

    def _check_running(self, outs, what):
        """running statistics and num_batches_tracked; the worst |err|/bound"""
        if not self.running:
            return 0.0
        mean, var, rstd, *_ = self.consts()
        rm, rv = running_ref(self.rm0.cuda(), self.rv0.cuda(), mean, var, self.count)
        unb = var * self.count / (self.count - 1)
        worst = check_elementwise(what + " running_mean", outs["running_mean"], rm,
                      8 * U * (self.rm0.cuda().double().abs() + mean.abs().sum(0)) + 1e-30)
        worst = max(worst, check_elementwise(what + " running_var", outs["running_var"], rv,
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
        worst = check_elementwise(what + " y", outs["y"], y, bound)
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
        worst = check_elementwise(what + " g_out", outs["g_out"], ref, bound)
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
        return check_elementwise(what + " dw", outs["dw"], ref, bound)

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
        worst = check_elementwise(what + " dz", outs["dz"], ref, bound)
        if c.db:
            rows = N * c.H * c.W
            worst = max(worst, check_elementwise(what + " db", outs["db"], ref.sum((0, 1, 2)),
                                     bound.sum((0, 1, 2)) + U * (rows + 16) * ref.abs().sum((0, 1, 2))))
        return worst

    def _check_tail_fwd(self, outs, what):
        c = self.c
        x, e = self.staged_x()
        out = x.permute(0, 2, 1) if c.nchw else x
        bnd = e.permute(0, 2, 1) if c.nchw else e
        worst = check_elementwise(what + " out", outs["out"], out, bnd)
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
        return self.arena.outputs()

    def check(self, what):
        outs = self.outputs()
        c = self.c
        C, K = c.C, c.K
        # forward
        out, pre, A, b = tail_fwd_ref(self.a, self.ss, self.w, self.bias, c.act_mid, c.act_out)
        bound = 2.0 ** -22 * (math.ceil(9 * C / 8) + 9 + 4) * A
        bound = bound + U * (pre.abs() + b.abs())
        worst = check_elementwise(what + " out", outs["out"], out, act_bound(c.act_out, pre, out, bound))
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
            worst = max(worst, check_elementwise(what + " dgamma", outs["dgb"][:C], r["s2"], bs2 + U * r["s2"].abs()))
            worst = max(worst, check_elementwise(what + " dbeta", outs["dgb"][C:], r["s1"], bs1 + U * r["s1"].abs()))
        sc = self.ss[:C].double()
        m1, m2 = r["s1"] / total, r["s2"] / total
        bda = sc.abs() * (bdz + bs1 / total + exh * m2.abs() + xh.abs() * bs2 / total +
                          4 * U * (dz.abs() + m1.abs() + (xh * m2).abs())) + U * r["da"].abs()
        if c.rtf:
            bda = bda + 2.0 ** -11 * (r["da"].abs() + bda)
        alt = torch.where(near0, ra["da"], torch.full_like(r["da"], float("nan"))) if ra is not None else None
        worst = max(worst, check_elementwise(what + " da", outs["da"], r["da"], bda, alt=alt))
        if c.rtf:
            assert ((outs["da"].view(torch.int32) & 0x1FFF) == 0).all(), f"{what}: round_tf32 da not TF32-representable"
        shape = (K, C, 3, 3)
        y_flip = (ra["y"] - r["y"]).abs() * near0 if ra is not None else torch.zeros_like(r["y"])
        bdw = U * (m + 4) * conv_wgrad(r["y"].abs(), gk.abs(), shape, 1, 1) + \
            conv_wgrad(U * r["pre"].abs() + y_flip, gk.abs(), shape, 1, 1)
        worst = max(worst, check_elementwise(what + " dw", outs["dw"], r["dw"], bdw))
        if c.db:
            worst = max(worst, check_elementwise(what + " db", outs["db"], r["db"], U * (m + 4) * S(gk.abs())))
        return worst


# ---- the per-case test ---------------------------------------------------------------------------------------------
# fp64 sums and fp32 atomics (tail.cu's backward: sums -> da, dgamma_dbeta; dw, db), running statistics from them;
# a chain wgrad's dw repeats only with the slab workspace
ALWAYS_VARIES = ("out_stats", "sums", "db", "ws", "dgb", "running_mean", "running_var", "nbt")
MAY_VARY = ("dw", "da")
FAMILY = ("nbk_", "tail_")


@pytest.mark.parametrize("case", ch.CASES, ids=lambda c: c.id)
def test_chain_case(case):
    run_case(ChainRun(case), case.id, first_grid(case.kernels, case.grid), refuse=(-2,) if case.error else (),
             varies=ALWAYS_VARIES + (() if case.deterministic else MAY_VARY), family=FAMILY, num_sms=ch.NUM_SMS)


@pytest.mark.parametrize("case", tl.CASES, ids=lambda c: c.id)
def test_tail_case(case):
    run_case(TailRun(case), case.id, first_grid(case.kernels, None), refuse=(-1, -2) if case.error else (),
             varies=ALWAYS_VARIES + MAY_VARY, family=FAMILY)
