"""Every case of tests/stream_cases.py (head.cu and index_ops.cu), element by element against torch float64.

Each case calls the C ABI on the guarded buffers of tests/conformance.py (Arena) and runs its protocol: inputs between
NaN guards, outputs started as NaN, sentinels around everything the library writes.  Adam's p, m and v are read and
written in place: they get the Arena's "io" role (their data, and sentinel guards); its step buffer starts at
(step0, 0) and must come back as (step0 + 1, 0).

Checks:
  - bit for bit: transpose, upsample forward, pad forward (also with round_tf32, against tf32_rna), the activation and
    the epilogue backward for none / LeakyReLU / ReLU, restated in fp32 with the kernel's operation order;
  - everything else against fp64 with a bound from the arithmetic, 2^-23 (n + s + 4) A as in the conv suite: A the
    same sum over |terms|, n the length of the kernel's longest fp32 chain and s the partials added outside it;
    tanh / sigmoid carried through with chain_cases.act_bound; Adam's bound counts its roundings per step;
  - the traced kernels, launch count and grids of the table;
  - a CUDA-graph replay, bit for bit but for the epilogue's atomically summed db;
  - refusals: the error code, untouched outputs, intact guards.
"""
import math

import pytest
import torch

import stream_cases as sc
from b200gan import _lib
from chain_cases import act_bound
from conformance import Arena, bits_equal, check_elementwise, not_vacuous, run_case, tf32_rna
from stream_cases import (ADAM, F32, SLOPE, U, act32_exact, act64, adam_ref, bce_grad_ref, bce_ref, grad32_exact, pad_grad_ref,
                          pad_ref, upsample_grad_ref, upsample_ref)

pytestmark = pytest.mark.gpu

ACT_CODE = {"none": _lib.ACT_NONE, "lrelu": _lib.ACT_LRELU, "relu": _lib.ACT_RELU, "tanh": _lib.ACT_TANH,
            "sigmoid": _lib.ACT_SIGMOID}


# ---- runs ------------------------------------------------------------------------------------------------------------
class Run:
    def __init__(self, c, seed=0):
        self.c, self.lib = c, _lib.load()
        self.gen = torch.Generator().manual_seed(seed)
        self.off = {}                     # name -> leading floats in front of the operand (misaligned pointers)
        specs, self.data = getattr(self, "setup_" + c.op)(c.dims, c.opt)
        self.arena = Arena(specs)

    # data helpers
    def randn(self, *s, scale=1.0):
        return (torch.randn(*s, generator=self.gen) * scale).cuda()

    def rand(self, *s):
        return torch.rand(*s, generator=self.gen).cuda()

    def add(self, specs, name, n, role, value=None, off=0):
        specs.append((name, n + off, F32, role))
        if off:
            self.off[name] = off
        if value is not None:
            lead = torch.full((off,), float("nan"), device="cuda")
            self.data[name] = torch.cat([lead, value.reshape(-1).float()])

    def p(self, name):
        if name not in self.arena.t:
            return None
        return self.arena.ptr(name) + 4 * self.off.get(name, 0)

    def t(self, name):
        return self.arena.t[name][self.off.get(name, 0):]

    def prepare(self):
        self.arena.prepare(self.data)

    def outputs(self):
        return self.arena.outputs()

    # ---- head.cu
    def setup_linear1(self, d, o):
        N, K = d
        specs, self.data = [], {}
        self.x, self.w = self.randn(N, K), self.randn(K, scale=1 / math.sqrt(K))
        self.b = self.randn(1) if o.get("b", True) else None
        self.dy = self.randn(N)
        if o.get("sparse"):   # every 64th row and the last: a 4096-term chain with 65 roundings
            rows = torch.arange(N, device="cuda")
            self.dy = torch.where((rows % 64 == 0) | (rows == N - 1), self.dy, torch.zeros_like(self.dy))
        self.add(specs, "x", N * K, "in", self.x, o.get("offset", 0))
        self.add(specs, "w", K, "in", self.w)
        if self.b is not None:
            self.add(specs, "b", 1, "in", self.b)
        self.add(specs, "dy", N, "in", self.dy)
        self.add(specs, "y", N, "out")
        if o.get("dx", True):
            self.add(specs, "dx", N * K, "out")
        self.add(specs, "dw", K, "out")
        if o.get("db", True):
            self.add(specs, "db", 1, "out")
        return specs, self.data

    def call_linear1(self, st):
        (N, K), a, p, L = self.c.dims, ACT_CODE[self.c.opt["act"]], self.p, self.lib
        if not self.c.error:
            rc = L.b200gan_linear1_fwd(p("x"), p("w"), p("b"), p("y"), N, K, a, st)
            if rc:
                return rc
        return L.b200gan_linear1_bwd(p("x"), p("w"), p("y"), p("dy"), p("dx"), p("dw"), p("db"), N, K, a, st)

    def check_linear1(self, what):
        (N, K), act = self.c.dims, self.c.opt["act"]
        x, w, dy = self.x.double(), self.w.double(), self.dy.double()
        b = self.b.double() if self.b is not None else torch.zeros(1, dtype=torch.float64, device="cuda")
        z = x @ w + b
        n = math.ceil(K / 128) + 4 + 9           # a thread's chain (float4: 4 products per step), 5 shuffles, 4 warps
        bound = U * (n + 1 + 4) * ((x.abs() @ w.abs()) + b.abs())
        y_ref = act64(act, z)
        worst = check_elementwise(what + " y", self.t("y"), y_ref, act_bound(act, z, y_ref, bound), "(n,)")
        not_vacuous(what + " y", bound, (x * w).abs())
        y = self.t("y").double()
        g = y * (1 - y) if act == "sigmoid" else torch.ones_like(y)
        dl = dy * g
        edl = 3 * U * dl.abs()
        nz = int((dl != 0).sum().item())          # fmaf(0, x, acc) == acc: zero terms do not round
        bdw = U * (nz + 4) * (x.abs().t() @ dl.abs()) + x.abs().t() @ edl
        worst = max(worst, check_elementwise(what + " dw", self.t("dw"), x.t() @ dl, bdw, "(k,)"))
        not_vacuous(what + " dw", bdw, (x * dl[:, None]).abs()[dl != 0])
        if "dx" in self.arena.t:
            dx = dl[:, None] * w[None, :]
            worst = max(worst, check_elementwise(what + " dx", self.t("dx"), dx, edl[:, None] * w.abs() + U * dx.abs(),
                                                 "(n, k)"))
        if "db" in self.arena.t:
            bdb = U * (math.ceil(N / 128) + 9 + 4) * dl.abs().sum() + edl.sum()
            worst = max(worst, check_elementwise(what + " db", self.t("db"), dl.sum().view(1), bdb.view(1), "()"))
        return worst

    def setup_bce(self, d, o):
        (n,) = d
        specs, self.data = [], {}
        v = 0.02 + 0.96 * self.rand(n)
        tv = o["t"]
        if tv == "mixed":
            t = torch.tensor([0.0, 1.0, 0.3], device="cuda")[torch.randint(0, 3, (n,), generator=self.gen).cuda()]
        else:
            t = torch.full((n,), float(tv), device="cuda")
        if o.get("edges"):
            v[0::4], v[1::4] = 0.0, 1.0
            t[:12] = torch.tensor([0.0, 0.0, 0, 0, 1, 1, 0, 0, 0.3, 0.3, 0, 0], device="cuda")
        self.v, self.tt, self.gout = v, t, torch.tensor([1.5], device="cuda")
        for name, val, role in (("v", v, "in"), ("t", t, "in"), ("gout", self.gout, "in")):
            self.add(specs, name, val.numel(), role, val)
        self.add(specs, "loss", 1, "out")
        self.add(specs, "dv", n, "out")
        return specs, self.data

    def call_bce(self, st):
        (n,), p, L = self.c.dims, self.p, self.lib
        return L.b200gan_bce_fwd(p("v"), p("t"), p("loss"), n, st) or \
            L.b200gan_bce_bwd(p("v"), p("t"), p("gout"), p("dv"), n, st)

    def check_bce(self, what):
        (n,) = self.c.dims
        loss, terms, lp, lq = bce_ref(self.v, self.tt)
        t = self.tt.double()
        # 128 thread chains of ceil(n / 128), 5 shuffles, 4 warps; 4 ulps per term from the logs and products; / n
        bound = (U * (math.ceil(n / 128) + 9 + 4) * terms.abs().sum() +
                 4 * U * ((t - 1).abs() * lq.abs() + t.abs() * lp.abs()).sum()) / n + U * loss.abs()
        worst = check_elementwise(what + " loss", self.t("loss"), loss.view(1), bound.view(1), "()")
        dv = bce_grad_ref(self.v, self.tt, self.gout.item())
        worst = max(worst, check_elementwise(what + " dv", self.t("dv"), dv, 8 * U * dv.abs(), "(i,)"))
        return worst

    # ---- index_ops.cu: data movement
    def setup_transpose(self, d, o):
        N, C, HW = d
        specs, self.data = [], {}
        self.x = self.randn(N * C * HW)
        self.add(specs, "x", N * C * HW, "in", self.x)
        self.add(specs, "y", N * C * HW, "out")
        return specs, self.data

    def call_transpose(self, st):
        (N, C, HW), p = self.c.dims, self.p
        f = self.lib.b200gan_nchw_to_nhwc if self.c.opt.get("to_nhwc", True) else self.lib.b200gan_nhwc_to_nchw
        return f(p("x"), p("y"), N, C, HW, st)

    def check_transpose(self, what):
        N, C, HW = self.c.dims
        src = self.x.view(N, C, HW) if self.c.opt.get("to_nhwc", True) else self.x.view(N, HW, C)
        bits_equal(what + " y", self.t("y"), src.transpose(1, 2))
        return 0.0

    def setup_upsample(self, d, o):
        N, H, W, C = d
        specs, self.data = [], {}
        self.x, self.dy = self.randn(N, H, W, C), self.randn(N, 2 * H, 2 * W, C)
        self.add(specs, "x", self.x.numel(), "in", self.x)
        self.add(specs, "dy", self.dy.numel(), "in", self.dy)
        self.add(specs, "y", self.dy.numel(), "out")
        self.add(specs, "dx", self.x.numel(), "out")
        return specs, self.data

    def call_upsample(self, st):
        (N, H, W, C), p, L = self.c.dims, self.p, self.lib
        return L.b200gan_upsample2x_fwd(p("x"), p("y"), N, H, W, C, st) or \
            L.b200gan_upsample2x_bwd(p("dy"), p("dx"), N, H, W, C, st)

    def check_upsample(self, what):
        bits_equal(what + " y", self.t("y"), upsample_ref(self.x))
        bound = U * (4 + 4) * upsample_grad_ref(self.dy.double().abs())
        worst = check_elementwise(what + " dx", self.t("dx"), upsample_grad_ref(self.dy.double()), bound, "(n,h,w,c)")
        not_vacuous(what + " dx", bound, self.dy.abs())
        return worst

    def setup_pad(self, d, o):
        N, H, W, C = d
        t, l, b, r = o["pads"]
        Ho, Wo = H + t + b, W + l + r
        specs, self.data = [], {}
        off = o.get("offset", 0)
        self.x, self.dy = self.randn(N, H, W, C), self.randn(N, Ho, Wo, C)
        self.add(specs, "x", self.x.numel(), "in", self.x, off)
        self.add(specs, "dy", self.dy.numel(), "in", self.dy, off)
        self.add(specs, "y", self.dy.numel(), "out", None, off)
        self.add(specs, "dx", self.x.numel(), "out", None, off)
        return specs, self.data

    def call_pad(self, st):
        (N, H, W, C), o, p, L = self.c.dims, self.c.opt, self.p, self.lib
        mode = _lib.PAD_REFLECT if o["mode"] == "reflect" else _lib.PAD_ZERO
        rc = L.b200gan_pad2d_fwd(p("x"), p("y"), N, H, W, C, *o["pads"], mode, int(o.get("rtf", False)), st)
        rb = L.b200gan_pad2d_bwd(p("dy"), p("dx"), N, H, W, C, *o["pads"], mode, st)
        if self.c.error:    # both entry points must refuse
            return rb if rc and rb else 0
        return rc or rb

    def check_pad(self, what):
        o = self.c.opt
        y = pad_ref(self.x, o["pads"], o["mode"])
        bits_equal(what + " y", self.t("y"), tf32_rna(y) if o.get("rtf") else y)
        if o.get("rtf"):
            assert ((self.t("y").view(torch.int32) & 0x1FFF) == 0).all(), f"{what}: round_tf32 y not TF32-representable"
        ref = pad_grad_ref(self.dy.double(), self.x.shape, o["pads"], o["mode"])
        bound = U * (9 + 4) * pad_grad_ref(self.dy.double().abs(), self.x.shape, o["pads"], o["mode"])
        worst = check_elementwise(what + " dx", self.t("dx"), ref, bound, "(n,h,w,c)")
        not_vacuous(what + " dx", bound, self.dy.abs())
        for name in ("y", "dx"):   # the float in front of a misaligned output is never written
            lead = self.arena.t[name][:self.off.get(name, 0)]
            assert torch.isnan(lead).all(), f"{what}: {name} written in front of its start"
        return worst

    # ---- index_ops.cu: activation, epilogue backward, bias gradient
    def setup_act(self, d, o):
        N, HW, C = d
        specs, self.data = [], {}
        self.x = self.randn(N, HW, C, scale=2.0)
        mk = o["mask"]
        self.mask = None
        if mk != "none":
            shape = (N, HW, C) if mk == "elem" else (N, 1, C)
            self.mask = torch.where(self.rand(*shape) < 0.3, 0.0, 1.25)
        self.add(specs, "x", self.x.numel(), "in", self.x)
        if self.mask is not None:
            self.add(specs, "mask", self.mask.numel(), "in", self.mask)
        self.add(specs, "y", self.x.numel(), "out")
        return specs, self.data

    def call_act(self, st):
        (N, HW, C), o, p = self.c.dims, self.c.opt, self.p
        return self.lib.b200gan_act_fwd(p("x"), p("mask"), int(o["mask"] == "chan"), ACT_CODE[o["act"]], SLOPE,
                                        N * HW * C, C, HW, p("y"), st)

    def check_act(self, what):
        act = self.c.opt["act"]
        mask = self.mask if self.mask is not None else torch.ones(1, device="cuda")
        if act in ("none", "lrelu", "relu"):
            bits_equal(what + " y", self.t("y"), act32_exact(act, self.x) * mask)
            return 0.0
        x = self.x.double()
        a = act64(act, x)
        y = a * mask.double()
        bound = act_bound(act, x, a, torch.zeros_like(x)) * mask.double().abs() + U * y.abs()
        return check_elementwise(what + " y", self.t("y"), y, bound, "(n, hw, c)")

    def setup_epilogue(self, d, o):
        N, PQ, K = d
        specs, self.data = [], {}
        act = o["act"]
        self.dy = self.randn(N, PQ, K)
        self.cs = torch.where(self.rand(N, 1, K) < 0.25, 0.0, 1.25) if o.get("cs") else None
        z = self.randn(N, PQ, K, scale=1.5)
        a = act64(act, z.double()).float()
        self.y = a * self.cs if self.cs is not None else a
        self.add(specs, "dy", self.dy.numel(), "in", self.dy)
        if act != "none":
            self.add(specs, "y", self.y.numel(), "in", self.y)
        if self.cs is not None:
            self.add(specs, "cs", self.cs.numel(), "in", self.cs)
        self.add(specs, "dz", self.dy.numel(), "out")
        self.add(specs, "db", K, "out")
        return specs, self.data

    def call_epilogue(self, st):
        (N, PQ, K), o, p, L = self.c.dims, self.c.opt, self.p, self.lib
        a = ACT_CODE[o["act"]]
        return L.b200gan_epilogue_bwd(p("dy"), p("y"), p("cs"), a, SLOPE, N * PQ * K, K, PQ, int(o.get("rtf", False)),
                                      p("dz"), st) or \
            L.b200gan_bias_grad(p("dy"), p("y"), p("cs"), a, SLOPE, N * PQ, K, PQ, p("db"), st)

    def check_epilogue(self, what):
        (N, PQ, K), o = self.c.dims, self.c.opt
        act, rtf = o["act"], o.get("rtf", False)
        worst = 0.0
        d32 = self.dy * self.cs if self.cs is not None else self.dy
        if act in ("none", "lrelu", "relu"):
            dz32 = d32 * grad32_exact(act, self.y)
            bits_equal(what + " dz", self.t("dz"), tf32_rna(dz32) if rtf else dz32)
            term, eterm = dz32.double(), U * dz32.double().abs()     # the product d * act' rounded once
        else:
            yv = self.y
            if self.cs is not None:
                yv = torch.where(self.cs != 0, self.y / self.cs, torch.zeros_like(self.y))
            yv = yv.double()
            g = 1 - yv * yv if act == "tanh" else yv * (1 - yv)
            term = d32.double() * g
            # act' from y: two roundings of at most |yv| (1 + |yv|), the product one more
            eterm = 3 * U * d32.double().abs() * (g.abs() + yv.abs() * (1 + yv.abs()))
            bound = eterm + (2.0 ** -11 * (term.abs() + eterm) if rtf else 0)
            worst = check_elementwise(what + " dz", self.t("dz"), term, bound, "(n, pq, k)")
        if rtf:
            assert ((self.t("dz").view(torch.int32) & 0x1FFF) == 0).all(), f"{what}: round_tf32 dz not TF32-representable"
        (gx, gy, _), rpb = sc.bias_grad_grid(N * PQ, K)
        n = math.ceil(rpb / 8) + 8 + gy            # a thread's rows, the 8 shared partials, the yb atomics
        rows = term.reshape(-1, K)
        bdb = U * (n + 4) * rows.abs().sum(0) + eterm.reshape(-1, K).sum(0)
        worst = max(worst, check_elementwise(what + " db", self.t("db"), rows.sum(0), bdb, "(k,)"))
        not_vacuous(what + " db", bdb, rows.abs())
        return worst

    # ---- index_ops.cu: Adam
    def setup_adam(self, d, o):
        specs, self.data = [], {}
        self.sizes = self.c.adam_sizes()
        self.st0 = float(o.get("step0", 0))
        for i, n in enumerate(self.sizes):
            self.add(specs, f"p{i}", n, "io", self.randn(n))
            self.add(specs, f"g{i}", n, "in", self.randn(n, scale=0.1 + i % 5))
            self.add(specs, f"m{i}", n, "io", self.randn(n, scale=0.1))
            self.add(specs, f"v{i}", n, "io", 0.01 * self.rand(n))
        self.add(specs, "step", 2, "io", torch.tensor([self.st0, 0.0], device="cuda"))
        return specs, self.data

    def call_adam(self, st):
        (count,), o, p = self.c.dims, self.c.opt, self.p
        table = (_lib.AdamTensor * max(len(self.sizes), 1))()
        bad_i, bad = o.get("bad", (-1, None))
        for i, n in enumerate(self.sizes):
            table[i].p, table[i].g, table[i].m, table[i].v, table[i].n = p(f"p{i}"), p(f"g{i}"), p(f"m{i}"), \
                p(f"v{i}"), n
            if i == bad_i:
                if bad == "n0":
                    table[i].n = 0
                else:
                    table[i].p = None
        return self.lib.b200gan_adam_multi(table, count, ADAM["lr"], ADAM["b1"], ADAM["b2"], ADAM["eps"],
                                           float(o.get("gscale", 1.0)), p("step"), st)

    def check_adam(self, what):
        o = self.c.opt
        step = self.t("step")
        assert step[0].item() == self.st0 + 1, f"{what}: step {step[0].item()} after one call from {self.st0}"
        assert step[1].view(torch.int32).item() == 0, f"{what}: the ticket step[1] is not back at 0"
        worst = 0.0
        for i, n in enumerate(self.sizes):
            d = self.data
            (p1, ep), (m1, em), (v1, ev) = adam_ref(d[f"p{i}"], d[f"g{i}"], d[f"m{i}"], d[f"v{i}"], self.st0,
                                                    o.get("gscale", 1.0))
            for name, ref, b in (("p", p1, ep), ("m", m1, em), ("v", v1, ev)):
                worst = max(worst, check_elementwise(f"{what} {name}{i}", self.t(f"{name}{i}"), ref, b, "(i,)"))
            not_vacuous(f"{what} p{i}", ep, (p1 - d[f"p{i}"].double()).abs())
        return worst

    def call(self, st):
        return getattr(self, "call_" + self.c.op)(st)

    def check(self, what):
        return getattr(self, "check_" + self.c.op)(what)


# ---- the per-case test ---------------------------------------------------------------------------------------------
FAMILY = tuple({k for c in sc.CASES for k in c.kernels})
VARIES = {"epilogue": ("db",)}


@pytest.mark.parametrize("case", sc.CASES, ids=lambda c: c.id)
def test_stream_case(case):
    run_case(Run(case), case.id, case.launches, refuse=(-2,) if case.error else (), varies=VARIES.get(case.op, ()),
             family=FAMILY, num_sms=sc.NUM_SMS)
