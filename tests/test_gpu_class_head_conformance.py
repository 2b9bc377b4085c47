"""Every case of tests/class_head_cases.py -- the class-head mode of linear1_{fwd,bwd}_kernel and the cross-entropy mode
of bce_{fwd,bwd}_kernel (csrc/head.cu) -- element by element against torch float64.

Each case calls the C ABI on the guarded buffers of tests/conformance.py (Arena) and runs its protocol: inputs between
NaN guards, outputs started as NaN, sentinels around everything the library writes.

Checks:
  - every output against fp64 with a bound from the arithmetic, 2^-23 (n + s) A as in the stream suite: A the same sum
    over |terms|, n the length of the kernel's longest fp32 chain and s the roundings outside it; the softmax carries
    the logits' bound through its derivative;
  - the traced kernels and grids of the table;
  - a CUDA-graph replay, bit for bit;
  - refusals: each entry point the case names returns B200GAN_E_BAD_ARG and writes nothing, the others accept the call.
The linear1 and BCE rows of the stream table, which share these kernels, run in tests/test_gpu_stream_conformance.py.
"""
import math

import pytest
import torch

import class_head_cases as hc
from b200gan import _lib
from class_head_cases import ce_grad_ref, ce_ref, head_grad_ref, head_ref
from conformance import Arena, check_elementwise, not_vacuous, run_case

pytestmark = pytest.mark.gpu

U = 2.0 ** -23
TINY = 2.0 ** -126      # fp32's smallest normal: what an underflowing expf may lose
F32, I64 = torch.float32, torch.int64


# ---- runs ------------------------------------------------------------------------------------------------------------
class Run:
    def __init__(self, c, seed=0):
        self.c, self.lib = c, _lib.load()
        self.gen = torch.Generator().manual_seed(seed)
        self.off, self.data, specs = {}, {}, []
        getattr(self, "setup_" + c.op)(specs, c.dims, c.opt)
        self.arena = Arena(specs)

    def randn(self, *s, scale=1.0):
        return (torch.randn(*s, generator=self.gen, dtype=torch.float64) * scale).float().cuda()

    def add(self, specs, name, n, role, value=None, off=0, dtype=F32):
        specs.append((name, max(n, 1) + off, dtype, role))
        if off:
            self.off[name] = off
        if value is not None:
            lead = torch.full((off,), float("nan"), device="cuda", dtype=dtype) if dtype == F32 else \
                torch.zeros(off, device="cuda", dtype=dtype)
            self.data[name] = torch.cat([lead, value.reshape(-1).to(dtype)])

    def p(self, name):
        if name == self.c.opt.get("null") or name not in self.arena.t:
            return None
        return self.arena.ptr(name) + self.arena.t[name].element_size() * self.off.get(name, 0)

    def t(self, name):
        return self.arena.t[name][self.off.get(name, 0):]

    def prepare(self):
        self.arena.prepare(self.data)

    def outputs(self):
        return self.arena.outputs()

    # ---- Linear(K, n) + Softmax
    def setup_head(self, specs, d, o):
        N, K, n = d
        Nr, Kr = max(N, 1), max(K, 1)
        self.x = self.randn(Nr, Kr, scale=o.get("xscale", 1.0))
        self.w = self.randn(n, Kr, scale=1 / math.sqrt(Kr))
        self.b = self.randn(n) if o.get("b", True) else None
        self.dy = self.randn(Nr, n)
        self.add(specs, "x", Nr * Kr, "in", self.x, o.get("offset", 0))
        self.add(specs, "w", n * Kr, "in", self.w)
        if self.b is not None:
            self.add(specs, "b", n, "in", self.b)
        self.add(specs, "dy", Nr * n, "in", self.dy)
        self.add(specs, "y", Nr * n, "out")
        if o.get("dx", True):
            self.add(specs, "dx", Nr * Kr, "out")
        self.add(specs, "dw", n * Kr, "out")
        if o.get("db", True):
            self.add(specs, "db", n, "out")

    def fwd_head(self, s):
        N, K, n = self.c.dims
        p = self.p
        return self.lib.b200gan_class_head_fwd(p("x"), p("w"), p("b"), p("y"), N, K, n, s)

    def bwd_head(self, s):
        N, K, n = self.c.dims
        p = self.p
        return self.lib.b200gan_class_head_bwd(p("x"), p("w"), p("y"), p("dy"), p("dx"), p("dw"), p("db"), N, K, n, s)

    def check_head(self, what):
        N, K, n = self.c.dims
        x, w, dy = self.x.double(), self.w.double(), self.dy.double()
        y_ref, z = head_ref(self.x, self.w, self.b)
        chain = math.ceil(K / 128) + 4 + 5 + 4        # a thread's float4 steps, 5 shuffles, the 4 warp partials
        ez = U * (chain + 2) * (x.abs() @ w.abs().t() + (0 if self.b is None else self.b.double().abs()))
        zm = (z - z.max(1, keepdim=True).values).abs()
        # y = exp(z - m) / s: the logits' error through the softmax, then z - m, expf (2 ulp), the 5-step sum, the divide;
        # below 2^-126 expf loses its precision to underflow
        ey = y_ref * (ez + (y_ref * ez).sum(1, keepdim=True) + U * (zm + (y_ref * zm).sum(1, keepdim=True)) + 12 * U) + \
            TINY
        worst = check_elementwise(what + " y", self.t("y"), y_ref, ey, "(r, j)")
        not_vacuous(what + " y", ey - TINY, y_ref)
        yk = self.t("y").view(N, n)
        dx_ref, dw_ref, db_ref, dz = head_grad_ref(self.x, self.w, yk, self.dy)
        yd = yk.double()
        s_abs = (yd * dy).abs().sum(1, keepdim=True)
        edz = yd.abs() * (U * (dy - (yd * dy).sum(1, keepdim=True)).abs() + (n + 2) * U * s_abs) + U * dz.abs()
        bdw = U * (N + 4) * (dz.abs().t() @ x.abs()) + edz.t() @ x.abs()
        worst = max(worst, check_elementwise(what + " dw", self.t("dw"), dw_ref, bdw, "(j, k)"))
        if "dx" in self.arena.t:
            bdx = U * (n + 4) * (dz.abs() @ w.abs()) + edz @ w.abs()
            worst = max(worst, check_elementwise(what + " dx", self.t("dx"), dx_ref, bdx, "(r, k)"))
        if "db" in self.arena.t:
            bdb = U * (N + 4) * dz.abs().sum(0) + edz.sum(0)
            worst = max(worst, check_elementwise(what + " db", self.t("db"), db_ref, bdb, "(j,)"))
        return worst

    # ---- CrossEntropyLoss
    def setup_ce(self, specs, d, o):
        N, C = d
        Nr, Cr = max(N, 1), max(C, 1)
        self.ignore = o.get("ignore", hc.IGNORE)
        self.x = self.randn(Nr, Cr, scale=o.get("xscale", 1.0)) + o.get("xshift", 0.0)
        t = torch.randint(0, Cr, (Nr,), generator=self.gen)
        if o.get("ignored"):
            drop = torch.rand(Nr, generator=self.gen) < o["ignored"]
            t = torch.where(drop, torch.full_like(t, self.ignore), t)
            if o["ignored"] < 1:
                t[0] = self.ignore            # at least one ignored row
                if self.ignore == 3:
                    t[1] = 3                  # ignore_index is a class: hit it on purpose
        for r, v in o.get("bad", ()):
            t[r] = v
        self.target = t.cuda()
        self.gout = torch.tensor([1.5], device="cuda")
        self.add(specs, "x", Nr * Cr, "in", self.x)
        self.add(specs, "target", Nr, "in", self.target, dtype=I64)
        self.add(specs, "gout", 1, "in", self.gout)
        self.add(specs, "out", 2, "out")
        self.add(specs, "dx", Nr * Cr, "out")

    def fwd_ce(self, s):
        N, C = self.c.dims
        p = self.p
        return self.lib.b200gan_cross_entropy_fwd(p("x"), p("target"), p("out"), N, C, self.ignore, s)

    def bwd_ce(self, s):
        N, C = self.c.dims
        p = self.p
        return self.lib.b200gan_cross_entropy_bwd(p("x"), p("target"), p("out"), p("gout"), p("dx"), N, C, self.ignore, s)

    def check_ce(self, what):
        N, C = self.c.dims
        x, t = self.x.double(), self.target
        keep = t != self.ignore
        bad = keep & ((t < 0) | (t >= C))
        out, dx = self.t("out"), self.t("dx").view(N, C)
        count = int(keep.sum().item())
        assert out[1].item() == count, f"{what}: count {out[1].item()}, expected {count}"
        loss, terms, _ = ce_ref(self.x, t, self.ignore)
        if bad.any() or count == 0:
            assert torch.isnan(out[0]), f"{what}: loss {out[0].item()}, expected NaN"
        else:
            m = x.max(1, keepdim=True).values
            p = torch.softmax(x, 1)
            xt = x.gather(1, t.clamp(0, C - 1)[:, None])
            lse_m = torch.log(torch.exp(x - m).sum(1, keepdim=True))
            # s = sum expf(x - m): each term rounded in x - m (U |x - m|) and expf (2 ulp), a lane's chain and 5 shuffles
            rel_s = U * (math.ceil(C / 32) + 5 + 3) + U * (p * (x - m).abs()).sum(1, keepdim=True)
            err = rel_s + U * ((m - xt).abs() + 2 * lse_m.abs() + (m - xt + lse_m).abs())
            bound = (err[:, 0] * keep).sum() / count + 2 * U * loss.abs()
            check_elementwise(what + " loss", out[:1], loss.view(1), bound.view(1), "()")
        g = self.gout.double().item()
        d_ref = ce_grad_ref(self.x, t, self.ignore, g, max(count, 1))
        d_ref = torch.where(bad[:, None], torch.full_like(d_ref, float("nan")), d_ref)
        assert torch.isnan(dx[bad]).all(), f"{what}: a row of an out-of-range target is not NaN"
        assert (dx[~keep] == 0).all(), f"{what}: an ignored row is not zero"
        ok = keep & ~bad
        if not ok.any():
            return 0.0
        m = x.max(1, keepdim=True).values
        p = torch.softmax(x, 1)
        rel_s = U * (math.ceil(C / 32) + 5 + 3) + U * (p * (x - m).abs()).sum(1, keepdim=True)
        ep = p * (U * (x - m).abs() + 4 * U + rel_s)
        bound = (g / count) * (ep + TINY) + 3 * U * d_ref.abs()
        return check_elementwise(what + " dx", dx[ok], d_ref[ok], bound[ok], "(r, j)")

    def call(self, s):
        if not self.c.error:
            return getattr(self, "fwd_" + self.c.op)(s) or getattr(self, "bwd_" + self.c.op)(s)
        # a refusal: each entry point the case names must refuse it; one it does not name accepts the call, and what
        # that wrote is reset, so that the refusals are seen to write nothing
        codes = []
        for side in ("fwd", "bwd"):
            rc = getattr(self, f"{side}_{self.c.op}")(s)
            torch.cuda.synchronize()
            if side in self.c.opt["refused_by"]:
                codes.append(rc)
            else:
                assert rc == 0, f"{self.c.id}: {side} rc {rc}: {self.lib.b200gan_last_error().decode()}"
                self.prepare()
        return next((rc for rc in codes if rc != -2), -2)

    def check(self, what):
        return getattr(self, "check_" + self.c.op)(what)


# ---- the per-case test ---------------------------------------------------------------------------------------------
FAMILY = tuple({k for c in hc.CASES for k in c.kernels})


@pytest.mark.parametrize("case", hc.CASES, ids=lambda c: c.id)
def test_class_head_case(case):
    run_case(Run(case), case.id, case.launches, refuse=(-2,) if case.error else (), family=FAMILY)
