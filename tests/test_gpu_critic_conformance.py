"""Every case of tests/critic_cases.py (mlp_critic.cu), element by element against torch float64.

Each case calls the C ABI on the guarded buffers of tests/conformance.py (Arena) and runs its protocol: inputs between
NaN guards, outputs and workspaces started as NaN, sentinels around everything the library writes.

The references are the closed forms of the header (fwd, bwd, dbwd, and the critic iteration with coef = 0 where an
input gradient is zero), in fp64; tests/test_cpu_kernel_coverage.py holds them to nn.Sequential autograd.  Bounds
follow the conv suite: an fp32 chain of n products with s partials added outside it is within 2^-23 (n + s + 4) A of
fp64, A the same sum over |terms|; tile_gemm has n = K, row_dots ceil(K / 32) + 5, col_sums R.  Errors of operands
computed earlier in the same launch are carried through (critic_cases.mm) to check the intermediates a launch keeps in its
workspace (dbwd's t and s, critic_step's stacked operands); the GEMMs that read them are checked against fp64 of the
kernel's own intermediates, so their bounds stay below one term of their sums.  A LeakyReLU mask may differ from the fp64 sign of
h only where |h| is within its bound; downstream the reference uses the kernel's masks (the forward's m1 / m2
outputs, critic_step's M1 / M2 workspace), so one such element cannot flip a whole row.
"""
import ctypes
import math

import pytest
import torch

import critic_cases as cr
from b200gan import _lib
from conformance import Arena, check_elementwise, first_grid, not_vacuous, run_case
from critic_cases import (F32, U, check_mask, critic_bwd_ref, critic_dbwd_ref, critic_fwd_ref, critic_step_ref, mask, mm,
                          rowdot_n, z)

pytestmark = pytest.mark.gpu


class Run:
    def __init__(self, c, seed=0):
        self.c, self.lib = c, _lib.load()
        g = torch.Generator().manual_seed(seed)
        rn = lambda *s, scale=1.0: (torch.randn(*s, generator=g) * scale).cuda()
        N, Din, H1, H2 = c.N, c.Din, c.H1, c.H2
        Nc, Dc, H1c, H2c = max(N, 1), max(Din, 1), max(H1, 1), max(H2, 1)
        self.d = _lib.MlpCriticDesc(N, Din, H1, H2, c.slope)
        P = dict(W1=rn(H1c, Dc, scale=1 / math.sqrt(Dc)), b1=rn(H1c, scale=0.2), W2=rn(H2c, H1c, scale=1 / math.sqrt(H1c)),
                 b2=rn(H2c, scale=0.2), W3=rn(1, H2c, scale=1 / math.sqrt(H2c)), b3=rn(1, scale=0.2))
        if c.zero_w3:
            P["W3"].zero_()
        if c.zero_row >= 0:
            P["b1"] = -0.5 - 0.1 * P["b1"].abs()
        self.P = P
        f32, specs, data = F32, [], dict(P)
        ins = lambda name, t: (specs.append((name, t.numel(), f32, "in")), data.__setitem__(name, t))
        outs = lambda name, n, role="out": specs.append((name, n, f32, role))
        for k, v in P.items():
            if not (c.no_w1 and k == "W1"):
                ins(k, v)
        if c.op == "fwd":
            ins("x", rn(Nc, Dc))
            for name, n in (("out", Nc), ("m1", Nc * H1c), ("a1", Nc * H1c), ("m2", Nc * H2c), ("a2", Nc * H2c)):
                outs(name, n)
        elif c.op in ("bwd", "dbwd"):
            x = rn(Nc, Dc)
            fw = critic_fwd_ref(x.double(), *(P[k].double() for k in ("W1", "b1", "W2", "b2", "W3", "b3")), c.slope)
            fw["m1"] = mask(fw["h1"], torch.tensor(c.slope, dtype=F32).item())
            fw["m2"] = mask(fw["h2"], torch.tensor(c.slope, dtype=F32).item())
            for k in ("m1", "a1", "m2", "a2"):
                ins(k, fw[k].float())
            ins("dout", rn(Nc))
            ins("x", x)
            if c.op == "bwd":
                for name, n in (("dx", Nc * Dc), ("dW1", H1c * Dc), ("db1", H1c), ("dW2", H2c * H1c), ("db2", H2c),
                                ("dW3", H2c), ("db3", 1), ("U1", Nc * H1c), ("U2", Nc * H2c)):
                    if name not in c.null:
                        outs(name, n)
            else:
                ins("u", rn(Nc, Dc))
                ins("U1", rn(Nc, H1c, scale=0.1))
                ins("U2", rn(Nc, H2c, scale=0.1))
                for name, n in (("dW1", H1c * Dc), ("dW2", H2c * H1c), ("dW3", H2c), ("ddout", Nc)):
                    if name not in c.null:
                        outs(name, n)
            nws = self.lib.b200gan_mlp_critic_bwd_workspace_floats(ctypes.byref(self.d))
            if not c.no_ws:
                outs("ws", max(nws, 1), "ws")
        else:
            real, fake = rn(Nc, Dc), rn(Nc, Dc)
            if c.zero_row >= 0:
                real[c.zero_row].zero_()
                fake[c.zero_row].zero_()
            alpha = {"rand": torch.rand(Nc, generator=g).cuda(), "zero": torch.zeros(Nc, device="cuda"),
                     "one": torch.ones(Nc, device="cuda")}[c.alpha]
            ins("real", real)
            ins("fake", fake)
            ins("alpha", alpha)
            for name, n in (("losses", 2), ("dW1", H1c * Dc), ("db1", H1c), ("dW2", H2c * H1c), ("db2", H2c),
                            ("dW3", H2c), ("db3", 1)):
                outs(name, n)
            if not c.no_ws:
                outs("ws", max(self.lib.b200gan_critic_step_workspace_floats(ctypes.byref(self.d)), 1), "ws")
        self.arena, self.data = Arena(specs), data

    def prepare(self):
        self.arena.prepare(self.data)

    def outputs(self):
        return self.arena.outputs()

    def call(self, st):
        p, d, L, c = self.arena.ptr, ctypes.byref(self.d), self.lib, self.c
        if c.op == "fwd":
            return L.b200gan_mlp_critic_fwd(d, p("x"), p("W1"), p("b1"), p("W2"), p("b2"), p("W3"), p("b3"), p("out"),
                                            p("m1"), p("a1"), p("m2"), p("a2"), st)
        if c.op == "bwd":
            return L.b200gan_mlp_critic_bwd(d, p("dout"), p("x"), p("W1"), p("W2"), p("W3"), p("m1"), p("a1"), p("m2"),
                                            p("a2"), p("dx"), p("dW1"), p("db1"), p("dW2"), p("db2"), p("dW3"),
                                            p("db3"), p("U1"), p("U2"), p("ws"), st)
        if c.op == "dbwd":
            return L.b200gan_mlp_critic_dbwd(d, p("u"), p("dout"), p("U1"), p("U2"), p("m1"), p("m2"), p("W1"), p("W2"),
                                             p("W3"), p("dW1"), p("dW2"), p("dW3"), p("ddout"), p("ws"), st)
        return L.b200gan_critic_step_mlp(d, c.lam, p("real"), p("fake"), p("alpha"), p("W1"), p("b1"), p("W2"),
                                         p("b2"), p("W3"), p("b3"), p("losses"), p("dW1"), p("db1"), p("dW2"),
                                         p("db2"), p("dW3"), p("db3"), p("ws"), st)

    def check(self, what):
        c, t, D = self.c, self.arena.t, {k: v.double() for k, v in self.data.items()}
        N, Din, H1, H2 = c.N, c.Din, c.H1, c.H2
        slope = torch.tensor(c.slope, dtype=F32).item()
        W = [D[k] for k in ("W1", "b1", "W2", "b2", "W3", "b3")]
        worst = 0.0
        if c.op == "fwd":
            x = D["x"]
            # layer by layer, each from the kernel's own previous layer
            h1 = x @ W[0].t() + W[1]
            eh1 = U * (Din + 5) * (x.abs() @ W[0].abs().t() + W[1].abs())
            check_mask(what + " m1", t["m1"], h1, eh1, slope)
            m1 = t["m1"].double().view(N, H1)
            worst = check_elementwise(what + " a1", t["a1"], h1 * m1, eh1 * m1 + U * (h1 * m1).abs(), "(n, i)")
            not_vacuous(what + " a1", eh1, (x.abs() @ W[0].abs().t()) / Din)
            a1 = t["a1"].double().view(N, H1)
            h2 = a1 @ W[2].t() + W[3]
            eh2 = U * (H1 + 5) * (a1.abs() @ W[2].abs().t() + W[3].abs())
            check_mask(what + " m2", t["m2"], h2, eh2, slope)
            m2 = t["m2"].double().view(N, H2)
            worst = max(worst, check_elementwise(what + " a2", t["a2"], h2 * m2, eh2 * m2 + U * (h2 * m2).abs(),
                                                 "(n, j)"))
            a2 = t["a2"].double().view(N, H2)
            out = (a2 @ W[4].t()).reshape(-1) + W[5]
            eo = U * (rowdot_n(H2) + 5) * ((a2.abs() @ W[4].abs().t()).reshape(-1) + W[5].abs())
            worst = max(worst, check_elementwise(what + " out", t["out"], out, eo, "(n,)"))
            return worst
        if c.op == "bwd":
            W1 = D.get("W1")
            r = critic_bwd_ref(D["dout"], D["x"], W1, D["W2"], D["W3"].view(-1), D["m1"].view(N, H1), D["a1"].view(N, H1),
                               D["m2"].view(N, H2), D["a2"].view(N, H2))

        elif c.op == "dbwd":
            r = critic_dbwd_ref(D["u"].view(N, Din), D["dout"], D["U1"].view(N, H1), D["U2"].view(N, H2),
                                D["m1"].view(N, H1), D["m2"].view(N, H2), D["W1"], D["W2"], D["W3"].view(-1))
            # t and s in the workspace against the chain from the inputs; the GEMMs that read them against fp64 of the
            # kernel's own t and s
            ws = t["ws"]
            want_s = "dW3" in c.outputs() or "ddout" in c.outputs()
            if want_s or "dW2" in c.outputs():
                tk = ws[:N * H1].double().view(N, H1)
                worst = max(worst, check_elementwise(what + " t", tk, *r["t"], "(n, i)"))
                r["dW2"] = mm(D["U2"].view(N, H2).t(), z(D["U2"].view(N, H2)).t(), tk, z(tk), N)
            if want_s:
                sk = ws[N * H1:N * (H1 + H2)].double().view(N, H2)
                worst = max(worst, check_elementwise(what + " s", sk, *r["s"], "(n, j)"))
                d = D["dout"].reshape(-1, 1)
                r["dW3"] = mm(sk.t(), z(sk).t(), d, z(d), N)
                w3 = D["W3"].reshape(-1, 1)
                r["ddout"] = mm(sk, z(sk), w3, z(w3), rowdot_n(H2))
        else:
            R = 3 * N
            ws = t["ws"]
            o = R * Din + 2 * R * H1
            M1, M2 = ws[o:o + R * H1].double().view(R, H1), ws[o + R * H1 + 2 * R * H2:o + R * H1 + 3 * R * H2]
            r = critic_step_ref(D["real"], D["fake"], D["alpha"], *W[:4], W[4], W[5], c.slope, c.lam, M1,
                                M2.double().view(R, H2))
            check_mask(what + " M1", M1, *r["h1"], slope)
            check_mask(what + " M2", M2, *r["h2"], slope)
            coef = ws[o + R * H1 + 3 * R * H2 + R:][:N]
            assert not torch.isnan(coef).any(), f"{what}: NaN coefficient (a zero input gradient)"
            worst = max(worst, check_elementwise(what + " coef", coef, r["coef"], r["ecoef"], "(n,)"))
            # the workspace operands of the last GEMMs against the chain from the inputs; the parameter gradients
            # against fp64 of those operands
            at = {"X3": 0, "A1": R * Din, "U1": R * Din + R * H1, "A2": R * Din + 3 * R * H1,
                  "U2": R * Din + 3 * R * H1 + R * H2}
            wk = {}
            for name, cols in (("X3", Din), ("A1", H1), ("U1", H1), ("A2", H2), ("U2", H2)):
                wk[name] = ws[at[name]:at[name] + R * cols].double().view(R, cols)
                worst = max(worst, check_elementwise(f"{what} {name}", wk[name], *r["ws"][name], "(row, col)"))
            d = r["dout"]
            r["dW1"] = mm(wk["U1"].t(), z(wk["U1"]).t(), wk["X3"], z(wk["X3"]), R)
            r["dW2"] = mm(wk["U2"].t(), z(wk["U2"]).t(), wk["A1"], z(wk["A1"]), R)
            r["dW3"] = tuple(v.reshape(1, -1) for v in mm(wk["A2"].t(), z(wk["A2"]).t(), d, z(d), R))
            for name, src in (("db1", "U1"), ("db2", "U2")):
                v = wk[src][:2 * N]
                r[name] = (v.sum(0), U * (2 * N + 4) * v.abs().sum(0))
        for name in c.outputs():
            if name not in r:
                continue
            val, b, *term = r[name]
            worst = max(worst, check_elementwise(f"{what} {name}", t[name], val.reshape(-1), b.reshape(-1), "(flat)"))
            if term:   # a GEMM output: the bound below one term of its sum
                not_vacuous(f"{what} {name}", b.reshape(-1), term[0].reshape(-1))
        return worst


# ---- the per-case test -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", cr.CASES, ids=lambda c: c.id)
def test_critic_case(case):
    run = Run(case)
    # atomically summed losses; workspace rows the step overwrites in place
    varies = ("losses", "ws") if case.deterministic else tuple(run.arena.t)
    run_case(run, case.id, first_grid(case.kernels, case.grid), refuse=(-2,) if case.error else (), varies=varies,
             family=tuple(cr.KERNEL.values()), num_sms=cr.NUM_SMS)
