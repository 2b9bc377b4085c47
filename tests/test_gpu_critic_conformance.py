"""Every case of tests/critic_cases.py (mlp_critic.cu), element by element against torch float64.

Each case calls the C ABI on the guarded buffers of the convolution conformance test (Arena): inputs between NaN
guards, outputs and workspaces started as NaN, sentinels around everything the library writes.

The references are the closed forms of the header (fwd, bwd, dbwd, and the critic iteration with coef = 0 where an
input gradient is zero), in fp64; tests/test_cpu_kernel_coverage.py holds them to nn.Sequential autograd.  Bounds
follow the conv suite: an fp32 chain of n products with s partials added outside it is within 2^-23 (n + s + 4) A of
fp64, A the same sum over |terms|; tile_gemm has n = K, row_dots ceil(K / 32) + 5, col_sums R.  Errors of operands
computed earlier in the same launch are carried through (mm below) to check the intermediates a launch keeps in its
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
from test_gpu_conv_conformance import Arena, check_elementwise, traced_kernels
from test_gpu_stream_conformance import not_vacuous

pytestmark = pytest.mark.gpu

U = 2.0 ** -23


# ---- fp64 references with their bounds (device-agnostic) -------------------------------------------------------------
def mm(A, eA, B, eB, n):
    """A @ B in fp64, the bound of an fp32 evaluation with chains of n terms from operands off by eA, eB, and the
    mean magnitude of one term of the sum"""
    S = A.abs() @ B.abs()
    return A @ B, U * (n + 4) * S + eA @ B.abs() + A.abs() @ eB, S / max(A.shape[-1], 1)


def mask(h, slope):
    return torch.where(h > 0, torch.ones_like(h), torch.full_like(h, slope))


def z(t):
    return torch.zeros_like(t)


def rowdot_n(K):
    return math.ceil(K / 32) + 5


def critic_fwd_ref(x, W1, b1, W2, b2, W3, b3, slope, m1=None, m2=None):
    """h1, m1, a1, h2, m2, a2, out; each layer from the previous layer's (given) masks; with bounds of h1, h2, out"""
    r = {}
    h1, e1, _ = mm(x, z(x), W1.t(), z(W1).t(), x.shape[1] + 1)
    r["h1"], r["eh1"] = h1 + b1, e1 + U * 5 * b1.abs()
    r["m1"] = mask(r["h1"], slope) if m1 is None else m1
    r["a1"] = r["h1"] * r["m1"]
    h2, e2, _ = mm(r["a1"], z(r["a1"]), W2.t(), z(W2).t(), W2.shape[1] + 1)
    r["h2"], r["eh2"] = h2 + b2, e2 + U * 5 * b2.abs()
    r["m2"] = mask(r["h2"], slope) if m2 is None else m2
    r["a2"] = r["h2"] * r["m2"]
    out, eo, _ = mm(r["a2"], z(r["a2"]), W3.t(), z(W3).t(), rowdot_n(W3.shape[1]) + 1)
    r["out"], r["eout"] = out.reshape(-1) + b3, eo.reshape(-1) + U * 5 * b3.abs()
    return r


def critic_bwd_ref(dout, x, W1, W2, W3, m1, a1, m2, a2):
    N = x.shape[0]
    d = dout.reshape(-1, 1)
    U2 = d * W3.reshape(1, -1) * m2
    eU2 = 2 * U * U2.abs()
    r = {"U2": (U2, eU2)}
    r["dW3"] = tuple(v.reshape(1, -1) for v in mm(a2.t(), z(a2).t(), d, z(d), N))
    r["db3"] = (d.sum().reshape(1), U * (N + 4) * d.abs().sum().reshape(1))
    r["dW2"] = mm(U2.t(), eU2.t(), a1, z(a1), N)
    v, e, _ = mm(U2, eU2, W2, z(W2), W2.shape[0])
    U1 = v * m1
    eU1 = e * m1.abs() + U * U1.abs()
    r["U1"] = (U1, eU1)
    r["db2"] = (U2.sum(0), U * (N + 4) * U2.abs().sum(0) + eU2.sum(0))
    r["dW1"] = mm(U1.t(), eU1.t(), x, z(x), N)
    r["dx"] = mm(U1, eU1, W1, z(W1), W1.shape[0])
    r["db1"] = (U1.sum(0), U * (N + 4) * U1.abs().sum(0) + eU1.sum(0))
    return r


def critic_dbwd_ref(u, dout, U1, U2, m1, m2, W1, W2, W3):
    N = u.shape[0]
    r = {"dW1": mm(U1.t(), z(U1).t(), u, z(u), N)}
    v, e, _ = mm(u, z(u), W1.t(), z(W1).t(), W1.shape[1])
    t, et = v * m1, e * m1.abs() + U * (v * m1).abs()
    r["dW2"] = mm(U2.t(), z(U2).t(), t, et, N)
    v, e, _ = mm(t, et, W2.t(), z(W2).t(), W2.shape[1])
    s, es = v * m2, e * m2.abs() + U * (v * m2).abs()
    d = dout.reshape(-1, 1)
    r["dW3"] = tuple(v.reshape(1, -1) for v in mm(s.t(), es.t(), d, z(d), N))
    r["ddout"] = tuple(v.reshape(-1) for v in mm(s, es, W3.reshape(-1, 1), z(W3).reshape(-1, 1), rowdot_n(s.shape[1])))
    r["t"], r["s"] = (t, et), (s, es)
    return r


def critic_step_ref(real, fake, alpha, W1, b1, W2, b2, W3, b3, slope, lam, M1=None, M2=None):
    """the critic iteration: losses [d_loss, lambda * gp] and the gradient of d_loss w.r.t. every parameter, each as
    (value, bound); M1 / M2 [3N][H]: the masks of the stacked rows (None: the fp64 signs)"""
    N, Din = real.shape
    R = 3 * N
    a = alpha.reshape(-1, 1)
    X = torch.cat([real, fake, a * real + (1 - a) * fake])
    eX = torch.cat([z(real), z(fake), 3 * U * (a.abs() * real.abs() + (1 - a).abs() * fake.abs())])
    f = critic_fwd_ref(X, W1, b1, W2, b2, W3, b3, slope, M1, M2)
    M1, M2 = f["m1"], f["m2"]
    eh1 = f["eh1"] + eX @ W1.abs().t()
    ea1 = eh1 * M1.abs() + U * f["a1"].abs()
    eh2 = f["eh2"] + ea1 @ W2.abs().t()
    ea2 = eh2 * M2.abs() + U * f["a2"].abs()
    eout = f["eout"] + (ea2 @ W3.abs().t()).reshape(-1)
    r = {"h1": (f["h1"], eh1), "h2": (f["h2"], eh2), "M1": M1, "M2": M2}
    # dout = (-1/N, +1/N, 1) per row group, as the kernel forms it in fp32
    dout = torch.cat([torch.full((N,), -1.0 / N), torch.full((N,), 1.0 / N), torch.ones(N)])
    dout = dout.float().double().to(real.device).reshape(-1, 1)
    out = f["out"][:2 * N]
    wterms = out * dout[:2 * N, 0]
    U2 = dout * W3.reshape(1, -1) * M2
    eU2 = 2 * U * U2.abs()
    v, e, _ = mm(U2, eU2, W2, z(W2), W2.shape[0])
    U1, eU1 = v * M1, e * M1.abs() + U * (v * M1).abs()
    g1, eg1 = U1[2 * N:], eU1[2 * N:]
    gx, egx, _ = mm(g1, eg1, W1, z(W1), W1.shape[0])
    s = (gx * gx).sum(1)
    es = U * (rowdot_n(Din) + 4) * s + 2 * (gx.abs() * egx).sum(1)
    rn = torch.sqrt(s)
    pos = rn > 0
    safe = torch.where(pos, rn, torch.ones_like(rn))
    er = torch.where(pos, es / (2 * safe) + U * rn, torch.zeros_like(rn))
    k = lam * 2.0 / N
    coef = torch.where(pos, k * (rn - 1) / safe, torch.zeros_like(rn))
    ecoef = torch.where(pos, abs(k) * er / (safe * safe) + 4 * U * coef.abs(), torch.zeros_like(rn))
    pterms = lam * (rn - 1) ** 2 / N
    epterms = abs(lam) / N * 2 * (rn - 1).abs() * er + 4 * U * pterms
    gp = pterms.sum()
    egp = epterms.sum() + U * (N + 4) * pterms.abs().sum()
    ew = (eout[:2 * N] * dout[:2 * N, 0].abs()).sum() + 2 * U * wterms.abs().sum()
    loss = wterms.sum() + gp
    eloss = ew + egp + U * (3 * N + 4) * (wterms.abs().sum() + pterms.abs().sum())
    r["losses"] = (torch.stack([loss, gp]), torch.stack([eloss, egp]))
    c = coef.reshape(-1, 1)
    ec = ecoef.reshape(-1, 1)
    g1s = c * g1
    eg1s = c.abs() * eg1 + ec * g1.abs() + U * g1s.abs()
    Ucat, eUcat = torch.cat([U1[:2 * N], g1s]), torch.cat([eU1[:2 * N], eg1s])
    Xcat, eXcat = torch.cat([X[:2 * N], gx]), torch.cat([z(X[:2 * N]), egx])
    r["dW1"] = mm(Ucat.t(), eUcat.t(), Xcat, eXcat, R)
    acc, eacc, _ = mm(gx, egx, W1.t(), z(W1).t(), Din)
    Mp = M1[2 * N:]
    t = acc * c * Mp
    et = (eacc * c.abs() + acc.abs() * ec) * Mp.abs() + 2 * U * t.abs()
    A1cat, eA1cat = torch.cat([f["a1"][:2 * N], t]), torch.cat([ea1[:2 * N], et])
    r["dW2"] = mm(U2.t(), eU2.t(), A1cat, eA1cat, R)
    v, e, _ = mm(t, et, W2.t(), z(W2).t(), W2.shape[1])
    sp, esp = v * M2[2 * N:], e * M2[2 * N:].abs() + U * (v * M2[2 * N:]).abs()
    A2cat, eA2cat = torch.cat([f["a2"][:2 * N], sp]), torch.cat([ea2[:2 * N], esp])
    r["dW3"] = tuple(v.reshape(1, -1) for v in mm(A2cat.t(), eA2cat.t(), dout, z(dout), R))
    r["db1"] = (U1[:2 * N].sum(0), U * (2 * N + 4) * U1[:2 * N].abs().sum(0) + eU1[:2 * N].sum(0))
    r["db2"] = (U2[:2 * N].sum(0), U * (2 * N + 4) * U2[:2 * N].abs().sum(0) + eU2[:2 * N].sum(0))
    r["db3"] = (dout[:2 * N].sum().reshape(1), U * (2 * N + 4) * dout[:2 * N].abs().sum().reshape(1))
    r["coef"], r["ecoef"] = coef, ecoef
    # the workspace rows the kernel's last GEMMs read: U1 (penalty rows scaled), X3 (penalty rows gx), U2, A1
    # (penalty rows t), A2 (penalty rows (t W2^T) * m2)
    r["ws"] = {"U1": (Ucat, eUcat), "X3": (Xcat, eXcat), "U2": (U2, eU2), "A1": (A1cat, eA1cat), "A2": (A2cat, eA2cat)}
    r["dout"] = dout
    return r


# ---- the case as tensors ----------------------------------------------------------------------------------------------
F32 = torch.float32


def check_mask(what, m, h, eh, slope):
    """the kernel's mask equals the fp64 sign of h wherever |h| exceeds its bound, and is 1 or slope everywhere"""
    m = m.double().view_as(h)
    ok = (m == 1) | (m == torch.tensor(slope, dtype=F32).item())
    assert ok.all(), f"{what}: mask value {m[~ok][0].item()} is neither 1 nor the slope"
    sure = h.abs() > eh
    bad = sure & (m != mask(h, torch.tensor(slope, dtype=F32).item()))
    assert not bad.any(), f"{what}: mask differs from the sign of h at {tuple(bad.nonzero()[0].tolist())}, " \
                          f"h {h[bad][0].item():.3e}, bound {eh[bad][0].item():.3e}"


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
        return {k: v.clone() for k, v in self.arena.t.items() if self.arena.layout[k][3] != "in"}

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
def check_route(run):
    c = run.c
    marker = torch.zeros(1, device="cuda")
    seen = []
    for _ in range(3):
        run.prepare()
        seen = [(n, tuple(g)) for n, g in traced_kernels(lambda: (marker.zero_(), run.call(
            torch.cuda.current_stream().cuda_stream))) if n in cr.KERNEL.values()]
        if [n for n, _ in seen] == list(c.kernels):
            break
    if not seen:
        return "the profiler recorded no CUDA kernel activity on this machine"
    assert [n for n, _ in seen] == list(c.kernels), f"{c.id}: trace {seen}, table {c.kernels}"
    if torch.cuda.get_device_properties(0).multi_processor_count == cr.NUM_SMS:
        assert seen[0][1] == c.grid, f"{c.id}: grid {seen[0][1]}, table {c.grid}"
    return None


@pytest.mark.parametrize("case", cr.CASES, ids=lambda c: c.id)
def test_critic_case(case):
    run = Run(case)
    lib = run.lib
    run.prepare()
    before = run.outputs()
    rc = run.call(torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    if case.error:
        assert rc == -2, f"{case.id}: expected B200GAN_E_BAD_ARG, rc {rc}"
        run.arena.check_guards(case.id)
        after = run.outputs()
        for k, v in before.items():
            assert torch.equal(v.view(torch.int32), after[k].view(torch.int32)), f"{case.id}: refused call wrote {k}"
        return
    assert rc == 0, f"{case.id}: rc {rc}: {lib.b200gan_last_error().decode()}"
    run.arena.check_guards(case.id)
    eager = run.outputs()
    worst = run.check(case.id + " eager")

    skip_reason = check_route(run)

    side = torch.cuda.Stream()
    run.prepare()
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=side):
        rc = run.call(side.cuda_stream)
    assert rc == 0, f"{case.id}: rc {rc} under capture: {lib.b200gan_last_error().decode()}"
    run.prepare()
    torch.cuda.synchronize()
    graph.replay()
    torch.cuda.synchronize()
    run.arena.check_guards(case.id + " graph")
    replay = run.outputs()
    if case.deterministic:
        for k, v in replay.items():
            if k in ("losses", "ws"):     # atomically summed losses; workspace rows the step overwrites in place
                continue
            same = v.view(torch.int32) == eager[k].view(torch.int32)
            assert same.all(), f"{case.id}: graph replay differs from the eager call in {k} (marked deterministic)"
    worst = max(worst, run.check(case.id + " graph"))
    print(f"\n{case.id}: worst |err|/bound {worst:.3g}, grid {case.grid}")
    if skip_reason:
        pytest.skip(skip_reason)
