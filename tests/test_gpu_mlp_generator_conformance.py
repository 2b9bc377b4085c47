"""Every case of tests/generator_cases.py (csrc/mlp_generator/mlp_generator.cu), element by element against fp64.

Each case calls the C ABI on the guarded buffers of the convolution conformance test (Arena): outputs and workspaces
started as NaN, sentinels around everything the library writes.  The running statistics are inputs the forward updates
in place; they are read back and checked against the fp64 update.

The forward is checked layer by layer: each layer's reference starts from the kernel's own previous activations (the
saved region), so a bound covers one layer's rounding.  A forward without a saved region (torch.no_grad()) is checked
from the last hidden activation it leaves in its workspace and must repeat the saved-mode call bit for bit.  The
backward reads a saved region formed from the fp64 forward and rounded to fp32, so its reference is exact in its
inputs; bounds follow the conv suite: an fp32 chain of n products with s partials added outside it is within
2^-23 (n + s + 4) A of fp64, A the same sum over |terms|, carried from layer to layer (mmr).
tests/test_cpu_mlp_generator.py holds the references to torch float64 autograd.
"""
import ctypes
import math
import re

import pytest
import torch

import generator_cases as gc
from b200gan import _lib
from test_gpu_conv_conformance import Arena, check_elementwise, traced_kernels
from test_gpu_critic_conformance import z
from test_gpu_stream_conformance import not_vacuous

pytestmark = pytest.mark.gpu

U = 2.0 ** -23
EPS, MOMENTUM = 0.8, 0.1     # BatchNorm1d(o, 0.8) of wgan_gp.py:49 / gan.py:45, torch's default momentum
F32 = torch.float32


def f32(v):
    return torch.tensor(v, dtype=F32).item()


# ---- inputs and fp64 references (device-agnostic) ------------------------------------------------------------------
def make(c, seed=0):
    """the case's fp32 inputs on the CPU: z, W{l}, b{l}, and per norm layer gamma, beta, rm, rv, nbt; dout"""
    g = torch.Generator().manual_seed(seed)
    rn = lambda *s, scale=1.0: torch.randn(*s, generator=g) * scale  # noqa: E731
    N, w = max(c.N, 1), c.widths
    P = {"z": rn(N, w[0])}
    for l in range(c.L):
        P[f"W{l}"] = rn(w[l + 1], w[l], scale=1 / math.sqrt(w[l]))
        P[f"b{l}"] = rn(w[l + 1], scale=0.2)
        if c.has_norm[l]:
            P[f"gamma{l}"] = 1 + rn(w[l + 1], scale=0.2)
            P[f"beta{l}"] = rn(w[l + 1], scale=0.2)
            P[f"rm{l}"] = rn(w[l + 1], scale=0.1)
            P[f"rv{l}"] = 1 + torch.rand(w[l + 1], generator=g)
            P[f"nbt{l}"] = torch.tensor([7], dtype=torch.int64)
    P["dout"] = rn(N, w[-1])
    return P


def mask(a, slope):
    return torch.where(a > 0, torch.ones_like(a), torch.full_like(a, slope))


def gen_fwd_ref(P, c, acts=None):
    """fp64 forward of case c from its (fp32) inputs P.  Per layer: x (the layer's input), h, and for a norm layer mean,
    var, rstd, xhat, the updated running statistics; y, a; and out.  acts: the kernel's activations, each layer then
    starts from the kernel's previous layer."""
    D = {k: v.double() for k, v in P.items() if v.is_floating_point()}
    slope, N = f32(c.slope), D["z"].shape[0]
    x, layers = D["z"], []
    for l in range(c.L):
        r = {"x": x, "h": x @ D[f"W{l}"].t() + D[f"b{l}"]}
        if l == c.L - 1:
            r["out"] = torch.tanh(r["h"])
        else:
            y = r["h"]
            if c.has_norm[l]:
                mean = y.mean(0)
                var = ((y - mean) ** 2).mean(0)
                r.update(mean=mean, var=var, rstd=1 / torch.sqrt(var + f32(EPS)))
                r["xhat"] = (y - mean) * r["rstd"]
                y = r["xhat"] * D[f"gamma{l}"] + D[f"beta{l}"]
                m = f32(MOMENTUM)
                r["rm"] = (1 - m) * D[f"rm{l}"] + m * mean
                r["rv"] = (1 - m) * D[f"rv{l}"] + m * var * N / (N - 1)
            r["y"], r["a"] = y, y * mask(y, slope)
            x = r["a"] if acts is None or acts[l] is None else acts[l].double()
        layers.append(r)
    return layers


def saved_of(c, layers):
    """the saved region (include/b200gan.h: a_l, then xhat and rstd of each norm layer) from a forward's layers"""
    hid = [layers[l] for l in range(c.L - 1)]
    parts = [r["a"] for r in hid] + [r["xhat"] for r, n in zip(hid, c.has_norm) if n] + \
        [r["rstd"] for r, n in zip(hid, c.has_norm) if n]
    return torch.cat([p.reshape(-1) for p in parts]) if parts else torch.zeros(0, dtype=torch.float64)


def split_saved(c, saved, N):
    """saved -> (acts, xhats, rstds), per hidden layer (None for layers without a norm)"""
    w, o = c.widths, 0
    acts, xh, rs = [], [None] * (c.L - 1), [None] * (c.L - 1)
    for l in range(c.L - 1):
        acts.append(saved[o:o + N * w[l + 1]].view(N, w[l + 1]))
        o += N * w[l + 1]
    for l in range(c.L - 1):
        if c.has_norm[l]:
            xh[l] = saved[o:o + N * w[l + 1]].view(N, w[l + 1])
            o += N * w[l + 1]
    for l in range(c.L - 1):
        if c.has_norm[l]:
            rs[l] = saved[o:o + w[l + 1]]
            o += w[l + 1]
    return acts, xh, rs


def mmr(A, eA, B, n):
    """A @ B in fp64 for an operand A off by eA and an exact B: the bound of the fp32 GEMM's own rounding, plus the
    operand errors carried as independent ones (root-sum-square); and the mean magnitude of one term"""
    S = A.abs() @ B.abs()
    return A @ B, U * (n + 4) * S + torch.sqrt((eA * eA) @ (B * B)), S / max(A.shape[-1], 1)


def rss(e, dim=0):
    return torch.sqrt((e * e).sum(dim))


def gen_bwd_ref(c, dout, out, z_, W, gamma, acts, xhat, rstd):
    """fp64 backward for dout with bounds: name -> (value, bound[, mean magnitude of one term]) for dz, dW{l}, db{l},
    dgamma{l}, dbeta{l}; every operand but the gradient itself is exact (the kernel reads the same fp32 values).  The
    gradient's own error is carried from layer to layer as independent per-element errors (mmr, rss): the worst case of
    correlated errors grows by the row sums of |W| per layer and is vacuous after five layers.  Each carried bound is
    itself a worst case of its layer's rounding, far above the error a kernel makes."""
    slope, N = f32(c.slope), dout.shape[0]
    g = dout * (1 - out * out)
    eg = U * (3 * g.abs() + 2 * dout.abs() * out * out)
    r = {}
    for l in range(c.L - 1, -1, -1):
        ain = z_ if l == 0 else acts[l - 1]
        r[f"dW{l}"] = mmr(g.t(), eg.t(), ain, N)
        r[f"db{l}"] = (g.sum(0), U * (N + 4) * g.abs().sum(0) + rss(eg))
        da, eda, _ = mmr(g, eg, W[l], W[l].shape[0])
        if l == 0:
            r["dz"] = (da, eda)
            break
        mk = mask(ain, slope)
        dy, edy = da * mk, eda * mk.abs() + U * (da * mk).abs()
        if c.has_norm[l - 1]:
            xh, k = xhat[l - 1], gamma[l - 1] * rstd[l - 1]
            s1, s2 = dy.sum(0), (dy * xh).sum(0)
            es1 = U * (N + 4) * dy.abs().sum(0) + rss(edy)
            es2 = U * (N + 4) * (dy * xh).abs().sum(0) + rss(edy * xh)
            r[f"dbeta{l - 1}"], r[f"dgamma{l - 1}"] = (s1, es1), (s2, es2)
            inner = dy - s1 / N - xh * s2 / N
            g = k * inner
            eg = k.abs() * (edy + es1 / N + xh.abs() * es2 / N
                            + 6 * U * (dy.abs() + (s1 / N).abs() + (xh * s2 / N).abs())) + 2 * U * g.abs()
        else:
            g, eg = dy, edy
    return r


# ---- the case as buffers ---------------------------------------------------------------------------------------------
def desc(c, ptr=None):
    d = _lib.MlpGenDesc()
    d.L, d.N = c.L, c.N
    for l, v in enumerate(c.widths):
        d.width[l] = v
    for l, v in enumerate(c.has_norm):
        d.has_norm[l] = int(v)
    d.slope, d.eps, d.momentum = c.slope, EPS, MOMENTUM
    if ptr is not None:
        for l in range(c.L):
            d.W[l], d.b[l] = ptr(f"W{l}"), ptr(f"b{l}")
            if c.has_norm[l]:
                d.gamma[l], d.beta[l] = ptr(f"gamma{l}"), ptr(f"beta{l}")
                d.running_mean[l], d.running_var[l] = ptr(f"rm{l}"), ptr(f"rv{l}")
                d.num_batches_tracked[l] = ptr(f"nbt{l}")
    return d


class Run:
    def __init__(self, c, seed=0):
        self.c, self.lib = c, _lib.load()
        self.P = make(c, seed)
        N = max(c.N, 1)
        d0 = desc(c)
        self.nsaved = self.lib.b200gan_mlp_gen_saved_floats(ctypes.byref(d0))
        self.nws = self.lib.b200gan_mlp_gen_workspace_floats(ctypes.byref(d0))
        specs, data = [], {}
        for k, v in self.P.items():
            if k != "dout" or c.op == "bwd":
                specs.append((k, v.numel(), v.dtype, "in"))
                data[k] = v.cuda()
        specs.append(("out", N * c.widths[-1], F32, "in" if c.op == "bwd" else "out"))
        if c.op == "fwd":
            if c.keep:
                specs.append(("saved", max(self.nsaved, 1), F32, "out"))
        else:
            # the backward's inputs: the fp64 forward rounded to fp32
            if c.error:
                data["out"], data["saved"] = torch.zeros(N, c.widths[-1]).cuda(), torch.zeros(1).cuda()
            else:
                layers = gen_fwd_ref(self.P, c)
                data["out"] = layers[-1]["out"].float().cuda()
                data["saved"] = saved_of(c, layers).float().cuda()
                if data["saved"].numel() == 0:   # L = 1: nothing is saved; the buffer holds one unread float
                    data["saved"] = torch.zeros(1, device="cuda")
            specs.append(("saved", max(data["saved"].numel(), 1), F32, "in"))
            for name in c.all_outputs():
                if name in c.outputs():
                    specs.append((name, self.numel(name), F32, "out"))
        if not c.no_ws:
            specs.append(("ws", max(self.nws, 1), F32, "ws"))
        self.arena, self.data = Arena(specs), data

    def numel(self, name):
        c, w = self.c, self.c.widths
        if name == "dz":
            return max(c.N, 1) * w[0]
        l = int(re.sub(r"\D", "", name))
        return w[l + 1] * w[l] if name.startswith("dW") else w[l + 1]

    def prepare(self):
        self.arena.prepare(self.data)

    def outputs(self):
        return {k: v.clone() for k, v in self.arena.t.items()
                if self.arena.layout[k][3] != "in" or k.startswith(("rm", "rv", "nbt"))}

    def call(self, st):
        c, p, L = self.c, self.arena.ptr, self.lib
        d = desc(c, p)
        if c.op == "fwd":
            return L.b200gan_mlp_gen_fwd(ctypes.byref(d), p("z"), p("out"), p("saved"), p("ws"), st)
        gr = _lib.MlpGenGrads()
        for l in range(c.L):
            for name in ("dW", "db", "dgamma", "dbeta"):
                getattr(gr, name)[l] = p(f"{name}{l}")
        return L.b200gan_mlp_gen_bwd(ctypes.byref(d), p("dout"), p("z"), p("out"), p("saved"), p("dz"),
                                     ctypes.byref(gr), p("ws"), st)

    def check(self, what):
        c, t, N = self.c, self.arena.t, self.c.N
        worst = 0.0
        if c.op == "bwd":
            D = {k: v.double() for k, v in self.data.items() if v.is_floating_point()}
            acts, xh, rs = split_saved(c, D["saved"], N)
            r = gen_bwd_ref(c, D["dout"].view(N, -1), D["out"].view(N, -1), D["z"].view(N, -1),
                            [D[f"W{l}"] for l in range(c.L)],
                            [D.get(f"gamma{l}") for l in range(c.L)], acts, xh, rs)
            for name in c.outputs():
                val, b, *term = r[name]
                worst = max(worst, check_elementwise(f"{what} {name}", t[name], val.reshape(-1), b.reshape(-1),
                                                     "(flat)"))
                if term:
                    not_vacuous(f"{what} {name}", b.reshape(-1), term[0].reshape(-1))
            return worst
        slope = f32(c.slope)
        if c.keep:
            acts = split_saved(c, t["saved"], N)[0]
        else:   # the activations ping-pong through workspace slabs 1 and 2; the last hidden one is still there
            slab = N * max(c.widths[1:])
            acts = [None] * (c.L - 1)
            if c.L > 1:
                l = c.L - 2
                o = (1 + (l & 1)) * slab
                acts[l] = t["ws"][o:o + N * c.widths[l + 1]].view(N, -1)
        layers = gen_fwd_ref(self.P, c, [a.cpu() if a is not None else None for a in acts])
        D = {k: v.double() for k, v in self.P.items() if v.is_floating_point()}
        for l, r in enumerate(layers):
            if not c.keep and l < c.L - 1:
                continue   # checked bit for bit against the saved-mode call instead
            x, W, b = r["x"], D[f"W{l}"], D[f"b{l}"]
            K = W.shape[1]
            eh = U * (K + 5) * (x.abs() @ W.abs().t() + b.abs())
            if l == c.L - 1:
                out = r["out"]
                eo = (1 - out ** 2 + 2 * eh).clamp(max=1) * eh + 4 * U * out.abs()
                worst = max(worst, check_elementwise(f"{what} out", t["out"].cpu(), out, eo, "(n, j)"))
                not_vacuous(f"{what} out", eo.reshape(-1), ((x.abs() @ W.abs().t()) / K).reshape(-1))
                continue
            if c.has_norm[l]:
                h, mean, var, rstd, xhat = r["h"], r["mean"], r["var"], r["rstd"], r["xhat"]
                d = h - mean
                em = eh.mean(0) + U * (N + 2) * h.abs().mean(0)
                ed = eh + em + U * d.abs()
                ev = 2 * (d.abs() * ed).mean(0) + (ed * ed).mean(0) + U * (N + 4) * var
                rel = ev / (2 * (var + f32(EPS))) + 3 * U
                exh = ed * rstd + xhat.abs() * rel + U * xhat.abs()
                gam = D[f"gamma{l}"]
                ey = gam.abs() * exh + 2 * U * ((gam * xhat).abs() + D[f"beta{l}"].abs())
                m, n1 = f32(MOMENTUM), N / (N - 1)
                erm = m * em + 4 * U * ((1 - m) * D[f"rm{l}"].abs() + m * mean.abs())
                erv = m * ev * n1 + 6 * U * ((1 - m) * D[f"rv{l}"].abs() + m * var * n1)
                if c.keep:
                    _, xs, rss = split_saved(c, t["saved"], N)
                    worst = max(worst, check_elementwise(f"{what} xhat{l}", xs[l].cpu(), xhat, exh, "(n, c)"))
                    worst = max(worst, check_elementwise(f"{what} rstd{l}", rss[l].cpu(), rstd, rstd * rel, "(c,)"))
                worst = max(worst, check_elementwise(f"{what} rm{l}", t[f"rm{l}"].cpu(), r["rm"], erm, "(c,)"))
                worst = max(worst, check_elementwise(f"{what} rv{l}", t[f"rv{l}"].cpu(), r["rv"], erv, "(c,)"))
                assert t[f"nbt{l}"].item() == self.P[f"nbt{l}"].item() + 1, f"{what}: num_batches_tracked{l}"
            else:
                ey = eh
            ea = (1 + slope) * ey + U * r["a"].abs()
            worst = max(worst, check_elementwise(f"{what} a{l}", acts[l].cpu(), r["a"], ea, "(n, c)"))
        return worst


# ---- the per-case test -----------------------------------------------------------------------------------------------
def check_route(run):
    c = run.c
    seen = []
    for _ in range(3):
        run.prepare()
        seen = [(n, tuple(g)) for n, g in traced_kernels(lambda: run.call(torch.cuda.current_stream().cuda_stream))
                if n in gc.KERNEL.values()]
        if [n for n, _ in seen] == list(c.kernels):
            break
    if not seen:
        return "the profiler recorded no CUDA kernel activity on this machine"
    assert [n for n, _ in seen] == list(c.kernels), f"{c.id}: trace {seen}, table {c.kernels}"
    if torch.cuda.get_device_properties(0).multi_processor_count == gc.NUM_SMS:
        assert seen[0][1] == c.grid, f"{c.id}: grid {seen[0][1]}, table {c.grid}"
    return None


@pytest.mark.parametrize("case", gc.CASES, ids=lambda c: c.id)
def test_generator_case(case):
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

    if case.op == "fwd" and not case.keep:
        # the same call with a saved region computes the same out and running statistics, bit for bit
        kept = Run(gc.Case(case.name, "fwd", case.N, case.widths, case.norms, case.slope))
        kept.prepare()
        assert kept.call(torch.cuda.current_stream().cuda_stream) == 0
        torch.cuda.synchronize()
        worst = max(worst, kept.check(case.id + " kept"))
        for k, v in kept.outputs().items():
            if k in eager and k != "ws":
                assert torch.equal(v.view(torch.int32), eager[k].view(torch.int32)), f"{case.id}: {k} differs " \
                    "from the forward that keeps a saved region"

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
    for k, v in run.outputs().items():
        if k == "ws":
            continue
        same = v.view(torch.int32) == eager[k].view(torch.int32)
        assert same.all(), f"{case.id}: graph replay differs from the eager call in {k}"
    worst = max(worst, run.check(case.id + " graph"))
    print(f"\n{case.id}: worst |err|/bound {worst:.3g}, grid {case.grid}")
    if skip_reason:
        pytest.skip(skip_reason)
