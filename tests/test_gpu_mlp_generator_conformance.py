"""Every case of tests/generator_cases.py (csrc/mlp_generator/mlp_generator.cu), element by element against fp64.

Each case calls the C ABI on the guarded buffers of tests/conformance.py (Arena) and runs its protocol: outputs and
workspaces started as NaN, sentinels around everything the library writes.  The running statistics are inputs the forward updates
in place; they are read back and checked against the fp64 update.

The forward is checked layer by layer: each layer's reference starts from the kernel's own previous activations (the
saved region), so a bound covers one layer's rounding.  A forward without a saved region (torch.no_grad()) is checked
from the last hidden activation it leaves in its workspace and must repeat the saved-mode call bit for bit.  The
backward reads a saved region formed from the fp64 forward and rounded to fp32, so its reference is exact in its
inputs; bounds follow the conv suite: an fp32 chain of n products with s partials added outside it is within
2^-23 (n + s + 4) A of fp64, A the same sum over |terms|, carried from layer to layer (generator_cases.mmr).
tests/test_cpu_mlp_generator.py holds the references to torch float64 autograd.
"""
import ctypes
import re

import pytest
import torch

import generator_cases as gc
from b200gan import _lib
from conformance import Arena, check_elementwise, first_grid, not_vacuous, run_case
from generator_cases import EPS, F32, MOMENTUM, U, f32, gen_bwd_ref, gen_fwd_ref, make, saved_of, split_saved

pytestmark = pytest.mark.gpu


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
        worst = self.check_against_kept(what) if c.op == "fwd" and not c.keep else 0.0
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


    def check_against_kept(self, what):
        """the same call with a saved region computes the same out and running statistics, bit for bit"""
        c = self.c
        kept = Run(gc.Case(c.name, "fwd", c.N, c.widths, c.norms, c.slope))
        kept.prepare()
        assert kept.call(torch.cuda.current_stream().cuda_stream) == 0
        torch.cuda.synchronize()
        worst = kept.check(what + " kept")
        mine = self.outputs()
        for k, v in kept.outputs().items():
            if k in mine and k != "ws":
                assert torch.equal(v.view(torch.int32), mine[k].view(torch.int32)), f"{what}: {k} differs " \
                    "from the forward that keeps a saved region"
        return worst


# ---- the per-case test -----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", gc.CASES, ids=lambda c: c.id)
def test_generator_case(case):
    run_case(Run(case), case.id, first_grid(case.kernels, case.grid), refuse=(-2,) if case.error else (),
             varies=("ws",), family=tuple(gc.KERNEL.values()), num_sms=gc.NUM_SMS)
