"""Case table of the normalisation entry points (b200gan_norm_stats / finalize / apply / bwd).

One geometry per edge of the apply and backward kernels' plan, each run with every fused activation, together with
what the library must launch for it: the vector width VEC of the norm_apply / norm_bwd_reduce / norm_bwd_apply
instances (4 when C % 4 == 0 and the streamed tensors are 16-byte aligned, else 1) and the number of channel slices
of at most 256 groups in gridDim.z.  Written from the launchers in pytorch-gan_b200/csrc/norm.cu, not from a run.

tests/test_cpu_norm_case_table.py checks it against the kernels the source declares and launches;
tests/test_gpu_norm_conformance.py runs every case against torch float64.
"""
import ctypes
from dataclasses import dataclass

import torch

from b200gan import _lib
from conformance import Arena, check_elementwise

ACTS = ("none", "lrelu", "relu", "tanh", "sigmoid")
KERNELS = {"norm_stats_kernel", "norm_finalize_kernel", "norm_apply_kernel", "norm_bwd_reduce_kernel",
           "norm_bwd_apply_kernel", "norm_bwd_params_kernel"}     # what norm.cu declares


@dataclass(frozen=True)
class Geom:
    name: str
    N: int
    C: int
    H: int
    W: int
    per_sample: bool      # InstanceNorm2d (groups n*C + c) rather than BatchNorm2d (groups c)
    affine: bool
    vec: int              # expected VEC of the apply / backward instances
    slices: int = 1       # expected gridDim.z
    offset: int = 0       # floats between x's aligned allocation and x (1 misaligns every float4)
    why: str = ""


GEOMS = (
    Geom("c3", 4, 3, 16, 16, False, True, vec=1, why="C % 4 != 0: 85 rows of 3 groups per block, 1 thread left over"),
    Geom("c5", 3, 5, 12, 12, True, False, vec=1, why="InstanceNorm with N > 1 at VEC 1: 51 rows of 5, 1 left over"),
    Geom("c16", 8, 16, 8, 8, False, True, vec=4, why="reference layer width: 4 groups, 64 rows per block"),
    Geom("c64", 2, 64, 16, 16, True, False, vec=4, why="reference InstanceNorm(64)"),
    Geom("c128", 4, 128, 8, 8, False, True, vec=4, why="reference BatchNorm(128)"),
    Geom("c512", 2, 512, 4, 4, True, False, vec=4, why="reference InstanceNorm(512): 128 groups, 2 rows per block"),
    Geom("c96", 4, 96, 8, 8, False, True, vec=4, why="256 % 24 != 0: 10 rows per block, 16 threads left over"),
    Geom("c768", 2, 768, 4, 4, True, False, vec=4, why="192 groups: one row per block, 64 threads left over"),
    Geom("c1280", 2, 1280, 4, 4, False, True, vec=4, slices=2, why="320 groups: slices of 256 and 64 groups"),
    Geom("c258", 2, 258, 4, 4, True, True, vec=1, slices=2,
         why="affine InstanceNorm at VEC 1 with slices of 256 and 2 channels: gamma indexed by channel"),
    Geom("c64_off", 4, 64, 8, 8, False, True, vec=1, offset=1, why="x one float past 16-byte alignment: VEC 1"),
    Geom("bn_hw1", 64, 128, 1, 1, False, True, vec=4, why="BatchNorm over a 1x1 map: the batch is the whole group"),
)


@dataclass(frozen=True)
class Case:
    geom: Geom
    act: str
    rtf: bool             # round_tf32 on y and dx

    @property
    def kernels(self):
        """the kernel instances a forward (stats, finalize, apply) and a backward launch, in order"""
        v = self.geom.vec
        return ("norm_stats_kernel", "norm_finalize_kernel", f"norm_apply_kernel<{v}>",
                f"norm_bwd_reduce_kernel<{v}>", f"norm_bwd_apply_kernel<{v}>", "norm_bwd_params_kernel")

    @property
    def id(self):
        return f"{self.geom.name}-{self.act}{'-rtf' if self.rtf else ''}"


# every geometry with every activation; round_tf32 alternates so that each activation runs with it on and off
CASES = tuple(Case(g, a, (i + j) % 2 == 1) for i, g in enumerate(GEOMS) for j, a in enumerate(ACTS))


# ---- runs and references -------------------------------------------------------------------------------------------
SLOPE = 0.2
MOMENTUM = 0.1
NBT0 = 7
ACT_CODE = {"none": _lib.ACT_NONE, "lrelu": _lib.ACT_LRELU, "relu": _lib.ACT_RELU, "tanh": _lib.ACT_TANH,
            "sigmoid": _lib.ACT_SIGMOID}


class Run:
    """one case on guarded buffers: stats -> finalize -> apply, then the backward"""

    def __init__(self, case, seed=0):
        self.c, g = case, case.geom
        self.lib = _lib.load()
        self.G = g.N * g.C if g.per_sample else g.C
        self.numel = g.N * g.H * g.W * g.C
        self.eps = 1e-5 if g.per_sample else 0.8
        gen = torch.Generator().manual_seed(seed)
        self.x = (torch.randn(g.N, g.H * g.W, g.C, generator=gen) * 2 + 0.5).cuda()
        self.dy = torch.randn(g.N, g.H * g.W, g.C, generator=gen).cuda()
        self.gamma = (1 + 0.5 * torch.randn(g.C, generator=gen)).cuda()
        self.beta = (0.3 * torch.randn(g.C, generator=gen)).cuda()
        self.rm0 = (0.1 * torch.randn(g.C, generator=gen)).cuda()
        self.rv0 = (1 + torch.rand(g.C, generator=gen)).cuda()
        f32, f64 = torch.float32, torch.float64
        specs = [("x", self.numel + g.offset, f32, "in"), ("dy", self.numel, f32, "in"),
                 ("y", self.numel, f32, "out"), ("mean_rstd", 2 * self.G, f32, "out"),
                 ("scale_shift", 2 * self.G, f32, "out"), ("dx", self.numel, f32, "out"),
                 ("stats", 2 * self.G, f64, "ws"), ("sums", 2 * self.G, f64, "ws")]
        if g.affine:
            specs += [("gamma", g.C, f32, "in"), ("beta", g.C, f32, "in"), ("dgb", 2 * self.G, f32, "out")]
        if not g.per_sample:
            specs += [("running_mean", g.C, f32, "ws"), ("running_var", g.C, f32, "ws"), ("nbt", 1, torch.int64, "in")]
        self.arena = Arena(specs)
        lead = torch.full((g.offset,), float("nan"), device="cuda")
        self.data = dict(x=torch.cat([lead, self.x.reshape(-1)]), dy=self.dy, gamma=self.gamma, beta=self.beta,
                         nbt=torch.tensor([NBT0], device="cuda"))
        self.d = _lib.NormDesc(g.N, g.H * g.W, g.C, int(g.per_sample), self.eps, MOMENTUM, ACT_CODE[case.act], SLOPE,
                               int(case.rtf))

    def prepare(self):
        a = self.arena
        a.prepare(self.data)
        a.t["stats"].zero_()
        a.t["sums"].zero_()
        if "running_mean" in a.t:
            a.t["running_mean"].copy_(self.rm0)
            a.t["running_var"].copy_(self.rv0)

    def ptr(self, name):
        p = self.arena.ptr(name)
        return p + 4 * self.c.geom.offset if name == "x" else p

    def outputs(self):
        return self.arena.outputs()

    def call(self, st):
        """forward then backward on stream st; the first failing return code, or 0"""
        lib, d, p, act = self.lib, ctypes.byref(self.d), self.ptr, self.c.act
        for rc in (lambda: lib.b200gan_norm_stats(d, p("x"), p("stats"), st),
                   lambda: lib.b200gan_norm_finalize(d, p("stats"), p("gamma"), p("beta"), p("mean_rstd"),
                                                     p("scale_shift"), p("running_mean"), p("running_var"), p("nbt"),
                                                     st),
                   lambda: lib.b200gan_norm_apply(d, p("x"), p("scale_shift"), p("y"), st),
                   lambda: lib.b200gan_norm_bwd(d, p("dy"), p("x"), p("y") if act in ("tanh", "sigmoid") else None,
                                                p("mean_rstd"), p("scale_shift") if act in ("lrelu", "relu") else None,
                                                p("gamma"), p("sums"), p("dx"), p("dgb"), st)):
            code = rc()
            if code:
                return code
        return 0


def mask(act, pre):
    if act == "lrelu":
        return torch.where(pre > 0, torch.ones_like(pre), torch.full_like(pre, SLOPE))
    if act == "relu":
        return (pre > 0).to(pre.dtype)
    return torch.ones_like(pre)


def closed_form(x, dy, gamma, beta, u, ugamma, ubeta, eps, act, per_sample, ap=None):
    """(dL/d(dy), dL/dx, dL/d(gamma) per channel or None) on NCHW tensors, any dtype; gamma/beta None = non-affine,
    ugamma/ubeta None = 0; ap: the activation's mask, else computed from the normalised x"""
    n, c = x.shape[:2]
    dims = (2, 3) if per_sample else (0, 2, 3)
    m = x[0, 0].numel() * (1 if per_sample else n)
    ch = (1, c, 1, 1)
    mean = x.mean(dims, keepdim=True)
    r = 1 / torch.sqrt(((x - mean) ** 2).mean(dims, keepdim=True) + eps)
    xh = (x - mean) * r
    ga = gamma.view(ch) if gamma is not None else 1.0
    be = beta.view(ch) if beta is not None else 0.0
    ap = mask(act, ga * xh + be) if ap is None else ap
    g = dy * ap
    A, B = g.sum(dims, keepdim=True) / m, (g * xh).sum(dims, keepdim=True) / m
    U, T, Q = u.sum(dims, keepdim=True), (u * xh).sum(dims, keepdim=True), (u * g).sum(dims, keepdim=True)
    ug = ugamma.view(ch) if ugamma is not None else 0.0
    ub = ubeta.view(ch) if ubeta is not None else 0.0
    gdy = ap * (ga * r * (u - U / m - xh * T / m) + ug * xh + ub)
    gx = ug * r * (g - A - xh * B) - (ga * r * r / m) * (xh * (Q - A * U - 3 * B * T) + T * (g - A) + B * (m * u - U))
    ggamma = None
    if gamma is not None:
        ggamma = (r * (Q - A * U - B * T)).sum(0).view(c)
    return gdy, gx, ggamma


# ---- element-wise checks of a run (tests/test_gpu_norm_conformance.py, tests/test_gpu_norm_statistics.py) ----------
TOL = 2.0 ** -16
U = 2.0 ** -23
LIPSCHITZ = {"none": 1.0, "lrelu": 1.0, "relu": 1.0, "tanh": 1.0, "sigmoid": 0.25}


def act_fwd(name, v):
    return {"none": lambda: v, "lrelu": lambda: torch.where(v > 0, v, v * SLOPE), "relu": lambda: v.clamp_min(0),
            "tanh": lambda: torch.tanh(v), "sigmoid": lambda: torch.sigmoid(v)}[name]()


def act_grad(name, y):
    """the derivative the library applies, from the kernel's output y"""
    return {"none": lambda: torch.ones_like(y), "lrelu": lambda: torch.where(y > 0, 1.0, SLOPE),
            "relu": lambda: (y > 0).double(), "tanh": lambda: 1 - y * y, "sigmoid": lambda: y * (1 - y)}[name]()


def check_outputs(run, what):
    """every output of a Run against fp64 (from run.x and run.dy); the worst |err|/bound.  Bounds are 2^-16 relative to
    the magnitudes that enter each value; the statistics themselves are held to their summation chains by
    tests/test_gpu_norm_statistics.py"""
    c, g, t = run.c, run.c.geom, run.arena.t
    x, dy = run.x.double(), run.dy.double()
    dims = (1,) if g.per_sample else (0, 1)
    count = g.H * g.W * (1 if g.per_sample else g.N)
    mean = x.mean(dims, keepdim=True)
    var = ((x - mean) ** 2).mean(dims, keepdim=True)
    rstd = 1 / torch.sqrt(var + run.eps)
    ga = run.gamma.double() if g.affine else torch.ones(g.C, dtype=torch.float64, device="cuda")
    be = run.beta.double() if g.affine else torch.zeros(g.C, dtype=torch.float64, device="cuda")

    # forward
    xhat = (x - mean) * rstd
    pre = xhat * ga + be
    y_ref = act_fwd(c.act, pre)
    b = LIPSCHITZ[c.act] * TOL * ((x.abs() + mean.abs()) * rstd * ga.abs() + be.abs()) + 4 * U * y_ref.abs()
    if c.rtf:
        b = b + 2.0 ** -11 * (y_ref.abs() + b)
    y = t["y"].view(g.N, g.H * g.W, g.C)
    worst = check_elementwise(f"{what} y", y, y_ref, b)
    if c.rtf:
        assert ((t["y"].view(torch.int32) & 0x1FFF) == 0).all(), f"{what}: round_tf32 y not TF32-representable"
    assert (t["stats"] == 0).all(), f"{what}: the statistics accumulator is not handed back zeroed"
    if not g.per_sample:
        m, v = mean.view(-1), var.view(-1) * count / max(count - 1, 1)
        rm = (1 - MOMENTUM) * run.rm0.double() + MOMENTUM * m
        rv = (1 - MOMENTUM) * run.rv0.double() + MOMENTUM * v
        worst = max(worst, check_elementwise(f"{what} running_mean", t["running_mean"], rm,
                                             TOL * (run.rm0.double().abs() + x.abs().mean(dims).view(-1))))
        worst = max(worst, check_elementwise(f"{what} running_var", t["running_var"], rv,
                                             TOL * (run.rv0.double().abs() + v.abs())))
        assert t["nbt"].item() == NBT0 + 1, f"{what}: num_batches_tracked {t['nbt'].item()}"

    # backward, through the derivative of the kernel's own output
    dz = dy * act_grad(c.act, y.double())
    m1, m2 = dz.mean(dims, keepdim=True), (dz * xhat).mean(dims, keepdim=True)
    dx_ref = ga * rstd * (dz - m1 - xhat * m2)
    a1, a2 = dz.abs().mean(dims, keepdim=True), (dz * xhat).abs().mean(dims, keepdim=True)
    b = TOL * ga.abs() * rstd * (dz.abs() + a1 + xhat.abs() * a2)
    if c.rtf:
        b = b + 2.0 ** -11 * (dx_ref.abs() + b)
    dx = t["dx"].view(g.N, g.H * g.W, g.C)
    worst = max(worst, check_elementwise(f"{what} dx", dx, dx_ref, b))
    if c.rtf:
        assert ((t["dx"].view(torch.int32) & 0x1FFF) == 0).all(), f"{what}: round_tf32 dx not TF32-representable"
    if g.affine:
        dgamma, dbeta = (dz * xhat).sum(dims).reshape(-1), dz.sum(dims).reshape(-1)
        worst = max(worst, check_elementwise(f"{what} dgamma", t["dgb"][:run.G], dgamma,
                                             TOL * (dz * xhat).abs().sum(dims).reshape(-1)))
        worst = max(worst, check_elementwise(f"{what} dbeta", t["dgb"][run.G:], dbeta,
                                             TOL * dz.abs().sum(dims).reshape(-1)))
    assert (t["sums"] == 0).all(), f"{what}: the backward's sums workspace is not handed back zeroed"
    return worst
