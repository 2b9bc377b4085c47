"""Every normalisation case of tests/norm_cases.py, element by element against torch float64.

Each case calls the C ABI directly on guarded buffers (the Arena of the convolution conformance test: NaN around
the inputs, outputs started as NaN, sentinels around everything the library writes): stats -> finalize -> apply,
then the backward.  A LeakyReLU / ReLU backward gets scale_shift and no saved output (the mask is recomputed from
x); a Tanh / Sigmoid backward gets the saved output y.  Checked:
  - y, running_mean / running_var, num_batches_tracked, dx, dgamma / dbeta against fp64;
  - the statistics accumulator and the backward's sums workspace come back zeroed;
  - round_tf32 outputs are TF32-representable;
  - the trace shows the kernel instances, sample count and channel slices the table names.
The reference takes the activation's derivative from the kernel's own y (the mask of x * scale + shift in fp32, or
the saved output the library differentiates through), so an element next to a sign change cannot flip.  Bounds are
2^-16 relative to the magnitudes that enter each value (fp32 sums of at most a few dozen terms, then fp64):
an indexing error, a wrong channel's parameters or a lost slice is O(1).
"""
import ctypes

import pytest
import torch

import norm_cases as nc
from b200gan import _lib
from test_gpu_conv_conformance import Arena, traced_kernels

pytestmark = pytest.mark.gpu

TOL = 2.0 ** -16
U = 2.0 ** -23
SLOPE = 0.2
MOMENTUM = 0.1
NBT0 = 7
ACT_CODE = {"none": _lib.ACT_NONE, "lrelu": _lib.ACT_LRELU, "relu": _lib.ACT_RELU, "tanh": _lib.ACT_TANH,
            "sigmoid": _lib.ACT_SIGMOID}
LIPSCHITZ = {"none": 1.0, "lrelu": 1.0, "relu": 1.0, "tanh": 1.0, "sigmoid": 0.25}


def act_fwd(name, v):
    return {"none": lambda: v, "lrelu": lambda: torch.where(v > 0, v, v * SLOPE), "relu": lambda: v.clamp_min(0),
            "tanh": lambda: torch.tanh(v), "sigmoid": lambda: torch.sigmoid(v)}[name]()


def act_grad(name, y):
    """the derivative the library applies, from the kernel's output y"""
    return {"none": lambda: torch.ones_like(y), "lrelu": lambda: torch.where(y > 0, 1.0, SLOPE),
            "relu": lambda: (y > 0).double(), "tanh": lambda: 1 - y * y, "sigmoid": lambda: y * (1 - y)}[name]()


class Run:
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

    def call(self):
        """forward then backward on the current stream; the first failing return code, or 0"""
        lib, d, p, act = self.lib, ctypes.byref(self.d), self.ptr, self.c.act
        st = torch.cuda.current_stream().cuda_stream
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


def check(what, got, ref, bound):
    got = got.double().view_as(ref)
    assert not torch.isnan(got).any(), f"{what}: NaN at {tuple(torch.isnan(got).nonzero()[0].tolist())} " \
                                       "(an element never written, or a guard read)"
    err = (got - ref).abs()
    bad = (err > bound).nonzero()
    if bad.numel():
        at = tuple(bad[0].tolist())
        raise AssertionError(f"{what}: |err| {err[at].item():.3e} > bound {bound[at].item():.3e} at {at}; "
                             f"got {got[at].item():.9g}, fp64 {ref[at].item():.9g}")


def check_outputs(run):
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
    check(f"{c.id} y", y, y_ref, b)
    if c.rtf:
        assert ((t["y"].view(torch.int32) & 0x1FFF) == 0).all(), f"{c.id}: round_tf32 y not TF32-representable"
    assert (t["stats"] == 0).all(), f"{c.id}: the statistics accumulator is not handed back zeroed"
    if not g.per_sample:
        m, v = mean.view(-1), var.view(-1) * count / max(count - 1, 1)
        rm = (1 - MOMENTUM) * run.rm0.double() + MOMENTUM * m
        rv = (1 - MOMENTUM) * run.rv0.double() + MOMENTUM * v
        check(f"{c.id} running_mean", t["running_mean"], rm,
              TOL * (run.rm0.double().abs() + x.abs().mean(dims).view(-1)))
        check(f"{c.id} running_var", t["running_var"], rv, TOL * (run.rv0.double().abs() + v.abs()))
        assert t["nbt"].item() == NBT0 + 1, f"{c.id}: num_batches_tracked {t['nbt'].item()}"

    # backward, through the derivative of the kernel's own output
    dz = dy * act_grad(c.act, y.double())
    m1, m2 = dz.mean(dims, keepdim=True), (dz * xhat).mean(dims, keepdim=True)
    dx_ref = ga * rstd * (dz - m1 - xhat * m2)
    a1, a2 = dz.abs().mean(dims, keepdim=True), (dz * xhat).abs().mean(dims, keepdim=True)
    b = TOL * ga.abs() * rstd * (dz.abs() + a1 + xhat.abs() * a2)
    if c.rtf:
        b = b + 2.0 ** -11 * (dx_ref.abs() + b)
    dx = t["dx"].view(g.N, g.H * g.W, g.C)
    check(f"{c.id} dx", dx, dx_ref, b)
    if c.rtf:
        assert ((t["dx"].view(torch.int32) & 0x1FFF) == 0).all(), f"{c.id}: round_tf32 dx not TF32-representable"
    if g.affine:
        dgamma, dbeta = (dz * xhat).sum(dims).reshape(-1), dz.sum(dims).reshape(-1)
        check(f"{c.id} dgamma", t["dgb"][:run.G], dgamma, TOL * (dz * xhat).abs().sum(dims).reshape(-1))
        check(f"{c.id} dbeta", t["dgb"][run.G:], dbeta, TOL * dz.abs().sum(dims).reshape(-1))
    assert (t["sums"] == 0).all(), f"{c.id}: the backward's sums workspace is not handed back zeroed"


def check_route(run):
    """one profiler session, read once: the norm kernels in launch order, and the grids of the templated ones"""
    c, g = run.c, run.c.geom
    # CUPTI hands a session its activity buffer while the session's first launch is in cudaLaunchKernel (the trace
    # shows an "Activity Buffer Request" inside that call), and once earlier sessions have run in the process the
    # kernel record of that launch is lost while its runtime record stays.  So the session's first launch is a
    # marker whose record the check does not need.
    marker = torch.zeros(1, device="cuda")
    run.prepare()
    seen = [(n, grid) for n, grid in traced_kernels(lambda: (marker.zero_(), run.call())) if n.startswith("norm_")]
    if not seen:
        return "the profiler recorded no CUDA kernel activity on this machine"
    names = [n for n, _ in seen]
    assert names == list(c.kernels), f"{c.id}: trace {names}, table {list(c.kernels)}"
    for n, grid in seen:
        if "<" in n:
            assert tuple(grid[1:]) == (g.N if g.per_sample else 1, g.slices), \
                f"{c.id}: {n} grid {grid}: (samples, channel slices) should be ({g.N if g.per_sample else 1}, " \
                f"{g.slices})"
    return None


@pytest.mark.parametrize("case", nc.CASES, ids=lambda c: c.id)
def test_norm_case(case):
    run = Run(case)
    run.prepare()
    rc = run.call()
    torch.cuda.synchronize()
    assert rc == 0, f"{case.id}: rc {rc}: {run.lib.b200gan_last_error().decode()}"
    run.arena.check_guards(case.id)
    check_outputs(run)
    skip_reason = check_route(run)
    if skip_reason:
        pytest.skip(skip_reason)
