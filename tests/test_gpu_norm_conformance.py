"""Every normalisation case of tests/norm_cases.py, element by element against torch float64.

Each case calls the C ABI directly on the guarded buffers of tests/conformance.py (Arena: NaN around the inputs,
outputs started as NaN, sentinels around everything the library writes) and runs its protocol: stats -> finalize ->
apply, then the backward, eagerly and replayed from a CUDA graph.  A LeakyReLU / ReLU backward gets scale_shift and no
saved output (the mask is recomputed from x); a Tanh / Sigmoid backward gets the saved output y.  Checked:
  - y, running_mean / running_var, num_batches_tracked, dx, dgamma / dbeta against fp64;
  - the statistics accumulator and the backward's sums workspace come back zeroed;
  - round_tf32 outputs are TF32-representable;
  - the trace shows the kernel instances, sample count and channel slices the table names.
The reference takes the activation's derivative from the kernel's own y (the mask of x * scale + shift in fp32, or
the saved output the library differentiates through), so an element next to a sign change cannot flip.  Bounds are
2^-16 relative to the magnitudes that enter each value (fp32 sums of at most a few dozen terms, then fp64):
an indexing error, a wrong channel's parameters or a lost slice is O(1).
"""
import pytest
import torch

import norm_cases as nc
from conformance import check_elementwise, run_case
from norm_cases import MOMENTUM, NBT0, SLOPE

pytestmark = pytest.mark.gpu

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
    """every output against fp64; the worst |err|/bound"""
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


class Run(nc.Run):
    def check(self, what):
        return check_outputs(self, what)


# the statistics and the backward's sums are fp64 atomics in no fixed order; everything formed from them may differ in
# its last bits between two calls
VARIES = ("y", "mean_rstd", "scale_shift", "dx", "dgb", "running_mean", "running_var")


def launches(c):
    """the table's kernel instances in launch order; a templated instance's grid has the samples (InstanceNorm: N) in y
    and the channel slices in z"""
    g = c.geom
    return [(k, (None, g.N if g.per_sample else 1, g.slices) if "<" in k else None) for k in c.kernels]


@pytest.mark.parametrize("case", nc.CASES, ids=lambda c: c.id)
def test_norm_case(case):
    run_case(Run(case), case.id, launches(case), varies=VARIES, family=("norm_",))
