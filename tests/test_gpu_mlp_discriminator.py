"""The vanilla GAN discriminator (gan.py:64-80, bgan.py:66-80, aae.py:90-104) on the MLP critic kernels' Sigmoid mode:
b200gan_mlp_disc_fwd / _bwd element by element against torch float64, then functional.MlpDiscriminatorFn end to end.

Conformance: each case calls the C ABI on the guarded buffers of tests/conformance.py (Arena), runs its protocol and is
checked with the critic's references and bounds (tests/critic_cases.py).  Bounds added here:
  y = sigmoid(z):  the fp64 logit z is within ez of the kernel's (the critic's row-dot bound); sigmoid' = y (1 - y)
                   changes by at most a factor exp(ez) over that interval; expf is within 2 ulp and 1 + e and the
                   division round once each: |y - sigmoid(z)| <= y (1 - y) ez exp(ez) + 4 u y.
  g = dout y (1 - y):  three roundings, 2 u |g|; it is read from the workspace, and the critic backward of the
                   kernel's own g (critic_bwd_ref) bounds the seven gradients.
The route assertion names the kernel and its grid from a trace; a CUDA-graph replay repeats every output bit for bit.

End to end, against stock torch fp32 on the GPU (TF32 off): Sequential + BCELoss (output, dx and the six parameter
gradients within 1e-4 norm-relative, DESIGN.md section 2's bound for fp32 FFMA kernels), a create_graph=True penalty,
CUDA-graph replays of train.gan_step against an eager twin, and tests/scripts/mini_gan under the launcher."""
import copy
import ctypes
import math
import os
from dataclasses import dataclass

import pytest
import torch

import critic_cases as cr
from b200gan import _lib
from conformance import Arena, check_elementwise, first_grid, not_vacuous, run_case
from conftest import rel_err
from critic_cases import U, check_mask, critic_bwd_ref, mask, rowdot_n

pytestmark = pytest.mark.gpu
F32 = torch.float32
GRADS = ("dx", "dW1", "db1", "dW2", "db2", "dW3", "db3")


# ---- the case table --------------------------------------------------------------------------------------------------
@dataclass(frozen=True)
class Case:
    name: str
    op: str                 # fwd | bwd
    N: int
    Din: int
    H1: int = 512
    H2: int = 256
    slope: float = 0.2
    logits: str = "rand"    # rand | near0 (|z| < 0.01) | sat_pos / sat_neg (|z| > 20)
    null: tuple = ()        # bwd outputs passed as NULL
    no_y: bool = False      # refusal: no saved output
    no_ws: bool = False     # refusal: no workspace
    error: bool = False
    why: str = ""

    @property
    def id(self):
        return f"{self.op}-{self.name}"

    @property
    def kernels(self):
        return () if self.error else (cr.KERNEL[self.op],)

    @property
    def grid(self):
        return None if self.error else cr.GRID

    def outputs(self):
        return ("y", "m1", "a1", "m2", "a2") if self.op == "fwd" else tuple(o for o in GRADS if o not in self.null)


def _only(out):
    return tuple(o for o in GRADS if o != out)


CASES = []
for _op in ("fwd", "bwd"):
    CASES += [
        Case("gan", _op, 64, 784, why="gan.py / bgan.py at their defaults: batch 64, 28 x 28"),
        Case("aae", _op, 64, 10, why="aae.py: Din = latent_dim = 10"),
        Case("din1024", _op, 64, 1024, slope=0.0, why="Din = 1024 (32 x 32 images), slope 0"),
        Case("n1", _op, 1, 784, why="N = 1: one row"),
        Case("n2", _op, 2, 10, slope=1.0, why="N = 2, slope 1"),
        Case("n300", _op, 300, 1024, why="N = 300: many tiles per block of the persistent grid"),
        Case("near0", _op, 64, 784, logits="near0", why="logits near 0: y ~ 1/2, g ~ dout / 4"),
        Case("sat_pos", _op, 64, 784, logits="sat_pos", why="logits > 20: y = 1 in fp32, g = 0"),
        Case("sat_neg", _op, 64, 10, logits="sat_neg", why="logits < -20: y ~ 1e-10, tiny gradients"),
    ]
CASES += [Case(f"{o}_only", "bwd", 33, 10, 64, 31, null=_only(o), why=f"{o} alone") for o in GRADS]
CASES += [
    Case("none", "bwd", 33, 10, 64, 31, null=GRADS, why="no gradient at all: g, U1, U2 only"),
    Case("zero_n", "bwd", 0, 10, 64, 31, error=True, why="N = 0 is refused"),
    Case("no_y", "bwd", 33, 10, 64, 31, no_y=True, error=True, why="no saved output y is refused"),
    Case("no_ws", "bwd", 33, 10, 64, 31, no_ws=True, error=True, why="no workspace is refused"),
    Case("zero_n", "fwd", 0, 10, 64, 31, error=True, why="N = 0 is refused"),
]


def test_case_table_covers_its_edges():
    ids = [c.id for c in CASES]
    assert len(ids) == len(set(ids)) and all(c.why for c in CASES)
    for op in ("fwd", "bwd"):
        ok = [c for c in CASES if c.op == op and not c.error]
        assert {1, 2, 64, 300} <= {c.N for c in ok} and {10, 784, 1024} <= {c.Din for c in ok}, op
        assert {0.0, 0.2, 1.0} <= {c.slope for c in ok} and {"near0", "sat_pos", "sat_neg"} <= {c.logits for c in ok}
    assert {f"{o}_only" for o in GRADS} <= {c.name for c in CASES if c.op == "bwd"}


# ---- one case as tensors ---------------------------------------------------------------------------------------------
def _fwd64(x, P, slope, m1=None, m2=None):
    """h1, h2 and the logit z in fp64, each layer from the given masks (None: the fp64 signs)"""
    h1 = x @ P["W1"].t() + P["b1"]
    m1 = mask(h1, slope) if m1 is None else m1
    a1 = h1 * m1
    h2 = a1 @ P["W2"].t() + P["b2"]
    m2 = mask(h2, slope) if m2 is None else m2
    a2 = h2 * m2
    return h1, m1, a1, h2, m2, a2, (a2 @ P["W3"].t()).reshape(-1) + P["b3"]


class Run:
    def __init__(self, c, seed=0):
        self.c, self.lib = c, _lib.load()
        g = torch.Generator().manual_seed(seed)
        rn = lambda *s, scale=1.0: (torch.randn(*s, generator=g) * scale).cuda()  # noqa: E731
        N, Din, H1, H2 = max(c.N, 1), c.Din, c.H1, c.H2
        self.d = _lib.MlpCriticDesc(c.N, Din, H1, H2, c.slope)
        P = dict(W1=rn(H1, Din, scale=1 / math.sqrt(Din)), b1=rn(H1, scale=0.2), W2=rn(H2, H1, scale=1 / math.sqrt(H1)),
                 b2=rn(H2, scale=0.2), W3=rn(1, H2, scale=1 / math.sqrt(H2)), b3=rn(1, scale=0.2))
        if c.logits == "near0":
            P["W3"] *= 1e-3
            P["b3"].zero_()
        elif c.logits in ("sat_pos", "sat_neg"):
            P["W3"] *= 0.1
            P["b3"].fill_(25.0 if c.logits == "sat_pos" else -25.0)
        specs, data = [], dict(P)
        ins = lambda name, t: (specs.append((name, t.numel(), F32, "in")), data.__setitem__(name, t))  # noqa: E731
        outs = lambda name, n, role="out": specs.append((name, n, F32, role))  # noqa: E731
        for k, v in P.items():
            ins(k, v)
        x = rn(N, Din)
        ins("x", x)
        slope32 = torch.tensor(c.slope, dtype=F32).item()
        f = _fwd64(x.double(), {k: v.double() for k, v in P.items()}, slope32)
        self.z64 = f[6]
        if c.op == "fwd":
            for name, n in (("y", N), ("m1", N * H1), ("a1", N * H1), ("m2", N * H2), ("a2", N * H2)):
                outs(name, n)
        else:
            for name, t in (("m1", f[1]), ("a1", f[2]), ("m2", f[4]), ("a2", f[5]), ("y", torch.sigmoid(f[6]))):
                if not (c.no_y and name == "y"):
                    ins(name, t.float())
            ins("dout", rn(N))
            for name, n in (("dx", N * Din), ("dW1", H1 * Din), ("db1", H1), ("dW2", H2 * H1), ("db2", H2),
                            ("dW3", H2), ("db3", 1)):
                if name not in c.null:
                    outs(name, n)
            if not c.no_ws:
                outs("ws", max(self.lib.b200gan_mlp_disc_bwd_workspace_floats(ctypes.byref(self.d)), 1), "ws")
        self.arena, self.data = Arena(specs), data

    def prepare(self):
        self.arena.prepare(self.data)

    def outputs(self):
        return self.arena.outputs()

    def call(self, st):
        p, d, L = self.arena.ptr, ctypes.byref(self.d), self.lib
        if self.c.op == "fwd":
            return L.b200gan_mlp_disc_fwd(d, p("x"), p("W1"), p("b1"), p("W2"), p("b2"), p("W3"), p("b3"), p("y"),
                                          p("m1"), p("a1"), p("m2"), p("a2"), st)
        return L.b200gan_mlp_disc_bwd(d, p("dout"), p("y"), p("x"), p("W1"), p("W2"), p("W3"), p("m1"), p("a1"),
                                      p("m2"), p("a2"), *[p(o) for o in GRADS], p("ws"), st)

    def check(self, what):
        c, t, D = self.c, self.arena.t, {k: v.double() for k, v in self.data.items()}
        N, Din, H1, H2 = c.N, c.Din, c.H1, c.H2
        slope = torch.tensor(c.slope, dtype=F32).item()
        if c.op == "fwd":
            x = D["x"]
            h1 = x @ D["W1"].t() + D["b1"]
            eh1 = U * (Din + 5) * (x.abs() @ D["W1"].abs().t() + D["b1"].abs())
            check_mask(what + " m1", t["m1"], h1, eh1, slope)
            m1 = t["m1"].double().view(N, H1)
            worst = check_elementwise(what + " a1", t["a1"], h1 * m1, eh1 * m1 + U * (h1 * m1).abs(), "(n, i)")
            a1 = t["a1"].double().view(N, H1)
            h2 = a1 @ D["W2"].t() + D["b2"]
            eh2 = U * (H1 + 5) * (a1.abs() @ D["W2"].abs().t() + D["b2"].abs())
            check_mask(what + " m2", t["m2"], h2, eh2, slope)
            m2 = t["m2"].double().view(N, H2)
            worst = max(worst, check_elementwise(what + " a2", t["a2"], h2 * m2, eh2 * m2 + U * (h2 * m2).abs(),
                                                 "(n, j)"))
            a2 = t["a2"].double().view(N, H2)
            z = (a2 @ D["W3"].t()).reshape(-1) + D["b3"]
            ez = U * (rowdot_n(H2) + 5) * ((a2.abs() @ D["W3"].abs().t()).reshape(-1) + D["b3"].abs())
            y = torch.sigmoid(z)
            ey = y * (1 - y) * ez * torch.exp(ez) + 4 * U * y
            return max(worst, check_elementwise(what + " y", t["y"], y, ey, "(n,)"))
        y, dout = D["y"], D["dout"]
        g = dout * y * (1 - y)
        gk = t["ws"][N * (H1 + H2):N * (H1 + H2 + 1)]
        worst = check_elementwise(what + " g", gk, g, 2 * U * g.abs(), "(n,)")
        r = critic_bwd_ref(gk.double(), D["x"], D["W1"], D["W2"], D["W3"].view(-1), D["m1"].view(N, H1),
                           D["a1"].view(N, H1), D["m2"].view(N, H2), D["a2"].view(N, H2))
        for name in c.outputs():
            val, b, *term = r[name]
            worst = max(worst, check_elementwise(f"{what} {name}", t[name], val.reshape(-1), b.reshape(-1), "(flat)"))
            if term:
                not_vacuous(f"{what} {name}", b.reshape(-1), term[0].reshape(-1))
        return worst


@pytest.mark.parametrize("case", CASES, ids=lambda c: c.id)
def test_disc_case(case):
    run = Run(case)
    z = run.z64
    if case.logits == "near0":
        assert z.abs().max() < 0.01, case.id
    elif case.logits.startswith("sat"):
        assert z.abs().min() > 20 and (z > 0).all() == (case.logits == "sat_pos"), case.id
    run_case(run, case.id, first_grid(case.kernels, case.grid), refuse=(-2,) if case.error else (),
             family=tuple(cr.KERNEL.values()), num_sms=cr.NUM_SMS)


# ---- the module path ------------------------------------------------------------------------------------------------
@pytest.fixture(autouse=True)
def _fp32():
    prev = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32 = prev


@pytest.fixture
def calls(monkeypatch):
    """Counts of the discriminator's forward and backward issued through ops."""
    from b200gan import ops
    n = {"fwd": 0, "bwd": 0}
    for k in n:
        fn = getattr(ops, "mlp_disc_" + k)

        def wrapped(*a, _fn=fn, _k=k, **kw):
            n[_k] += 1
            return _fn(*a, **kw)
        monkeypatch.setattr(ops, "mlp_disc_" + k, wrapped)
    return n


def _pair(din, seed=0):
    from b200gan import zoo
    torch.manual_seed(seed)
    ref = zoo.GANDiscriminator((din,), nn=zoo.namespace(stock=True)).cuda()
    ours = zoo.GANDiscriminator((din,)).cuda()
    ours.load_state_dict(ref.state_dict())
    return ref, ours


@pytest.mark.parametrize("din", [784, 10], ids=["gan", "aae"])
def test_sequential_with_bce_against_stock(din, calls):
    from b200gan import nn as bnn
    ref, ours = _pair(din, seed=1)
    assert isinstance(ours.model, bnn.Sequential)
    x = torch.randn(64, din, device="cuda") * 0.5
    target = (torch.rand(64, 1, device="cuda") > 0.5).float()
    xr, xo = x.clone().requires_grad_(True), x.clone().requires_grad_(True)
    yr, yo = ref(xr), ours(xo)
    assert calls == {"fwd": 1, "bwd": 0} and rel_err(yo, yr) < 1e-4
    bnn.BCELoss()(yo, target).backward()
    torch.nn.BCELoss()(yr, target).backward()
    assert calls == {"fwd": 1, "bwd": 1}
    assert rel_err(xo.grad, xr.grad) < 1e-4
    for (k, po), (_, pr) in zip(ours.named_parameters(), ref.named_parameters()):
        assert rel_err(po.grad, pr.grad) < 1e-4, k
    with torch.no_grad():   # no node, the same forward
        y = ours(xo)
    assert y.grad_fn is None and calls["fwd"] == 2 and rel_err(y, yr) < 1e-4


def test_create_graph_penalty_matches_stock(calls):
    """a gradient penalty through the discriminator (autograd.grad(create_graph=True)) recomputes the six modules with
    torch ops: the penalty and every parameter gradient of loss + penalty match stock fp32"""
    ref, ours = _pair(784, seed=2)
    x = torch.randn(32, 784, device="cuda") * 0.5
    out = []
    for net in (ref, ours):
        xi = x.clone().requires_grad_(True)
        y = net(xi)
        gx, = torch.autograd.grad(y, xi, torch.ones_like(y), create_graph=True)
        gp = ((gx.norm(2, dim=1) - 1) ** 2).mean()
        (y.mean() + 10.0 * gp).backward()
        out.append((gp.detach(), [p.grad.clone() for p in net.parameters()]))
    # the penalty's backward ran the torch recomputation; the first-order backward of y.mean() the kernel
    assert calls == {"fwd": 1, "bwd": 1}
    assert rel_err(out[1][0], out[0][0]) < 1e-4
    for go, gr in zip(out[1][1], out[0][1]):
        assert rel_err(go, gr) < 1e-4


def test_gan_step_graph_replays_match_an_eager_twin(calls):
    """train.gan_step (gan.py:124-161) at batch 64, 28 x 28, with the capturable Adam, captured with train.GraphedStep:
    the replays match an eager twin step for step, parameters and running statistics included"""
    from b200gan import optim, train, zoo
    torch.manual_seed(0)
    g = zoo.WGANGPGenerator((1, 28, 28)).cuda()
    d = zoo.GANDiscriminator((1, 28, 28)).cuda()
    g2, d2 = copy.deepcopy(g), copy.deepcopy(d)

    def make_step(g, d):
        og = optim.Adam(g.parameters(), lr=2e-4, betas=(0.5, 0.999))
        od = optim.Adam(d.parameters(), lr=2e-4, betas=(0.5, 0.999))

        def step(imgs, z):
            gl, dl, _ = train.gan_step(g, d, og, od, imgs, z)
            return torch.stack([gl, dl])
        return step

    def inputs(seed):
        gen = torch.Generator("cuda").manual_seed(seed)
        return (torch.rand(64, 1, 28, 28, device="cuda", generator=gen) * 2 - 1,
                torch.randn(64, 100, device="cuda", generator=gen))

    graphed = train.GraphedStep(make_step(g, d), inputs(0))
    assert calls == {"fwd": 12, "bwd": 12}      # three D passes and three D backwards per step, four steps
    eager = make_step(g2, d2)
    for _ in range(3):
        eager(*inputs(0))
    for seed in (1, 2, 3):
        a = graphed(*inputs(seed)).clone()
        b = eager(*inputs(seed))
        assert rel_err(a, b) < 1e-5, seed
    torch.cuda.synchronize()
    # the bias of a Linear in front of a BatchNorm1d gets a gradient that is zero but for rounding, whose sign Adam turns
    # into +-lr: there two evaluations may differ by up to 2 lr per element and step
    pre_norm = {f"model.{i}.bias" for i, m in enumerate(g.model) if isinstance(m, torch.nn.Linear)
                and i + 1 < len(g.model) and isinstance(g.model[i + 1], torch.nn.BatchNorm1d)}
    for (k, x), (_, y) in zip(list(g.named_parameters()) + list(g.named_buffers()) + list(d.named_parameters()),
                              list(g2.named_parameters()) + list(g2.named_buffers()) + list(d2.named_parameters())):
        if k in pre_norm:
            assert (x - y).abs().max().item() <= 2 * 2e-4 * 6 * 1.01, k
        else:
            assert rel_err(x, y) < 1e-5, k


def test_gan_step_against_stock(calls):
    """three train.gan_step steps on the drop-ins against the stock modules (fp32, torch Adam on both)"""
    from b200gan import train, zoo
    torch.manual_seed(4)
    g_ref = zoo.WGANGPGenerator((1, 28, 28), nn=zoo.namespace(stock=True)).cuda()
    d_ref = zoo.GANDiscriminator((1, 28, 28), nn=zoo.namespace(stock=True)).cuda()
    g, d = zoo.WGANGPGenerator((1, 28, 28)).cuda(), zoo.GANDiscriminator((1, 28, 28)).cuda()
    g.load_state_dict(g_ref.state_dict())
    d.load_state_dict(d_ref.state_dict())
    opt = lambda ps: torch.optim.Adam(ps, lr=2e-4, betas=(0.5, 0.999))  # noqa: E731
    ogr, odr, og, od = opt(g_ref.parameters()), opt(d_ref.parameters()), opt(g.parameters()), opt(d.parameters())
    for it in range(3):
        gen = torch.Generator("cuda").manual_seed(10 + it)
        imgs = torch.rand(64, 1, 28, 28, device="cuda", generator=gen) * 2 - 1
        z = torch.randn(64, 100, device="cuda", generator=gen)
        glr, dlr, _ = train.gan_step(g_ref, d_ref, ogr, odr, imgs, z)
        gl, dl, _ = train.gan_step(g, d, og, od, imgs, z)
        assert abs(gl.item() - glr.item()) < 1e-3 * abs(glr.item()), it
        assert abs(dl.item() - dlr.item()) < 1e-3 * abs(dlr.item()), it
    assert calls == {"fwd": 9, "bwd": 9}
    for (k, po), (_, pr) in zip(d.named_parameters(), d_ref.named_parameters()):
        assert rel_err(po, pr) < 1e-3, k


def test_reference_idiom_gan_script_under_the_launcher_on_cuda(calls):
    """launch.run() of tests/scripts/mini_gan (Linear / LeakyReLU / Sigmoid discriminator) on the GPU: stock torch
    against the drop-ins, same seeds: the printed losses agree and the patched run called the discriminator ops"""
    from b200gan import launch
    script = os.path.join(os.path.dirname(os.path.abspath(__file__)), "scripts", "mini_gan", "mini_gan.py")
    args = ["--epochs", "1", "--batch_size", "32"]
    ref = launch.run(script, args, iters=3, seed=0, stock=True, quiet=True)
    assert calls == {"fwd": 0, "bwd": 0}
    ours = launch.run(script, args, iters=3, seed=0, stock=False, quiet=True)
    assert calls == {"fwd": 9, "bwd": 9}

    def losses(run):
        rows = [line for line in run["__b200_stdout__"].splitlines() if "[D " in line]
        return [(float(r.split("[D ")[1].split("]")[0]), float(r.split("[G ")[1].split("]")[0])) for r in rows]
    lr, lo = losses(ref), losses(ours)
    assert len(lr) == len(lo) == 3
    for (dr, gr), (do, go) in zip(lr, lo):
        assert abs(do - dr) < 2e-3 * max(abs(dr), 1.0) and abs(go - gr) < 2e-3 * max(abs(gr), 1.0), (lr, lo)
