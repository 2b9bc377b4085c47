"""Gradient penalties through training-mode BatchNorm2d / InstanceNorm2d (SURVEY.md 8f N2) on the GPU.

C ABI: b200gan_norm_dbwd on every geometry of tests/norm_cases.py with none / LeakyReLU / ReLU, on guarded buffers
(the Arena of tests/conformance.py), against the fp64 closed form of tests/norm_cases.py (held to torch float64 double
backward by tests/test_cpu_norm_double_backward.py) taking the mask from the kernel's own forward output (so an element next to a sign change cannot flip).  Bounds are
2^-16 relative to the magnitudes that enter each value, as in test_gpu_norm_conformance.py.  Also: every output asked for
alone, the workspace handed back zeroed, Tanh / Sigmoid refused, a bit-identical CUDA-graph replay, and the kernel
instances of every case, traced in one profiler session.

Modules: the DRAGAN penalty (dragan.py:144-167) on the DCGAN discriminator as a fused chain and unfused, a mixed loss on
one forward, and the DualGAN WGAN-GP critic (dualgan/models.py:102-123) with BatchNorm2d(.8) and with an affine
InstanceNorm2d, each against stock fp32 torch on the same GPU with the same seeds; the refusals; a captured critic
iteration; and a script in the reference's idiom under the launcher.
"""
import copy
import ctypes
import os

import pytest
import torch

import norm_cases as nc
from b200gan import _lib
from conformance import Arena, check_elementwise, check_route
from conftest import rel_err
from norm_cases import ACT_CODE, SLOPE, Run, closed_form

pytestmark = pytest.mark.gpu

TOL = 2.0 ** -16
ACTS = ("none", "lrelu", "relu")
CASES = [nc.Case(g, a, False) for g in nc.GEOMS for a in ACTS]


def nchw(t, g):
    return t.double().view(g.N, g.H, g.W, g.C).permute(0, 3, 1, 2)


class DRun:
    """The forward of Run (stats, finalize, apply), then b200gan_norm_dbwd on a second guarded arena"""

    def __init__(self, case):
        self.fwd = Run(case, seed=1)
        self.fwd.prepare()
        assert self.fwd.call(torch.cuda.current_stream().cuda_stream) == 0
        torch.cuda.synchronize()
        g, f = case.geom, self.fwd
        self.c, self.g, self.G, self.lib = case, g, f.G, f.lib
        gen = torch.Generator().manual_seed(7)
        self.u = torch.randn(g.N, g.H * g.W, g.C, generator=gen).cuda()
        self.ugb = torch.randn(2 * g.C, generator=gen).cuda() if g.affine else None
        f32, f64 = torch.float32, torch.float64
        specs = [("x", f.numel + g.offset, f32, "in"), ("dy", f.numel, f32, "in"), ("u", f.numel, f32, "in"),
                 ("mean_rstd", 2 * f.G, f32, "in"), ("scale_shift", 2 * f.G, f32, "in"),
                 ("gx", f.numel, f32, "out"), ("gdy", f.numel, f32, "out"), ("sums", 5 * f.G, f64, "ws")]
        if g.affine:
            specs += [("gamma", g.C, f32, "in"), ("ugb", 2 * g.C, f32, "in"), ("gg", f.G, f32, "out")]
        self.arena = Arena(specs)
        t = f.arena.t
        self.data = dict(x=f.data["x"], dy=f.dy, u=self.u, mean_rstd=t["mean_rstd"].clone(), gamma=f.gamma, ugb=self.ugb,
                         scale_shift=t["scale_shift"].clone())
        self.y = t["y"].clone()
        self.d = _lib.NormDesc(g.N, g.H * g.W, g.C, int(g.per_sample), f.eps, 0.0, ACT_CODE[case.act], SLOPE, 0)

    def prepare(self):
        self.arena.prepare(self.data)
        self.arena.t["sums"].zero_()

    def ptr(self, name):
        p = self.arena.ptr(name)
        return p + 4 * self.g.offset if name == "x" else p

    def call(self, want=("gx", "gdy", "gg"), act=None):
        a, p = self.arena, self.ptr
        d = self.d if act is None else _lib.NormDesc(self.g.N, self.g.H * self.g.W, self.g.C, int(self.g.per_sample),
                                                     self.fwd.eps, 0.0, act, SLOPE, 0)
        return self.lib.b200gan_norm_dbwd(ctypes.byref(d), p("dy"), p("x"), p("mean_rstd"),
                                          p("scale_shift"), p("gamma"), p("u"), p("ugb"), p("sums"),
                                          p("gx") if "gx" in want else None, p("gdy") if "gdy" in want else None,
                                          p("gg") if "gg" in want and "gg" in a.t else None,
                                          torch.cuda.current_stream().cuda_stream)

    def reference(self):
        """(gdy, gx, ggamma per group, and their bounds) in fp64, NCHW"""
        g, f = self.g, self.fwd
        x, dy, u = nchw(f.x, g), nchw(f.dy, g), nchw(self.u, g)
        ap = {"none": lambda y: torch.ones_like(y),
              "lrelu": lambda y: torch.where(y > 0, torch.ones_like(y), torch.full_like(y, SLOPE)),
              "relu": lambda y: (y > 0).double()}[self.c.act](nchw(self.y, g))
        gamma = f.gamma.double() if g.affine else None
        beta = f.beta.double() if g.affine else None
        ug, ub = (self.ugb[:g.C].double(), self.ugb[g.C:].double()) if g.affine else (None, None)
        eps = f.eps
        gdy, gx, _ = closed_form(x, dy, gamma, beta, u, ug, ub, eps, "none", g.per_sample, ap=ap)
        dims = (2, 3) if g.per_sample else (0, 2, 3)
        m = g.H * g.W * (1 if g.per_sample else g.N)
        mean = x.mean(dims, keepdim=True)
        r = 1 / torch.sqrt(((x - mean) ** 2).mean(dims, keepdim=True) + eps)
        xh = (x - mean) * r
        xa = (x.abs() + mean.abs()) * r                     # magnitude of xhat as the kernel forms it
        gr = dy * ap
        S = lambda t: t.sum(dims, keepdim=True)  # noqa: E731
        A, B, U, T, Q = S(gr) / m, S(gr * xh) / m, S(u), S(u * xh), S(u * gr)
        Aa, Ba, Ua, Ta, Qa = S(gr.abs()) / m, S((gr * xa).abs()) / m, S(u.abs()), S((u * xa).abs()), S((u * gr).abs())
        ch = (1, g.C, 1, 1)
        gaa = gamma.abs().view(ch) if g.affine else 1.0
        uga = ug.abs().view(ch) if g.affine else 0.0
        uba = ub.abs().view(ch) if g.affine else 0.0
        b_gdy = ap.abs() * (gaa * r * (u.abs() + Ua / m + xa * Ta / m) + uga * xa + uba)
        b_gx = uga * r * (gr.abs() + Aa + xa * Ba) + (gaa * r * r / m) * (
            xa * (Qa + Aa * Ua + 3 * Ba * Ta) + Ta * (gr.abs() + Aa) + Ba * (m * u.abs() + Ua))
        gg = gg_b = None
        if g.affine:  # per group: [1, C] for BatchNorm, [N, C] for InstanceNorm
            gg = (r * (Q - A * U - B * T)).view(-1, g.C).reshape(-1)
            gg_b = (r * (Qa + Aa * Ua + Ba * Ta)).view(-1, g.C).reshape(-1)
        return gdy, gx, gg, TOL * b_gdy, TOL * b_gx, None if gg_b is None else TOL * gg_b


@pytest.mark.parametrize("case", CASES, ids=lambda c: c.id)
def test_norm_dbwd_case(case):
    run = DRun(case)
    g, t = case.geom, run.arena.t
    run.prepare()
    rc = run.call()
    torch.cuda.synchronize()
    assert rc == 0, f"{case.id}: rc {rc}: {run.lib.b200gan_last_error().decode()}"
    run.arena.check_guards(case.id)
    assert (t["sums"] == 0).all(), f"{case.id}: the workspace is not handed back zeroed"
    gdy, gx, gg, b_gdy, b_gx, b_gg = run.reference()
    check_elementwise(f"{case.id} gdy", nchw(t["gdy"], g), gdy, b_gdy)
    check_elementwise(f"{case.id} gx", nchw(t["gx"], g), gx, b_gx)
    if g.affine:
        check_elementwise(f"{case.id} ggamma", t["gg"], gg, b_gg)
    full = {k: t[k].clone() for k in ("gx", "gdy", "gg") if k in t}

    # each output alone: bit-identical to the full call, the others never written
    for want in full:
        run.prepare()
        assert run.call(want=(want,)) == 0
        torch.cuda.synchronize()
        run.arena.check_guards(f"{case.id} {want} alone")
        assert torch.equal(t[want], full[want]), f"{case.id}: {want} alone differs from the full call"
        for other in full:
            if other != want:
                assert torch.isnan(t[other]).all(), f"{case.id}: {other} written although not asked for"
        assert (t["sums"] == 0).all()

    # CUDA-graph replay
    run.prepare()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        with torch.cuda.graph(graph, stream=s):
            run.call()
    torch.cuda.current_stream().wait_stream(s)
    graph.replay()
    torch.cuda.synchronize()
    for k, v in full.items():
        assert torch.equal(t[k], v), f"{case.id}: graph replay of {k} is not bit-identical"


def expected_instances(case):
    """the launches of one b200gan_norm_dbwd call: the first-order backward's instances, the reduce twice"""
    v = case.geom.vec
    return [f"norm_bwd_reduce_kernel<{v}>", f"norm_bwd_reduce_kernel<{v}>", f"norm_bwd_apply_kernel<{v}>",
            "norm_bwd_params_kernel"]


def test_norm_dbwd_traced_instances():
    """Every case's calls in ONE profiler session (few sessions per process keep the activity records complete): the
    kernel instances in launch order, and the (samples, channel slices) of each templated launch."""
    runs = [DRun(c) for c in CASES]
    launches = [(n, (None, c.geom.N if c.geom.per_sample else 1, c.geom.slices) if "<" in n else None)
                for c in CASES for n in expected_instances(c)]
    check_route("norm_dbwd", lambda: [r.call() for r in runs], launches, family=("norm_",),
                prepare=lambda: [r.prepare() for r in runs])


@pytest.mark.parametrize("act", ["tanh", "sigmoid"])
def test_norm_dbwd_refuses_tanh_and_sigmoid(act):
    run = DRun(nc.Case(nc.GEOMS[2], "none", False))
    run.prepare()
    assert run.call(act=ACT_CODE[act]) == -1  # B200GAN_E_UNSUPPORTED
    torch.cuda.synchronize()
    assert torch.isnan(run.arena.t["gx"]).all() and (run.arena.t["sums"] == 0).all()


# ---- modules ----------------------------------------------------------------------------------------------------
def _dragan_penalty(d, x_hat, seed):
    torch.manual_seed(seed)                         # the same Dropout2d masks in both implementations
    out = d(x_hat)
    grads = torch.autograd.grad(out, x_hat, torch.ones_like(out), create_graph=True, retain_graph=True)[0]
    return 10.0 * ((grads.norm(2, dim=1) - 1) ** 2).mean(), out


def _interpolates(x, seed):
    gen = torch.Generator(device="cuda").manual_seed(seed)
    alpha = torch.rand(x.shape, generator=gen, device="cuda")
    return alpha * x + (1 - alpha) * (x + 0.5 * x.std() * torch.rand(x.shape, generator=gen, device="cuda"))


def _dcgan_pair(img=32):
    from b200gan import zoo
    torch.manual_seed(11)
    ref = zoo.DCGANDiscriminator(img, 1, nn=zoo.namespace(stock=True)).cuda().train()
    with torch.no_grad():
        for m in ref.modules():
            if isinstance(m, torch.nn.BatchNorm2d):
                m.weight.normal_(1.0, 0.2)
                m.bias.normal_(0.0, 0.2)
    ours = zoo.DCGANDiscriminator(img, 1).cuda().train()
    ours.load_state_dict(ref.state_dict())
    return ref, ours


def _compare_dragan(mixed, fused=True, steps=2):
    """fp32 against fp32: the fused chain's kernels are fp32, and the unfused run takes the fp32 SIMT convolutions"""
    from b200gan import ops
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    prev = ops.Config.fuse_narrow_chain, ops.Config.algo
    ops.Config.fuse_narrow_chain = fused
    ops.Config.algo = "auto" if fused else "simt"
    try:
        ref, ours = _dcgan_pair()
        if fused:
            assert [type(s).__name__ for s in ours.model._plan()] == ["_ChainStep"]
        for step in range(steps):
            x = torch.rand(16, 1, 32, 32, device="cuda") * 2 - 1
            xh0 = _interpolates(x, 100 + step)
            res = []
            for net in (ref, ours):
                net.zero_grad()
                xh = xh0.clone().requires_grad_(True)
                gp, out = _dragan_penalty(net, xh, 200 + step)
                loss = out.mean() + gp if mixed else gp
                loss.backward()
                res.append((gp.detach(), [(k, p.grad) for k, p in net.named_parameters()]))
            assert abs(res[1][0].item() - res[0][0].item()) < 1e-3 * abs(res[0][0].item()), (res[1][0], res[0][0])
            for (k, go), (_, gr) in zip(res[1][1], res[0][1]):
                assert go is not None, k
                assert rel_err(go, gr) < 1e-3, f"step {step} {k}: {rel_err(go, gr):.2e}"
        # one running-statistics update per forward
        for (k, bo), (_, br) in zip(ours.named_buffers(), ref.named_buffers()):
            if k.endswith("num_batches_tracked"):
                assert bo.item() == br.item() == steps, (k, bo.item(), br.item())
            else:
                assert rel_err(bo, br) < 1e-5, k
    finally:
        ops.Config.fuse_narrow_chain, ops.Config.algo = prev


def test_dragan_penalty_fused_chain():
    _compare_dragan(mixed=False)


def test_dragan_penalty_unfused():
    _compare_dragan(mixed=False, fused=False)


def test_dragan_mixed_loss_on_one_forward():
    _compare_dragan(mixed=True)
    _compare_dragan(mixed=True, fused=False)


def _dualgan_critic(ns, instance=False):
    def block(i, o, normalize=True):
        layers = [ns.Conv2d(i, o, 4, stride=2, padding=1)]
        if normalize:
            layers.append(ns.InstanceNorm2d(o, affine=True) if instance else ns.BatchNorm2d(o, 0.8))
        layers.append(ns.LeakyReLU(0.2, inplace=True))
        return layers
    return ns.Sequential(*block(3, 64, normalize=False), *block(64, 128), *block(128, 256), ns.ZeroPad2d((1, 0, 1, 0)),
                         ns.Conv2d(256, 1, kernel_size=4))


@pytest.mark.parametrize("instance", [False, True], ids=["batchnorm", "instancenorm"])
def test_dualgan_wgan_gp_critic(instance):
    from b200gan import zoo
    torch.manual_seed(23)
    ref = _dualgan_critic(zoo.namespace(stock=True), instance).cuda().train()
    with torch.no_grad():
        for m in ref.modules():
            if getattr(m, "weight", None) is not None and m.weight.dim() == 1:
                m.weight.normal_(1.0, 0.2)
                m.bias.normal_(0.0, 0.2)
    ref_t = copy.deepcopy(ref)
    ours = _dualgan_critic(zoo.namespace(), instance).cuda().train()
    ours.load_state_dict(ref.state_dict())
    real, fake = torch.randn(8, 3, 64, 64, device="cuda"), torch.randn(8, 3, 64, 64, device="cuda")
    alpha = torch.rand(8, 1, 1, 1, device="cuda")
    res = {}
    for name, net, tf32 in (("fp32", ref, False), ("tf32", ref_t, True), ("ours", ours, False)):
        torch.backends.cudnn.allow_tf32 = tf32
        xh = (alpha * real + (1 - alpha) * fake).requires_grad_(True)
        out = net(xh)
        grads = torch.autograd.grad(out, xh, torch.ones_like(out), create_graph=True, retain_graph=True)[0]
        gp = ((grads.reshape(grads.size(0), -1).norm(2, dim=1) - 1) ** 2).mean()
        loss = -net(real).mean() + net(fake).mean() + 10.0 * gp       # dualgan.py:116-135
        loss.backward()
        res[name] = (gp.detach().reshape(1), [(k, p.grad) for k, p in net.named_parameters()])
    torch.backends.cudnn.allow_tf32 = False
    e_o, e_t = rel_err(res["ours"][0], res["fp32"][0]), rel_err(res["tf32"][0], res["fp32"][0])
    assert e_o < max(2e-3, 1.5 * e_t), f"gp: ours {e_o:.2e}, stock TF32 {e_t:.2e}"
    top = max(g.double().norm().item() for _, g in res["fp32"][1])
    for (k, go), (_, gr), (_, gt) in zip(res["ours"][1], res["fp32"][1], res["tf32"][1]):
        if gr.double().norm().item() < 1e-5 * top:   # conv bias in front of a norm: analytically zero
            continue
        e_o, e_t = rel_err(go, gr), rel_err(gt, gr)
        assert e_o < max(2e-3, 1.5 * e_t), f"{k}: ours {e_o:.2e}, stock TF32 {e_t:.2e}"


# ---- refusals ------------------------------------------------------------------------------------------------------
def _grad_of_grad(net, x):
    x = x.clone().requires_grad_(True)
    out = net(x)
    g = torch.autograd.grad(out, x, torch.ones_like(out), create_graph=True)[0]
    g.square().sum().backward()


def test_refusals_under_create_graph():
    from b200gan import ops, zoo
    ns = zoo.namespace()
    x = torch.randn(4, 8, 16, 16, device="cuda")
    with pytest.raises(NotImplementedError, match="tanh / sigmoid"):
        _grad_of_grad(ns.Sequential(ns.BatchNorm2d(8), ns.Tanh()).cuda(), x)
    with pytest.raises(NotImplementedError, match="tanh / sigmoid"):
        _grad_of_grad(ns.Sequential(ns.InstanceNorm2d(8), ns.Sigmoid()).cuda(), x)
    # the generator tail: BatchNorm2d -> LeakyReLU -> Conv2d(64, 1, 3, 1, 1) -> Tanh
    from b200gan import nn as bnn
    tail = ns.Sequential(ns.Conv2d(8, 64, 3, 1, 1), ns.BatchNorm2d(64, 0.8), ns.LeakyReLU(0.2), ns.Conv2d(64, 1, 3, 1, 1),
                         ns.Tanh()).cuda()
    if any(isinstance(s, bnn._TailStep) for s in tail._plan()):
        with pytest.raises(NotImplementedError, match="generator tail"):
            _grad_of_grad(tail, torch.randn(4, 8, 32, 32, device="cuda"))
    # a fused chain under ops.bn_groups(2)
    _, d = _dcgan_pair()
    with pytest.raises(NotImplementedError, match="bn_groups"):
        with ops.bn_groups(2):
            xh = torch.randn(16, 1, 32, 32, device="cuda", requires_grad=True)
            out = d.model(xh)
        torch.autograd.grad(out.sum(), xh, create_graph=True)


# ---- graph capture -----------------------------------------------------------------------------------------------
def _dragan_penalty_nodrop(d, x_hat):
    out = d(x_hat)
    grads = torch.autograd.grad(out, x_hat, torch.ones_like(out), create_graph=True, retain_graph=True)[0]
    return 10.0 * ((grads.norm(2, dim=1) - 1) ** 2).mean(), out


def test_captured_dragan_critic_iteration_replays_bit_identically():
    """D(real) under BCE plus the DRAGAN penalty and d_loss.backward(), captured once and replayed: the loss and the
    penalty are bit-identical between replays.  The parameter gradients agree to fp32 rounding: the SIMT weight
    gradient sums its pixel splits with fp32 atomics, whose order is not fixed."""
    _, d = _dcgan_pair()
    for m in d.modules():  # each replay would draw new Dropout2d masks
        if isinstance(m, torch.nn.Dropout2d):
            m.p = 0.0
    real = torch.rand(16, 1, 32, 32, device="cuda") * 2 - 1
    xh0 = _interpolates(real, 5)
    bce = torch.nn.BCELoss()
    params = list(d.parameters())

    def iteration():
        for p in params:
            if p.grad is not None:
                p.grad.zero_()
        xh = xh0.detach().requires_grad_(True)
        gp, _ = _dragan_penalty_nodrop(d, xh)
        out = d(real)
        loss = bce(out, torch.ones_like(out)) + gp
        loss.backward()
        return loss.detach(), gp.detach()

    eager = iteration()
    eager = (eager[0].clone(), eager[1].clone(), [p.grad.clone() for p in params])
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        iteration()
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        loss, gp = iteration()
    results = []
    for _ in range(2):
        graph.replay()
        torch.cuda.synchronize()
        results.append((loss.clone(), gp.clone(), [p.grad.clone() for p in params]))
    for r in results:
        assert torch.equal(r[0], eager[0]) and torch.equal(r[1], eager[1]), (r[0], r[1], eager[0], eager[1])
        for a, b in zip(r[2], eager[2]):
            assert rel_err(a, b) < 1e-6


# ---- a script in the reference's idiom -----------------------------------------------------------------------------
def test_mini_dragan_script_under_the_launcher():
    from b200gan import launch
    script = os.path.join(os.path.dirname(os.path.abspath(__file__)), "scripts", "mini_dragan", "mini_dragan.py")
    args = ["--img_size", "32", "--batch_size", "16"]
    torch.backends.cudnn.allow_tf32 = False
    ref = launch.run(script, args, iters=3, seed=3, stock=True, quiet=True)
    ours = launch.run(script, args, iters=3, seed=3, stock=False, quiet=True)
    assert ref["losses"] and len(ours["losses"]) == len(ref["losses"])
    for a, b in zip(ours["losses"], ref["losses"]):
        for k in b:
            assert abs(a[k] - b[k]) <= 2e-3 * max(1.0, abs(b[k])), (k, a[k], b[k])
