"""The MLP critic under autograd (functional.MlpCriticFn / MlpCriticGradFn, csrc/mlp_critic.cu) against stock torch.nn
modules with the same weights, fp32 on the same GPU with TF32 off.  Bound: 1e-4 norm-relative -- summation order
only.  Covers the forward and first-order backward, the script-form WGAN-GP and WGAN-div critic losses with their own
autograd.grad(create_graph=True) penalties, repeated back-propagation, the gradient w.r.t. grad_outputs, the refusal of a
penalty on parameter gradients, CUDA-graph capture, and an unmodified reference-idiom script under the launcher."""
import copy
import os

import pytest
import torch

from conftest import rel_err

pytestmark = pytest.mark.gpu
TOL = 1e-4


@pytest.fixture(autouse=True)
def _fp32():
    prev = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32 = prev


@pytest.fixture
def calls(monkeypatch):
    """Counts of the three new entry points issued through ops."""
    from b200gan import ops
    n = {"fwd": 0, "bwd": 0, "dbwd": 0}
    for k in n:
        fn = getattr(ops, "mlp_critic_" + k)

        def wrapped(*a, _fn=fn, _k=k, **kw):
            n[_k] += 1
            return _fn(*a, **kw)
        monkeypatch.setattr(ops, "mlp_critic_" + k, wrapped)
    return n


def _pair(din, h1, h2, slope=0.2, seed=0):
    """(stock critic, drop-in critic) with identical weights, on the GPU."""
    from b200gan import nn as bnn
    torch.manual_seed(seed)
    ref = torch.nn.Sequential(torch.nn.Linear(din, h1), torch.nn.LeakyReLU(slope, inplace=True),
                              torch.nn.Linear(h1, h2), torch.nn.LeakyReLU(slope, inplace=True), torch.nn.Linear(h2, 1))
    ours = bnn.Sequential(bnn.Linear(din, h1), bnn.LeakyReLU(slope, inplace=True), bnn.Linear(h1, h2),
                          bnn.LeakyReLU(slope, inplace=True), bnn.Linear(h2, 1))
    ours.load_state_dict(ref.state_dict())
    return ref.cuda(), ours.cuda()


def _grads(*nets):
    return [p.grad for net in nets for p in net.parameters()]


def _check_grads(ours, ref, what):
    assert len(ours) == len(ref)
    for i, (a, b) in enumerate(zip(ours, ref)):
        assert a is not None and b is not None, (what, i)
        if b.double().norm().item() < 1e-9:
            assert a.abs().max().item() < 1e-6, (what, i)
        else:
            assert rel_err(a, b) < TOL, (what, i, rel_err(a, b))


@pytest.mark.parametrize("n,din,h1,h2", [(64, 1024, 512, 256), (7, 784, 100, 50), (33, 256, 96, 33)])
def test_forward_and_first_order_backward(n, din, h1, h2, calls):
    ref, ours = _pair(din, h1, h2, seed=n)
    x = torch.randn(n, din, device="cuda")
    xr, xo = x.clone().requires_grad_(True), x.clone().requires_grad_(True)
    yr, yo = ref(xr), ours(xo)
    assert calls["fwd"] == 1 and yo.shape == yr.shape == (n, 1)
    assert rel_err(yo, yr) < TOL
    dy = torch.randn(n, 1, device="cuda")
    yr.backward(dy)
    yo.backward(dy)
    assert calls["bwd"] == 1
    assert rel_err(xo.grad, xr.grad) < TOL
    _check_grads(_grads(ours), _grads(ref), "first order")


def _wgan_gp_loss(critic, real, fake, alpha, lam=10.0):
    """wgan_gp.py:119-138,164-171 in script form."""
    real_validity, fake_validity = critic(real), critic(fake)
    interpolates = (alpha * real.data + (1 - alpha) * fake.data).requires_grad_(True)
    d_int = critic(interpolates)
    grads = torch.autograd.grad(outputs=d_int, inputs=interpolates, grad_outputs=torch.ones_like(d_int),
                                create_graph=True, retain_graph=True, only_inputs=True)[0]
    gp = ((grads.view(grads.size(0), -1).norm(2, dim=1) - 1) ** 2).mean()
    return -torch.mean(real_validity) + torch.mean(fake_validity) + lam * gp


def test_wgan_gp_critic_loss_in_script_form(calls):
    ref, ours = _pair(1024, 512, 256, seed=1)
    torch.manual_seed(2)
    real, fake = torch.randn(64, 1024, device="cuda"), torch.randn(64, 1024, device="cuda")
    alpha = torch.rand(64, 1, device="cuda")
    lr = _wgan_gp_loss(ref, real, fake, alpha)
    lr.backward()
    lo = _wgan_gp_loss(ours, real, fake, alpha)
    lo.backward()
    assert calls == {"fwd": 3, "bwd": 3, "dbwd": 1}
    assert abs(lo.item() - lr.item()) < TOL * max(abs(lr.item()), 1.0)
    _check_grads(_grads(ours), _grads(ref), "wgan-gp")


def test_wgan_gp_critic_loss_with_fake_attached_to_a_generator(calls):
    ref, ours = _pair(256, 96, 33, seed=3)
    torch.manual_seed(4)
    g_ref = torch.nn.Sequential(torch.nn.Linear(16, 64), torch.nn.LeakyReLU(0.2), torch.nn.Linear(64, 256),
                                torch.nn.Tanh()).cuda()
    g_ours = copy.deepcopy(g_ref)
    real, z, alpha = torch.randn(33, 256, device="cuda"), torch.randn(33, 16, device="cuda"), torch.rand(33, 1,
                                                                                                          device="cuda")
    lr = _wgan_gp_loss(ref, real, g_ref(z), alpha)
    lr.backward()
    lo = _wgan_gp_loss(ours, real, g_ours(z), alpha)
    lo.backward()
    assert calls["dbwd"] == 1
    assert abs(lo.item() - lr.item()) < TOL * max(abs(lr.item()), 1.0)
    _check_grads(_grads(ours, g_ours), _grads(ref, g_ref), "wgan-gp, fake attached")


def _wgan_div_loss(critic, real, fake, k=2.0, p=6.0):
    """wgan_div.py:143-163: ||dD/dx||^p on the real and the fake batch, real images requiring grad."""
    real_validity, fake_validity = critic(real), critic(fake)
    ones = torch.ones(real.shape[0], 1, device=real.device)
    rg = torch.autograd.grad(real_validity, real, ones, create_graph=True, retain_graph=True, only_inputs=True)[0]
    rgn = rg.view(rg.size(0), -1).pow(2).sum(1) ** (p / 2)
    fg = torch.autograd.grad(fake_validity, fake, ones, create_graph=True, retain_graph=True, only_inputs=True)[0]
    fgn = fg.view(fg.size(0), -1).pow(2).sum(1) ** (p / 2)
    return -torch.mean(real_validity) + torch.mean(fake_validity) + torch.mean(rgn + fgn) * k / 2


def test_wgan_div_critic_loss(calls):
    ref, ours = _pair(784, 100, 50, slope=0.2, seed=5)
    torch.manual_seed(6)
    real = torch.randn(7, 784, device="cuda")
    g_ref = torch.nn.Sequential(torch.nn.Linear(12, 784), torch.nn.Tanh()).cuda()
    g_ours = copy.deepcopy(g_ref)
    z = torch.randn(7, 12, device="cuda")
    rr, ro = real.clone().requires_grad_(True), real.clone().requires_grad_(True)
    lr = _wgan_div_loss(ref, rr, g_ref(z))
    lr.backward()
    lo = _wgan_div_loss(ours, ro, g_ours(z))
    lo.backward()
    assert calls["dbwd"] == 2
    assert abs(lo.item() - lr.item()) < TOL * max(abs(lr.item()), 1.0)
    assert rel_err(ro.grad, rr.grad) < TOL
    _check_grads(_grads(ours, g_ours), _grads(ref, g_ref), "wgan-div")


def test_backward_twice_with_retain_graph():
    ref, ours = _pair(256, 96, 33, seed=7)
    x = torch.randn(9, 256, device="cuda")
    dy = torch.randn(9, 1, device="cuda")
    for net in (ref, ours):
        y = net(x)
        y.backward(dy, retain_graph=True)
        y.backward(2 * dy)
    _check_grads(_grads(ours), _grads(ref), "twice")


def test_gradient_of_requires_grad_grad_outputs(calls):
    ref, ours = _pair(256, 96, 33, seed=8)
    x = torch.randn(12, 256, device="cuda", requires_grad=True)
    out = {}
    for name, net in (("ref", ref), ("ours", ours)):
        go = torch.randn(12, 1, device="cuda", generator=torch.Generator("cuda").manual_seed(9)).requires_grad_(True)
        g = torch.autograd.grad(net(x), x, go, create_graph=True)[0]
        ((g - 0.5) ** 2).sum().backward()
        out[name] = (go.grad, _grads(net))
    assert calls["dbwd"] == 1
    assert rel_err(out["ours"][0], out["ref"][0]) < TOL
    weights = [0, 2, 4]  # the biases get no gradient from a penalty on dD/dx (torch: None)
    _check_grads([out["ours"][1][i] for i in weights], [out["ref"][1][i] for i in weights], "weights")


def test_a_penalty_on_parameter_gradients_is_refused():
    _, ours = _pair(64, 32, 16, seed=10)
    x = torch.randn(5, 64, device="cuda")
    gw = torch.autograd.grad(ours(x).sum(), ours[0].weight, create_graph=True)[0]
    with pytest.raises(NotImplementedError, match="parameter gradients"):
        (gw ** 2).sum().backward()


def test_critic_iteration_replayed_from_a_cuda_graph_matches_eager():
    from b200gan import train
    _, ours = _pair(1024, 512, 256, seed=11)
    params = list(ours.parameters())

    def step(real, fake, alpha):
        loss = _wgan_gp_loss(ours, real, fake, alpha)
        return (loss,) + torch.autograd.grad(loss, params)

    def inputs(seed):
        gen = torch.Generator("cuda").manual_seed(seed)
        return (torch.randn(64, 1024, device="cuda", generator=gen), torch.randn(64, 1024, device="cuda", generator=gen),
                torch.rand(64, 1, device="cuda", generator=gen))

    graphed = train.GraphedStep(step, inputs(0))
    for seed in (1, 2):
        replay = [t.clone() for t in graphed(*inputs(seed))]
        eager = step(*inputs(seed))
        for i, (a, b) in enumerate(zip(replay, eager)):
            assert rel_err(a, b) < 1e-6, (seed, i)


@pytest.mark.parametrize("penalty", ["gp", "div"])
def test_reference_idiom_wgan_script_runs_under_the_launcher(penalty, calls):
    """launch.run() of tests/scripts/mini_wgangp (autograd.grad(create_graph=True) penalty, n_critic, .data
    interpolates): stock torch vs the drop-ins, same seeds: the printed losses agree and the patched run issued the
    fused critic passes, double backward included."""
    from b200gan import launch
    script = os.path.join(os.path.dirname(os.path.abspath(__file__)), "scripts", "mini_wgangp", "mini_wgangp.py")
    args = ["--epochs", "1", "--batch_size", "16", "--side", "16", "--penalty", penalty]
    ref = launch.run(script, args, iters=4, seed=5, stock=True, quiet=True)
    assert calls == {"fwd": 0, "bwd": 0, "dbwd": 0}
    ours = launch.run(script, args, iters=4, seed=5, stock=False, quiet=True)
    iters, g_steps = 4, 2
    per_iter = 3 if penalty == "gp" else 2
    assert calls["fwd"] == iters * per_iter + g_steps and calls["dbwd"] == iters * (1 if penalty == "gp" else 2)
    assert len(ref["history"]) == len(ours["history"]) == g_steps
    # relative for losses of magnitude >= 1, absolute below (the generator loss of a young critic is near zero)
    for (cr, gr), (co, go) in zip(ref["history"], ours["history"]):
        assert abs(co - cr) < 2e-3 * max(abs(cr), 1.0) and abs(go - gr) < 2e-3 * max(abs(gr), 1.0), (
            ref["history"], ours["history"])
