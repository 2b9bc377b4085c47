"""The MLP generator on the fused kernels (functional.MlpGeneratorFn, csrc/mlp_generator) end to end on the GPU: the
WGAN-GP critic iterations and generator step against stock torch fp32 with TF32 off, a reference-idiom MLP GAN script
under the launcher, the benchmark's critic iteration captured in a CUDA graph, and the refusal of a double backward."""
import copy
import os

import pytest
import torch

from conftest import rel_err
from oracle import ref_models

pytestmark = pytest.mark.gpu
TOL = 1e-3
LR = 2e-4


@pytest.fixture(autouse=True)
def _fp32():
    prev = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32 = prev


@pytest.fixture
def calls(monkeypatch):
    """Counts of the generator's forward and backward issued through ops."""
    from b200gan import ops
    n = {"fwd": 0, "bwd": 0}
    for k in n:
        fn = getattr(ops, "mlp_gen_" + k)

        def wrapped(*a, _fn=fn, _k=k, **kw):
            n[_k] += 1
            return _fn(*a, **kw)
        monkeypatch.setattr(ops, "mlp_gen_" + k, wrapped)
    return n


def _build(img=32, seed=0):
    from b200gan import zoo
    g_ref, d_ref = ref_models.build_wgan_gp(img, seed=seed)
    g, d = zoo.WGANGPGenerator((1, img, img)), zoo.WGANGPDiscriminator((1, img, img))
    g.load_state_dict(g_ref.state_dict())
    d.load_state_dict(d_ref.state_dict())
    return g_ref.cuda(), d_ref.cuda(), g.cuda(), d.cuda()


def _biases_in_front_of_a_norm(g):
    return {f"model.{i}.bias" for i, m in enumerate(g.model) if isinstance(m, torch.nn.Linear)
            and i + 1 < len(g.model) and isinstance(g.model[i + 1], torch.nn.BatchNorm1d)}


def test_wgan_gp_critic_iterations_and_generator_step(calls):
    """Five critic iterations (G under torch.no_grad()) and one generator step (wgan_gp.py:146-193): the drop-in G on
    the fused kernels and the one-kernel critic iteration against stock torch fp32 on the GPU."""
    from b200gan import train
    g_ref, d_ref, g, d = _build(32, seed=2)
    opt = lambda ps: torch.optim.Adam(ps, lr=LR, betas=(0.5, 0.999))  # noqa: E731
    od_r, og_r, od, og = opt(d_ref.parameters()), opt(g_ref.parameters()), opt(d.parameters()), opt(g.parameters())
    n = 64
    for it in range(5):
        real = ref_models.synthetic_images(n, 1, 32, 32, seed=40 + it).cuda()
        z = ref_models.synthetic_z(n, seed=40 + it).cuda()
        alpha = ref_models.synthetic_alpha(n, seed=40 + it).cuda()
        dl_r, gp_r = train.wgan_gp_critic_step(g_ref, d_ref, od_r, real, z, alpha, 10.0, fused_gp=False)
        dl, gp = train.wgan_gp_critic_step(g, d, od, real, z, alpha, 10.0, fused_gp="step")
        assert abs(dl.item() - dl_r.item()) < TOL * max(abs(dl_r.item()), 1.0), it
        assert abs(gp.item() - gp_r.item()) < TOL * abs(gp_r.item()), it
    assert calls == {"fwd": 5, "bwd": 0}
    gl_r = train.wgan_gp_generator_step(g_ref, d_ref, og_r, z)
    gl = train.wgan_gp_generator_step(g, d, og, z)
    assert calls == {"fwd": 6, "bwd": 1}
    assert abs(gl.item() - gl_r.item()) < TOL * max(abs(gl_r.item()), 1.0)
    for (k, po), (_, pr) in zip(d.named_parameters(), d_ref.named_parameters()):
        assert rel_err(po, pr) < TOL, k
    for (k, po), (_, pr) in zip(g.named_parameters(), g_ref.named_parameters()):
        if k in _biases_in_front_of_a_norm(g):
            # the bias of a Linear in front of a BatchNorm1d gets a gradient that is zero but for rounding, whose sign
            # Adam's first step turns into +-lr: any two fp32 evaluations differ there by up to 2 lr per element
            assert (po - pr).abs().max().item() <= 2 * LR * 1.01, k
        else:
            assert rel_err(po, pr) < TOL, k
    for (k, bo), (_, br) in zip(g.named_buffers(), g_ref.named_buffers()):
        if k.endswith("num_batches_tracked"):
            assert bo.item() == br.item() == 6, k
        else:
            assert rel_err(bo, br) < TOL, k


def test_generator_forward_and_backward_against_stock(calls):
    """gan.py's widths (-> 784) with every gradient, dz included, against the stock modules"""
    from b200gan import nn as bnn, zoo
    torch.manual_seed(3)
    ref = ref_models.WGANGPGenerator((1, 28, 28), 100).cuda()
    ours = zoo.WGANGPGenerator((1, 28, 28), nn=zoo.namespace()).cuda()
    ours.load_state_dict(ref.state_dict())
    assert isinstance(ours.model, bnn.Sequential) and bnn.mlp_generator_layers(list(ours.model), 100) is not None
    z = torch.randn(64, 100, device="cuda")
    zr, zo = z.clone().requires_grad_(True), z.clone().requires_grad_(True)
    yr, yo = ref(zr), ours(zo)
    assert calls["fwd"] == 1 and rel_err(yo, yr) < 1e-4
    dy = torch.randn_like(yr)
    yr.backward(dy)
    yo.backward(dy)
    assert calls["bwd"] == 1
    assert rel_err(zo.grad, zr.grad) < 1e-4
    for (k, po), (_, pr) in zip(ours.named_parameters(), ref.named_parameters()):
        if k in _biases_in_front_of_a_norm(ours):   # their gradient is zero but for rounding
            assert po.grad.abs().max().item() < 1e-5 and pr.grad.abs().max().item() < 1e-5, k
        else:
            assert rel_err(po.grad, pr.grad) < 1e-4, k


def test_double_backward_through_the_generator_is_refused():
    from b200gan import zoo
    g = zoo.WGANGPGenerator((1, 8, 8)).cuda()
    z = torch.randn(4, 100, device="cuda", requires_grad=True)
    with pytest.raises(NotImplementedError, match="not twice differentiable"):
        torch.autograd.grad(g(z).sum(), z, create_graph=True)


def test_reference_idiom_mlp_gan_script_under_the_launcher_on_cuda(calls):
    """launch.run() of tests/scripts/mini_mlpgan (Linear / BatchNorm1d / LeakyReLU generator) on the GPU: stock torch
    against the drop-ins, same seeds: the printed losses agree and the patched run issued the generator kernels."""
    from b200gan import launch
    script = os.path.join(os.path.dirname(os.path.abspath(__file__)), "scripts", "mini_mlpgan", "mini_mlpgan.py")
    args = ["--epochs", "1", "--batch_size", "32"]
    ref = launch.run(script, args, iters=3, seed=0, stock=True, quiet=True)
    assert calls == {"fwd": 0, "bwd": 0}
    ours = launch.run(script, args, iters=3, seed=0, stock=False, quiet=True)
    assert calls == {"fwd": 3, "bwd": 3}

    def losses(run):
        rows = [l for l in run["__b200_stdout__"].splitlines() if "[D " in l]
        return [(float(r.split("[D ")[1].split("]")[0]), float(r.split("[G ")[1].split("]")[0])) for r in rows]
    lr, lo = losses(ref), losses(ours)
    assert len(lr) == len(lo) == 3
    for (dr, gr), (do, go) in zip(lr, lo):
        assert abs(do - dr) < 2e-3 * max(abs(dr), 1.0) and abs(go - gr) < 2e-3 * max(abs(gr), 1.0), (lr, lo)


def test_bench_critic_iteration_captured_in_a_cuda_graph(calls):
    """bench.py --config wgan_gp's step (drop-in G under torch.no_grad(), the one-kernel critic iteration, the fused
    Adam) captured with train.GraphedStep: replays match an eager twin, running statistics included."""
    from b200gan import optim, train, zoo
    torch.manual_seed(0)
    g = zoo.WGANGPGenerator((1, 32, 32), nn=zoo.namespace()).cuda()
    d = zoo.WGANGPDiscriminator((1, 32, 32), nn=zoo.namespace()).cuda()
    g2, d2 = copy.deepcopy(g), copy.deepcopy(d)

    def make_step(g, d):
        od = optim.Adam(d.parameters(), lr=LR, betas=(0.5, 0.999))

        def step(imgs, z, alpha):
            dl, gp = train.wgan_gp_critic_step(g, d, od, imgs, z, alpha, 10.0, fused_gp="step")
            return torch.stack([dl, gp])
        return step

    def inputs(seed):
        gen = torch.Generator("cuda").manual_seed(seed)
        return (torch.rand(64, 1, 32, 32, device="cuda", generator=gen) * 2 - 1,
                torch.randn(64, 100, device="cuda", generator=gen), torch.rand(64, 1, 1, 1, device="cuda", generator=gen))

    graphed = train.GraphedStep(make_step(g, d), inputs(0))
    assert calls["fwd"] == 4          # three warm-up steps and the captured one
    eager = make_step(g2, d2)
    for _ in range(3):                # the warm-up steps GraphedStep ran
        eager(*inputs(0))
    for seed in (1, 2, 3):
        a = graphed(*inputs(seed)).clone()
        b = eager(*inputs(seed))
        assert rel_err(a, b) < 1e-5, seed
    torch.cuda.synchronize()
    for (k, x), (_, y) in zip(list(g.named_buffers()) + list(d.named_parameters()),
                              list(g2.named_buffers()) + list(d2.named_parameters())):
        if k.endswith("num_batches_tracked"):
            assert x.item() == y.item() == 6, k
        else:
            assert rel_err(x, y) < 1e-5, k
