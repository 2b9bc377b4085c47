"""GPU parity for BASELINE config 2: the WGAN-GP gradient penalty built with autograd.grad(create_graph=True) on the
drop-in critic (its double backward on the fused MLP-critic kernels) and the whole critic iteration in one kernel
(b200gan_critic_step_mlp), against the reference's golden vectors and against autograd on stock torch."""
import os

import pytest
import torch

from conftest import rel_err
from oracle import ref_models

pytestmark = pytest.mark.gpu
TOL = 1e-3


@pytest.fixture
def calls(monkeypatch):
    """Counts of the MLP-critic forward, backward and double backward issued through ops."""
    from b200gan import ops
    n = {"fwd": 0, "bwd": 0, "dbwd": 0}
    for k in n:
        fn = getattr(ops, "mlp_critic_" + k)

        def wrapped(*a, _fn=fn, _k=k, **kw):
            n[_k] += 1
            return _fn(*a, **kw)
        monkeypatch.setattr(ops, "mlp_critic_" + k, wrapped)
    return n


def _build(img=32, seed=0):
    from b200gan import zoo
    g_ref, d_ref = ref_models.build_wgan_gp(img, seed=seed)
    g, d = zoo.WGANGPGenerator((1, img, img)), zoo.WGANGPDiscriminator((1, img, img))
    g.load_state_dict(g_ref.state_dict())
    d.load_state_dict(d_ref.state_dict())
    return g_ref.cuda(), d_ref.cuda(), g.cuda(), d.cuda()


def _no_grad(p):
    return p.grad is None or not p.grad.any()


def test_gp_double_backward_against_reference_golden(golden_dir, calls):
    """The reference's compute_gradient_penalty on the drop-in critic: one fused forward, one fused backward under
    create_graph=True, and gp.backward() as one fused double backward."""
    fix = torch.load(os.path.join(golden_dir, "wgan_gp_32_b64.pt"), weights_only=False)
    _, _, _, d = _build(fix["img_size"], fix["seed"])
    real, fake, alpha = fix["real"].cuda(), fix["fake"].cuda(), fix["alpha"].cuda()
    lam = fix["lambda_gp"]
    gp = lam * ref_models.compute_gradient_penalty(d, real, fake, alpha)
    assert abs(gp.item() - lam * fix["gp"].item()) < 1e-4 * abs(gp.item())
    gp.backward()
    assert calls == {"fwd": 1, "bwd": 1, "dbwd": 1}
    assert rel_err(d.model[4].weight.grad, fix["dW3"]) < TOL
    assert rel_err(d.model[0].weight.grad[:4], fix["dW1_head"]) < TOL
    assert rel_err(d.model[2].weight.grad[:8], fix["dW2_head"]) < TOL
    assert abs(d.model[0].weight.grad.double().norm().item() - fix["dW1_norm"]) < TOL * fix["dW1_norm"]
    assert abs(d.model[2].weight.grad.double().norm().item() - fix["dW2_norm"]) < TOL * fix["dW2_norm"]
    assert _no_grad(d.model[0].bias) and _no_grad(d.model[4].bias)  # bias gradients are exactly zero


@pytest.mark.parametrize("batch,img", [(64, 32), (7, 28), (33, 16)])
def test_gp_double_backward_vs_stock_autograd(batch, img, calls):
    """Same D, same interpolates: the penalty's double backward on the fused kernels (drop-in critic) vs autograd on
    stock torch, both through autograd.grad(create_graph=True) + backward on the GPU."""
    torch.backends.cuda.matmul.allow_tf32 = False
    _, d_ref, _, d = _build(img, seed=3)
    xi = torch.randn(batch, 1, img, img, device="cuda")
    ones = torch.ones(batch, 1, 1, 1, device="cuda")
    gp_ref = 10.0 * ref_models.compute_gradient_penalty(d_ref, xi, xi, ones)
    gp_ref.backward()
    gp = 10.0 * ref_models.compute_gradient_penalty(d, xi, xi, ones)
    gp.backward()
    assert calls["dbwd"] == 1
    assert abs(gp.item() - gp_ref.item()) < 1e-4 * abs(gp_ref.item())
    for i in (0, 2, 4):
        assert rel_err(d.model[i].weight.grad, d_ref.model[i].weight.grad) < TOL, i


def test_wgan_gp_critic_and_generator_steps():
    """Five critic iterations + one generator step (wgan_gp.py:146-193), the one-kernel critic iteration
    (fused_gp=True) vs the reference formulation (oracle restatement, stock torch on the GPU): losses and post-Adam
    parameters."""
    from b200gan import train
    torch.backends.cuda.matmul.allow_tf32 = False
    g_ref, d_ref, g, d = _build(32, seed=0)
    od_r = torch.optim.Adam(d_ref.parameters(), lr=2e-4, betas=(0.5, 0.999))
    og_r = torch.optim.Adam(g_ref.parameters(), lr=2e-4, betas=(0.5, 0.999))
    od = torch.optim.Adam(d.parameters(), lr=2e-4, betas=(0.5, 0.999))
    og = torch.optim.Adam(g.parameters(), lr=2e-4, betas=(0.5, 0.999))
    n = 64
    for it in range(5):
        real = ref_models.synthetic_images(n, 1, 32, 32, seed=20 + it).cuda()
        z = ref_models.synthetic_z(n, seed=20 + it).cuda()
        alpha = ref_models.synthetic_alpha(n, seed=20 + it).cuda()
        dl_r, gp_r = train.wgan_gp_critic_step(g_ref, d_ref, od_r, real, z, alpha, 10.0, fused_gp=False)
        dl, gp = train.wgan_gp_critic_step(g, d, od, real, z, alpha, 10.0, fused_gp=True)
        assert abs(dl.item() - dl_r.item()) < TOL * max(abs(dl_r.item()), 1.0), it
        assert abs(gp.item() - gp_r.item()) < TOL * abs(gp_r.item()), it
    gl_r = train.wgan_gp_generator_step(g_ref, d_ref, og_r, z)
    gl = train.wgan_gp_generator_step(g, d, og, z)
    assert abs(gl.item() - gl_r.item()) < TOL * max(abs(gl_r.item()), 1.0)
    for (k, po), (_, pr) in zip(d.named_parameters(), d_ref.named_parameters()):
        assert rel_err(po, pr) < TOL, k


@pytest.mark.parametrize("batch,img", [(64, 32), (5, 28), (7, 28), (33, 16)])
def test_whole_critic_iteration_in_one_kernel(batch, img):
    """b200gan_critic_step_mlp: -mean(D(real)) + mean(D(fake)) + lambda * gp and all six parameter gradients against
    autograd on stock torch (the oracle's compute_gradient_penalty, wgan_gp.py:119-138,164-173)."""
    from b200gan import functional as F
    torch.backends.cuda.matmul.allow_tf32 = False
    _, d_ref, _, d = _build(img, seed=4)
    torch.manual_seed(12)
    real = torch.randn(batch, 1, img, img, device="cuda")
    fake = torch.randn(batch, 1, img, img, device="cuda")
    alpha = torch.rand(batch, 1, 1, 1, device="cuda")
    gp_ref = ref_models.compute_gradient_penalty(d_ref, real, fake, alpha)
    loss_ref = -torch.mean(d_ref(real)) + torch.mean(d_ref(fake)) + 10.0 * gp_ref
    loss_ref.backward()
    loss, gp = F.critic_step_mlp(d.model, real, fake, alpha, 10.0)
    loss.backward()
    assert abs(loss.item() - loss_ref.item()) < 1e-4 * max(abs(loss_ref.item()), 1.0)
    assert abs(gp.item() - 10.0 * gp_ref.item()) < 1e-4 * abs(10.0 * gp_ref.item())
    for (k, po), (_, pr) in zip(d.named_parameters(), d_ref.named_parameters()):
        den = pr.grad.double().norm().item()
        if den < 1e-9:     # the last bias: -1 + 1 = 0 exactly
            assert po.grad.abs().max().item() < 1e-6, k
        else:
            assert rel_err(po.grad, pr.grad) < TOL, k


def test_wgan_gp_critic_steps_with_the_one_kernel_iteration():
    from b200gan import optim, train
    torch.backends.cuda.matmul.allow_tf32 = False
    g_ref, d_ref, g, d = _build(32, seed=1)
    od_r = torch.optim.Adam(d_ref.parameters(), lr=2e-4, betas=(0.5, 0.999))
    od = optim.Adam(d.parameters(), lr=2e-4, betas=(0.5, 0.999))
    n = 64
    for it in range(4):
        real = ref_models.synthetic_images(n, 1, 32, 32, seed=30 + it).cuda()
        z = ref_models.synthetic_z(n, seed=30 + it).cuda()
        alpha = ref_models.synthetic_alpha(n, seed=30 + it).cuda()
        dl_r, gp_r = train.wgan_gp_critic_step(g_ref, d_ref, od_r, real, z, alpha, 10.0, fused_gp=False)
        dl, gp = train.wgan_gp_critic_step(g, d, od, real, z, alpha, 10.0, fused_gp="step")
        assert abs(dl.item() - dl_r.item()) < TOL * max(abs(dl_r.item()), 1.0), it
        assert abs(gp.item() - gp_r.item()) < TOL * abs(gp_r.item()), it
    for (k, po), (_, pr) in zip(d.named_parameters(), d_ref.named_parameters()):
        assert rel_err(po, pr) < TOL, k
