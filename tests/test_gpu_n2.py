"""SURVEY.md section 8(f) N2: gradient penalty of a CONV critic (stargan/stargan.py:142-161, models.py:87-115: Conv2d k4 s2
+ LeakyReLU(0.01), no normalisation) -- autograd.grad(create_graph=True) through the drop-in convolutions, then backward
through that graph.  The conv is bilinear, so the double backward reuses fprop / dgrad / wgrad (functional.ConvDgradFn /
ConvWgradFn); compared with stock torch fp32 on the same GPU."""
import pytest
import torch

from conftest import rel_err

pytestmark = pytest.mark.gpu


def _critic(ns, chans=(3, 32, 64, 128)):
    layers = []
    for cin, cout in zip(chans[:-1], chans[1:]):
        layers += [ns.Conv2d(cin, cout, 4, stride=2, padding=1), ns.LeakyReLU(0.01)]
    layers.append(ns.Conv2d(chans[-1], 1, 3, stride=1, padding=1, bias=False))
    return ns.Sequential(*layers)


def _penalty(d, x_hat):
    out = d(x_hat)
    grad = torch.autograd.grad(outputs=out, inputs=x_hat, grad_outputs=torch.ones_like(out), retain_graph=True,
                               create_graph=True, only_inputs=True)[0]
    return ((grad.reshape(grad.size(0), -1).norm(2, dim=1) - 1) ** 2).mean(), out


def _transposed_critic(ns):
    # a ConvTranspose2d too narrow for the tensor cores: its data gradient and double backward run the SIMT kernels
    return ns.Sequential(ns.Conv2d(3, 8, 4, stride=2, padding=1), ns.LeakyReLU(0.01),
                         ns.ConvTranspose2d(8, 6, 4, stride=2, padding=1), ns.LeakyReLU(0.01),
                         ns.Conv2d(6, 1, 3, stride=1, padding=1))


@pytest.mark.parametrize("algo", ["simt", "auto"])
def test_conv_critic_gradient_penalty(algo):
    _check_gradient_penalty(_critic, algo)


@pytest.mark.parametrize("algo", ["simt", "auto"])
def test_transposed_conv_critic_gradient_penalty(algo):
    _check_gradient_penalty(_transposed_critic, algo)


def _check_gradient_penalty(make_critic, algo):
    import b200gan
    from b200gan import zoo
    torch.backends.cudnn.allow_tf32 = False
    torch.manual_seed(19)
    prev = b200gan.Config.algo
    b200gan.Config.algo = algo
    try:
        ref = make_critic(zoo.namespace(stock=True)).cuda()
        ours = make_critic(zoo.namespace()).cuda()
        ours.load_state_dict(ref.state_dict())
        x = torch.randn(4, 3, 32, 32, device="cuda")
        res = []
        for net in (ref, ours):
            xh = x.clone().requires_grad_(True)
            gp, out = _penalty(net, xh)
            loss = out.mean() + 10.0 * gp          # Wasserstein term + penalty, as in the critic loss
            loss.backward()
            res.append((gp.detach(), [p.grad.clone() for p in net.parameters()]))
        tol = 1e-4 if algo == "simt" else 2e-2     # TF32 tensor cores on the 32/64/128-channel layers
        assert abs(res[1][0].item() - res[0][0].item()) < tol * abs(res[0][0].item())
        for go, gr in zip(res[1][1], res[0][1]):
            assert rel_err(go, gr) < tol
    finally:
        b200gan.Config.algo = prev
