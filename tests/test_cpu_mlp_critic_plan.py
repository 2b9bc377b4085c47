"""Which module lists the drop-in Sequential runs as the fused MLP critic (functional.MlpCriticFn): exactly
Linear(Din, H1) -> LeakyReLU(s) -> Linear(H1, H2) -> LeakyReLU(s) -> Linear(H2, 1), all with biases, one slope
(wgan_gp.py:72-78, wgan_div.py:72-78).  Everything else keeps the per-layer path."""
import pytest
import torch

from b200gan import nn as bnn

DIN = 784


def _critic(ns, din=DIN, h1=512, h2=256, slopes=(0.2, 0.2), biases=(True, True, True), out=1, act=None):
    act = act or ns.LeakyReLU
    return [ns.Linear(din, h1, bias=biases[0]), act(slopes[0]) if act is ns.LeakyReLU else act(),
            ns.Linear(h1, h2, bias=biases[1]), ns.LeakyReLU(slopes[1]), ns.Linear(h2, out, bias=biases[2])]


@pytest.mark.parametrize("ns", [torch.nn, bnn], ids=["stock", "dropin"])
def test_accepts_the_wgan_gp_and_wgan_div_critic(ns):
    mods = _critic(ns)
    plan = bnn.mlp_critic_layers(mods, DIN)
    assert plan is not None
    l1, l2, l3, slope = plan
    assert (l1, l2, l3) == (mods[0], mods[2], mods[4]) and slope == 0.2
    inplace = [ns.Linear(DIN, 64), ns.LeakyReLU(0.2, inplace=True), ns.Linear(64, 33), ns.LeakyReLU(0.2, inplace=True),
               ns.Linear(33, 1)]
    assert bnn.mlp_critic_layers(inplace, DIN) is not None


@pytest.mark.parametrize("ns", [torch.nn, bnn], ids=["stock", "dropin"])
def test_rejects_everything_else(ns):
    reject = {
        "trailing sigmoid": _critic(ns) + [ns.Sigmoid()],
        "different slopes": _critic(ns, slopes=(0.2, 0.1)),
        "missing bias": _critic(ns, biases=(True, False, True)),
        "two outputs": _critic(ns, out=2),
        "relu": _critic(ns, act=ns.ReLU),
        "extra layer": _critic(ns)[:4] + [ns.Linear(256, 256), ns.LeakyReLU(0.2), ns.Linear(256, 1)],
    }
    for what, mods in reject.items():
        assert bnn.mlp_critic_layers(mods, DIN) is None, what
    assert bnn.mlp_critic_layers(_critic(ns), DIN + 1) is None, "mismatched input width"


def test_rejects_hooked_layers_and_has_no_side_effects():
    mods = _critic(torch.nn)
    state = {k: v.clone() for k, v in torch.nn.Sequential(*mods).state_dict().items()}
    h = mods[2].register_forward_pre_hook(lambda m, a: None)
    assert bnn.mlp_critic_layers(mods, DIN) is None
    h.remove()
    assert bnn.mlp_critic_layers(mods, DIN) is not None
    for k, v in torch.nn.Sequential(*mods).state_dict().items():
        assert torch.equal(v, state[k]) and v.grad is None, k


def test_fused_critic_step_refuses_what_the_plan_rejects(monkeypatch):
    """functional.critic_step_mlp (the one-kernel WGAN-GP critic iteration) accepts exactly what mlp_critic_layers
    accepts: a hooked critic, whose hooks the kernel would skip, and a non-critic are refused before any launch."""
    from b200gan import functional as F, ops

    def launched(*a, **kw):
        raise AssertionError("critic_step_mlp launched")
    monkeypatch.setattr(ops, "critic_step_mlp", launched)
    real = fake = torch.zeros(2, 1, 28, 28)
    alpha = torch.zeros(2, 1, 1, 1)
    hooked = _critic(bnn)
    hooked[0].register_forward_hook(lambda m, a, out: None)
    for what, mods in {"hooked": hooked, "trailing sigmoid": _critic(bnn) + [bnn.Sigmoid()]}.items():
        with pytest.raises(NotImplementedError):
            F.critic_step_mlp(bnn.Sequential(*mods), real, fake, alpha, 10.0)
    with pytest.raises(AssertionError, match="launched"):  # the same critic without the hook goes to the kernel
        F.critic_step_mlp(bnn.Sequential(*_critic(bnn)), real, fake, alpha, 10.0)
