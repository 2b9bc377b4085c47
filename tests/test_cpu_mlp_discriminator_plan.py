"""Which module lists the drop-in Sequential runs as the vanilla GAN discriminator (functional.MlpDiscriminatorFn):
exactly Linear(Din, H1) -> LeakyReLU(s) -> Linear(H1, H2) -> LeakyReLU(s) -> Linear(H2, 1) -> Sigmoid, all with biases,
one slope >= 0 (gan.py:64-80, bgan.py:66-80 with Din 784; aae.py:90-104 with Din = latent_dim = 10).  Everything else
keeps its other paths.  Also: the discriminator's entry points launch only the MLP critic's kernels."""
import os
import re

import pytest
import torch

import critic_cases as cr
from b200gan import nn as bnn
from conformance import CSRC, declared, functions

MC_CU = os.path.join(CSRC, "mlp_critic.cu")


def _disc(ns, din=784, h1=512, h2=256, slopes=(0.2, 0.2), biases=(True, True, True), out=1, inplace=True,
          last=None):
    mods = [ns.Linear(din, h1, bias=biases[0]), ns.LeakyReLU(slopes[0], inplace=inplace),
            ns.Linear(h1, h2, bias=biases[1]), ns.LeakyReLU(slopes[1], inplace=inplace),
            ns.Linear(h2, out, bias=biases[2])]
    return mods + [last() if last else ns.Sigmoid()]


@pytest.mark.parametrize("ns", [torch.nn, bnn], ids=["stock", "dropin"])
@pytest.mark.parametrize("din", [784, 10], ids=["gan_bgan", "aae"])
@pytest.mark.parametrize("inplace", [True, False])
def test_accepts_the_gan_bgan_and_aae_discriminators(ns, din, inplace):
    mods = _disc(ns, din, inplace=inplace)
    plan = bnn.mlp_discriminator_layers(mods, din)
    assert plan is not None
    l1, l2, l3, slope = plan
    assert (l1, l2, l3) == (mods[0], mods[2], mods[4]) and slope == 0.2
    assert bnn.mlp_critic_layers(mods, din) is None, "the critic recogniser still refuses a trailing Sigmoid"
    for s in (0.0, 1.0):
        assert bnn.mlp_discriminator_layers(_disc(ns, din, slopes=(s, s)), din)[3] == s


@pytest.mark.parametrize("ns", [torch.nn, bnn], ids=["stock", "dropin"])
def test_rejects_everything_else(ns):
    reject = {
        "trailing tanh": _disc(ns, last=ns.Tanh),
        "no activation at the end": _disc(ns)[:5],
        "different slopes": _disc(ns, slopes=(0.2, 0.1)),
        "negative slope": _disc(ns, slopes=(-0.2, -0.2)),
        "missing bias 1": _disc(ns, biases=(False, True, True)),
        "missing bias 2": _disc(ns, biases=(True, False, True)),
        "missing bias 3": _disc(ns, biases=(True, True, False)),
        "two outputs": _disc(ns, out=2),
        "relu": _disc(ns)[:1] + [ns.ReLU()] + _disc(ns)[2:],
        "two Linears": [ns.Linear(784, 512), ns.LeakyReLU(0.2), ns.Linear(512, 1), ns.Sigmoid()],
        "four Linears": _disc(ns)[:4] + [ns.Linear(256, 128), ns.LeakyReLU(0.2), ns.Linear(128, 1), ns.Sigmoid()],
        "sigmoid twice": _disc(ns) + [ns.Sigmoid()],
        "dropout": _disc(ns)[:2] + [ns.Dropout(0.4)] + _disc(ns)[2:],
    }
    for what, mods in reject.items():
        assert bnn.mlp_discriminator_layers(mods, 784) is None, what
    assert bnn.mlp_discriminator_layers(_disc(ns), 785) is None, "mismatched input width"
    assert bnn.mlp_discriminator_layers(_disc(ns, din=10), 784) is None, "mismatched input width"


@pytest.mark.parametrize("at", range(6))
@pytest.mark.parametrize("kind", ["forward", "forward_pre", "full_backward"])
def test_rejects_hooks_on_any_module(at, kind):
    mods = _disc(bnn)
    m = mods[at]
    if kind == "forward":
        h = m.register_forward_hook(lambda m_, a, o: None)
    elif kind == "forward_pre":
        h = m.register_forward_pre_hook(lambda m_, a: None)
    else:
        h = m.register_full_backward_hook(lambda m_, gi, go: None)
    assert bnn.mlp_discriminator_layers(mods, 784) is None
    h.remove()
    assert bnn.mlp_discriminator_layers(mods, 784) is not None


def test_plan_has_no_side_effects():
    mods = _disc(bnn)
    seq = torch.nn.Sequential(*mods)
    state = {k: v.clone() for k, v in seq.state_dict().items()}
    assert bnn.mlp_discriminator_layers(mods, 784) is not None
    assert bnn.mlp_discriminator_layers(mods, 785) is None
    for k, v in seq.state_dict().items():
        assert torch.equal(v, state[k]), k
    assert all(p.grad is None for p in seq.parameters())
    assert [m.training for m in mods] == [True] * 6


def test_the_discriminator_on_the_cpu_is_the_stock_module():
    """the drop-in Sequential on a CPU tensor runs the stock modules, bit for bit"""
    torch.manual_seed(0)
    ours = bnn.Sequential(*_disc(bnn, din=10))
    torch.manual_seed(0)
    ref = torch.nn.Sequential(*_disc(torch.nn, din=10))
    x = torch.randn(7, 10)
    assert torch.equal(ours(x), ref(x))


# ---- the entry points and the kernels they launch --------------------------------------------------------------------
def _launched(fns, name, seen=()):
    body = fns[name]
    assert "<<<" not in body, name
    kernels = set(re.findall(r"launch_coop\(\s*(\w+)", body))
    for callee in set(re.findall(r"\b(\w+)\s*\(", body)) & set(fns):
        if callee != name and callee not in seen:
            kernels |= _launched(fns, callee, seen + (name,))
    return kernels


def test_mlp_critic_cu_declares_only_the_critic_kernels_and_the_disc_entry_points_launch_them():
    assert declared(MC_CU) == set(cr.KERNEL.values())
    fns = functions(open(MC_CU).read())
    assert {"b200gan_mlp_disc_fwd", "b200gan_mlp_disc_bwd", "b200gan_mlp_disc_bwd_workspace_floats"} <= set(fns)
    assert _launched(fns, "b200gan_mlp_disc_fwd") == {cr.KERNEL["fwd"]}
    assert _launched(fns, "b200gan_mlp_disc_bwd") == {cr.KERNEL["bwd"]}
    assert _launched(fns, "b200gan_mlp_disc_bwd_workspace_floats") == set()
    # the critic entry points launch the same kernels as before
    assert _launched(fns, "b200gan_mlp_critic_fwd") == {cr.KERNEL["fwd"]}
    assert _launched(fns, "b200gan_mlp_critic_bwd") == {cr.KERNEL["bwd"]}
