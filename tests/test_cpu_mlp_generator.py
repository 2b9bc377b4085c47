"""The MLP generator (csrc/mlp_generator/mlp_generator.cu, functional.MlpGeneratorFn) without a GPU: the fp64
references of tests/generator_cases.py against torch float64 autograd for every case of the table, which module lists
the drop-in Sequential routes to the kernels, the BatchNorm1d drop-in on the CPU, and ptxas's registers and spills."""
import math
import os

import pytest
import torch

import generator_cases as gc
from b200gan import nn as bnn
from conformance import CSRC, declared, needs_nvcc, ptxas_report, table_kernels

GEN_CU = os.path.join(CSRC, "mlp_generator", "mlp_generator.cu")


# ---- the fp64 references against torch float64 autograd -------------------------------------------------------------
def _stock(c, P):
    """nn.Sequential float64 of the case, with its parameters and running statistics"""
    tnn, mods = torch.nn, []
    for l in range(c.L):
        lin = tnn.Linear(c.widths[l], c.widths[l + 1]).double()
        with torch.no_grad():
            lin.weight.copy_(P[f"W{l}"])
            lin.bias.copy_(P[f"b{l}"])
        mods.append(lin)
        if l == c.L - 1:
            mods.append(tnn.Tanh())
            break
        if c.has_norm[l]:
            # the kernel's eps and momentum are fp32
            bn = tnn.BatchNorm1d(c.widths[l + 1], gc.f32(gc.EPS), momentum=gc.f32(gc.MOMENTUM)).double()
            with torch.no_grad():
                for name, key in (("weight", "gamma"), ("bias", "beta"), ("running_mean", "rm"), ("running_var", "rv"),
                                  ("num_batches_tracked", "nbt")):
                    getattr(bn, name).copy_(P[f"{key}{l}"].reshape(()) if key == "nbt" else P[f"{key}{l}"])
            mods.append(bn)
        mods.append(tnn.LeakyReLU(gc.f32(c.slope), inplace=True))
    return tnn.Sequential(*mods)


@pytest.mark.parametrize("case", [c for c in gc.CASES if not c.error and (c.op == "fwd" or c.only is None)],
                         ids=lambda c: c.id)
def test_references_are_torch_float64_autograd(case):
    c, P = case, gc.make(case, seed=0)
    net = _stock(c, P)
    z = P["z"].double().requires_grad_(True)
    out = net(z)
    layers = gc.gen_fwd_ref(P, c)
    torch.testing.assert_close(layers[-1]["out"], out.detach(), rtol=1e-12, atol=1e-12)
    bns = [m for m in net if isinstance(m, torch.nn.BatchNorm1d)]
    for l, bn in zip([l for l in range(c.L - 1) if c.has_norm[l]], bns):
        torch.testing.assert_close(layers[l]["rm"], bn.running_mean, rtol=1e-12, atol=1e-12)
        torch.testing.assert_close(layers[l]["rv"], bn.running_var, rtol=1e-12, atol=1e-12)
        assert bn.num_batches_tracked.item() == P[f"nbt{l}"].item() + 1
    dout = P["dout"].double()
    params = list(net.parameters())
    want = dict(zip(["dz"] + [n for l in range(c.L) for n in (f"dW{l}", f"db{l}") +
                              ((f"dgamma{l}", f"dbeta{l}") if c.has_norm[l] else ())],
                    torch.autograd.grad(out, [z] + params, dout)))
    acts, xh, rs = gc.split_saved(c, gc.saved_of(c, layers), c.N)
    r = gc.gen_bwd_ref(c, dout, layers[-1]["out"], P["z"].double(), [P[f"W{l}"].double() for l in range(c.L)],
                         [P[f"gamma{l}"].double() if c.has_norm[l] else None for l in range(c.L)], acts, xh, rs)
    assert set(r) == set(c.all_outputs()) == set(want)
    for name, w in want.items():
        torch.testing.assert_close(r[name][0].reshape(w.shape), w, rtol=1e-9, atol=1e-11, msg=name)


# ---- the case table --------------------------------------------------------------------------------------------------
def test_generator_table_covers_its_edges():
    ids = [c.id for c in gc.CASES]
    assert len(ids) == len(set(ids)) and all(c.why for c in gc.CASES)
    assert declared(GEN_CU) == set(gc.KERNEL.values()) == table_kernels(gc.CASES)
    for op in ("fwd", "bwd"):
        ok = [c for c in gc.CASES if c.op == op and not c.error]
        assert any(c.N == 64 and c.widths == gc.WGAN for c in ok) and any(c.widths == gc.GAN for c in ok), op
        assert any(any(w % 32 for w in c.widths) for c in ok) and any(c.N == 2 for c in ok), op
        assert any(c.L == 1 for c in ok) and {0.0, 0.2, 1.0} <= {c.slope for c in ok}, op
        assert any(math.ceil(c.N / 32) * math.ceil(max(c.widths) / 32) > 2 * gc.GRID[0] for c in ok), op
        err = {c.name for c in gc.CASES if c.op == op and c.error}
        assert {"n1", "wide", "no_ws"} <= err, op
    single = gc.Case("", "bwd", 0, gc.SMALL, (1, 1)).all_outputs()
    assert {f"{o}_only" for o in single} <= {c.name for c in gc.CASES if c.op == "bwd"}
    assert any(not c.keep for c in gc.CASES if c.op == "fwd" and not c.error)


def test_build_compiles_every_source_at_any_depth():
    import build as b200_build
    assert os.path.join("mlp_generator", "mlp_generator.cu") in b200_build.sources()
    assert all(os.path.isfile(os.path.join(CSRC, f)) for f in b200_build._files())


@needs_nvcc
def test_generator_kernels_do_not_spill_and_the_grid_follows_from_the_registers():
    rep = ptxas_report(GEN_CU)
    for name, r in rep.items():
        assert r["stack"] == r["spills"] == 0, f"{name}: {r}"
    regs = {k: r["registers"] for k, r in rep.items()}
    assert regs == gc.REGISTERS, f"ptxas {regs}, table {gc.REGISTERS}"
    assert [r["smem"] for r in rep.values()] == [gc.SMEM_BYTES] * 2
    per_sm = min(gc.blocks_per_sm(v) for v in regs.values())
    assert gc.GRID == (gc.NUM_SMS * min(2, per_sm), 1, 1)
    assert all(c.grid == gc.GRID for c in gc.CASES if not c.error)


# ---- which Sequentials run on the generator kernels ------------------------------------------------------------------
def _gen(ns, widths=(100, 128, 256, 512, 1024, 784), norms=(False, True, True, True), slopes=None, bias=True):
    slopes = slopes or (0.2,) * len(norms)
    mods = []
    for l, (i, o) in enumerate(zip(widths[:-2], widths[1:-1])):
        mods.append(ns.Linear(i, o, bias=bias))
        if norms[l]:
            mods.append(ns.BatchNorm1d(o, 0.8))
        mods.append(ns.LeakyReLU(slopes[l], inplace=True))
    return mods + [ns.Linear(widths[-2], widths[-1]), ns.Tanh()]


@pytest.mark.parametrize("ns", [torch.nn, bnn], ids=["stock", "dropin"])
def test_accepts_the_wgan_gp_and_gan_generators(ns):
    for widths in ((100, 128, 256, 512, 1024, 1024), (100, 128, 256, 512, 1024, 784)):
        mods = _gen(ns, widths)
        plan = bnn.mlp_generator_layers(mods, 100)
        assert plan is not None
        layers, slope = plan
        assert slope == 0.2 and [lin for lin, _ in layers] == [m for m in mods if isinstance(m, torch.nn.Linear)]
        assert [bn is not None for _, bn in layers] == [False, True, True, True, False]
    assert bnn.mlp_generator_layers([ns.Linear(100, 784), ns.Tanh()], 100) is not None, "L = 1"


def _modify(mods, what):
    bns = [m for m in mods if isinstance(m, torch.nn.BatchNorm1d)]
    if what == "eval":
        bns[0].eval()
    elif what == "momentum None":
        bns[1].momentum = None
    elif what == "hook":
        mods[0].register_forward_hook(lambda m, a, o: None)
    elif what == "bn hook":
        bns[0].register_forward_pre_hook(lambda m, a: None)
    return mods


@pytest.mark.parametrize("ns", [torch.nn, bnn], ids=["stock", "dropin"])
def test_rejects_everything_else(ns):
    reject = {
        "hook": _modify(_gen(ns), "hook"),
        "bn hook": _modify(_gen(ns), "bn hook"),
        "bias-less Linear": _gen(ns, bias=False),
        "eval mode": _modify(_gen(ns), "eval"),
        "momentum None": _modify(_gen(ns), "momentum None"),
        "affine False": _gen(ns)[:2] + [ns.Linear(128, 256), ns.BatchNorm1d(256, 0.8, affine=False)] + _gen(ns)[4:],
        "untracked": _gen(ns)[:2] + [ns.Linear(128, 256), ns.BatchNorm1d(256, 0.8, track_running_stats=False)] +
        _gen(ns)[4:],
        "other eps": _gen(ns)[:2] + [ns.Linear(128, 256), ns.BatchNorm1d(256, 1e-5)] + _gen(ns)[4:],
        "mixed slopes": _gen(ns, slopes=(0.2, 0.2, 0.1, 0.2)),
        "negative slope": _gen(ns, slopes=(-0.2,) * 4),
        "no tanh": _gen(ns)[:-1],
        "sigmoid": _gen(ns)[:-1] + [ns.Sigmoid()],
        "one output": _gen(ns, widths=(100, 128, 256, 512, 1024, 1)),
        "relu": _gen(ns)[:1] + [ns.ReLU()] + _gen(ns)[2:],
        "dropout": _gen(ns)[:2] + [ns.Dropout(0.5)] + _gen(ns)[2:],
        "nine layers": _gen(ns, widths=(100,) + (64,) * 9, norms=(True,) * 8),
        "too wide": _gen(ns, widths=(100, 8193, 784), norms=(True,)),
    }
    for what, mods in reject.items():
        assert bnn.mlp_generator_layers(mods, 100) is None, what
    assert bnn.mlp_generator_layers(_gen(ns), 101) is None, "mismatched input width"


def test_plan_has_no_side_effects():
    mods = _gen(bnn)
    state = {k: v.clone() for k, v in torch.nn.Sequential(*mods).state_dict().items()}
    assert bnn.mlp_generator_layers(mods, 100) is not None
    for k, v in torch.nn.Sequential(*mods).state_dict().items():
        assert torch.equal(v, state[k]), k


def test_batchnorm1d_drop_in_is_the_stock_module_on_the_cpu():
    torch.manual_seed(0)
    ours, ref = bnn.BatchNorm1d(33, 0.8), torch.nn.BatchNorm1d(33, 0.8)
    assert type(ours).__name__ == "BatchNorm1d" and bnn.REPLACEMENTS["BatchNorm1d"] is bnn.BatchNorm1d
    assert ours.state_dict().keys() == ref.state_dict().keys()
    x = torch.randn(9, 33)
    assert torch.equal(ours(x), ref(x))
    for k, v in ref.state_dict().items():
        assert torch.equal(ours.state_dict()[k], v), k
    torch.manual_seed(1)
    seq_ours = bnn.Sequential(*_gen(bnn, widths=(20, 64, 128, 64), norms=(False, True)))
    torch.manual_seed(1)
    seq_ref = torch.nn.Sequential(*_gen(torch.nn, widths=(20, 64, 128, 64), norms=(False, True)))
    z = torch.randn(5, 20)
    assert torch.equal(seq_ours(z), seq_ref(z))
    with pytest.raises(ValueError, match="Expected more than 1 value per channel"):
        seq_ours(z[:1])
