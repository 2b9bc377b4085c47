"""SURVEY.md section 8(f) N1: the ConvTranspose2d + BatchNorm2d(.8) + ReLU stacks of context_encoder/models.py:10-37 and
ccgan/models.py:10-42 (the stack BASELINE's north star names), including the 1x1 bottleneck Conv2d(512, 4000, 1)
(context_encoder/models.py:30): fusion plan and parity of outputs / every parameter gradient against stock torch fp32,
with the stock-TF32 yardstick (these layers all run on wgmma)."""
import copy

import pytest
import torch

from conftest import rel_err

pytestmark = pytest.mark.gpu


def _decoder(ns):
    def up(i, o):
        return [ns.ConvTranspose2d(i, o, 4, 2, 1), ns.BatchNorm2d(o, 0.8), ns.ReLU()]

    def down(i, o, normalize=True):
        layers = [ns.Conv2d(i, o, 4, 2, 1)]
        if normalize:
            layers.append(ns.BatchNorm2d(o, 0.8))
        layers.append(ns.LeakyReLU(0.2))
        return layers
    # context_encoder/models.py:23-37 with the channel widths of its deepest stages
    return ns.Sequential(*down(64, 128), *down(128, 512), ns.Conv2d(512, 4000, 1), *up(4000, 512), *up(512, 128),
                         ns.Conv2d(128, 32, 3, 1, 1), ns.Tanh())


def test_plan_fuses_conv_transpose_batchnorm_relu_and_pairs_norm_conv():
    from b200gan import nn as bnn, zoo
    m = _decoder(zoo.namespace())
    plan = m._plan()
    # a BatchNorm2d in front of a stride-1 Conv2d pairs with it (functional.NormConvFn); the others stay single steps
    assert [type(s).__name__ for s in plan] == ["_ConvStep", "_NormStep", "_ConvStep", "_NormConvStep", "_ConvStep",
                                                "_NormStep", "_ConvStep", "_NormConvStep"]
    steps = [p for s in plan for p in (s.fallback if isinstance(s, bnn._NormConvStep) else [s])]
    kinds = [(type(s).__name__, getattr(s, "stats", None)) for s in steps]
    # every (transposed) conv in front of a BatchNorm carries the fused statistics; the norm steps take them
    assert kinds == [("_ConvStep", False), ("_NormStep", None), ("_ConvStep", False), ("_NormStep", None),
                     ("_ConvStep", None), ("_ConvStep", False), ("_NormStep", None), ("_ConvStep", False),
                     ("_NormStep", None), ("_ConvStep", None)]
    assert all(s.takes_stats for s in steps if isinstance(s, bnn._NormStep))
    assert steps[5].conv.__class__.__name__ == "ConvTranspose2d" and steps[6].act == 2   # ReLU fused into the norm


def test_conv_transpose_bn_relu_stack_matches_stock_torch():
    from b200gan import zoo
    torch.manual_seed(13)
    ref = _decoder(zoo.namespace(stock=True)).cuda().train()
    ours = _decoder(zoo.namespace()).cuda().train()
    ours.load_state_dict(ref.state_dict())
    ref_t = copy.deepcopy(ref)
    x = torch.randn(8, 64, 32, 32, device="cuda")
    res = {}
    for name, m, tf32 in (("fp32", ref, False), ("tf32", ref_t, True), ("ours", ours, False)):
        torch.backends.cudnn.allow_tf32 = tf32
        torch.backends.cuda.matmul.allow_tf32 = tf32
        xi = x.clone().requires_grad_(True)
        y = m(xi)
        y.square().mean().backward()
        res[name] = (y.detach(), xi.grad, [(k, p.grad) for k, p in m.named_parameters()])
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    for i, nm in enumerate(("y", "dx")):
        e_o, e_t = rel_err(res["ours"][i], res["fp32"][i]), rel_err(res["tf32"][i], res["fp32"][i])
        assert e_o < max(2e-3, 1.5 * e_t), f"{nm}: ours {e_o:.2e}, stock TF32 {e_t:.2e}"
    top = max(g.double().norm().item() for _, g in res["fp32"][2])
    for (k, go), (_, gr), (_, gt) in zip(res["ours"][2], res["fp32"][2], res["tf32"][2]):
        if gr.double().norm().item() < 1e-5 * top:   # conv bias in front of BatchNorm: analytically zero
            continue
        e_o, e_t = rel_err(go, gr), rel_err(gt, gr)
        assert e_o < max(3e-3, 1.5 * e_t), f"{k}: ours {e_o:.2e}, stock TF32 {e_t:.2e}"
