"""GPU parity of the fused Generator tail (csrc/tail.cu): BatchNorm2d -> LeakyReLU/ReLU -> Conv2d(C, K<=3, 3, 1, 1)
-> Tanh (dcgan.py:60-63) against stock torch fp32 on the same GPU: output, the gradient that flows into the preceding
conv, and every parameter gradient.  The forward conv runs on wgmma (TF32 operands): 1e-3 on the output; the backward
kernels are fp32, so the gradients only see the TF32 forward through tanh'."""
import pytest
import torch

from conftest import rel_err

pytestmark = pytest.mark.gpu

CASES = [  # N, C, K, H, W, mid activation, out activation
    (4, 64, 1, 32, 32, "lrelu", "tanh"),
    (2, 64, 1, 64, 64, "lrelu", "tanh"),      # the BASELINE geometry (batch reduced)
    (3, 64, 1, 20, 16, "relu", "tanh"),       # ragged bands, 8 rows per tile
    (2, 32, 3, 30, 32, "lrelu", "none"),
    (2, 128, 3, 17, 64, "lrelu", "tanh"),
    (1, 64, 2, 5, 128, "none", "sigmoid"),
]


def _mods(ns, c, k, mid, out):
    layers = [ns.Conv2d(8, c, 3, 1, 1), ns.BatchNorm2d(c, 0.8)]
    if mid == "lrelu":
        layers.append(ns.LeakyReLU(0.2, inplace=True))
    elif mid == "relu":
        layers.append(ns.ReLU(inplace=True))
    layers.append(ns.Conv2d(c, k, 3, stride=1, padding=1))
    if out == "tanh":
        layers.append(ns.Tanh())
    elif out == "sigmoid":
        layers.append(ns.Sigmoid())
    return ns.Sequential(*layers)


@pytest.fixture(autouse=True)
def _fp32_reference():
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    yield


@pytest.mark.parametrize("case", CASES, ids=[str(c) for c in CASES])
def test_tail_matches_stock_torch(case):
    from b200gan import nn as bnn, zoo
    n, c, k, h, w, mid, out = case
    torch.manual_seed(3)
    ref = _mods(zoo.namespace(stock=True), c, k, mid, out).cuda().train()
    ours = _mods(zoo.namespace(), c, k, mid, out).cuda().train()
    with torch.no_grad():
        ref[1].weight.normal_(1.0, 0.2)
        ref[1].bias.normal_(0.0, 0.2)
    ours.load_state_dict(ref.state_dict())
    assert any(type(s).__name__ == "_TailStep" for s in ours._plan())
    x = torch.randn(n, 8, h, w, device="cuda")
    xr, xo = x.clone().requires_grad_(True), x.clone().requires_grad_(True)
    yr, yo = ref(xr), ours(xo)
    assert yo.shape == yr.shape
    assert rel_err(yo, yr) < 1e-3
    gy = torch.randn_like(yr)
    yr.backward(gy)
    yo.backward(gy)
    for (name, po), (_, pr) in zip(ours.named_parameters(), ref.named_parameters()):
        if name == "0.bias":  # conv bias in front of BatchNorm: exactly-zero gradient, fp noise only
            continue
        assert rel_err(po.grad, pr.grad) < 3e-3, name
    assert rel_err(xo.grad, xr.grad) < 3e-3
    for key in ("1.running_mean", "1.running_var", "1.num_batches_tracked"):
        assert rel_err(ours.state_dict()[key].float(), ref.state_dict()[key].float()) < 1e-4, key


def test_tail_falls_back_in_eval_mode_and_keeps_the_accumulators_clean():
    """ADVICE r1: conv -> BatchNorm2d(eval) must not leave partial sums in the shared statistics accumulator."""
    from b200gan import zoo
    torch.manual_seed(4)
    ref = _mods(zoo.namespace(stock=True), 64, 1, "lrelu", "tanh").cuda()
    ours = _mods(zoo.namespace(), 64, 1, "lrelu", "tanh").cuda()
    ours.load_state_dict(ref.state_dict())
    x = torch.randn(2, 8, 32, 32, device="cuda")
    ref.eval(); ours.eval()
    with torch.no_grad():
        assert rel_err(ours(x), ref(x)) < 1e-3
    ref.train(); ours.train()
    xr, xo = x.clone().requires_grad_(True), x.clone().requires_grad_(True)
    yr, yo = ref(xr), ours(xo)
    assert rel_err(yo, yr) < 1e-3
    yr.sum().backward(); yo.sum().backward()
    assert rel_err(ours[1].weight.grad, ref[1].weight.grad) < 3e-3
    assert rel_err(xo.grad, xr.grad) < 3e-3
