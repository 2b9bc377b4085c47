"""GPU parity of the fused Generator tail (csrc/tail.cu) at sizes that exercise how the backward splits its work into
per-block pixel ranges, against stock torch fp32 with the bounds of test_gpu_tail.py: the full DCGAN geometry, ranges
that start mid-image with H not dividing evenly, fewer pixels than one ring stage, one-row images (a zero separator
row in the staged output gradient after every row), and enough pixels that the staged output gradient caps the range
length and the grid has more blocks than resident slots."""
import pytest
import torch

from conftest import rel_err
from tail_cases import mods

pytestmark = pytest.mark.gpu

CASES = [  # N, C, K, H, W, mid activation, out activation
    (128, 64, 1, 64, 64, "lrelu", "tanh"),    # the DCGAN geometry
    (7, 128, 3, 37, 32, "lrelu", "tanh"),     # ranges start mid-image; 37 rows
    (1, 32, 2, 3, 16, "relu", "tanh"),        # 48 pixels: less than one ring stage, one block
    (5, 64, 1, 1, 64, "lrelu", "none"),       # one-row images
    (8000, 32, 1, 1, 128, "lrelu", "tanh"),   # range length capped by the staged g: 334 blocks for 264 slots
]


@pytest.fixture(autouse=True)
def _fp32_reference():
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    yield


@pytest.mark.parametrize("case", CASES, ids=[str(c) for c in CASES])
def test_tail_ranges_match_stock_torch(case):
    from b200gan import zoo
    n, c, k, h, w, mid, out = case
    torch.manual_seed(5)
    ref = mods(zoo.namespace(stock=True), c, k, mid, out).cuda().train()
    ours = mods(zoo.namespace(), c, k, mid, out).cuda().train()
    with torch.no_grad():
        ref[1].weight.normal_(1.0, 0.2)
        ref[1].bias.normal_(0.0, 0.2)
    ours.load_state_dict(ref.state_dict())
    assert any(type(s).__name__ == "_TailStep" for s in ours._plan())
    x = torch.randn(n, 8, h, w, device="cuda")
    xr, xo = x.clone().requires_grad_(True), x.clone().requires_grad_(True)
    yr, yo = ref(xr), ours(xo)
    assert rel_err(yo, yr) < 1e-3
    gy = torch.randn_like(yr)
    yr.backward(gy)
    yo.backward(gy)
    for (name, po), (_, pr) in zip(ours.named_parameters(), ref.named_parameters()):
        if name == "0.bias":  # conv bias in front of BatchNorm: exactly-zero gradient, fp noise only
            continue
        assert rel_err(po.grad, pr.grad) < 3e-3, name
    assert rel_err(xo.grad, xr.grad) < 3e-3
