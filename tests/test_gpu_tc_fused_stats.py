"""Fused BatchNorm / InstanceNorm statistics of the wgmma convolutions at sizes with more output tiles than an H100 has
SMs (ragged maps, one image per tile, 256-wide tiles, the all-phase Upsample(2x)+Conv3x3 kernel), with bias, LeakyReLU
and a Dropout2d scale in the same epilogue, against fp32 torch.  Per-sample sums are also returned when a 128-pixel
tile spans several images (the library then adds a statistics pass)."""
import pytest
import torch
import torch.nn.functional as F

from conftest import rel_err

pytestmark = pytest.mark.gpu

TOL = 1e-3


@pytest.fixture(autouse=True)
def _fp32_reference():
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    yield


def _sums(y, per_sample):
    y = y.double()
    dims = (2, 3) if per_sample else (0, 2, 3)
    return torch.cat([y.sum(dims).flatten(), (y * y).sum(dims).flatten()])


# (name, N, C, K, H, W, up, per_sample, dropout scale): each launches more tiles than an H100 has SMs
CASES = [
    # 20x20 map in 32x4 tiles: 12 of every 32 columns are outside the output (ragged, TMA-clipped)
    ("batchnorm_ragged", 64, 64, 128, 20, 20, 1, False, True),
    # 16x16 map: two tiles per image, so per-sample sums change group at every image
    ("instancenorm_one_image_per_tile", 128, 64, 64, 16, 16, 1, True, False),
    # 256 output channels and enough tiles for the 256-wide tile
    ("batchnorm_bn256", 96, 64, 256, 16, 16, 1, False, False),
    # folded Upsample(2x)+Conv3x3 with 64 output channels: the all-phase kernel, per-sample sums over four phases
    ("allphase_instancenorm", 128, 128, 64, 16, 16, 2, True, True),
    ("allphase_batchnorm", 128, 128, 64, 32, 32, 2, False, False),
    # 8x8 map: a tile holds two images, so per-sample sums cannot be fused into the epilogue
    ("instancenorm_tile_spans_images", 512, 64, 64, 8, 8, 1, True, False),
    # all-phase kernel at 4x4 per phase: eight images per tile
    ("allphase_instancenorm_tile_spans_images", 2048, 128, 64, 4, 4, 2, True, True),
]


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_fused_statistics_over_many_tiles_per_cta(case):
    from b200gan import ops
    from b200gan._lib import ACT_LRELU, ALGO_TC, PACK_TC_FPROP, PACK_TC_FPROP_UP2
    _, n, c, k, h, w, up, per_sample, drop = case
    torch.manual_seed(0)
    x = torch.randn(n, c, h, w, device="cuda").contiguous(memory_format=torch.channels_last)
    wt = torch.randn(k, c, 3, 3, device="cuda") * (1.0 / (3 * c ** 0.5))
    bias = torch.randn(k, device="cuda") * 0.5 + 0.5
    scale = (torch.rand(n, k, device="cuda") < 0.8).float() * 1.25 if drop else None
    g, _ = ops.make_geom(tuple(x.shape), tuple(wt.shape), 1, (1, 1, 1, 1), 0, up, False)
    assert ops.tc_supported(g, 0)
    packed = ops.pack_weights(g, wt, PACK_TC_FPROP_UP2 if up == 2 else PACK_TC_FPROP)
    stats = torch.zeros(2 * (n * k if per_sample else k), device="cuda", dtype=torch.float64)
    y = ops.conv_fprop(g, x, packed, ALGO_TC, bias=bias, act=ACT_LRELU, slope=0.2, chan_scale=scale, stats=stats,
                       stats_per_sample=per_sample)
    xr = F.interpolate(x, scale_factor=2, mode="nearest") if up == 2 else x
    yr = F.leaky_relu(F.conv2d(xr, wt, bias, padding=1), 0.2)
    if drop:
        yr = yr * scale[:, :, None, None]
    torch.cuda.synchronize()
    assert rel_err(y, yr) < TOL
    assert rel_err(stats, _sums(yr, per_sample)) < TOL
