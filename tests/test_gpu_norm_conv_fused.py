"""BatchNorm2d [-> LeakyReLU / ReLU] -> Upsample x2 -> Conv2d backward on fused kernels, end to end: three SGD steps of
the DCGAN generator take functional.NormConvFn for both generator blocks and agree with stock fp32 torch.

The entry points themselves (b200gan_conv2d_dgrad_norm, b200gan_norm_bwd_from_sums and the fused bias gradient of
b200gan_conv2d_wgrad_fused_bias) are checked element by element against fp64 in tests/test_gpu_norm_conv_conformance.py
and tests/test_gpu_conv_conformance.py."""
import copy

import pytest
import torch

from conftest import rel_err

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _fp32_reference():
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    yield


# ---- end to end: DCGAN steps --------------------------------------------------------------------------------------
def _generator_steps(model, steps, batch, img):
    from oracle import ref_models
    opt = torch.optim.SGD(model.parameters(), lr=0.05)
    out = []
    for step in range(steps):
        z = ref_models.synthetic_z(batch, seed=10 + step).cuda()
        target = ref_models.synthetic_images(batch, 1, img, img, seed=10 + step).cuda()
        opt.zero_grad()
        gen = model(z)
        ((gen - target) ** 2).mean().backward()
        out.append((gen.detach(), {k: p.grad.detach().clone() for k, p in model.named_parameters()}))
        opt.step()
    return out


def _set_tf32(on):
    torch.backends.cudnn.allow_tf32 = on
    torch.backends.cuda.matmul.allow_tf32 = on


def test_dcgan_generator_steps_take_the_fused_norm_conv_and_match_stock_fp32(monkeypatch):
    """Three SGD steps of the 64x64 generator; bounds of tests/test_gpu_dcgan.py (output 1e-3; gradients 2e-3 or 1.5x
    what stock TF32 torch reaches against stock fp32)."""
    from oracle import ref_models
    from b200gan import functional as F, zoo
    img, batch, steps = 64, 128, 3   # batch 128: conv1's data gradient is not split over CTAs (at 64 it is)
    g_cpu, _ = ref_models.build_dcgan(img, seed=0)
    _set_tf32(False)
    fp32 = _generator_steps(copy.deepcopy(g_cpu).cuda(), steps, batch, img)
    _set_tf32(True)
    tf32 = _generator_steps(copy.deepcopy(g_cpu).cuda(), steps, batch, img)
    _set_tf32(False)
    g = zoo.DCGANGenerator(img)
    g.load_state_dict(g_cpu.state_dict())
    applied = []
    orig = F.NormConvFn.apply

    def spy(*a):
        applied.append(True)
        return orig(*a)

    monkeypatch.setattr(F.NormConvFn, "apply", spy)
    ours = _generator_steps(g.cuda(), steps, batch, img)
    assert len(applied) == 2 * steps, "both generator norms should run as NormConvFn in every step"
    for step in range(steps):
        assert rel_err(ours[step][0], fp32[step][0]) < 1e-3, f"step {step}: generator output"
        for k, ref in fp32[step][1].items():
            if ref.double().norm().item() < 1e-7:  # conv bias in front of BatchNorm: exactly-zero gradient
                continue
            bound = max(2e-3, 1.5 * rel_err(tf32[step][1][k], ref))
            e = rel_err(ours[step][1][k], ref)
            assert e < bound, f"step {step}: {k}: rel err {e:.2e} exceeds {bound:.2e}"
