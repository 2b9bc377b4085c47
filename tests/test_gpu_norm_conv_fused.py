"""BatchNorm2d [-> LeakyReLU / ReLU] [-> Upsample x2] -> Conv2d backward on fused kernels, against fp64:

  * b200gan_conv2d_dgrad_norm: the conv's data gradient, bit-identical to b200gan_conv2d_dgrad, with the norm backward's
    sums (sum dy', sum dy' * xhat) accumulated in the same epilogue -- DCGAN's two generator geometries, activations
    none / LeakyReLU / ReLU, up 1 and 2, ragged maps with pixels outside the output in a tile -- and its refusals;
  * b200gan_norm_bwd_from_sums: dx and dgamma / dbeta from those sums, the sums handed back zeroed;
  * the bias gradient the tensor-core weight gradient now produces itself, on up2 and plain geometries with several
    pixel splits (each dy pixel counted once);
  * the kernels each call launches, one CUDA-graph replay, and DCGAN training steps against stock fp32 torch.

Outputs land in NaN-filled buffers between NaN guard regions: every element must be written, nothing around it."""
import ctypes
import copy

import pytest
import torch
import torch.nn.functional as tf

from conformance import check_route, traced_kernels
from conftest import rel_err

pytestmark = pytest.mark.gpu

CL = torch.channels_last
GUARD = 64
EPS32 = 2.0 ** -24


@pytest.fixture(autouse=True)
def _fp32_reference():
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    yield


def _guarded(shape, dtype=torch.float32, cl=True):
    """(buffer with NaN guards, view of the payload): a NaN-filled payload between two NaN guard regions."""
    n = 1
    for s in shape:
        n *= s
    buf = torch.full((n + 2 * GUARD,), float("nan"), device="cuda", dtype=dtype)
    body = buf[GUARD:GUARD + n]
    if len(shape) == 4 and cl:
        nn_, c, h, w = shape
        view = body.view(nn_, h, w, c).permute(0, 3, 1, 2)
    else:
        view = body.view(shape)
    return buf, view


def _guards_intact(buf):
    return bool(torch.isnan(buf[:GUARD]).all()) and bool(torch.isnan(buf[-GUARD:]).all())


# (id, N, C, K, H, W, up, act, slope): C = norm channels = conv input channels, K = conv output channels
CASES = [
    ("dcgan_bn128_up_conv128", 128, 128, 128, 16, 16, 2, 0, 0.0),      # dcgan.py:53-55
    ("dcgan_bn128_lrelu_up_conv64", 128, 128, 64, 32, 32, 2, 1, 0.2),  # dcgan.py:56-59
    ("relu_up1_3x3", 96, 64, 64, 16, 16, 1, 2, 0.0),
    ("lrelu_up1_ragged_12x12", 96, 64, 32, 12, 12, 1, 1, 0.1),         # 16x8 tiles over 12x12: invalid rows/columns
    ("none_up2_ragged_10x10", 80, 64, 64, 10, 10, 2, 0, 0.0),          # 16x8 tiles over 10x10 per phase grid
    ("relu_up2_k32", 128, 64, 32, 16, 16, 2, 2, 0.0),
]
EXPECTED_DGRAD = {128: "conv_tc_kernel<128, 6>", 64: "conv_tc_kernel<64, 8>", 32: "conv_tc_kernel<32, 8>"}


class Setup:
    def __init__(self, case, seed=0):
        from b200gan import ops
        from b200gan._lib import PACK_TC_DGRAD, PACK_TC_DGRAD_UP2
        _, n, c, k, h, w, up, act, slope = case
        self.case, self.act, self.slope, self.up = case, act, slope, up
        gen = torch.Generator(device="cuda").manual_seed(seed)
        self.x = (torch.randn(n, c, h, w, device="cuda", generator=gen) * 1.5 + 0.3).contiguous(memory_format=CL)
        self.gamma = torch.rand(c, device="cuda", generator=gen) + 0.5
        self.beta = torch.randn(c, device="cuda", generator=gen) * 0.2
        self.eps = 0.8 if c == 128 else 1e-5
        _, self.mean_rstd, self.scale_shift = ops.norm_forward(self.x, self.gamma, self.beta, None, None, None, False,
                                                               self.eps, 0.0, act, slope, return_scale_shift=True)
        self.g, oshape = ops.make_geom((n, c, h, w), (k, c, 3, 3), 1, (1, 1, 1, 1), 0, up, False)
        self.wt = torch.randn(k, c, 3, 3, device="cuda", generator=gen) / (3 * c ** 0.5)
        self.packed = ops.pack_weights(self.g, self.wt, PACK_TC_DGRAD_UP2 if up == 2 else PACK_TC_DGRAD)
        self.dy = torch.randn(*oshape, device="cuda", generator=gen).contiguous(memory_format=CL)
        self.desc = ops._norm_desc(self.x.shape, False, self.eps, 0.0, act, slope, False)

    def dgrad_norm(self, dx, sums, stream=None):
        from b200gan import _lib, ops
        return _lib.load().b200gan_conv2d_dgrad_norm(
            ctypes.byref(self.g), ctypes.byref(self.desc), self.dy.data_ptr(), self.packed.data_ptr(), self.x.data_ptr(),
            self.mean_rstd.data_ptr(), self.scale_shift.data_ptr(), sums.data_ptr(), dx.data_ptr(),
            stream if stream is not None else ops._stream())

    def from_sums(self, da, sums, dx, dgb, stream=None):
        from b200gan import _lib, ops
        return _lib.load().b200gan_norm_bwd_from_sums(
            ctypes.byref(self.desc), da.data_ptr(), self.x.data_ptr(), self.mean_rstd.data_ptr(),
            self.scale_shift.data_ptr(), self.gamma.data_ptr(), sums.data_ptr(), dx.data_ptr(), dgb.data_ptr(),
            stream if stream is not None else ops._stream())

    def terms64(self, da):
        """fp64 dy' and xhat from the data gradient da (the same mask rule as the kernels: from x * scale + shift)"""
        c = self.x.shape[1]
        x = self.x.double()
        sc, sh = self.scale_shift[:c].double().view(1, -1, 1, 1), self.scale_shift[c:].double().view(1, -1, 1, 1)
        mean, rstd = self.mean_rstd[:c].double().view(1, -1, 1, 1), self.mean_rstd[c:].double().view(1, -1, 1, 1)
        pre = x * sc + sh
        if self.act == 1:
            mask = torch.where(pre > 0, 1.0, float(torch.tensor(self.slope, dtype=torch.float32)))
        elif self.act == 2:
            mask = (pre > 0).double()
        else:
            mask = torch.ones_like(pre)
        return da.double() * mask, (x - mean) * rstd


def _dgrad_plain(s):
    from b200gan import ops
    from b200gan._lib import ALGO_TC
    return ops.conv_dgrad(s.g, s.dy, s.packed, ALGO_TC)


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_dgrad_norm_sums_and_apply_from_sums_vs_fp64(case):
    from b200gan import ops
    s = Setup(case)
    assert ops.conv_dgrad_norm_supported(s.g), f"{case[0]}: geometry should take the fused data gradient"
    n, c, h, w = s.x.shape
    buf, da = _guarded((n, c, h, w))
    sums = torch.zeros(2 * c, device="cuda", dtype=torch.float64)
    assert s.dgrad_norm(da, sums) == 0
    torch.cuda.synchronize()
    assert _guards_intact(buf) and not torch.isnan(da).any(), f"{case[0]}: dx written outside / not everywhere"
    # the data gradient is the unfused one, bit for bit
    ref_da = _dgrad_plain(s)
    assert torch.equal(da.contiguous(memory_format=CL).view(torch.int32), ref_da.view(torch.int32)), case[0]
    # and matches the fp64 convolution gradient within TF32 operand rounding
    x64 = torch.zeros(n, c, h, w, dtype=torch.float64, device="cuda", requires_grad=True)
    inp = tf.interpolate(x64, scale_factor=2, mode="nearest") if s.up == 2 else x64
    tf.conv2d(inp, s.wt.double(), padding=1).backward(s.dy.double())
    assert rel_err(da, x64.grad) < 2e-3
    # sums against fp64 over the data gradient the kernel produced; bound: fp32 partial sums of <= 128 terms per
    # column of a tile (warp transpose + four warps), added in fp64 -- 8 roundings of the absolute sum, with margin 4x
    dz, xhat = s.terms64(da)
    want = torch.cat([dz.sum((0, 2, 3)), (dz * xhat).sum((0, 2, 3))])
    absum = torch.cat([dz.abs().sum((0, 2, 3)), (dz * xhat).abs().sum((0, 2, 3))])
    bound = 32 * EPS32 * absum + 1e-30
    err = (sums - want).abs()
    assert (err <= bound).all(), f"{case[0]}: sums off by {(err / bound).max().item():.2f} x the bound"
    # norm apply from these sums vs fp64; the workspace comes back zeroed
    bx, dx = _guarded((n, c, h, w))
    bg, dgb = _guarded((2 * c,), cl=False)
    assert s.from_sums(da.contiguous(memory_format=CL), sums, dx, dgb) == 0
    torch.cuda.synchronize()
    assert _guards_intact(bx) and _guards_intact(bg) and not torch.isnan(dx).any() and not torch.isnan(dgb).any()
    assert (sums == 0).all(), "norm_bwd_from_sums must hand the sums back zeroed"
    count = n * h * w
    m1, m2 = (want[:c] / count).view(1, -1, 1, 1), (want[c:] / count).view(1, -1, 1, 1)
    gr = (s.gamma.double() * s.mean_rstd[c:].double()).view(1, -1, 1, 1)
    dx_ref = gr * (dz - m1 - xhat * m2)
    assert rel_err(dx, dx_ref) < 1e-5
    assert rel_err(dgb[:c], want[c:]) < 1e-6 and rel_err(dgb[c:], want[:c]) < 1e-6
    # the unfused norm backward on the same gradient agrees
    dx_unfused, dgb_unfused = ops.norm_backward(da.contiguous(memory_format=CL), s.x, None, s.mean_rstd, s.gamma, False,
                                                s.eps, s.act, s.slope, True, False, s.scale_shift)
    assert rel_err(dx, dx_unfused) < 1e-5 and rel_err(dgb, dgb_unfused) < 1e-5


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_dgrad_norm_kernels_and_graph_replay(case):
    s = Setup(case)
    n, c, h, w = s.x.shape
    da = torch.empty_like(s.x, memory_format=CL)
    dx = torch.empty_like(s.x, memory_format=CL)
    dgb = torch.empty(2 * c, device="cuda")
    sums = torch.zeros(2 * c, device="cuda", dtype=torch.float64)

    def both(stream=None):
        assert s.dgrad_norm(da, sums, stream) == 0
        assert s.from_sums(da, sums, dx, dgb, stream) == 0

    check_route(case[0], both, [(EXPECTED_DGRAD[c], None), ("norm_bwd_apply_kernel<4>", None),
                                ("norm_bwd_params_kernel", None)])
    eager = (da.clone(), dx.clone(), dgb.clone())
    side = torch.cuda.Stream()
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=side):
        both(side.cuda_stream)
    for t in (da, dx, dgb):
        t.fill_(float("nan"))
    torch.cuda.synchronize()
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(da.view(torch.int32), eager[0].view(torch.int32))
    assert rel_err(dx, eager[1]) < 1e-6 and rel_err(dgb, eager[2]) < 1e-6
    assert (sums == 0).all()


def test_dgrad_norm_refusals():
    from b200gan import _lib, ops
    from b200gan._lib import PAD_REFLECT
    lib = _lib.load()
    base = CASES[0]
    s = Setup(base)
    c = s.x.shape[1]
    sums = torch.zeros(2 * c, device="cuda", dtype=torch.float64)
    da = torch.empty_like(s.x, memory_format=CL)
    # per-sample (InstanceNorm) statistics
    s.desc.per_sample = 1
    assert s.dgrad_norm(da, sums) == -1
    s.desc.per_sample = 0
    # reflection padding
    g = _lib.ConvGeom.from_buffer_copy(s.g)
    g.pad_mode, g.up = PAD_REFLECT, 1
    g.P, g.Q = g.H, g.W
    assert not lib.b200gan_conv2d_dgrad_norm_supported(ctypes.byref(g))
    # a layer with so few output tiles that the contraction is split over CTAs
    gs, _ = ops.make_geom((2, 64, 8, 8), (64, 64, 3, 3), 1, (1, 1, 1, 1), 0, 2, False)
    assert ops.tc_supported(gs, 1) and not ops.conv_dgrad_norm_supported(gs)
    # fewer than 32 channels on the norm side: no tensor-core data gradient
    gn, _ = ops.make_geom((64, 16, 16, 16), (64, 16, 3, 3), 1, (1, 1, 1, 1), 0, 1, False)
    assert not ops.conv_dgrad_norm_supported(gn)
    # stride 2 writes its gradient through a phase view
    g2, _ = ops.make_geom((64, 64, 16, 16), (64, 64, 3, 3), 2, (1, 1, 1, 1), 0, 1, False)
    assert ops.tc_supported(g2, 1) and not ops.conv_dgrad_norm_supported(g2)
    # the entry point itself refuses what the query refuses
    s2 = Setup(("split", 2, 64, 64, 8, 8, 2, 0, 0.0))
    sums2 = torch.zeros(128, device="cuda", dtype=torch.float64)
    assert s2.dgrad_norm(torch.empty_like(s2.x, memory_format=CL), sums2) == -1
    torch.cuda.synchronize()
    assert (sums == 0).all() and (sums2 == 0).all()


# ---- bias gradient inside the tensor-core weight gradient ----------------------------------------------------------
# (id, N, C, K, H, W, up, stride): dy is the A operand (K % 128 == 0) or the B operand (K in {32, 64})
WGRAD_CASES = [
    ("dcgan_up2_conv128", 128, 128, 128, 16, 16, 2, 1),
    ("dcgan_up2_conv64", 128, 128, 64, 32, 32, 2, 1),
    ("plain_k128_many_splits", 256, 64, 128, 16, 16, 1, 1),
    ("plain_k32_b_operand", 64, 128, 32, 20, 20, 1, 1),
    ("stride2_k128", 64, 64, 128, 32, 32, 1, 2),
]


@pytest.mark.parametrize("case", WGRAD_CASES, ids=[c[0] for c in WGRAD_CASES])
def test_tc_wgrad_bias_gradient_vs_fp64(case):
    from b200gan import _lib, ops
    from b200gan._lib import ALGO_AUTO
    _, n, c, k, h, w, up, stride = case
    gen = torch.Generator(device="cuda").manual_seed(3)
    x = torch.randn(n, c, h, w, device="cuda", generator=gen).contiguous(memory_format=CL)
    g, oshape = ops.make_geom((n, c, h, w), (k, c, 3, 3), stride, (1, 1, 1, 1), 0, up, False)
    assert ops.tc_supported(g, 2)
    dy = (torch.randn(*oshape, device="cuda", generator=gen) + 0.25).contiguous(memory_format=CL)
    lib = _lib.load()
    nws = lib.b200gan_conv2d_wgrad_workspace_floats(ctypes.byref(g), ALGO_AUTO)
    ws = torch.empty(nws, device="cuda")
    dw = torch.empty(k, c, 3, 3, device="cuda")
    bb, db = _guarded((k,), cl=False)

    def call():
        assert lib.b200gan_conv2d_wgrad_fused_bias(ctypes.byref(g), x.data_ptr(), dy.data_ptr(), dw.data_ptr(), db.data_ptr(),
                                        ws.data_ptr(), ALGO_AUTO, ops._stream()) == 0

    names = []
    for _ in range(3):  # a profiler session now and then loses a kernel record; a wrong route repeats
        names = [nm for nm, _ in traced_kernels(call)]
        assert not any("colsum" in nm for nm in names), names
        if any(nm.startswith("wgrad_tc_kernel") for nm in names):
            break
    assert any(nm.startswith("wgrad_tc_kernel") for nm in names), names
    torch.cuda.synchronize()
    assert _guards_intact(bb) and not torch.isnan(db).any()
    d64 = dy.double()
    want = d64.sum((0, 2, 3))
    # fp32 partial sums per thread over its pixel range (at most the whole map), shuffles, fp32 atomics per CTA
    bound = (h * w * n * (up * up) * EPS32 + 64 * EPS32) * d64.abs().sum((0, 2, 3))
    assert ((db.double() - want).abs() <= bound).all()
    assert rel_err(db, want) < 1e-6
    # the weight gradient itself is unchanged by the fused sum
    dw_ref, _ = ops.conv_wgrad(g, x, dy, (k, c, 3, 3), False, ALGO_AUTO)
    assert rel_err(dw, dw_ref) < 1e-6


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
