"""GPU parity tests (-m gpu): every CUDA kernel, through the C ABI, against (a) stock torch fp32 on
the same device (cuDNN with TF32 disabled = the reference's own operator path at full precision),
(b) the golden vectors produced by the reference on CPU, (c) size-independent properties.

Tolerances: 1e-3 norm-relative for floating point (BASELINE.json north star); exact equality
(torch.equal) for shape / index ops.
"""
import os

import pytest
import torch

from conftest import rel_err

pytestmark = pytest.mark.gpu

TOL = 1e-3


@pytest.fixture(autouse=True)
def _fp32_reference():
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    yield


def _mods():
    from b200gan import nn as bnn
    return bnn


def _cl(x):
    return x.contiguous(memory_format=torch.channels_last)


CONV_CASES = [  # cin, cout, k, stride, pad, H, W, N   -- every geometry of SURVEY.md section 0.6
    (1, 16, 3, 2, 1, 64, 64, 4),     # dcgan D block 1
    (16, 32, 3, 2, 1, 32, 32, 4),
    (64, 128, 3, 2, 1, 8, 8, 4),
    (64, 1, 3, 1, 1, 32, 32, 3),     # dcgan G output conv (small-K kernel)
    (128, 3, 4, 1, 1, 17, 17, 2),    # pix2pix final conv geometry
    (3, 64, 4, 2, 1, 32, 32, 2),     # pix2pix down1
    (6, 64, 4, 2, 1, 16, 16, 2),
    (3, 8, 7, 1, 0, 22, 22, 2),      # cyclegan 7x7 (after reflection pad)
    (32, 32, 3, 1, 0, 10, 10, 2),    # residual block conv
    (5, 7, 3, 1, 1, 9, 11, 3),       # odd everything
    (64, 64, 3, 1, 1, 16, 16, 2),    # tensor-core eligible
    (128, 128, 3, 1, 1, 32, 32, 2),
    (128, 64, 3, 1, 1, 24, 20, 3),   # tensor-core with ragged tiles
    (256, 256, 3, 1, 0, 18, 18, 1),  # cyclegan residual conv on a padded map
    (64, 128, 7, 1, 3, 16, 16, 1),
    (64, 256, 3, 1, 1, 64, 48, 7),   # 256-wide tiles in fprop (>= 132 tiles), ragged
    (256, 32, 3, 2, 1, 64, 64, 8),   # ... and in the (scatter-form, four-phase) data gradient
]


@pytest.mark.parametrize("algo", ["simt", "auto"])
@pytest.mark.parametrize("case", CONV_CASES, ids=lambda c: "c%d_k%d_%dx%ds%dp%d_%dx%d" % (c[0], c[1], c[2], c[2], c[3], c[4], c[5], c[6]))
def test_conv2d_fwd_bwd(case, algo):
    import b200gan
    cin, cout, k, s, p, h, w, n = case
    prev = b200gan.Config.algo
    if algo == "auto" and prev == "simt":
        pytest.skip("B200GAN_ALGO=simt")
    b200gan.Config.algo = algo
    try:
        torch.manual_seed(1)
        ref = torch.nn.Conv2d(cin, cout, k, s, p).cuda()
        ours = _mods().Conv2d(cin, cout, k, s, p).cuda()
        ours.load_state_dict(ref.state_dict())
        x = torch.randn(n, cin, h, w, device="cuda")
        xr = x.clone().requires_grad_(True)
        xo = _cl(x).clone().requires_grad_(True)
        yr = ref(xr)
        yo = ours(xo)
        assert yo.shape == yr.shape
        assert rel_err(yo, yr) < TOL
        gy = torch.randn_like(yr)
        yr.backward(gy)
        yo.backward(_cl(gy))
        assert rel_err(xo.grad, xr.grad) < TOL
        assert rel_err(ours.weight.grad, ref.weight.grad) < TOL
        assert rel_err(ours.bias.grad, ref.bias.grad) < TOL
    finally:
        b200gan.Config.algo = prev


@pytest.mark.parametrize("case", [(6, 4, 5, 6, 2), (512, 64, 2, 2, 2), (64, 32, 8, 8, 3), (128, 64, 16, 16, 2)])
def test_conv_transpose2d_fwd_bwd(case):
    cin, cout, h, w, n = case
    torch.manual_seed(2)
    ref = torch.nn.ConvTranspose2d(cin, cout, 4, 2, 1, bias=False).cuda()
    ours = _mods().ConvTranspose2d(cin, cout, 4, 2, 1, bias=False).cuda()
    ours.load_state_dict(ref.state_dict())
    x = torch.randn(n, cin, h, w, device="cuda")
    xr = x.clone().requires_grad_(True)
    xo = _cl(x).clone().requires_grad_(True)
    yr, yo = ref(xr), ours(xo)
    assert yo.shape == yr.shape == (n, cout, 2 * h, 2 * w)
    assert rel_err(yo, yr) < TOL
    gy = torch.randn_like(yr)
    yr.backward(gy)
    yo.backward(_cl(gy))
    assert rel_err(xo.grad, xr.grad) < TOL
    assert rel_err(ours.weight.grad, ref.weight.grad) < TOL


def test_conv_golden_vectors_from_torch_cpu(golden_dir):
    """Fixtures written by oracle/make_golden.py (stock torch CPU) -- forward, dx, dw, db."""
    bnn = _mods()
    for c in torch.load(os.path.join(golden_dir, "ops_conv.pt"), weights_only=False):
        cls = bnn.ConvTranspose2d if c["transposed"] else bnn.Conv2d
        w = c["w"]
        cin, cout = (w.shape[0], w.shape[1]) if c["transposed"] else (w.shape[1], w.shape[0])
        m = cls(cin, cout, w.shape[2], c["stride"], c["pad"]).cuda()
        with torch.no_grad():
            m.weight.copy_(w)
            m.bias.copy_(c["b"])
        x = c["x"].cuda().requires_grad_(True)
        y = m(x)
        assert rel_err(y, c["y"]) < TOL, c["name"]
        y.backward(c["gy"].cuda())
        assert rel_err(x.grad, c["gx"]) < TOL, c["name"]
        assert rel_err(m.weight.grad, c["gw"]) < TOL, c["name"]
        assert rel_err(m.bias.grad, c["gb"]) < TOL, c["name"]


@pytest.mark.parametrize("cin,cout,h,w,n", [(128, 128, 16, 16, 4), (128, 64, 32, 32, 2), (64, 64, 8, 8, 3),
                                            (32, 16, 6, 5, 2)])
def test_upsample_conv_folded(cin, cout, h, w, n):
    """Upsample(x2) -> Conv3x3 inside a Sequential: the 4-phase fold (wgmma) or the gather (SIMT)."""
    bnn = _mods()
    torch.manual_seed(3)
    ref = torch.nn.Sequential(torch.nn.Upsample(scale_factor=2), torch.nn.Conv2d(cin, cout, 3, 1, 1)).cuda()
    ours = bnn.Sequential(bnn.Upsample(scale_factor=2), bnn.Conv2d(cin, cout, 3, 1, 1)).cuda()
    ours.load_state_dict(ref.state_dict())
    x = torch.randn(n, cin, h, w, device="cuda")
    xr = x.clone().requires_grad_(True)
    xo = x.clone().requires_grad_(True)
    yr, yo = ref(xr), ours(xo)
    assert yo.shape == yr.shape
    assert rel_err(yo, yr) < TOL
    gy = torch.randn_like(yr)
    yr.backward(gy)
    yo.backward(gy)
    assert rel_err(xo.grad, xr.grad) < TOL
    assert rel_err(ours[1].weight.grad, ref[1].weight.grad) < TOL
    assert rel_err(ours[1].bias.grad, ref[1].bias.grad) < TOL


@pytest.mark.parametrize("slope", [1.0, 0.2])
@pytest.mark.parametrize("norm,cin,cout,h,w,n", [("bn", 64, 64, 6, 5, 3), ("bn", 128, 64, 16, 16, 2),
                                                 ("in", 32, 64, 16, 8, 2), ("bn", 32, 192, 4, 4, 5)])
def test_upsample_conv_norm_act_all_phase_kernel(norm, cin, cout, h, w, n, slope):
    """Upsample -> Conv3x3 -> BatchNorm/InstanceNorm -> LeakyReLU (dcgan.py:54-57; cyclegan/models.py:73-78).  With
    64 (mod 128) output channels the forward runs in the all-phase wgmma kernel: 9 shifted operand tiles feed four
    register accumulators, the norm statistics are summed over the four phases in the epilogue.  Ragged and < 128-pixel
    maps exercise TMA clipping; the InstanceNorm case needs one image per tile.

    Gradients: a TF32 forward leaves a few pre-activations with |norm(z)| < 5e-4 on the other side of the LeakyReLU
    kink, and every such flip changes dz by 0.8 * dy at that element (tools/tf32_kink_emulation.py: 3e-3 .. 1.3e-2 of
    the gradient norm, for ANY TF32 convolution).  To test the kernels and not the kink, the fp32 reference gradient
    is taken with OUR forward's sign pattern (LeakyReLU written as a product with a fixed 1/slope mask); slope 1.0
    has no kink at all."""
    bnn = _mods()
    torch.manual_seed(11)
    mk = (lambda nn_: nn_.BatchNorm2d(cout, 0.8)) if norm == "bn" else (lambda nn_: nn_.InstanceNorm2d(cout))
    ref = torch.nn.Sequential(torch.nn.Upsample(scale_factor=2), torch.nn.Conv2d(cin, cout, 3, 1, 1), mk(torch.nn)).cuda()
    ours = bnn.Sequential(bnn.Upsample(scale_factor=2), bnn.Conv2d(cin, cout, 3, 1, 1), mk(bnn),
                          bnn.LeakyReLU(slope, inplace=True)).cuda()
    ours.load_state_dict(ref.state_dict())
    x = torch.randn(n, cin, h, w, device="cuda")
    gy = torch.randn(n, cout, 2 * h, 2 * w, device="cuda")
    xo = x.clone().requires_grad_(True)
    yo = ours(xo)
    yo.backward(gy)
    xr = x.clone().requires_grad_(True)
    pre = ref(xr)
    yr = torch.nn.functional.leaky_relu(pre, slope)
    assert rel_err(yo, yr) < TOL
    if norm == "bn":
        assert rel_err(ours[2].running_mean, ref[2].running_mean) < TOL
        assert rel_err(ours[2].running_var, ref[2].running_var) < TOL
    mask = torch.where(yo.detach() > 0, 1.0, slope)
    flips = (mask != torch.where(pre.detach() > 0, 1.0, slope)).sum().item()
    assert flips <= 1e-3 * mask.numel()  # the kink flips are rare (expected ~2e-4 of the elements)
    (pre * mask).backward(gy)
    assert rel_err(xo.grad, xr.grad) < 2 * TOL
    assert rel_err(ours[1].weight.grad, ref[1].weight.grad) < 2 * TOL
    # (the conv bias gradient is analytically zero behind a normalisation: nothing to compare)
    if norm == "bn":
        assert rel_err(ours[2].weight.grad, ref[2].weight.grad) < 2 * TOL
        assert rel_err(ours[2].bias.grad, ref[2].bias.grad) < 2 * TOL


def test_padded_convs_in_sequential():
    """ReflectionPad2d(3) -> Conv7x7 (cyclegan/models.py:49-50) and Upsample -> ZeroPad2d((1,0,1,0)) ->
    Conv4x4 p1 -> Tanh (pix2pix/models.py:76-81)."""
    bnn = _mods()
    torch.manual_seed(4)
    for ref, ours, shape in [
        (torch.nn.Sequential(torch.nn.ReflectionPad2d(3), torch.nn.Conv2d(3, 16, 7), torch.nn.InstanceNorm2d(16),
                             torch.nn.ReLU(inplace=True)),
         bnn.Sequential(bnn.ReflectionPad2d(3), bnn.Conv2d(3, 16, 7), bnn.InstanceNorm2d(16), bnn.ReLU(inplace=True)),
         (2, 3, 20, 20)),
        (torch.nn.Sequential(torch.nn.Upsample(scale_factor=2), torch.nn.ZeroPad2d((1, 0, 1, 0)),
                             torch.nn.Conv2d(8, 3, 4, padding=1), torch.nn.Tanh()),
         bnn.Sequential(bnn.Upsample(scale_factor=2), bnn.ZeroPad2d((1, 0, 1, 0)), bnn.Conv2d(8, 3, 4, padding=1),
                        bnn.Tanh()),
         (2, 8, 9, 9)),
        (torch.nn.Sequential(torch.nn.ReflectionPad2d(1), torch.nn.Conv2d(32, 32, 3), torch.nn.InstanceNorm2d(32),
                             torch.nn.ReLU(inplace=True), torch.nn.ReflectionPad2d(1), torch.nn.Conv2d(32, 32, 3),
                             torch.nn.InstanceNorm2d(32)),
         bnn.Sequential(bnn.ReflectionPad2d(1), bnn.Conv2d(32, 32, 3), bnn.InstanceNorm2d(32), bnn.ReLU(inplace=True),
                        bnn.ReflectionPad2d(1), bnn.Conv2d(32, 32, 3), bnn.InstanceNorm2d(32)),
         (2, 32, 12, 12)),
    ]:
        ref, ours = ref.cuda(), ours.cuda()
        ours.load_state_dict(ref.state_dict())
        x = torch.randn(*shape, device="cuda")
        xr, xo = x.clone().requires_grad_(True), x.clone().requires_grad_(True)
        yr, yo = ref(xr), ours(xo)
        assert yo.shape == yr.shape
        assert rel_err(yo, yr) < TOL
        gy = torch.randn_like(yr)
        yr.backward(gy)
        yo.backward(gy)
        assert rel_err(xo.grad, xr.grad) < TOL
        for (k, po), (_, pr) in zip(ours.named_parameters(), ref.named_parameters()):
            if not k.endswith("bias"):  # conv bias in front of a norm: exactly-zero gradient (fp noise only)
                assert rel_err(po.grad, pr.grad) < TOL, k


@pytest.mark.parametrize("eps", [1e-5, 0.8])
@pytest.mark.parametrize("shape", [(8, 16, 8, 8), (4, 128, 16, 16), (3, 5, 7, 3)])
def test_batchnorm2d_train(shape, eps):
    bnn = _mods()
    torch.manual_seed(5)
    c = shape[1]
    ref = torch.nn.BatchNorm2d(c, eps).cuda()
    ours = bnn.BatchNorm2d(c, eps).cuda()
    with torch.no_grad():
        ref.weight.normal_(1, 0.2)
        ref.bias.normal_(0, 0.2)
    ours.load_state_dict(ref.state_dict())
    for _ in range(2):
        x = torch.randn(*shape, device="cuda") * 2 + 0.5
        xr, xo = x.clone().requires_grad_(True), x.clone().requires_grad_(True)
        yr, yo = ref(xr), ours(xo)
        assert rel_err(yo, yr) < 1e-5
        gy = torch.randn_like(yr)
        yr.backward(gy)
        yo.backward(gy)
        assert rel_err(xo.grad, xr.grad) < 1e-4
        assert rel_err(ours.weight.grad, ref.weight.grad) < 1e-4
        assert rel_err(ours.bias.grad, ref.bias.grad) < 1e-4
        ref.zero_grad()
        ours.zero_grad()
    assert rel_err(ours.running_mean, ref.running_mean) < 1e-5
    assert rel_err(ours.running_var, ref.running_var) < 1e-5   # unbiased variance in the running stat
    assert int(ours.num_batches_tracked) == int(ref.num_batches_tracked) == 2
    ref.eval()
    ours.eval()
    x = torch.randn(*shape, device="cuda")
    assert rel_err(ours(x), ref(x)) < 1e-5


def test_instancenorm2d():
    bnn = _mods()
    torch.manual_seed(6)
    for shape in [(2, 16, 8, 8), (3, 7, 5, 9), (2, 64, 32, 32)]:
        ref = torch.nn.InstanceNorm2d(shape[1]).cuda()
        ours = bnn.InstanceNorm2d(shape[1]).cuda()
        x = torch.randn(*shape, device="cuda") * 3 - 1
        xr, xo = x.clone().requires_grad_(True), x.clone().requires_grad_(True)
        yr, yo = ref(xr), ours(xo)
        assert rel_err(yo, yr) < 1e-5
        gy = torch.randn_like(yr)
        yr.backward(gy)
        yo.backward(gy)
        assert rel_err(xo.grad, xr.grad) < 1e-4
    with pytest.raises(ValueError):  # pix2pix down8 has normalize=False because IN on 1x1 raises
        bnn.InstanceNorm2d(4).cuda()(torch.randn(2, 4, 1, 1, device="cuda"))


def test_shape_ops_bit_exact():
    bnn = _mods()
    x = torch.randn(3, 6, 7, 5, device="cuda")
    assert torch.equal(bnn.Upsample(scale_factor=2)(x), torch.nn.Upsample(scale_factor=2)(x))
    assert torch.equal(bnn.ZeroPad2d((1, 0, 1, 0))(x), torch.nn.ZeroPad2d((1, 0, 1, 0))(x))
    assert torch.equal(bnn.ReflectionPad2d(3)(x), torch.nn.ReflectionPad2d(3)(x))
    assert torch.equal(bnn.ReflectionPad2d(1)(x), torch.nn.ReflectionPad2d(1)(x))
    from b200gan import ops
    xc = ops.to_cl(x)
    assert xc.is_contiguous(memory_format=torch.channels_last) and torch.equal(xc, x)
    back = ops.to_nchw(xc)
    assert back.is_contiguous() and torch.equal(back, x)
    # gradients of the index ops: compare with autograd of the stock modules (sums of <= 4 terms)
    for ours, ref in [(bnn.Upsample(scale_factor=2), torch.nn.Upsample(scale_factor=2)),
                      (bnn.ReflectionPad2d(2), torch.nn.ReflectionPad2d(2)),
                      (bnn.ZeroPad2d((1, 0, 1, 0)), torch.nn.ZeroPad2d((1, 0, 1, 0)))]:
        xo, xr = x.clone().requires_grad_(True), x.clone().requires_grad_(True)
        yo, yr = ours(xo), ref(xr)
        gy = torch.randn_like(yr)
        yo.backward(gy)
        yr.backward(gy)
        assert rel_err(xo.grad, xr.grad) < 1e-6


def test_activations_and_dropout2d_mask_identical():
    bnn = _mods()
    x = torch.randn(4, 8, 6, 6, device="cuda")
    for ours, ref in [(bnn.LeakyReLU(0.2), torch.nn.LeakyReLU(0.2)), (bnn.ReLU(), torch.nn.ReLU()),
                      (bnn.Tanh(), torch.nn.Tanh()), (bnn.Sigmoid(), torch.nn.Sigmoid())]:
        xo, xr = x.clone().requires_grad_(True), x.clone().requires_grad_(True)
        yo, yr = ours(xo), ref(xr)
        assert rel_err(yo, yr) < 1e-6
        gy = torch.randn_like(yr)
        yo.backward(gy)
        yr.backward(gy)
        assert rel_err(xo.grad, xr.grad) < 1e-5
    # Dropout2d: same torch RNG call as F.dropout2d -> bit-identical masks under the same seed
    d_ours, d_ref = bnn.Dropout2d(0.25), torch.nn.Dropout2d(0.25)
    torch.manual_seed(7)
    yo = d_ours(x)
    torch.manual_seed(7)
    yr = d_ref(x)
    assert torch.equal(yo == 0, yr == 0)
    assert rel_err(yo, yr) < 1e-6
    d_ours.eval()
    assert d_ours(x) is x


def test_conv_linearity_and_adjointness_full_size():
    """Size-independent properties at the BASELINE sizes (dcgan conv2: [128,128,32,32] after upsample):
    linearity in x, and <conv(x), dy> == <x, dgrad(dy)> == <w, wgrad(x, dy)>."""
    bnn = _mods()
    torch.manual_seed(8)
    seq = bnn.Sequential(bnn.Upsample(scale_factor=2), bnn.Conv2d(128, 128, 3, 1, 1, bias=False)).cuda()
    x1 = torch.randn(128, 128, 16, 16, device="cuda", requires_grad=True)
    x2 = torch.randn(128, 128, 16, 16, device="cuda")
    y1 = seq(x1)
    y2 = seq(x2)
    y12 = seq(x1.detach() + 2 * x2)
    assert rel_err(y12, y1 + 2 * y2) < TOL
    dy = torch.randn_like(y1)
    (dx, dw) = torch.autograd.grad(y1, [x1, seq[1].weight], dy)
    lhs = (y1.double() * dy.double()).sum().item()
    assert abs((x1.double() * dx.double()).sum().item() - lhs) < 2e-3 * abs(lhs) + 1.0
    assert abs((seq[1].weight.double() * dw.double()).sum().item() - lhs) < 2e-3 * abs(lhs) + 1.0


def test_empty_batch_and_errors():
    bnn = _mods()
    conv = bnn.Conv2d(4, 4, 3, 1, 1).cuda()
    y = conv(torch.zeros(0, 4, 8, 8, device="cuda"))
    assert y.shape == (0, 4, 8, 8)
    with pytest.raises(RuntimeError):
        conv(torch.zeros(1, 5, 8, 8, device="cuda"))
    with pytest.raises(NotImplementedError):
        bnn.Conv2d(4, 4, 3, 1, 1, groups=2).cuda()(torch.zeros(1, 4, 8, 8, device="cuda"))


def test_discriminator_head_and_bce_match_stock_torch():
    """Sequential(Linear(2048, 1), Sigmoid) + BCELoss (dcgan.py:92,103): one kernel per direction each."""
    from b200gan import nn as bnn
    torch.manual_seed(11)
    ref = torch.nn.Sequential(torch.nn.Linear(2048, 1), torch.nn.Sigmoid()).cuda()
    ours = bnn.Sequential(bnn.Linear(2048, 1), bnn.Sigmoid()).cuda()
    ours.load_state_dict(ref.state_dict())
    for n in (128, 7):
        x = torch.randn(n, 2048, device="cuda") * 0.5
        for tgt in (1.0, 0.0, 0.3):
            t = torch.full((n, 1), tgt, device="cuda")
            xr, xo = x.clone().requires_grad_(True), x.clone().requires_grad_(True)
            ref.zero_grad(); ours.zero_grad()
            vr, vo = ref(xr), ours(xo)
            assert rel_err(vo, vr) < 1e-5
            lr_, lo = torch.nn.BCELoss()(vr, t), bnn.BCELoss()(vo, t)
            assert abs(lo.item() - lr_.item()) < 1e-5 * abs(lr_.item())
            lr_.backward(); lo.backward()
            assert rel_err(xo.grad, xr.grad) < 1e-5
            assert rel_err(ours[0].weight.grad, ref[0].weight.grad) < 1e-5
            assert rel_err(ours[0].bias.grad, ref[0].bias.grad) < 1e-5
    # saturated inputs: the clamps of torch's BCE (log >= -100, denominator >= 1e-12)
    v = torch.tensor([[0.0], [1.0], [1e-30], [0.5]], device="cuda")
    t = torch.tensor([[1.0], [0.0], [0.0], [1.0]], device="cuda")
    vr, vo = v.clone().requires_grad_(True), v.clone().requires_grad_(True)
    lr_, lo = torch.nn.BCELoss()(vr, t), bnn.BCELoss()(vo, t)
    assert abs(lo.item() - lr_.item()) < 1e-5 * abs(lr_.item())
    lr_.backward(); lo.backward()
    assert rel_err(vo.grad, vr.grad) < 1e-5


def test_all_phase_kernel_unmasked_gradient_vs_stock_cudnn_tf32():
    """VERDICT r1 (weak #2): the un-masked comparison.  Upsample -> Conv(128, 64) -> BatchNorm(.8) -> LeakyReLU at
    [8,128,32,32] -> 64x64, a size where cuDNN really runs TF32 kernels.  The fp32 reference (stock torch, allow_tf32 =
    False) is the truth; the yardstick is the SAME stock module with allow_tf32 = True (the reference's default GPU
    path).  Our input gradient / weight gradient must deviate from fp32 by no more than 1.5x what cuDNN-TF32 does (or
    2e-3): if cuDNN showed no kink deviation and we did, the kernel would be wrong.  The measured numbers are printed
    so that the round's log carries them."""
    bnn = _mods()
    torch.manual_seed(21)

    def build(ns):
        return ns.Sequential(ns.Upsample(scale_factor=2), ns.Conv2d(128, 64, 3, 1, 1), ns.BatchNorm2d(64, 0.8),
                             ns.LeakyReLU(0.2, inplace=True))
    ref = build(torch.nn).cuda()
    ours = build(bnn).cuda()
    ours.load_state_dict(ref.state_dict())
    import copy
    ref_t = copy.deepcopy(ref)
    x = torch.randn(8, 128, 32, 32, device="cuda")
    gy = torch.randn(8, 64, 64, 64, device="cuda")
    res = {}
    for name, m, tf32 in (("fp32", ref, False), ("tf32", ref_t, True), ("ours", ours, False)):
        torch.backends.cudnn.allow_tf32 = tf32
        xi = x.clone().requires_grad_(True)
        y = m(xi)
        y.backward(gy)
        res[name] = (y.detach(), xi.grad, m[1].weight.grad, m[2].weight.grad, m[2].bias.grad)
    torch.backends.cudnn.allow_tf32 = False
    names = ("y", "dx", "dW", "dgamma", "dbeta")
    line = []
    for i, nm in enumerate(names):
        e_t, e_o = rel_err(res["tf32"][i], res["fp32"][i]), rel_err(res["ours"][i], res["fp32"][i])
        line.append(f"{nm}: cudnn-tf32 {e_t:.2e} ours {e_o:.2e}")
        assert e_o < max(2e-3, 1.5 * e_t), f"{nm}: ours {e_o:.2e} vs stock TF32 {e_t:.2e}"
    print("all-phase yardstick [8,128,32,32]->64: " + "; ".join(line))


@pytest.mark.parametrize("n,hw", [(4, 8), (16, 4), (2, 16)])
def test_deep_unet_layers_split_k(n, hw):
    """pix2pix/models.py:62-73: Conv2d(C, C, 4, 2, 1, bias=False) -> InstanceNorm2d -> LeakyReLU and ConvTranspose2d(...,
    bias=False) -> InstanceNorm2d -> ReLU at 4x4 .. 16x16 pixels: a handful of output tiles, so the wgmma kernel splits
    the (tap, k-chunk) loop over CTAs and adds raw partial tiles with TMA reduce-stores; the norm statistics then come
    from a separate pass.  Forward, input gradient, weight gradients vs stock torch fp32."""
    bnn = _mods()
    torch.manual_seed(17)

    def build(ns):
        return ns.Sequential(ns.Conv2d(256, 256, 4, 2, 1, bias=False), ns.InstanceNorm2d(256), ns.LeakyReLU(0.2),
                             ns.ConvTranspose2d(256, 128, 4, 2, 1, bias=False), ns.InstanceNorm2d(128), ns.ReLU(inplace=True))
    import copy
    ref, ours = build(torch.nn).cuda(), build(bnn).cuda()
    ours.load_state_dict(ref.state_dict())
    yard = copy.deepcopy(ref)                # stock torch with TF32 convolutions: the reference's default GPU arithmetic
    x = torch.randn(n, 256, hw, hw, device="cuda")
    xr, xo, xt = (x.clone().requires_grad_(True) for _ in range(3))
    prev = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    try:
        yr = ref(xr)
        torch.backends.cudnn.allow_tf32 = True
        yt = yard(xt)
        torch.backends.cudnn.allow_tf32 = False
        yo = ours(xo)
        assert rel_err(yo, yr) < max(2 * TOL, 1.5 * rel_err(yt, yr))
        gy = torch.randn_like(yr)
        yr.backward(gy)
        torch.backends.cudnn.allow_tf32 = True
        yt.backward(gy)
        torch.backends.cudnn.allow_tf32 = False
        yo.backward(gy)
    finally:
        torch.backends.cudnn.allow_tf32 = prev
    # Through two InstanceNorms over 4..64 pixels with TF32 operands: an activation within TF32 rounding of the
    # LeakyReLU / ReLU kink flips its mask and moves single gradient elements by O(1) (the measured deviation is a few
    # 1e-2, the same for cuDNN's TF32 kernels) -- the bound is what stock TF32 shows on the same inputs, x2.
    for nm, o, r, t in (("dx", xo.grad, xr.grad, xt.grad),
                        ("dw0", ours[0].weight.grad, ref[0].weight.grad, yard[0].weight.grad),
                        ("dw3", ours[3].weight.grad, ref[3].weight.grad, yard[3].weight.grad)):
        e_o, e_t = rel_err(o, r), rel_err(t, r)
        assert e_o < max(1e-2, 2.0 * e_t), f"{nm}: ours {e_o:.2e} vs stock TF32 {e_t:.2e}"
