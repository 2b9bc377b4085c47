"""Host-side logic of the C ABI and of the module planner, without a GPU: geometry validation, which pass of which
reference layer the wgmma path takes, workspace / packed sizes, error reporting.  None of these calls launches a
kernel (the library's host entry points validate before they touch CUDA)."""
import ctypes
import itertools

import pytest
import torch


def _lib_ops():
    from b200gan import _lib, ops
    return _lib, ops


def _geom(x_shape, w_shape, stride, pad, up=1, transposed=False, pads=None):
    _, ops = _lib_ops()
    return ops.make_geom(x_shape, w_shape, stride, pads or (pad, pad, pad, pad), 0, up, transposed)


# every convolution of the DCGAN step at BASELINE configs[1] (dcgan.py:54-62 generator, :75-88 discriminator)
# name, x_shape, w_shape, stride, pad, up, (fprop, dgrad, wgrad) on tensor cores
DCGAN_LAYERS = [
    ("G conv1 up2 128->128 @16", (128, 128, 16, 16), (128, 128, 3, 3), 1, 1, 2, (True, True, True)),
    ("G conv2 up2 128->64 @32", (128, 128, 32, 32), (64, 128, 3, 3), 1, 1, 2, (True, True, True)),
    # (fused into the tail kernels in the step; stand-alone, its forward takes the narrow-output wgmma form)
    ("G conv3 64->1 @64", (128, 64, 64, 64), (1, 64, 3, 3), 1, 1, 1, (True, False, False)),
    ("D conv1 1->16 s2 @64", (128, 1, 64, 64), (16, 1, 3, 3), 2, 1, 1, (False, False, False)),
    ("D conv2 16->32 s2 @32", (128, 16, 32, 32), (32, 16, 3, 3), 2, 1, 1, (False, False, False)),
    ("D conv3 32->64 s2 @16", (128, 32, 16, 16), (64, 32, 3, 3), 2, 1, 1, (True, True, False)),
    ("D conv4 64->128 s2 @8", (128, 64, 8, 8), (128, 64, 3, 3), 2, 1, 1, (True, True, True)),
]


@pytest.mark.parametrize("name,xs,ws,stride,pad,up,expect", DCGAN_LAYERS, ids=[l[0] for l in DCGAN_LAYERS])
def test_which_dcgan_layers_ride_the_tensor_cores(name, xs, ws, stride, pad, up, expect):
    _lib, ops = _lib_ops()
    g, out = _geom(xs, ws, stride, pad, up)
    ref = torch.nn.functional.conv2d(torch.zeros(1, xs[1], xs[2] * up, xs[3] * up), torch.zeros(ws), None, stride, pad)
    assert out[1:] == tuple(ref.shape[1:])
    assert tuple(ops.tc_supported(g, p) for p in (0, 1, 2)) == expect
    for p in (0, 1, 2):  # the fp32 SIMT path takes everything
        assert _lib.load().b200gan_conv2d_supported(ctypes.byref(g), p, _lib.ALGO_SIMT) == 1


def test_planner_mirror_never_claims_more_than_the_library():
    """nn._tc_like() decides where operands are RN-rounded to TF32; it must imply library support for the forward
    pass on even-sized maps (odd maps at stride 2 fall back to SIMT inside the library, which is always correct)."""
    from b200gan import nn as bnn
    _lib, ops = _lib_ops()
    for cin, cout, k, stride, up, tr in itertools.product((1, 3, 16, 32, 64, 96, 128, 256), (1, 3, 16, 32, 64, 128, 192),
                                                          (3, 4), (1, 2), (1, 2), (False, True)):
        if up == 2 and (tr or stride != 1 or k != 3):
            continue
        conv = (bnn.ConvTranspose2d if tr else bnn.Conv2d)(cin, cout, k, stride, 1)
        g, out = _geom((2, cin, 16, 16), tuple(conv.weight.shape), stride, 1, up, tr)
        if stride == 2 and tr and out[2] % 2:
            continue  # odd full-resolution side (k3 s2 transposed): no parity view, SIMT inside the library
        claimed = bnn._tc_like(conv, up)
        actual = ops.tc_supported(g, 0)
        if claimed:
            assert actual, (cin, cout, k, stride, up, tr)
        narrow = cout < 32 and cin % 32 == 0 and stride == 1 and up == 1 and not tr   # forward-only wgmma form
        if (cin % 32 or cout % 32) and not narrow:
            assert not actual
        if narrow:
            assert actual and not ops.tc_supported(g, 1) and not ops.tc_supported(g, 2)


def test_pix2pix_and_cyclegan_hot_layers_are_tensor_core_eligible():
    """pix2pix/models.py:23 (Conv 4x4 s2), :39 (ConvTranspose 4x4 s2); cyclegan/models.py:28 (3x3 after reflection
    pad -> explicit pad + unpadded conv), :60 (3x3 s2), :75 (Upsample + 3x3)."""
    _, ops = _lib_ops()
    cases = [
        ((1, 64, 128, 128), (128, 64, 4, 4), 2, 1, 1, False),      # UNetDown 64->128
        ((1, 512, 2, 2), (512, 512, 4, 4), 2, 1, 1, False),         # down8
        ((1, 512, 1, 1), (512, 512, 4, 4), 2, 1, 1, True),          # up1 (ConvTranspose 1x1 -> 2x2)
        ((1, 256, 64, 64), (256, 128, 4, 4), 2, 1, 1, True),        # up6
        ((2, 256, 18, 18), (256, 256, 3, 3), 1, 0, 1, False),       # residual conv on the reflection-padded map
        ((2, 64, 64, 64), (128, 64, 3, 3), 2, 1, 1, False),         # cyclegan downsampling
        ((2, 256, 16, 16), (128, 256, 3, 3), 1, 1, 2, False),       # cyclegan upsampling
        ((2, 128, 32, 32), (64, 128, 3, 3), 1, 1, 2, False),        # cyclegan upsampling (all-phase kernel: 64 outputs)
    ]
    for xs, ws, stride, pad, up, tr in cases:
        g, _ = _geom(xs, ws, stride, pad, up, tr)
        assert ops.tc_supported(g, 0) and ops.tc_supported(g, 1), (xs, ws)
    # 3-channel image inputs stay on the fp32 path
    for xs, ws, stride, pad in [((1, 6, 256, 256), (64, 6, 4, 4), 2, 1), ((2, 3, 70, 70), (64, 3, 7, 7), 1, 0)]:
        g, _ = _geom(xs, ws, stride, pad)
        assert not ops.tc_supported(g, 0)
    # few-output-channel layers: forward on wgmma (narrow form), gradients fp32 -- the 1-channel PatchGAN head
    # (pix2pix/models.py:127) and the 3-channel output conv (cyclegan/models.py:82, on the reflection-padded map)
    for xs, ws, stride, pad in [((1, 512, 17, 17), (1, 512, 4, 4), 1, 1), ((2, 64, 70, 70), (3, 64, 7, 7), 1, 0)]:
        g, _ = _geom(xs, ws, stride, pad)
        assert ops.tc_supported(g, 0) and not ops.tc_supported(g, 1) and not ops.tc_supported(g, 2)


def test_geometry_validation_and_error_reporting():
    _lib, ops = _lib_ops()
    lib = _lib.load()
    g, _ = _geom((4, 32, 8, 8), (32, 32, 3, 3), 1, 1)
    # null pointers are refused before anything is launched, with a message (thread-local last error)
    rc = lib.b200gan_conv2d_fprop(ctypes.byref(g), None, None, None, None, _lib.ALGO_TC, None)
    assert rc < 0 and b"null pointer" in lib.b200gan_last_error()
    with pytest.raises(RuntimeError, match="null pointer"):
        _lib.check(rc, "conv2d_fprop")
    # inconsistent output size
    g.P = 5
    assert lib.b200gan_conv2d_supported(ctypes.byref(g), 0, _lib.ALGO_SIMT) == 0
    rc = lib.b200gan_conv2d_fprop(ctypes.byref(g), None, None, None, None, _lib.ALGO_SIMT, None)
    assert rc < 0 and b"output size mismatch" in lib.b200gan_last_error()
    # channel mismatch is caught in the Python shim with the reference's wording style
    with pytest.raises(RuntimeError, match="channels"):
        ops.make_geom((1, 3, 8, 8), (8, 4, 3, 3), 1, (1, 1, 1, 1))
    # reflection padding wider than the map is invalid (torch raises too)
    g2, _ = ops.make_geom((1, 4, 3, 3), (4, 4, 3, 3), 1, (3, 3, 3, 3), _lib.PAD_REFLECT)
    assert lib.b200gan_conv2d_supported(ctypes.byref(g2), 0, _lib.ALGO_SIMT) == 0


def test_packed_and_workspace_sizes():
    _lib, ops = _lib_ops()
    lib = _lib.load()
    g, _ = _geom((128, 128, 32, 32), (64, 128, 3, 3), 1, 1, 2)
    for pack in (_lib.PACK_SIMT_FPROP, _lib.PACK_SIMT_DGRAD, _lib.PACK_TC_FPROP, _lib.PACK_TC_DGRAD):
        assert lib.b200gan_packed_weight_floats(ctypes.byref(g), pack) == 9 * 128 * 64
    for pack in (_lib.PACK_TC_FPROP_UP2, _lib.PACK_TC_DGRAD_UP2):  # four phases x four pre-summed 2x2 taps
        assert lib.b200gan_packed_weight_floats(ctypes.byref(g), pack) == 16 * 128 * 64
    # wgmma weight gradient: one [Cin x Cout] partial per (phase, tap) job; SIMT accumulates in place
    assert lib.b200gan_conv2d_wgrad_workspace_floats(ctypes.byref(g), _lib.ALGO_TC) == 16 * 128 * 64
    assert lib.b200gan_conv2d_wgrad_workspace_floats(ctypes.byref(g), _lib.ALGO_SIMT) == 0
    # wgmma dgrad of the fold writes dx directly; the SIMT path goes through the upsampled gradient
    assert lib.b200gan_conv2d_dgrad_workspace_floats(ctypes.byref(g), _lib.ALGO_TC) == 0
    assert lib.b200gan_conv2d_dgrad_workspace_floats(ctypes.byref(g), _lib.ALGO_SIMT) == 128 * 128 * 64 * 64
    g1, _ = _geom((128, 64, 8, 8), (128, 64, 3, 3), 2, 1)
    assert lib.b200gan_conv2d_dgrad_workspace_floats(ctypes.byref(g1), _lib.ALGO_SIMT) == 0


def test_algo_override_switches_the_planner_mirror():
    from b200gan import nn as bnn
    _, ops = _lib_ops()
    conv = bnn.Conv2d(64, 64, 3, 1, 1)
    g, _ = _geom((2, 64, 8, 8), (64, 64, 3, 3), 1, 1)
    old = ops.Config.algo
    try:
        ops.Config.algo = "simt"
        assert not bnn._tc_like(conv, 1) and not ops.tc_supported(g, 0)
        ops.Config.algo = "auto"
        assert bnn._tc_like(conv, 1) and ops.tc_supported(g, 0)
    finally:
        ops.Config.algo = old


def test_patch_dispatches_adam_and_resets_pack_caches_on_apply():
    """patch(): torch.optim.Adam -> the one-launch Adam only when every parameter is a CUDA fp32 tensor (gan.py on CPU,
    BASELINE config 0, keeps the stock optimizer); Module.apply drops the packed-weight caches (name-based init writes
    parameters through .data, which does not bump the version counter the caches key on; dcgan.py:36-42)."""
    import torch
    import b200gan
    from b200gan import nn as bnn
    stock_adam = torch.optim.Adam
    with b200gan.patched():
        net = torch.nn.Sequential(torch.nn.Conv2d(3, 4, 3), torch.nn.Linear(4, 2))
        opt = torch.optim.Adam(net.parameters(), lr=2e-4, betas=(0.5, 0.999))
        assert type(opt) is stock_adam and isinstance(opt, torch.optim.Optimizer)       # CPU parameters: stock
        assert isinstance(net[0], bnn.Conv2d)
        net[0].__dict__["_b200_cache"] = object()
        net.apply(lambda m: None)
        assert "_b200_cache" not in net[0].__dict__
        sched = torch.optim.lr_scheduler.LambdaLR(opt, lr_lambda=lambda e: 1.0)         # cyclegan.py:93-101 still works
        assert sched.get_last_lr() == [2e-4]
    assert torch.optim.Adam is stock_adam and torch.nn.Module.apply.__qualname__ == "Module.apply"


def test_grouped_discriminator_pass_eligibility_is_decided_on_the_host():
    """train.dcgan_step batches discriminator(real) and discriminator(fake) (dcgan.py:178-179) into one grouped pass only
    when the fused chain covers the whole conv stack at that shape AND every layer has a tile plan whose tiles stay inside
    one statistics group (b200gan_nb_groups_supported: host-side planner, no GPU needed)."""
    import ctypes
    from b200gan import _lib, nn as bnn, ops, zoo
    d = zoo.DCGANDiscriminator(64)
    assert bnn.groups_eligible(d.model, (256, 1, 64, 64), 2)          # BASELINE: 2 x 128 images
    assert bnn.groups_eligible(d.model, (64, 1, 32, 32), 2)
    assert not bnn.groups_eligible(d.model, (255, 1, 64, 64), 2)      # does not split evenly
    assert not bnn.groups_eligible(d.model, (256, 3, 64, 64), 2)      # wrong channel count: the chain does not qualify
    wide = bnn.Sequential(bnn.Conv2d(256, 256, 3, 1, 1), bnn.BatchNorm2d(256))
    assert not bnn.groups_eligible(wide, (4, 256, 8, 8), 2)           # tensor-core territory, not a fused chain
    assert ops.bn_groups.active == 1                                  # the probe leaves no state behind
    lib = _lib.load()
    g, _ = ops.make_geom((6, 64, 8, 8), (128, 64, 3, 3), 2, (1, 1, 1, 1))
    assert lib.b200gan_nb_supported(ctypes.byref(g)) == 1
    # 3 images per group at 16 output pixels each: every plan needs tiles of >= 2 images, which would straddle the groups
    assert lib.b200gan_nb_groups_supported(ctypes.byref(g), 2) == 0
    assert lib.b200gan_nb_groups_supported(ctypes.byref(g), 1) == 1
    g2, _ = ops.make_geom((8, 64, 8, 8), (128, 64, 3, 3), 2, (1, 1, 1, 1))
    assert lib.b200gan_nb_groups_supported(ctypes.byref(g2), 2) == 1
    assert lib.b200gan_nb_groups_supported(ctypes.byref(g2), 5) == 0  # more groups than the kernels take


def test_negative_leaky_relu_slope_is_refused():
    """the fused backward kernels take LeakyReLU's derivative from the sign of its output y: with a negative slope y is
    positive on the negative side too, so such a module is refused rather than given the derivative 1 there"""
    from b200gan import nn as bnn
    with pytest.raises(NotImplementedError):
        bnn._act_of(torch.nn.LeakyReLU(-0.1))
    assert bnn._act_of(torch.nn.LeakyReLU(0.2)) == (bnn.ACT_LRELU, 0.2)
    assert bnn._act_of(torch.nn.LeakyReLU(0.0)) == (bnn.ACT_LRELU, 0.0)


@pytest.mark.parametrize("state", ["tracked", "untracked", "buffers_none", "momentum_none", "eval"])
def test_running_statistics_every_batchnorm_path_updates(state):
    """What a batch-statistics BatchNorm2d hands its kernels to update -- the same on the stand-alone path, the fused
    tail and the fused chain: its running buffers and momentum only if it tracks them AND has them.  A norm whose
    buffers were set to None updates nothing (not even num_batches_tracked); momentum=None with buffers is refused."""
    from b200gan import nn as bnn
    bn = bnn.BatchNorm2d(8, 0.8, momentum=None if state == "momentum_none" else 0.1,
                         track_running_stats=state != "untracked").train(state != "eval")
    if state == "buffers_none":
        bn.running_mean = bn.running_var = None
    if state == "momentum_none":
        with pytest.raises(NotImplementedError, match="momentum=None"):
            bnn._running_stats(bn)
        with pytest.raises(NotImplementedError, match="momentum=None"):
            bnn._batch_norm_spec(bn, False, 0, 0.0, False, False)
        return
    expected = (None, None, None, 0.0)
    if state in ("tracked", "eval"):
        expected = (bn.running_mean, bn.running_var, bn.num_batches_tracked, 0.1)
    assert bnn._running_stats(bn) == expected
    spec, rm, rv, nbt = bnn._batch_norm_spec(bn, False, 0, 0.0, False, False)
    if state == "eval":  # an eval-mode norm normalises with batch statistics only without buffers: no update then
        expected = (None, None, None, 0.0)
    assert (rm, rv, nbt, spec.momentum) == expected
