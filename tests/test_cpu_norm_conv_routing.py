"""Which nn.Sequential runs take functional.NormConvFn (BatchNorm2d [-> LeakyReLU/ReLU] [-> Upsample x2] -> Conv2d with
the norm's backward sums from the conv's data-gradient epilogue) and which keep the NormFn -> ConvFn pair, decided on
the host WITHOUT a GPU: the autograd nodes are replaced by recorders and the library's support query by a stub."""
import pytest
import torch
import torch.nn as tnn

from b200gan import _lib


@pytest.fixture
def calls(monkeypatch):
    from b200gan import functional as F, nn as bnn, ops
    log = []

    def conv_out(x, w, spec):
        g, shape = ops.make_geom(tuple(x.shape), tuple(w.shape), spec.stride, spec.pads, spec.pad_mode, spec.up,
                                 spec.transposed)
        y = torch.zeros(shape)
        return (y, torch.zeros(2 * shape[1], dtype=torch.float64)) if spec.stats is not None else y

    def norm_block(x, gamma, beta, stats, rm, rv, nbt, spec):
        log.append(("norm", spec.act))
        return x

    def conv_block(x, w, b, chan_scale, spec, cache):
        log.append(("conv", spec.up))
        return conv_out(x, w, spec)

    def norm_conv(x, gamma, beta, stats, rm, rv, nbt, w, b, chan_scale, nspec, cspec, cache):
        log.append(("norm_conv", nspec.act, cspec.up, cspec.stats))
        return conv_out(x, w, cspec)

    monkeypatch.setattr(bnn, "_on_device", lambda x: True)
    monkeypatch.setattr(F, "norm_block", norm_block)
    monkeypatch.setattr(F, "conv_block", conv_block)
    def affine(x, scale_shift, act, slope):  # eval-mode BatchNorm2d
        log.append(("affine", act))
        return x

    monkeypatch.setattr(F.NormConvFn, "apply", norm_conv)
    monkeypatch.setattr(F.AffineActFn, "apply", affine)
    monkeypatch.setattr(ops, "tail_supported", lambda *a: False)
    supported = {"ok": True}
    monkeypatch.setattr(ops, "conv_dgrad_norm_supported", lambda g: supported["ok"])
    monkeypatch.setattr(ops.Config, "algo", "auto")
    return log, supported


def _gen():
    from b200gan import zoo
    return zoo.DCGANGenerator(64).train()


def _run(seq, shape):
    return seq(torch.zeros(shape).contiguous(memory_format=torch.channels_last))


def test_dcgan_generator_norms_take_the_fused_node(calls):
    log, _ = calls
    g = _gen()
    _run(g.conv_blocks, (4, 128, 16, 16))
    # the tail (dcgan.py:60-63) is stubbed as unsupported here, so its norm and conv pair up as well
    assert log == [("norm_conv", _lib.ACT_NONE, 2, False), ("norm_conv", _lib.ACT_LRELU, 2, False),
                   ("norm_conv", _lib.ACT_LRELU, 1, None)]


def test_eval_generator_keeps_the_pair(calls):
    log, _ = calls
    g = _gen().eval()
    with torch.no_grad():
        _run(g.conv_blocks, (4, 128, 16, 16))
    assert not any(e[0] == "norm_conv" for e in log)


def test_geometry_without_fused_data_gradient_keeps_the_pair(calls):
    log, supported = calls
    supported["ok"] = False
    _run(_gen().conv_blocks, (4, 128, 16, 16))
    assert [e[0] for e in log] == ["norm", "conv", "norm", "conv", "norm", "conv"]


def test_eval_mode_keeps_the_pair_even_when_supported(calls):
    log, _ = calls
    g = _gen()
    g.conv_blocks[0].eval()
    _run(g.conv_blocks, (4, 128, 16, 16))
    assert [e[0] for e in log][:2] == ["affine", "conv"]


def test_hooks_keep_the_pair(calls):
    log, _ = calls
    g = _gen()
    g.conv_blocks[2].register_forward_hook(lambda *a: None)
    _run(g.conv_blocks, (4, 128, 16, 16))
    assert [e[0] for e in log][:3] == ["norm", "conv", "norm_conv"]


@pytest.mark.parametrize("make", [
    lambda: [tnn.InstanceNorm2d(32), tnn.Conv2d(32, 32, 3, 1, 1)],                    # per-sample statistics
    lambda: [tnn.BatchNorm2d(32), tnn.Conv2d(32, 32, 3, 2, 1)],                      # stride 2
    lambda: [tnn.BatchNorm2d(32), tnn.Tanh(), tnn.Conv2d(32, 32, 3, 1, 1)],          # activation without a mask from x
    lambda: [tnn.BatchNorm2d(32), tnn.ConvTranspose2d(32, 32, 4, 2, 1)],
], ids=["instancenorm", "stride2", "tanh", "convtranspose"])
def test_other_norm_conv_pairs_keep_the_pair(calls, make):
    import b200gan
    log, _ = calls
    with b200gan.patched():
        seq = tnn.Sequential(*make()).train()
    _run(seq, (2, 32, 8, 8))
    assert not any(e[0] == "norm_conv" for e in log), log


def test_plain_batchnorm_relu_conv_takes_the_fused_node(calls):
    import b200gan
    log, _ = calls
    with b200gan.patched():
        seq = tnn.Sequential(tnn.BatchNorm2d(32), tnn.ReLU(), tnn.Conv2d(32, 64, 3, 1, 1)).train()
    _run(seq, (2, 32, 8, 8))
    assert log == [("norm_conv", _lib.ACT_RELU, 1, None)]
