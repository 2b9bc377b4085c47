"""Which library entry points each conv / norm autograd node of functional.py launches, in which order and with which key
arguments -- forward, first-order backward and backward under create_graph=True -- pinned on the host WITHOUT a GPU.
Every `ops` launch wrapper is replaced by a recorder that logs "name(key arguments)" and returns zeros of the right shape
and layout; the support queries are stubbed so that each route is taken on purpose, in both directions.  What the kernels
compute is checked by the GPU tests; this pins the wiring: the same launches, no more and no fewer."""
import functools
import json
import pathlib

import pytest
import torch

from b200gan import _lib, zoo

CL = torch.channels_last
ALGO = {_lib.ALGO_AUTO: "auto", _lib.ALGO_SIMT: "simt", _lib.ALGO_TC: "tc"}
PACK = dict(zip(range(6), ("simt_fprop", "simt_dgrad", "tc_fprop", "tc_dgrad", "tc_fprop_up2", "tc_dgrad_up2")))
ACT = {_lib.ACT_NONE: None, _lib.ACT_LRELU: "lrelu", _lib.ACT_RELU: "relu", _lib.ACT_TANH: "tanh",
       _lib.ACT_SIGMOID: "sigmoid"}
LRELU, RELU, TANH, NONE = _lib.ACT_LRELU, _lib.ACT_RELU, _lib.ACT_TANH, _lib.ACT_NONE


def fmt(name, *pos, **flags):
    """name(positional descriptors, then every flag that is set: `k` for True, `k=v` otherwise)"""
    parts = [str(p) for p in pos] + [k if v is True else f"{k}={v}" for k, v in flags.items()
                                     if v is not None and v is not False]
    return f"{name}({','.join(parts)})"


def _cl(*shape, dtype=torch.float32):
    t = torch.zeros(shape, dtype=dtype)
    return t.contiguous(memory_format=CL) if t.dim() == 4 else t


def _stats_kind(stats, per_sample):
    return None if stats is None else ("sample" if per_sample else "chan")


class Recorder:
    """The launch log plus the answers of the support queries (tc: tensor-core conv, dgn: conv_dgrad_norm, tail:
    the fused generator tail, nb: the fused narrow chain)."""

    def __init__(self):
        self.log = []
        self.tc = self.dgn = self.tail = self.nb = True

    def take(self):
        out, self.log = self.log, []
        return out

    def install(self, monkeypatch):
        from b200gan import nn as bnn, ops
        rec = self

        def add(name, *pos, **flags):
            rec.log.append(fmt(name, *pos, **flags))

        def conv_fprop(g, x, packed, algo, bias=None, act=NONE, slope=0.0, chan_scale=None, stats=None,
                       stats_per_sample=False, round_tf32=False):
            add("conv_fprop", ALGO[algo], act=ACT[act], bias=bias is not None, scale=chan_scale is not None,
                stats=_stats_kind(stats, stats_per_sample), rtf=bool(round_tf32))
            return _cl(g.N, g.K, g.P, g.Q)

        def conv_dgrad(g, dy, packed, algo):
            add("conv_dgrad", ALGO[algo])
            return _cl(g.N, g.C, g.H, g.W)

        def conv_wgrad(g, x, dy, weight_shape, need_bias, algo):
            add("conv_wgrad", ALGO[algo], db=bool(need_bias))
            return torch.zeros(weight_shape), (torch.zeros(g.K) if need_bias else None)

        def pack_weights(g, w, kind, out=None):
            add("pack_weights", PACK[kind], into=out is not None)
            return torch.zeros(1) if out is None else out

        def epilogue_bwd(dy, y, chan_scale, act, slope, round_tf32=False):
            add("epilogue_bwd", act=ACT[act], y=y is not None, scale=chan_scale is not None, rtf=bool(round_tf32))
            return _cl(*dy.shape)

        def bias_grad(dy, y, chan_scale, act, slope):
            add("bias_grad", act=ACT[act], scale=chan_scale is not None)
            return torch.zeros(dy.shape[1])

        def groups(x, per_sample):
            return x.shape[0] * x.shape[1] if per_sample else x.shape[1]

        def norm_forward(x, gamma, beta, running_mean, running_var, nbt, per_sample, eps, momentum, act=NONE,
                         slope=0.0, stats=None, round_tf32=False, return_scale_shift=False):
            add("norm_forward", "in" if per_sample else "bn", act=ACT[act], affine=gamma is not None,
                running=running_mean is not None, stats=stats is not None, rtf=bool(round_tf32))
            gr = groups(x, per_sample)
            out = (_cl(*x.shape), torch.zeros(2 * gr), torch.zeros(2 * gr))
            return out if return_scale_shift else out[:2]

        def norm_stats(x, per_sample):
            add("norm_stats", "in" if per_sample else "bn")
            return torch.zeros(2 * groups(x, per_sample), dtype=torch.float64)

        def norm_finalize(x_shape, stats, gamma, beta, running_mean, running_var, nbt, per_sample, eps, momentum,
                          device):
            add("norm_finalize", "in" if per_sample else "bn", affine=gamma is not None,
                running=running_mean is not None)
            return torch.zeros(stats.numel()), torch.zeros(stats.numel())

        def norm_backward(dy, x, y, mean_rstd, gamma, per_sample, eps, act=NONE, slope=0.0, need_params=False,
                          round_tf32=False, scale_shift=None):
            add("norm_backward", "in" if per_sample else "bn", act=ACT[act], y=y is not None, affine=gamma is not None,
                params=bool(need_params), rtf=bool(round_tf32), ss=scale_shift is not None)
            return _cl(*x.shape), (torch.zeros(mean_rstd.numel()) if need_params else None)

        def norm_double_backward(dy, x, mean_rstd, scale_shift, gamma, u, ugamma_ubeta, per_sample, act, slope,
                                 need_gx, need_gdy, need_ggamma):
            add("norm_double_backward", "in" if per_sample else "bn", act=ACT[act], affine=gamma is not None,
                ugb=ugamma_ubeta is not None, gx=bool(need_gx), gdy=bool(need_gdy), ggamma=bool(need_ggamma))
            gr = mean_rstd.numel() // 2
            return (_cl(*x.shape) if need_gx else None, _cl(*x.shape) if need_gdy else None,
                    torch.zeros(gr) if need_ggamma else None)

        def conv_dgrad_norm(g, dy, packed, x, mean_rstd, scale_shift, act, slope):
            add("conv_dgrad_norm", act=ACT[act])
            return _cl(g.N, g.C, g.H, g.W), torch.zeros(2 * g.C, dtype=torch.float64)

        def norm_backward_from_sums(dy, x, mean_rstd, gamma, sums, eps, act=NONE, slope=0.0, need_params=False,
                                    round_tf32=False, scale_shift=None):
            add("norm_backward_from_sums", act=ACT[act], affine=gamma is not None, params=bool(need_params),
                rtf=bool(round_tf32), ss=scale_shift is not None)
            return _cl(*x.shape), (torch.zeros(sums.numel()) if need_params else None)

        def tail_fprop(d, a, scale_shift, w, bias):
            add("tail_fprop", mid=ACT[d.act_mid], out=ACT[d.act_out], bias=bias is not None)
            return _cl(d.N, d.K, d.H, d.W)

        def tail_bwd(d, a, mean_rstd, scale_shift, w, g, need_affine, need_bias, round_tf32):
            add("tail_bwd", affine=bool(need_affine), db=bool(need_bias), rtf=bool(round_tf32))
            return (_cl(*a.shape), torch.zeros(2 * d.C) if need_affine else None, torch.zeros(d.K, d.C, 3, 3),
                    torch.zeros(d.K) if need_bias else None)

        def norm_apply_affine(x, scale_shift, per_sample, act=NONE, slope=0.0):
            add("norm_apply_affine", act=ACT[act])
            return _cl(*x.shape)

        def act_forward(x, act, slope, mask=None, mask_per_channel=False):
            add("act_forward", act=ACT[act], mask=("chan" if mask_per_channel else "elem") if mask is not None else None)
            return _cl(*x.shape)

        def upsample2x(x):
            add("upsample2x")
            n, c, h, w = x.shape
            return _cl(n, c, 2 * h, 2 * w)

        def upsample2x_bwd(dy):
            add("upsample2x_bwd")
            n, c, h, w = dy.shape
            return _cl(n, c, h // 2, w // 2)

        def pad2d(x, pads, mode, round_tf32=False):
            add("pad2d", pads, mode=mode, rtf=bool(round_tf32))
            n, c, h, w = x.shape
            return _cl(n, c, h + pads[0] + pads[2], w + pads[1] + pads[3])

        def pad2d_bwd(dy, pads, mode):
            add("pad2d_bwd", pads, mode=mode)
            n, c, h, w = dy.shape
            return _cl(n, c, h - pads[0] - pads[2], w - pads[1] - pads[3])

        def nb_fprop(g, x, packed, bias, act, slope, chan_scale, in_edge, running_mean, running_var, nbt, momentum,
                     want_stats, groups=1):
            add("nb_fprop", act=ACT[act], bias=bias is not None, scale=chan_scale is not None, in_bn=in_edge is not None,
                running=running_mean is not None, stats=bool(want_stats), groups=groups if groups != 1 else None)
            return _cl(g.N, g.K, g.P, g.Q), (torch.zeros(groups * 2 * g.K, dtype=torch.float64) if want_stats else None)

        def nb_dz(g_in, a, chan_scale, act, slope, out_edge, want_db):
            add("nb_dz", act=ACT[act], scale=chan_scale is not None, out_bn=out_edge is not None, db=bool(want_db))
            return _cl(*a.shape), (torch.zeros(a.shape[1]) if want_db else None)

        def nb_wgrad(g, x, dz, in_edge, weight_shape):
            add("nb_wgrad", in_bn=in_edge is not None)
            return torch.zeros(weight_shape)

        def nb_dgrad(g, dz, packed, in_edge, a_prev):
            add("nb_dgrad", in_bn=in_edge is not None)
            sums = torch.zeros(in_edge.groups * 2 * g.C, dtype=torch.float64) if in_edge is not None else None
            return _cl(g.N, g.C, g.H, g.W), sums

        def nb_tail_fwd(a, edge, running_mean, running_var, nbt, momentum, nchw):
            add("nb_tail_fwd", running=running_mean is not None, nchw=bool(nchw))
            return torch.zeros(a.shape) if nchw else _cl(*a.shape)

        def nb_tail_bwd(a, edge, dout, nchw):
            add("nb_tail_bwd", nchw=bool(nchw))
            return _cl(*a.shape), torch.zeros(edge.groups * 2 * a.shape[1], dtype=torch.float64)

        def to_cl(x):
            add("to_cl")
            return x.contiguous(memory_format=CL)

        def to_nchw(x):
            add("to_nchw")
            return x.contiguous()

        for fn in (conv_fprop, conv_dgrad, conv_wgrad, pack_weights, epilogue_bwd, bias_grad, norm_forward, norm_stats,
                   norm_finalize, norm_backward, norm_double_backward, conv_dgrad_norm, norm_backward_from_sums,
                   tail_fprop, tail_bwd, norm_apply_affine, act_forward, upsample2x, upsample2x_bwd, pad2d, pad2d_bwd,
                   nb_fprop, nb_dz, nb_wgrad, nb_dgrad, nb_tail_fwd, nb_tail_bwd, to_cl, to_nchw):
            monkeypatch.setattr(ops, fn.__name__, fn)
        monkeypatch.setattr(ops, "pack_weights_multi", None)  # not a node launch: must not be reached
        monkeypatch.setattr(ops, "tc_supported", lambda g, pas: rec.tc)
        monkeypatch.setattr(ops, "conv_dgrad_norm_supported", lambda g: rec.dgn)
        monkeypatch.setattr(ops, "tail_supported", lambda *a: rec.tail)
        monkeypatch.setattr(ops, "nb_supported", lambda g: rec.nb)
        monkeypatch.setattr(ops, "_require_cuda", lambda t, name="tensor": None)
        monkeypatch.setattr(ops.Config, "algo", "auto")
        monkeypatch.setattr(ops.Config, "weight_cache", True)
        monkeypatch.setattr(ops.Config, "fuse_narrow_chain", True)
        monkeypatch.setattr(bnn, "_on_device", lambda x: True)
        return self


@pytest.fixture
def rec(monkeypatch):
    return Recorder().install(monkeypatch)


def _leaf(t, grad=True):
    return t.requires_grad_(grad)


def _phases(rec, run, inputs, grad_out):
    """(forward, backward, create_graph backward) launch lists of out = run() differentiated w.r.t. `inputs`"""
    out = run()
    fwd = rec.take()
    y = out[0] if isinstance(out, tuple) else out
    torch.autograd.grad(y, inputs, grad_out(y), retain_graph=True, allow_unused=True)
    bwd = rec.take()
    torch.autograd.grad(y, inputs, grad_out(y), create_graph=True, allow_unused=True)
    return fwd, bwd, rec.take()


def _cg_refused(rec, run, inputs, match):
    y = run()
    y = y[0] if isinstance(y, tuple) else y
    rec.take()
    with pytest.raises(NotImplementedError, match=match):
        torch.autograd.grad(y, inputs, _cl(*y.shape), create_graph=True, allow_unused=True)


# ---- ConvFn ------------------------------------------------------------------------------------------------------
def _conv_setup(bias, scale, need_x, need_w, c=32, k=32, n=2, hw=8):
    x = _leaf(_cl(n, c, hw, hw), need_x)
    w = _leaf(torch.zeros(k, c, 3, 3), need_w)
    b = _leaf(torch.zeros(k), need_w) if bias else None
    cs = torch.zeros(n, k) if scale else None
    inputs = [t for t in (x, w, b) if t is not None and t.requires_grad]
    return x, w, b, cs, inputs


def _conv_bwd_expected(tc, act, bias, scale, rtf_dz, need_x, need_w, dgrad):
    out = []
    epi = act != NONE or scale
    if epi:
        out.append(fmt("epilogue_bwd", act=ACT[act], y=act != NONE, scale=scale, rtf=rtf_dz))
    out += dgrad
    want_db = bias and need_w
    if want_db and epi and rtf_dz:
        out.append(fmt("bias_grad", act=ACT[act], scale=scale))
        want_db = False
    if need_w or want_db:
        out.append(fmt("conv_wgrad", "auto", db=want_db))
    return out


@pytest.mark.parametrize("tc", [True, False], ids=["tc", "simt"])
@pytest.mark.parametrize("stats", [None, False, True], ids=["nostats", "chanstats", "samplestats"])
@pytest.mark.parametrize("rtf_dz", [False, True], ids=["dz", "rtfdz"])
@pytest.mark.parametrize("scale", [False, True], ids=["noscale", "scale"])
@pytest.mark.parametrize("act", [NONE, LRELU, TANH], ids=["none", "lrelu", "tanh"])
@pytest.mark.parametrize("bias", [False, True], ids=["nobias", "bias"])
def test_conv_fn(rec, tc, stats, rtf_dz, scale, act, bias):
    from b200gan import functional as F
    rec.tc = tc
    x, w, b, cs, inputs = _conv_setup(bias, scale, True, True)
    spec = F.ConvSpec(stride=1, pads=(1, 1, 1, 1), act=act, slope=0.2, stats=stats, rtf_out=tc, rtf_dz=rtf_dz)
    run = lambda: F.conv_block(x, w, b, cs, spec, F.PackCache())  # noqa: E731
    algo, pf, pd = ("tc", "tc_fprop", "tc_dgrad") if tc else ("simt", "simt_fprop", "simt_dgrad")
    if scale and act == TANH:
        _cg_refused(rec, run, inputs, "Dropout2d fused with tanh")
        cg = None
    else:
        fwd, bwd, cg = _phases(rec, run, inputs, lambda y: _cl(*y.shape))
    fwd_expected = [fmt("pack_weights", pf),
                    fmt("conv_fprop", algo, act=ACT[act], bias=bias, scale=scale,
                        stats=_stats_kind(stats, stats), rtf=tc)]
    if cg is None:
        return
    assert fwd == fwd_expected
    # each _phases call runs the forward once: the second backward finds its packed copy in the cache
    assert bwd == _conv_bwd_expected(tc, act, bias, scale, rtf_dz, True, True,
                                     [fmt("pack_weights", pd), fmt("conv_dgrad", algo)])
    assert cg == [fmt("pack_weights", pd), fmt("conv_dgrad", algo), fmt("conv_wgrad", "auto")]


@pytest.mark.parametrize("need", ["frozen", "input_const"])
@pytest.mark.parametrize("rtf_dz", [False, True], ids=["dz", "rtfdz"])
def test_conv_fn_partial_gradients(rec, need, rtf_dz):
    from b200gan import functional as F
    need_x, need_w = need != "input_const", need != "frozen"
    x, w, b, cs, inputs = _conv_setup(True, True, need_x, need_w)
    if not inputs:
        return
    spec = F.ConvSpec(stride=1, pads=(1, 1, 1, 1), act=LRELU, slope=0.2, rtf_dz=rtf_dz)
    fwd, bwd, cg = _phases(rec, lambda: F.conv_block(x, w, b, cs, spec, F.PackCache()), inputs,
                           lambda y: _cl(*y.shape))
    assert fwd == ["pack_weights(tc_fprop)", "conv_fprop(tc,act=lrelu,bias,scale)"]
    dgrad = ["pack_weights(tc_dgrad)", "conv_dgrad(tc)"] if need_x else []
    assert bwd == _conv_bwd_expected(True, LRELU, True, True, rtf_dz, need_x, need_w, dgrad)
    if need == "frozen":
        assert bwd == ["epilogue_bwd(act=lrelu,y,scale" + (",rtf)" if rtf_dz else ")"),
                       "pack_weights(tc_dgrad)", "conv_dgrad(tc)"]
        assert cg == ["pack_weights(tc_dgrad)", "conv_dgrad(tc)"]
    else:
        assert cg == ["conv_wgrad(auto)"]


def test_conv_fn_nchw_input_and_gradient(rec):
    from b200gan import functional as F
    x = torch.zeros(2, 32, 8, 8, requires_grad=True)
    w = torch.zeros(32, 32, 3, 3, requires_grad=True)
    y = F.conv_block(x, w, None, None, F.ConvSpec(stride=1, pads=(1, 1, 1, 1)), F.PackCache())
    assert rec.take() == ["to_cl()", "pack_weights(tc_fprop)", "conv_fprop(tc)"]
    torch.autograd.grad(y, [x, w], torch.zeros(2, 32, 8, 8))
    assert rec.take() == ["to_cl()", "pack_weights(tc_dgrad)", "conv_dgrad(tc)", "conv_wgrad(auto)"]


def test_conv_fn_repacks_an_updated_weight_in_place(rec):
    from b200gan import functional as F
    x, w = _cl(2, 32, 8, 8), torch.zeros(32, 32, 3, 3)
    cache, spec = F.PackCache(), F.ConvSpec(stride=1, pads=(1, 1, 1, 1))
    F.conv_block(x, w, None, None, spec, cache)
    F.conv_block(x, w, None, None, spec, cache)
    w.add_(1.0)
    F.conv_block(x, w, None, None, spec, cache)
    assert rec.take() == ["pack_weights(tc_fprop)", "conv_fprop(tc)", "conv_fprop(tc)",
                          "pack_weights(tc_fprop,into)", "conv_fprop(tc)"]


@pytest.mark.parametrize("up,mode", [(2, _lib.PAD_ZERO), (1, _lib.PAD_REFLECT)], ids=["up2", "reflect"])
def test_conv_fn_folded_upsample_or_reflection_refuses_double_backward(rec, up, mode):
    from b200gan import functional as F
    x, w = _leaf(_cl(2, 32, 8, 8)), _leaf(torch.zeros(32, 32, 3, 3))
    spec = F.ConvSpec(stride=1, pads=(1, 1, 1, 1), pad_mode=mode, up=up)
    _cg_refused(rec, lambda: F.conv_block(x, w, None, None, spec, F.PackCache()), [x, w], "folded upsample")


# ---- NormFn ------------------------------------------------------------------------------------------------------
def _norm_setup(per_sample, affine, running, need_x, need_p, c=32, n=2, hw=8):
    x = _leaf(_cl(n, c, hw, hw), need_x)
    gamma = _leaf(torch.ones(c), need_p) if affine else None
    beta = _leaf(torch.zeros(c), need_p) if affine else None
    rm, rv, nbt = (torch.zeros(c), torch.ones(c), torch.zeros((), dtype=torch.long)) if running else (None,) * 3
    inputs = [t for t in (x, gamma, beta) if t is not None and t.requires_grad]
    return x, gamma, beta, rm, rv, nbt, inputs


@pytest.mark.parametrize("rtf", [False, True], ids=["plain", "rtf"])
@pytest.mark.parametrize("stats", [False, True], ids=["ownstats", "fusedstats"])
@pytest.mark.parametrize("act", [NONE, LRELU, RELU, TANH], ids=["none", "lrelu", "relu", "tanh"])
@pytest.mark.parametrize("affine", [True, False], ids=["affine", "nonaffine"])
@pytest.mark.parametrize("kind", ["bn", "bn_running", "in"])
def test_norm_fn(rec, rtf, stats, act, affine, kind):
    from b200gan import functional as F
    per_sample, running = kind == "in", kind == "bn_running"
    x, gamma, beta, rm, rv, nbt, inputs = _norm_setup(per_sample, affine, running, True, True)
    st = torch.zeros(2 * (2 * 32 if per_sample else 32), dtype=torch.float64) if stats else None
    spec = F.NormSpec(per_sample=per_sample, eps=0.8, momentum=0.1 if running else 0.0, act=act, slope=0.2,
                      rtf_out=rtf, rtf_dx=rtf)
    run = lambda: F.norm_block(x, gamma, beta, st, rm, rv, nbt, spec)  # noqa: E731
    mask_from_x = act in (LRELU, RELU)
    fwd_expected = [fmt("norm_forward", kind[:2], act=ACT[act], affine=affine, running=running, stats=stats, rtf=rtf)]
    bwd_expected = [fmt("norm_backward", kind[:2], act=ACT[act], y=act == TANH, affine=affine, params=affine,
                        rtf=rtf, ss=mask_from_x)]
    if act == TANH:
        _cg_refused(rec, run, inputs, "normalisation fused with tanh")
        y = run()
        assert rec.take() == fwd_expected
        torch.autograd.grad(y, inputs, _cl(*y.shape))
        assert rec.take() == bwd_expected
        return
    fwd, bwd, cg = _phases(rec, run, inputs, lambda y: _cl(*y.shape))
    assert fwd == fwd_expected
    assert bwd == bwd_expected
    assert cg == [fmt("norm_backward", kind[:2], act=ACT[act], affine=affine, params=affine, rtf=rtf, ss=mask_from_x)]


@pytest.mark.parametrize("need", ["frozen", "input_const"])
@pytest.mark.parametrize("per_sample", [False, True], ids=["bn", "in"])
def test_norm_fn_partial_gradients(rec, need, per_sample):
    from b200gan import functional as F
    x, gamma, beta, rm, rv, nbt, inputs = _norm_setup(per_sample, True, False, need != "input_const", need != "frozen")
    spec = F.NormSpec(per_sample=per_sample, act=LRELU, slope=0.2)
    fwd, bwd, cg = _phases(rec, lambda: F.norm_block(x, gamma, beta, None, rm, rv, nbt, spec), inputs,
                           lambda y: _cl(*y.shape))
    k = "in" if per_sample else "bn"
    assert fwd == [f"norm_forward({k},act=lrelu,affine)"]
    params = ",params" if need != "frozen" else ""
    assert bwd == [f"norm_backward({k},act=lrelu,affine{params},ss)"]
    assert cg == [f"norm_backward({k},act=lrelu,affine{params},ss)"]


@pytest.mark.parametrize("per_sample", [False, True], ids=["bn", "in"])
def test_norm_fn_second_order(rec, per_sample):
    """The penalty's own backward: the backward of NormBwdFn is one norm_double_backward."""
    from b200gan import functional as F
    x, gamma, beta, rm, rv, nbt, inputs = _norm_setup(per_sample, True, False, True, True)
    y = F.norm_block(x, gamma, beta, None, rm, rv, nbt, F.NormSpec(per_sample=per_sample, act=LRELU, slope=0.2))
    dx, dgamma, dbeta = torch.autograd.grad(y, inputs, _cl(*y.shape), create_graph=True)
    rec.take()
    torch.autograd.grad(dx.sum() + dgamma.sum(), inputs, allow_unused=True)
    k = "in" if per_sample else "bn"
    # the incoming gradient of dx.sum() is an expanded tensor, not channels_last
    assert rec.take() == ["to_cl()", f"norm_double_backward({k},act=lrelu,affine,ugb,gx,ggamma)"]


# ---- NormConvFn --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("tc", [True, False], ids=["tc", "simt"])
@pytest.mark.parametrize("stats", [None, False, True], ids=["nostats", "chanstats", "samplestats"])
@pytest.mark.parametrize("rtf_dz", [False, True], ids=["dz", "rtfdz"])
@pytest.mark.parametrize("scale", [False, True], ids=["noscale", "scale"])
@pytest.mark.parametrize("cact", [NONE, LRELU, TANH], ids=["none", "lrelu", "tanh"])
@pytest.mark.parametrize("bias", [False, True], ids=["nobias", "bias"])
@pytest.mark.parametrize("nact", [NONE, LRELU], ids=["bn", "bnlrelu"])
@pytest.mark.parametrize("affine", [True, False], ids=["affine", "nonaffine"])
def test_norm_conv_fn(rec, tc, stats, rtf_dz, scale, cact, bias, nact, affine):
    from b200gan import functional as F
    rec.tc = tc
    x, gamma, beta, rm, rv, nbt, _ = _norm_setup(False, affine, True, True, True)
    _, w, b, cs, _ = _conv_setup(bias, scale, True, True)
    inputs = [t for t in (x, gamma, beta, w, b) if t is not None]
    nspec = F.NormSpec(eps=0.8, momentum=0.1, act=nact, slope=0.2, rtf_out=tc, rtf_dx=False)
    cspec = F.ConvSpec(stride=1, pads=(1, 1, 1, 1), act=cact, slope=0.2, stats=stats, rtf_out=tc, rtf_dz=rtf_dz)
    run = lambda: F.NormConvFn.apply(x, gamma, beta, None, rm, rv, nbt, w, b, cs, nspec, cspec,  # noqa: E731
                                     F.PackCache())
    algo, pf, pd = ("tc", "tc_fprop", "tc_dgrad") if tc else ("simt", "simt_fprop", "simt_dgrad")
    fwd_expected = [fmt("norm_forward", "bn", act=ACT[nact], affine=affine, running=True, rtf=tc),
                    fmt("pack_weights", pf),
                    fmt("conv_fprop", algo, act=ACT[cact], bias=bias, scale=scale, stats=_stats_kind(stats, stats),
                        rtf=tc)]
    if scale and cact == TANH:
        _cg_refused(rec, run, inputs, "Dropout2d fused with tanh")
        return
    fwd, bwd, cg = _phases(rec, run, inputs, lambda y: _cl(*y.shape))
    assert fwd == fwd_expected
    dgrad = [fmt("pack_weights", pd), fmt("conv_dgrad_norm", act=ACT[nact]),
             fmt("norm_backward_from_sums", act=ACT[nact], affine=affine, params=affine, ss=True)]
    assert bwd == _conv_bwd_expected(tc, cact, bias, scale, rtf_dz, True, True, dgrad)
    assert cg == [fmt("norm_forward", "bn", act=ACT[nact], affine=affine, rtf=tc),
                  fmt("pack_weights", pd), fmt("conv_dgrad", algo), fmt("conv_wgrad", "auto"),
                  fmt("norm_backward", "bn", act=ACT[nact], affine=affine, params=affine, ss=True)]


@pytest.mark.parametrize("need", ["frozen", "frozen_conv", "input_const", "input_const_frozen_norm"])
def test_norm_conv_fn_partial_gradients(rec, need):
    from b200gan import functional as F
    need_x = not need.startswith("input_const")
    need_p = need not in ("frozen", "input_const_frozen_norm")
    need_w = need != "frozen"
    x, gamma, beta, rm, rv, nbt, _ = _norm_setup(False, True, False, need_x, need_p)
    _, w, b, cs, _ = _conv_setup(True, False, True, need_w)
    inputs = [t for t in (x, gamma, beta, w, b) if t.requires_grad]
    nspec = F.NormSpec(act=LRELU, slope=0.2)
    cspec = F.ConvSpec(stride=1, pads=(1, 1, 1, 1), rtf_dz=True)
    fwd, bwd, cg = _phases(rec, lambda: F.NormConvFn.apply(x, gamma, beta, None, rm, rv, nbt, w, b, cs, nspec, cspec,
                                                           F.PackCache()), inputs, lambda y: _cl(*y.shape))
    assert fwd == ["norm_forward(bn,act=lrelu,affine)", "pack_weights(tc_fprop)", "conv_fprop(tc,bias)"]
    wgrad = ["conv_wgrad(auto,db)"] if need_w else []
    if need_x or need_p:
        p = ",params" if need_p else ""
        assert bwd == ["pack_weights(tc_dgrad)", "conv_dgrad_norm(act=lrelu)",
                       f"norm_backward_from_sums(act=lrelu,affine{p},ss)"] + wgrad
        assert cg == ["norm_forward(bn,act=lrelu,affine)", "pack_weights(tc_dgrad)", "conv_dgrad(tc)"] + \
            (["conv_wgrad(auto)"] if need_w else []) + [f"norm_backward(bn,act=lrelu,affine{p},ss)"]
    else:
        assert bwd == wgrad
        assert cg == ["norm_forward(bn,act=lrelu,affine)", "conv_wgrad(auto)"]


def test_norm_conv_fn_refusals(rec):
    from b200gan import functional as F
    x, gamma, beta, rm, rv, nbt, _ = _norm_setup(False, True, False, True, True)
    _, w, b, cs, _ = _conv_setup(False, False, True, True)
    inputs = [x, gamma, beta, w]
    up = F.ConvSpec(stride=1, pads=(1, 1, 1, 1), up=2)
    _cg_refused(rec, lambda: F.NormConvFn.apply(x, gamma, beta, None, rm, rv, nbt, w, None, None, F.NormSpec(), up,
                                                F.PackCache()), inputs, "folded upsample")
    tanh = F.NormSpec(act=TANH)
    plain = F.ConvSpec(stride=1, pads=(1, 1, 1, 1))
    _cg_refused(rec, lambda: F.NormConvFn.apply(x, gamma, beta, None, rm, rv, nbt, w, None, None, tanh, plain,
                                                F.PackCache()), inputs, "normalisation fused with tanh")


# ---- TailFn ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("rtf", [False, True], ids=["plain", "rtf"])
@pytest.mark.parametrize("act_out", [NONE, TANH], ids=["out", "tanh"])
@pytest.mark.parametrize("act_mid", [NONE, LRELU, RELU], ids=["mid", "lrelu", "relu"])
@pytest.mark.parametrize("bias", [False, True], ids=["nobias", "bias"])
@pytest.mark.parametrize("stats", [False, True], ids=["ownstats", "fusedstats"])
@pytest.mark.parametrize("norm", ["affine", "nonaffine", "running", "frozen", "input_const"])
def test_tail_fn(rec, rtf, act_out, act_mid, bias, stats, norm):
    from b200gan import functional as F
    affine, running = norm != "nonaffine", norm == "running"
    need_p, need_x = norm != "frozen", norm != "input_const"
    a, gamma, beta, rm, rv, nbt, _ = _norm_setup(False, affine, running, need_x, need_p, c=64)
    w = _leaf(torch.zeros(3, 64, 3, 3), need_p)
    b = _leaf(torch.zeros(3), need_p) if bias else None
    inputs = [t for t in (a, gamma, beta, w, b) if t is not None and t.requires_grad]
    st = torch.zeros(128, dtype=torch.float64) if stats else None
    spec = F.TailSpec(eps=0.8, momentum=0.1 if running else 0.0, act_mid=act_mid, slope=0.2, act_out=act_out,
                      rtf_dx=rtf)
    run = lambda: F.TailFn.apply(a, st, gamma, beta, rm, rv, nbt, w, b, spec)  # noqa: E731
    y = run()
    assert rec.take() == ([] if stats else ["norm_stats(bn)"]) + \
        [fmt("norm_finalize", "bn", affine=affine, running=running),
         fmt("tail_fprop", mid=ACT[act_mid], out=ACT[act_out], bias=bias)]
    torch.autograd.grad(y, inputs, _cl(*y.shape))
    need_affine = affine and need_p
    assert rec.take() == ([fmt("epilogue_bwd", act="tanh", y=True)] if act_out == TANH else []) + \
        [fmt("tail_bwd", affine=need_affine, db=bias and need_p, rtf=rtf)]
    _cg_refused(rec, run, inputs, "fused generator tail")


# ---- AffineActFn (eval-mode BatchNorm2d) -------------------------------------------------------------------------
@pytest.mark.parametrize("act", [NONE, LRELU, RELU, TANH], ids=["none", "lrelu", "relu", "tanh"])
def test_affine_act_fn(rec, act):
    from b200gan import functional as F
    x = _leaf(_cl(2, 32, 8, 8))
    run = lambda: F.AffineActFn.apply(x, torch.zeros(64), act, 0.2)  # noqa: E731
    if act == TANH:
        _cg_refused(rec, run, [x], "eval-mode BatchNorm2d fused with tanh")
        y = run()
        assert rec.take() == ["norm_apply_affine(act=tanh)"]
        torch.autograd.grad(y, [x], _cl(*y.shape))
        assert rec.take() == ["epilogue_bwd(act=tanh,y)", "norm_apply_affine()"]
        return
    fwd, bwd, cg = _phases(rec, run, [x], lambda y: _cl(*y.shape))
    assert fwd == [fmt("norm_apply_affine", act=ACT[act])]
    assert bwd == ([fmt("epilogue_bwd", act=ACT[act], y=True)] if act != NONE else []) + ["norm_apply_affine()"]
    assert cg == []


# ---- through nn.Sequential: the fused chain (NbConvFn / NbTailFn), the tail, the norm-conv pair -------------------------
def _chain(bnn_ns, bias, p, affine, running):
    layers = []
    for i, (cin, cout) in enumerate([(4, 16), (16, 32), (32, 64)]):
        layers += [bnn_ns.Conv2d(cin, cout, 3, 2, 1, bias=bias), bnn_ns.LeakyReLU(0.2), bnn_ns.Dropout2d(p)]
        if i > 0:
            layers.append(bnn_ns.BatchNorm2d(cout, 0.8, affine=affine, track_running_stats=running))
    return bnn_ns.Sequential(*layers).train()


def _chain_expected(bias, p, affine, running, need_x, need_p, nchw):
    """DCGAN's discriminator blocks: the first without a norm, the next two with one"""
    s = ",scale" if p else ""
    b = ",bias" if bias else ""
    r = ",running" if running else ""
    nchw_flag = "nchw" if nchw else ""
    fwd = (["to_cl()"] if nchw else []) + ["pack_weights(simt_fprop)", f"nb_fprop(act=lrelu{b}{s})",
           "pack_weights(simt_fprop)", f"nb_fprop(act=lrelu{b}{s},stats)",
           "pack_weights(simt_fprop)", f"nb_fprop(act=lrelu{b}{s},in_bn{r},stats)",
           "nb_tail_fwd(" + ",".join(f for f in (r[1:], nchw_flag) if f) + ")"]
    db = ",db" if bias and need_p else ""
    wgrad = lambda in_bn: [f"nb_wgrad({in_bn})"] if need_p else []  # noqa: E731
    dgrad = lambda in_bn: ["pack_weights(simt_dgrad)", f"nb_dgrad({in_bn})"]  # noqa: E731
    bwd = [f"nb_tail_bwd({nchw_flag})",
           f"nb_dz(act=lrelu{s},out_bn{db})"] + wgrad("in_bn") + dgrad("in_bn") + [
           f"nb_dz(act=lrelu{s},out_bn{db})"] + wgrad("") + dgrad("") + [
           f"nb_dz(act=lrelu{s}{db})"] + wgrad("") + (dgrad("") if need_x else [])
    return fwd, bwd


@pytest.mark.parametrize("grads", ["all", "frozen", "input_const"])
@pytest.mark.parametrize("nchw", [False, True], ids=["nhwc", "nchw"])
@pytest.mark.parametrize("running", [True, False], ids=["running", "norunning"])
@pytest.mark.parametrize("affine", [True, False], ids=["affine", "nonaffine"])
@pytest.mark.parametrize("p", [0.0, 0.25], ids=["nodrop", "drop"])
@pytest.mark.parametrize("bias", [True, False], ids=["bias", "nobias"])
def test_chain_nodes(rec, grads, nchw, running, affine, p, bias):
    import b200gan
    with b200gan.patched():
        seq = _chain(torch.nn, bias, p, affine, running)
    if grads == "frozen":
        seq.requires_grad_(False)
    need_x, need_p = grads != "input_const", grads != "frozen"
    x = torch.zeros(4, 4, 16, 16)
    x = x if nchw else x.contiguous(memory_format=CL)
    x.requires_grad_(need_x)
    inputs = ([x] if need_x else []) + [q for q in seq.parameters() if q.requires_grad]
    assert [type(s).__name__ for s in seq._plan()] == ["_ChainStep"]
    y = seq(x)
    fwd_expected, bwd_expected = _chain_expected(bias, p, affine, running, need_x, need_p, nchw)
    assert rec.take() == fwd_expected
    torch.autograd.grad(y, inputs, torch.zeros(y.shape) if nchw else _cl(*y.shape))
    assert rec.take() == bwd_expected


def test_chain_create_graph_and_true_gradients_after_it(rec):
    """A penalty through the chain: create_graph=True rebuilds each layer from differentiable nodes; every first-order
    backward of the same forward after it finishes the norm backward per node (true gradients)."""
    import b200gan
    with b200gan.patched():
        seq = _chain(torch.nn, True, 0.0, True, True)
    x = _leaf(_cl(4, 4, 16, 16))
    params = list(seq.parameters())
    y = seq(x)
    rec.take()
    torch.autograd.grad(y, [x] + params, _cl(*y.shape), create_graph=True, retain_graph=True)
    simt_nodes = ["pack_weights(simt_dgrad)", "conv_dgrad(simt)", "conv_wgrad(simt)"]
    nbwd = "norm_backward(bn,affine,params,ss)"
    # the last layer reads a BatchNorm output: recomputed, and its backward a NormBwdFn; a layer next to a chain
    # BatchNorm keeps the fp32 kernels; the first layer, with no norm on either side, routes as ConvFn does
    assert rec.take() == ["norm_stats(bn)", "norm_finalize(bn,affine)", nbwd,
                          "norm_forward(bn,affine)"] + simt_nodes + [nbwd] + simt_nodes + [
                          "pack_weights(tc_dgrad)", "conv_dgrad(tc)", "conv_wgrad(auto)"]
    torch.autograd.grad(y, [x] + params, _cl(*y.shape))
    finish = ["norm_stats(bn)", "norm_finalize(bn,affine)", "norm_backward_from_sums(affine,params)"]
    assert rec.take() == ["nb_tail_bwd()"] + finish + [
        "nb_dz(act=lrelu,db)", "nb_wgrad(in_bn)", "pack_weights(simt_dgrad)", "nb_dgrad(in_bn)"] + finish + [
        "nb_dz(act=lrelu,db)", "nb_wgrad()", "pack_weights(simt_dgrad)", "nb_dgrad()",
        "nb_dz(act=lrelu,db)", "nb_wgrad()", "pack_weights(simt_dgrad)", "nb_dgrad()"]


def test_chain_refuses_create_graph_under_groups(rec):
    import b200gan
    from b200gan import ops
    with b200gan.patched():
        seq = _chain(torch.nn, True, 0.0, True, True)
    x = _leaf(_cl(4, 4, 16, 16))
    with ops.bn_groups(2):
        y = seq(x)
    assert rec.take()[3] == "nb_fprop(act=lrelu,bias,stats,groups=2)"
    with pytest.raises(NotImplementedError, match="bn_groups"):
        torch.autograd.grad(y, [x], _cl(*y.shape), create_graph=True)


@pytest.mark.parametrize("supported", [True, False], ids=["fused", "unfused"])
@pytest.mark.parametrize("state", ["running", "norunning", "frozen"])
def test_generator_tail_through_sequential(rec, supported, state):
    import b200gan
    rec.tail = supported
    rec.dgn = False   # unfused, the norm and the conv stay two nodes
    with b200gan.patched():
        seq = torch.nn.Sequential(torch.nn.Conv2d(64, 64, 3, 1, 1), torch.nn.BatchNorm2d(64, 0.8),
                                  torch.nn.LeakyReLU(0.2), torch.nn.Conv2d(64, 3, 3, 1, 1), torch.nn.Tanh()).train()
    if state == "norunning":
        seq[1].track_running_stats = False
        seq[1].running_mean = seq[1].running_var = seq[1].num_batches_tracked = None
    if state == "frozen":
        seq.requires_grad_(False)
    x = _leaf(_cl(2, 64, 8, 8))
    params = [q for q in seq.parameters() if q.requires_grad]
    y = seq(x)
    r = ",running" if state != "norunning" else ""
    head = ["pack_weights(tc_fprop)", "conv_fprop(tc,bias,stats=chan)"]
    if supported:
        assert rec.take() == head + [f"norm_finalize(bn,affine{r})", "tail_fprop(mid=lrelu,out=tanh,bias)"]
    else:
        assert rec.take() == head + [f"norm_forward(bn,act=lrelu,affine{r},stats,rtf)", "pack_weights(tc_fprop)",
                                     "conv_fprop(tc,act=tanh,bias)"]
    torch.autograd.grad(y, [x] + params, _cl(*y.shape))
    p = state != "frozen"
    wgrad = ["conv_wgrad(auto,db)"] if p else []
    head_bwd = ["pack_weights(tc_dgrad)", "conv_dgrad(tc)"] + wgrad
    if supported:
        assert rec.take() == ["epilogue_bwd(act=tanh,y)", f"tail_bwd({'affine,db,rtf' if p else 'rtf'})"] + head_bwd
    else:
        assert rec.take() == ["epilogue_bwd(act=tanh,y)", "pack_weights(tc_dgrad)", "conv_dgrad(tc)"] + wgrad + [
            f"norm_backward(bn,act=lrelu,affine{',params' if p else ''},rtf,ss)"] + head_bwd


@pytest.mark.parametrize("supported", [True, False], ids=["fused", "unfused"])
@pytest.mark.parametrize("next_norm", ["bn", "bn_eval", "in"])
def test_norm_conv_pair_through_sequential(rec, supported, next_norm):
    import b200gan
    rec.dgn = supported
    rec.tail = False
    with b200gan.patched():
        nxt = torch.nn.InstanceNorm2d(32) if next_norm == "in" else torch.nn.BatchNorm2d(32)
        seq = torch.nn.Sequential(torch.nn.BatchNorm2d(32), torch.nn.ReLU(), torch.nn.Conv2d(32, 32, 3, 1, 1),
                                  torch.nn.LeakyReLU(0.2), torch.nn.Dropout2d(0.5), nxt).train()
    if next_norm == "bn_eval":
        nxt.eval()
    x = _leaf(_cl(2, 32, 8, 8))
    params = list(seq.parameters())
    y = seq(x)
    st = {"bn": ",stats=chan", "in": ",stats=sample", "bn_eval": ""}[next_norm]
    conv = f"conv_fprop(tc,act=lrelu,bias,scale{st})"
    last = {"bn": "norm_forward(bn,affine,running,stats)", "in": "norm_forward(in,stats)",
            "bn_eval": "norm_apply_affine()"}[next_norm]
    # NormConvFn or NormFn -> ConvFn: the same forward launches
    assert rec.take() == ["norm_forward(bn,act=relu,affine,running,rtf)", "pack_weights(tc_fprop)", conv, last]
    torch.autograd.grad(y, [x] + params, _cl(*y.shape), allow_unused=True)
    first = {"bn": ["norm_backward(bn,affine,params)"], "in": ["norm_backward(in)"],
             "bn_eval": ["norm_apply_affine()"]}[next_norm]
    conv_bwd = ["epilogue_bwd(act=lrelu,y,scale,rtf)", "pack_weights(tc_dgrad)"]
    if supported:
        assert rec.take() == first + conv_bwd + ["conv_dgrad_norm(act=relu)",
                                                 "norm_backward_from_sums(act=relu,affine,params,ss)",
                                                 "bias_grad(act=lrelu,scale)", "conv_wgrad(auto)"]
    else:
        assert rec.take() == first + conv_bwd + ["conv_dgrad(tc)", "bias_grad(act=lrelu,scale)", "conv_wgrad(auto)",
                                                 "norm_backward(bn,act=relu,affine,params,ss)"]


# ---- whole networks through nn.Sequential: every planned step, fused and fallen back ---------------------------------
# The launch log of a forward and a backward through each network below, compared with tests/golden/
# sequential_launch_logs.json.  The networks are run in training and eval mode, on NCHW and channels_last input, with
# the four support queries all answering yes and all answering no; the small hand-built Sequentials, which pin the
# order in which fused steps fall back, also with only `nb` or only `tail` answering no.
GOLDEN_LOGS = pathlib.Path(__file__).parent / "golden" / "sequential_launch_logs.json"
SUPPORT = {"all": (True, True, True, True), "none": (False, False, False, False),
           "no_nb": (True, True, True, False), "no_tail": (True, True, False, True)}   # (tc, dgn, tail, nb)


def _dragan_critic(ns, rec):
    """the body of tests/scripts/mini_dragan's Critic: three strided conv blocks, the last two with a BatchNorm2d"""
    layers = []
    for i, (cin, cout) in enumerate(((1, 16), (16, 32), (32, 64))):
        layers += [ns.Conv2d(cin, cout, 3, 2, 1), ns.LeakyReLU(0.2, inplace=True), ns.Dropout2d(0.25)]
        if i:
            layers.append(ns.BatchNorm2d(cout, 0.8))
    return ns.Sequential(*layers)


def _n1_decoder(ns, rec):
    """tests/test_gpu_n1.py's ConvTranspose2d -> BatchNorm2d -> ReLU decoder, at narrower widths"""
    def up(i, o):
        return [ns.ConvTranspose2d(i, o, 4, 2, 1), ns.BatchNorm2d(o, 0.8), ns.ReLU()]

    def down(i, o):
        return [ns.Conv2d(i, o, 4, 2, 1), ns.BatchNorm2d(o, 0.8), ns.LeakyReLU(0.2)]
    return ns.Sequential(*down(64, 128), *down(128, 256), ns.Conv2d(256, 512, 1), *up(512, 256), *up(256, 128),
                         ns.Conv2d(128, 32, 3, 1, 1), ns.Tanh())


def _hooked(rec, m):
    m.register_forward_hook(lambda mod, inp, out: rec.log.append(f"hook({type(mod).__name__})"))
    return m


NETS = {  # name: (builder(ns, rec), input shape, hand-built)
    "dcgan_g": (lambda ns, rec: zoo.DCGANGenerator(16, nn=ns).conv_blocks, (2, 128, 4, 4), False),
    "dcgan_d": (lambda ns, rec: zoo.DCGANDiscriminator(16, nn=ns).model, (2, 1, 16, 16), False),
    "dragan_critic": (_dragan_critic, (2, 1, 16, 16), False),
    "pix2pix_down": (lambda ns, rec: zoo.UNetDown(64, 128, dropout=0.5, nn=ns).model, (2, 64, 8, 8), False),
    "pix2pix_up": (lambda ns, rec: zoo.UNetUp(128, 64, dropout=0.5, nn=ns).model, (2, 128, 4, 4), False),
    "pix2pix_final": (lambda ns, rec: ns.Sequential(ns.Upsample(scale_factor=2), ns.ZeroPad2d((1, 0, 1, 0)),
                                                    ns.Conv2d(128, 3, 4, padding=1), ns.Tanh()), (2, 128, 8, 8), False),
    "cyclegan_g": (lambda ns, rec: zoo.GeneratorResNet((3, 16, 16), 1, nn=ns).model, (2, 3, 16, 16), False),
    "n1_decoder": (_n1_decoder, (2, 64, 16, 16), False),
    # a chain of three convs whose parts hold a BatchNorm2d -> stride-1 Conv2d pair
    "chain_with_pair": (lambda ns, rec: ns.Sequential(
        ns.Conv2d(4, 16, 3, 2, 1), ns.LeakyReLU(0.2), ns.Conv2d(16, 32, 3, 2, 1), ns.LeakyReLU(0.2),
        ns.BatchNorm2d(32), ns.Conv2d(32, 32, 3, 1, 1), ns.LeakyReLU(0.2), ns.BatchNorm2d(32)), (2, 4, 16, 16), True),
    # a BatchNorm2d directly in front of a chain whose first conv has stride 1
    "norm_before_chain": (lambda ns, rec: ns.Sequential(
        ns.BatchNorm2d(4), ns.Conv2d(4, 16, 3, 1, 1), ns.LeakyReLU(0.2), ns.Conv2d(16, 32, 3, 2, 1),
        ns.LeakyReLU(0.2), ns.BatchNorm2d(32)), (2, 4, 16, 16), True),
    # a chain ending in a BatchNorm2d, followed by an Upsample -> Conv2d the chain cannot take
    "chain_then_conv": (lambda ns, rec: ns.Sequential(
        ns.Conv2d(4, 16, 3, 2, 1), ns.LeakyReLU(0.2), ns.Conv2d(16, 32, 3, 2, 1), ns.LeakyReLU(0.2),
        ns.BatchNorm2d(32), ns.Upsample(scale_factor=2), ns.Conv2d(32, 32, 3, 1, 1)), (2, 4, 16, 16), True),
    "tail": (lambda ns, rec: ns.Sequential(
        ns.Conv2d(64, 64, 3, 1, 1), ns.BatchNorm2d(64, 0.8), ns.LeakyReLU(0.2), ns.Conv2d(64, 3, 3, 1, 1),
        ns.Tanh()), (2, 64, 8, 8), True),
    "hooked_pair_norm": (lambda ns, rec: ns.Sequential(
        _hooked(rec, ns.BatchNorm2d(32)), ns.ReLU(), ns.Conv2d(32, 32, 3, 1, 1)), (2, 32, 8, 8), True),
    "hooked_pair_conv": (lambda ns, rec: ns.Sequential(
        ns.BatchNorm2d(32), ns.ReLU(), _hooked(rec, ns.Conv2d(32, 32, 3, 1, 1))), (2, 32, 8, 8), True),
    "hooked_before_pair": (lambda ns, rec: ns.Sequential(
        _hooked(rec, ns.Conv2d(32, 32, 3, 1, 1)), ns.BatchNorm2d(32), ns.ReLU(), ns.Conv2d(32, 32, 3, 1, 1)),
        (2, 32, 8, 8), True),
}
SEQUENTIAL_CASES = [f"{name}-{mode}-{layout}-{sup}" for name, (_, _, hand) in NETS.items()
                    for mode in ("train", "eval") for layout in ("nchw", "cl")
                    for sup in (SUPPORT if hand else ("all", "none"))]
SEQUENTIAL_CASES += [f"{name}-train-cl-{sup}-groups2" for name in ("dcgan_d", "dragan_critic", "tail")
                     for sup in ("all", "none")]
SEQUENTIAL_CASES += [f"{name}-train-cl-{sup}-create_graph" for name in ("dcgan_d", "dragan_critic")
                     for sup in ("all", "no_nb")]


def sequential_log(rec, case):
    """{"fwd": launches, "bwd": launches, "out": shape and layout}; a raised error ends its phase's list"""
    from b200gan import ops
    name, mode, layout, sup, *extra = case.split("-")
    build, shape, _ = NETS[name]
    rec.tc, rec.dgn, rec.tail, rec.nb = SUPPORT[sup]
    torch.manual_seed(0)
    seq = build(zoo.namespace(), rec).train(mode == "train")
    x = torch.zeros(shape)
    x = (x if layout == "nchw" else x.contiguous(memory_format=CL)).requires_grad_(True)
    inputs = [x] + [q for q in seq.parameters() if q.requires_grad]
    log = {}
    with ops.bn_groups(2 if "groups2" in extra else 1):
        try:
            y = seq(x)
        except (RuntimeError, NotImplementedError, ValueError) as e:
            return {"fwd": rec.take() + [f"raise {type(e).__name__}: {e}"]}
        log["fwd"] = rec.take()
        log["out"] = [list(y.shape), "nchw" if y.is_contiguous() else "cl"]
        try:
            torch.autograd.grad(y, inputs, torch.zeros_like(y), allow_unused=True,
                                create_graph="create_graph" in extra)
            log["bwd"] = rec.take()
        except (RuntimeError, NotImplementedError) as e:
            log["bwd"] = rec.take() + [f"raise {type(e).__name__}: {e}"]
    return log


@functools.lru_cache(maxsize=None)
def _golden_logs():
    return json.loads(GOLDEN_LOGS.read_text())


def test_every_sequential_case_has_a_golden_log():
    assert sorted(_golden_logs()) == sorted(SEQUENTIAL_CASES)


@pytest.mark.parametrize("case", SEQUENTIAL_CASES)
def test_sequential_launch_log(rec, case):
    assert sequential_log(rec, case) == _golden_logs()[case]
