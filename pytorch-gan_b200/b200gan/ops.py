"""Tensor-level wrappers over the C ABI (include/b200gan.h).

Activations are torch tensors of logical shape [N, C, H, W] whose memory is NHWC
(`torch.channels_last`).  Nothing here differentiates; autograd lives in functional.py.
PyTorch is used for device memory (caching allocator), streams and tensor plumbing only.
"""
import ctypes
import os

import torch

from . import _lib
from ._lib import (ACT_NONE, ALGO_AUTO, ALGO_SIMT, ALGO_TC, PACK_SIMT_DGRAD, PACK_SIMT_FPROP, PACK_TC_DGRAD,
                   PACK_TC_DGRAD_UP2, PACK_TC_FPROP, PACK_TC_FPROP_UP2, PAD_REFLECT, PAD_ZERO, ConvGeom, Epilogue,
                   MlpCriticDesc, MlpGenDesc, MlpGenGrads, NbBn, NormDesc, PixelLossDesc, TailDesc)

CL = torch.channels_last


class Config:
    """Global switches. `algo`: 'auto' (wgmma TF32 where the geometry qualifies) or 'simt'."""
    algo = os.environ.get("B200GAN_ALGO", "auto")
    weight_cache = True
    # a fused Sequential fed an NCHW-contiguous tensor returns an NCHW-contiguous tensor (what a script may .view,
    # dcgan.py:96) only for feature maps of at most this many pixels; larger maps stay channels_last
    contiguous_hw_limit = 64
    # [Conv2d -> LeakyReLU -> Dropout2d -> BatchNorm2d] runs of narrow layers as the fused chain (csrc/narrow_block.cu)
    fuse_narrow_chain = os.environ.get("B200GAN_FUSE_CHAIN", "1") not in ("", "0")


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _ptr(t):
    return 0 if t is None else t.data_ptr()


def _require_cuda(t, name="tensor"):
    if not t.is_cuda:
        raise RuntimeError(f"b200gan: {name} is on {t.device}; the b200gan product path runs on CUDA only "
                           "(no CPU fallback)")
    if t.dtype != torch.float32:
        raise RuntimeError(f"b200gan: {name} has dtype {t.dtype}; fp32 expected")


def is_cl(x):
    return x.dim() == 4 and x.is_contiguous(memory_format=CL)


def empty_cl(n, c, h, w, device):
    return torch.empty((n, c, h, w), device=device, dtype=torch.float32, memory_format=CL)


def to_cl(x):
    """NCHW-contiguous -> NHWC memory (our transpose kernel); no-op if already channels_last."""
    _require_cuda(x, "input")
    if is_cl(x):
        return x
    if x.dim() == 4 and x.stride(1) == 1 and not x.is_contiguous():
        # channel-innermost but not dense: a channel slice of a channels_last tensor (the gradient of one input of
        # torch.cat(..., 1), pix2pix/models.py:50,132).  One strided copy, coalesced along C -- not a round trip
        # through NCHW.
        y = empty_cl(*x.shape, x.device)
        y.copy_(x)
        return y
    if not x.is_contiguous():
        x = x.contiguous()
    n, c, h, w = x.shape
    y = empty_cl(n, c, h, w, x.device)
    if x.numel() == 0:
        return y
    _lib.check(_lib.load().b200gan_nchw_to_nhwc(x.data_ptr(), y.data_ptr(), n, c, h * w, _stream()), "nchw_to_nhwc")
    return y


def to_nchw(x):
    """NHWC memory -> NCHW-contiguous tensor (needed where scripts call .view, dcgan.py:96)."""
    _require_cuda(x, "input")
    if x.is_contiguous():
        return x
    if not is_cl(x):
        return x.contiguous()
    n, c, h, w = x.shape
    y = torch.empty((n, c, h, w), device=x.device, dtype=torch.float32)
    if x.numel() == 0:
        return y
    _lib.check(_lib.load().b200gan_nhwc_to_nchw(x.data_ptr(), y.data_ptr(), n, c, h * w, _stream()), "nhwc_to_nchw")
    return y


# ---- convolution -------------------------------------------------------------------------------
def make_geom(x_shape, weight_shape, stride, pads, pad_mode=PAD_ZERO, up=1, transposed=False):
    """pads = (top, left, bottom, right) of the virtual input. Returns (ConvGeom, out_shape)."""
    n, c, h, w = x_shape
    g = ConvGeom()
    g.N, g.H, g.W, g.C = n, h, w, c
    if transposed:
        cin, cout, r, s = weight_shape
    else:
        cout, cin, r, s = weight_shape
    if cin != c:
        raise RuntimeError(f"b200gan conv: input has {c} channels, weight expects {cin}")
    g.K, g.R, g.S, g.stride = cout, r, s, stride
    g.pad_t, g.pad_l, g.pad_b, g.pad_r = pads
    g.pad_mode, g.up, g.transposed = pad_mode, up, int(transposed)
    if transposed:
        g.P = (h - 1) * stride - 2 * pads[0] + r
        g.Q = (w - 1) * stride - 2 * pads[1] + s
    else:
        g.P = (h * up + pads[0] + pads[2] - r) // stride + 1
        g.Q = (w * up + pads[1] + pads[3] - s) // stride + 1
    return g, (n, cout, g.P, g.Q)


def tc_supported(g, pas):
    if Config.algo == "simt":
        return False
    return bool(_lib.load().b200gan_conv2d_supported(ctypes.byref(g), pas, ALGO_TC))


def conv_plan(g, pas, chan_scale=None):
    """(algo, packed layout) of pass `pas` (0 fprop, 1 dgrad, 2 wgrad) of a convolution: the one place that decides
    which kernel family runs it and which packed weight copy that kernel reads.  The layout follows the pass, whether or
    not the conv is transposed.  The weight gradient reads no packed copy (layout None) and lets the library route it.
    `chan_scale`: the forward carries a Dropout2d scale, which the narrow-output (K < 32) wgmma form does not fuse."""
    if pas == 2:
        return (ALGO_SIMT if Config.algo == "simt" else ALGO_AUTO), None
    tc = tc_supported(g, pas) and not (pas == 0 and g.K < 32 and chan_scale is not None)
    if not tc:
        return ALGO_SIMT, (PACK_SIMT_FPROP if pas == 0 else PACK_SIMT_DGRAD)
    if pas == 0:
        return ALGO_TC, (PACK_TC_FPROP_UP2 if g.up == 2 else PACK_TC_FPROP)
    return ALGO_TC, (PACK_TC_DGRAD_UP2 if g.up == 2 else PACK_TC_DGRAD)


def pack_weights(g, w, kind, out=None):
    lib = _lib.load()
    if out is None:
        n = lib.b200gan_packed_weight_floats(ctypes.byref(g), kind)
        out = torch.empty(n, device=w.device, dtype=torch.float32)
    _lib.check(lib.b200gan_pack_weights(ctypes.byref(g), kind, w.data_ptr(), out.data_ptr(), _stream()), "pack_weights")
    return out


def pack_weights_multi(jobs):
    """jobs: [(ConvGeom, kind, weight tensor, packed buffer)] -- one launch for all of them."""
    table = (_lib.PackJob * len(jobs))()
    for i, (g, kind, w, packed) in enumerate(jobs):
        table[i].w, table[i].packed, table[i].geom, table[i].pack = w.data_ptr(), packed.data_ptr(), g, kind
    _lib.check(_lib.load().b200gan_pack_weights_multi(table, len(jobs), _stream()), "pack_weights_multi")


def conv_fprop(g, x, packed, algo, bias=None, act=ACT_NONE, slope=0.0, chan_scale=None, stats=None,
               stats_per_sample=False, round_tf32=False):
    y = empty_cl(g.N, g.K, g.P, g.Q, x.device)
    if g.N == 0:
        return y
    ep = Epilogue()
    ep.bias, ep.act, ep.slope = _ptr(bias), act, slope
    ep.chan_scale, ep.stats = _ptr(chan_scale), _ptr(stats)
    ep.stats_per_sample, ep.round_tf32 = int(stats_per_sample), int(round_tf32)
    _lib.check(_lib.load().b200gan_conv2d_fprop(ctypes.byref(g), ctypes.byref(ep), x.data_ptr(), packed.data_ptr(),
                                                y.data_ptr(), algo, _stream()), "conv2d_fprop")
    return y


def conv_dgrad(g, dy, packed, algo):
    lib = _lib.load()
    dx = empty_cl(g.N, g.C, g.H, g.W, dy.device)
    nws = lib.b200gan_conv2d_dgrad_workspace_floats(ctypes.byref(g), algo)
    ws = torch.empty(nws, device=dy.device, dtype=torch.float32) if nws else None
    _lib.check(lib.b200gan_conv2d_dgrad(ctypes.byref(g), dy.data_ptr(), packed.data_ptr(), dx.data_ptr(), _ptr(ws),
                                        algo, _stream()), "conv2d_dgrad")
    return dx


def conv_wgrad(g, x, dy, weight_shape, need_bias, algo):
    lib = _lib.load()
    dw = torch.empty(weight_shape, device=x.device, dtype=torch.float32)
    db = torch.empty(g.K, device=x.device, dtype=torch.float32) if need_bias else None
    nws = lib.b200gan_conv2d_wgrad_workspace_floats(ctypes.byref(g), algo)
    ws = torch.empty(nws, device=x.device, dtype=torch.float32) if nws else None
    _lib.check(lib.b200gan_conv2d_wgrad_fused_bias(ctypes.byref(g), x.data_ptr(), dy.data_ptr(), dw.data_ptr(),
                                                   _ptr(db), _ptr(ws), algo, _stream()), "conv2d_wgrad")
    return dw, db


def conv_wgrad_phase_major(g):
    """whether the tensor-core weight gradient of g computes the four taps of an upsample phase per CTA"""
    return bool(_lib.load().b200gan_conv2d_wgrad_phase_major(ctypes.byref(g)))


def epilogue_bwd(dy, y, chan_scale, act, slope, round_tf32=False):
    n, k, p, q = dy.shape
    dz = torch.empty_like(dy, memory_format=CL)
    _lib.check(_lib.load().b200gan_epilogue_bwd(dy.data_ptr(), _ptr(y), _ptr(chan_scale), act, slope, dy.numel(), k,
                                                p * q, int(round_tf32), dz.data_ptr(), _stream()), "epilogue_bwd")
    return dz


def bias_grad(dy, y, chan_scale, act, slope):
    """Bias gradient of a fused conv block from unrounded values (see include/b200gan.h)."""
    n, k, p, q = dy.shape
    db = torch.empty(k, device=dy.device, dtype=torch.float32)
    _lib.check(_lib.load().b200gan_bias_grad(dy.data_ptr(), _ptr(y), _ptr(chan_scale), act, slope, n * p * q, k, p * q,
                                             db.data_ptr(), _stream()), "bias_grad")
    return db


# ---- normalisation -----------------------------------------------------------------------------
def _norm_desc(shape, per_sample, eps, momentum, act, slope, round_tf32):
    n, c, h, w = shape
    d = NormDesc()
    d.N, d.HW, d.C, d.per_sample = n, h * w, c, int(per_sample)
    d.eps, d.momentum, d.act, d.slope, d.round_tf32 = eps, momentum, act, slope, int(round_tf32)
    return d


_zero_scratch = {}


def zero_scratch(device, numel):
    """Persistent fp64 accumulator that is zero whenever it is handed out: every kernel that consumes it
    (norm_finalize, norm_bwd) zeroes it again, so no fill kernel is launched per use.  One buffer per
    (device, size) suffices because producer -> consumer pairs never interleave on the stream."""
    key = (device, numel)
    t = _zero_scratch.get(key)
    if t is None:
        t = torch.zeros(numel, device=device, dtype=torch.float64)
        _zero_scratch[key] = t
    return t


def reset_scratch():
    """Re-zero the accumulators (only needed after an exception interrupted a producer/consumer pair)."""
    for t in _zero_scratch.values():
        t.zero_()


def new_stats(x, per_sample):
    n, c = x.shape[0], x.shape[1]
    return zero_scratch(x.device, 2 * (n * c if per_sample else c))


def norm_forward(x, gamma, beta, running_mean, running_var, nbt, per_sample, eps, momentum, act=ACT_NONE, slope=0.0,
                 stats=None, round_tf32=False, return_scale_shift=False):
    """Training-mode BatchNorm2d / InstanceNorm2d.  Returns (y, mean_rstd)."""
    if stats is None:
        stats = norm_stats(x, per_sample)
    mean_rstd, scale_shift = norm_finalize(x.shape, stats, gamma, beta, running_mean, running_var, nbt, per_sample, eps,
                                           momentum, x.device)
    d = _norm_desc(x.shape, per_sample, eps, momentum, act, slope, round_tf32)
    y = torch.empty_like(x, memory_format=CL)
    _lib.check(_lib.load().b200gan_norm_apply(ctypes.byref(d), x.data_ptr(), scale_shift.data_ptr(), y.data_ptr(),
                                              _stream()), "norm_apply")
    if return_scale_shift:
        return y, mean_rstd, scale_shift
    return y, mean_rstd


def norm_finalize(x_shape, stats, gamma, beta, running_mean, running_var, nbt, per_sample, eps, momentum, device):
    """Batch statistics -> (mean_rstd, scale_shift); updates the running statistics.  `stats` is consumed (zeroed)."""
    d = _norm_desc(x_shape, per_sample, eps, momentum, ACT_NONE, 0.0, False)
    groups = stats.numel() // 2
    mean_rstd = torch.empty(2 * groups, device=device, dtype=torch.float32)
    scale_shift = torch.empty(2 * groups, device=device, dtype=torch.float32)
    _lib.check(_lib.load().b200gan_norm_finalize(ctypes.byref(d), stats.data_ptr(), _ptr(gamma), _ptr(beta),
                                                 mean_rstd.data_ptr(), scale_shift.data_ptr(), _ptr(running_mean),
                                                 _ptr(running_var), _ptr(nbt), _stream()), "norm_finalize")
    return mean_rstd, scale_shift


def norm_stats(x, per_sample):
    d = _norm_desc(x.shape, per_sample, 0.0, 0.0, ACT_NONE, 0.0, False)
    stats = new_stats(x, per_sample)
    _lib.check(_lib.load().b200gan_norm_stats(ctypes.byref(d), x.data_ptr(), stats.data_ptr(), _stream()), "norm_stats")
    return stats


# ---- Generator tail: BatchNorm2d -> act -> Conv2d(C, K<=3, 3, 1, 1) -> act (csrc/tail.cu) -------------------
def tail_desc(a_shape, k, act_mid, slope, act_out):
    n, c, h, w = a_shape
    d = TailDesc()
    d.N, d.H, d.W, d.C, d.K = n, h, w, c, k
    d.act_mid, d.slope, d.act_out = act_mid, slope, act_out
    return d


def tail_supported(a_shape, k, act_mid, slope, act_out):
    if Config.algo == "simt":
        return False
    return bool(_lib.load().b200gan_tail_supported(ctypes.byref(tail_desc(a_shape, k, act_mid, slope, act_out))))


def tail_fprop(d, a, scale_shift, w, bias):
    out = empty_cl(d.N, d.K, d.H, d.W, a.device)
    _lib.check(_lib.load().b200gan_tail_fprop(ctypes.byref(d), a.data_ptr(), scale_shift.data_ptr(), w.data_ptr(),
                                              _ptr(bias), out.data_ptr(), _stream()), "tail_fprop")
    return out


def tail_bwd(d, a, mean_rstd, scale_shift, w, g, need_affine, need_bias, round_tf32):
    lib = _lib.load()
    nws = lib.b200gan_tail_bwd_workspace_bytes(ctypes.byref(d))
    ws = torch.empty((nws + 7) // 8, device=a.device, dtype=torch.float64)
    da = torch.empty_like(a, memory_format=CL)
    dgb = torch.empty(2 * d.C, device=a.device, dtype=torch.float32) if need_affine else None
    dw = torch.empty((d.K, d.C, 3, 3), device=a.device, dtype=torch.float32)
    db = torch.empty(d.K, device=a.device, dtype=torch.float32) if need_bias else None
    _lib.check(lib.b200gan_tail_bwd(ctypes.byref(d), a.data_ptr(), mean_rstd.data_ptr(), scale_shift.data_ptr(),
                                    w.data_ptr(), g.data_ptr(), ws.data_ptr(), da.data_ptr(), _ptr(dgb), dw.data_ptr(),
                                    _ptr(db), int(round_tf32), _stream()), "tail_bwd")
    return da, dgb, dw, db


def norm_apply_affine(x, scale_shift, per_sample, act=ACT_NONE, slope=0.0):
    """y = act(x * scale + shift) with precomputed per-group scale/shift (eval-mode BatchNorm)."""
    d = _norm_desc(x.shape, per_sample, 0.0, 0.0, act, slope, False)
    y = torch.empty_like(x, memory_format=CL)
    _lib.check(_lib.load().b200gan_norm_apply(ctypes.byref(d), x.data_ptr(), scale_shift.data_ptr(), y.data_ptr(),
                                              _stream()), "norm_apply")
    return y


def norm_backward(dy, x, y, mean_rstd, gamma, per_sample, eps, act=ACT_NONE, slope=0.0, need_params=False,
                  round_tf32=False, scale_shift=None):
    lib = _lib.load()
    d = _norm_desc(x.shape, per_sample, eps, 0.0, act, slope, round_tf32)
    groups = mean_rstd.numel() // 2
    sums = zero_scratch(x.device, 2 * groups)
    dx = torch.empty_like(x, memory_format=CL)
    dgb = torch.empty(2 * groups, device=x.device, dtype=torch.float32) if need_params else None
    _lib.check(lib.b200gan_norm_bwd(ctypes.byref(d), dy.data_ptr(), x.data_ptr(), _ptr(y), mean_rstd.data_ptr(),
                                    _ptr(scale_shift), _ptr(gamma), sums.data_ptr(), dx.data_ptr(), _ptr(dgb), _stream()),
               "norm_bwd")
    return dx, dgb


def norm_double_backward(dy, x, mean_rstd, scale_shift, gamma, u, ugamma_ubeta, per_sample, act, slope, need_gx,
                         need_gdy, need_ggamma):
    """Backward of norm_backward (act NONE / LRELU / RELU): (gx, gdy, ggamma per group), each None unless asked for.
    u: the gradient w.r.t. dx; ugamma_ubeta: [2][C] gradients w.r.t. dgamma, dbeta, or None (= 0)."""
    d = _norm_desc(x.shape, per_sample, 0.0, 0.0, act, slope, False)
    groups = mean_rstd.numel() // 2
    sums = zero_scratch(x.device, 5 * groups)
    gx = torch.empty_like(x, memory_format=CL) if need_gx else None
    gdy = torch.empty_like(x, memory_format=CL) if need_gdy else None
    gg = torch.empty(groups, device=x.device, dtype=torch.float32) if need_ggamma else None
    _lib.check(_lib.load().b200gan_norm_dbwd(ctypes.byref(d), dy.data_ptr(), x.data_ptr(), mean_rstd.data_ptr(),
                                             _ptr(scale_shift), _ptr(gamma), u.data_ptr(), _ptr(ugamma_ubeta),
                                             sums.data_ptr(), _ptr(gx), _ptr(gdy), _ptr(gg), _stream()), "norm_dbwd")
    return gx, gdy, gg


# ---- BatchNorm2d [act] [Upsample x2] Conv2d backward: the norm's sums from the conv's data-gradient epilogue ----------
def conv_dgrad_norm_supported(g):
    if Config.algo == "simt":
        return False
    return bool(_lib.load().b200gan_conv2d_dgrad_norm_supported(ctypes.byref(g)))


def conv_dgrad_norm(g, dy, packed, x, mean_rstd, scale_shift, act, slope):
    """(dx, sums): the conv's data gradient (tensor cores) and, from the same epilogue, the fp64 [2][C] sums the
    BatchNorm backward of its input x needs.  `sums` is a zero_scratch buffer for norm_backward_from_sums to consume."""
    d = _norm_desc(x.shape, False, 0.0, 0.0, act, slope, False)
    sums = zero_scratch(x.device, 2 * g.C)
    dx = empty_cl(g.N, g.C, g.H, g.W, dy.device)
    _lib.check(_lib.load().b200gan_conv2d_dgrad_norm(ctypes.byref(g), ctypes.byref(d), dy.data_ptr(), packed.data_ptr(),
                                                     x.data_ptr(), mean_rstd.data_ptr(), scale_shift.data_ptr(),
                                                     sums.data_ptr(), dx.data_ptr(), _stream()), "conv2d_dgrad_norm")
    return dx, sums


def norm_backward_from_sums(dy, x, mean_rstd, gamma, sums, eps, act=ACT_NONE, slope=0.0, need_params=False,
                            round_tf32=False, scale_shift=None):
    """norm_backward (batch statistics) given the sums conv_dgrad_norm produced; hands `sums` back zeroed."""
    d = _norm_desc(x.shape, False, eps, 0.0, act, slope, round_tf32)
    dx = torch.empty_like(x, memory_format=CL)
    dgb = torch.empty(sums.numel(), device=x.device, dtype=torch.float32) if need_params else None
    _lib.check(_lib.load().b200gan_norm_bwd_from_sums(ctypes.byref(d), dy.data_ptr(), x.data_ptr(), mean_rstd.data_ptr(),
                                                      _ptr(scale_shift), _ptr(gamma), sums.data_ptr(), dx.data_ptr(),
                                                      _ptr(dgb), _stream()), "norm_bwd_from_sums")
    return dx, dgb


# ---- shape ops ------------------------------------------------------------------------------------
def upsample2x(x):
    n, c, h, w = x.shape
    y = empty_cl(n, c, 2 * h, 2 * w, x.device)
    _lib.check(_lib.load().b200gan_upsample2x_fwd(x.data_ptr(), y.data_ptr(), n, h, w, c, _stream()), "upsample2x_fwd")
    return y


def upsample2x_bwd(dy):
    n, c, h2, w2 = dy.shape
    dx = empty_cl(n, c, h2 // 2, w2 // 2, dy.device)
    _lib.check(_lib.load().b200gan_upsample2x_bwd(dy.data_ptr(), dx.data_ptr(), n, h2 // 2, w2 // 2, c, _stream()),
               "upsample2x_bwd")
    return dx


def pad2d(x, pads, mode, round_tf32=False):
    n, c, h, w = x.shape
    t, l, b, r = pads
    y = empty_cl(n, c, h + t + b, w + l + r, x.device)
    _lib.check(_lib.load().b200gan_pad2d_fwd(x.data_ptr(), y.data_ptr(), n, h, w, c, t, l, b, r, mode, int(round_tf32),
                                             _stream()), "pad2d_fwd")
    return y


def pad2d_bwd(dy, pads, mode):
    n, c, ho, wo = dy.shape
    t, l, b, r = pads
    h, w = ho - t - b, wo - l - r
    dx = empty_cl(n, c, h, w, dy.device)
    _lib.check(_lib.load().b200gan_pad2d_bwd(dy.data_ptr(), dx.data_ptr(), n, h, w, c, t, l, b, r, mode, _stream()),
               "pad2d_bwd")
    return dx


def act_forward(x, act, slope, mask=None, mask_per_channel=False):
    n, c, h, w = x.shape
    y = torch.empty_like(x, memory_format=CL)
    _lib.check(_lib.load().b200gan_act_fwd(x.data_ptr(), _ptr(mask), int(mask_per_channel), act, slope, x.numel(), c,
                                           h * w, y.data_ptr(), _stream()), "act_fwd")
    return y


# ---- Discriminator conv blocks as a fused chain (csrc/narrow_block.cu) ------------------------------------------
class BnEdge:
    """A training-mode BatchNorm2d between two fused convs: its batch statistics (fp64 sums of the producer's output)
    and parameters.  `sums` is filled by the consumer's backward (sum g, sum g * ahat) for the producer's backward."""

    def __init__(self, stats, gamma, beta, eps, count, groups=1):
        """stats: [groups][2][C] fp64; count: elements per channel and group (see b200gan_nb_bn in include/b200gan.h)."""
        self.stats, self.gamma, self.beta, self.eps, self.count = stats, gamma, beta, float(eps), float(count)
        self.groups = int(groups)
        self.sums = None

    def c_struct(self):
        b = NbBn()
        b.stats, b.gamma, b.beta = self.stats.data_ptr(), _ptr(self.gamma), _ptr(self.beta)
        b.eps, b.count, b.groups, b.reserved = self.eps, self.count, self.groups, 0
        return b


class bn_groups:
    """`with ops.bn_groups(G):` -- the batch entering the drop-in modules is G equal runs of images that are to be treated
    as G separate forward passes of the reference sharing the weights: independent BatchNorm batch statistics (running
    statistics updated G times, in order), Dropout2d masks drawn in the order of G separate passes, parameter gradients
    summed.  Used by train.dcgan_step to run discriminator(real_imgs) and discriminator(gen_imgs.detach())
    (dcgan.py:178-179) as one launch per layer.  Only the fused chain honours it: every other normalisation /
    dropout module raises while it is active (train.py checks eligibility first)."""

    active = 1

    def __init__(self, groups):
        self.groups = int(groups)

    def __enter__(self):
        self.prev = bn_groups.active
        bn_groups.active = self.groups
        return self

    def __exit__(self, *exc):
        bn_groups.active = self.prev


def nb_supported(g):
    if not Config.fuse_narrow_chain:
        return False
    lib = _lib.load()
    if bn_groups.active > 1:
        return bool(lib.b200gan_nb_groups_supported(ctypes.byref(g), bn_groups.active))
    return bool(lib.b200gan_nb_supported(ctypes.byref(g)))


def _bn_ref(edge):
    return ctypes.byref(edge.c_struct()) if edge is not None else None


def nb_fprop(g, x, packed, bias, act, slope, chan_scale, in_edge, running_mean, running_var, nbt, momentum, want_stats,
             groups=1):
    y = empty_cl(g.N, g.K, g.P, g.Q, x.device)
    stats = torch.empty(groups * 2 * g.K, device=x.device, dtype=torch.float64) if want_stats else None
    _lib.check(_lib.load().b200gan_nb_fprop(ctypes.byref(g), _bn_ref(in_edge), _ptr(running_mean), _ptr(running_var),
                                            _ptr(nbt), float(momentum), x.data_ptr(), packed.data_ptr(), _ptr(bias),
                                            act, slope, _ptr(chan_scale), y.data_ptr(), _ptr(stats), int(groups),
                                            _stream()), "nb_fprop")
    return y, stats


def nb_dz(g_in, a, chan_scale, act, slope, out_edge, want_db):
    n, k, p, q = a.shape
    dz = torch.empty_like(a, memory_format=CL)
    db = torch.empty(k, device=a.device, dtype=torch.float32) if want_db else None
    sums = out_edge.sums if out_edge is not None else None
    _lib.check(_lib.load().b200gan_nb_dz(n, p * q, k, g_in.data_ptr(), a.data_ptr(), _ptr(chan_scale), act, slope,
                                         _bn_ref(out_edge), _ptr(sums), dz.data_ptr(), _ptr(db), _stream()), "nb_dz")
    return dz, db


def nb_wgrad(g, x, dz, in_edge, weight_shape):
    dw = torch.empty(weight_shape, device=x.device, dtype=torch.float32)
    lib = _lib.load()
    nws = int(lib.b200gan_nb_wgrad_workspace_floats(ctypes.byref(g)))
    ws = torch.empty(nws, device=x.device, dtype=torch.float32) if nws else None
    _lib.check(lib.b200gan_nb_wgrad(ctypes.byref(g), _bn_ref(in_edge), x.data_ptr(), dz.data_ptr(), dw.data_ptr(), _ptr(ws),
                                    _stream()), "nb_wgrad")
    return dw


def nb_dgrad(g, dz, packed, in_edge, a_prev):
    gout = empty_cl(g.N, g.C, g.H, g.W, dz.device)
    sums = (torch.empty(in_edge.groups * 2 * g.C, device=dz.device, dtype=torch.float64)
            if in_edge is not None else None)
    _lib.check(_lib.load().b200gan_nb_dgrad(ctypes.byref(g), dz.data_ptr(), packed.data_ptr(), _bn_ref(in_edge),
                                            _ptr(a_prev) if in_edge is not None else 0, gout.data_ptr(), _ptr(sums),
                                            _stream()), "nb_dgrad")
    return gout, sums


def nb_tail_fwd(a, edge, running_mean, running_var, nbt, momentum, nchw):
    n, c, h, w = a.shape
    if nchw:
        out = torch.empty((n, c, h, w), device=a.device, dtype=torch.float32)
    else:
        out = torch.empty_like(a, memory_format=CL)
    _lib.check(_lib.load().b200gan_nb_tail_fwd(n, h * w, c, _bn_ref(edge), _ptr(running_mean), _ptr(running_var), _ptr(nbt),
                                               float(momentum), a.data_ptr(), out.data_ptr(), int(nchw), _stream()),
               "nb_tail_fwd")
    return out


def nb_tail_bwd(a, edge, dout, nchw):
    n, c, h, w = a.shape
    g = torch.empty_like(a, memory_format=CL)
    sums = torch.empty(edge.groups * 2 * c, device=a.device, dtype=torch.float64)
    _lib.check(_lib.load().b200gan_nb_tail_bwd(n, h * w, c, _bn_ref(edge), a.data_ptr(), dout.data_ptr(), int(nchw),
                                               g.data_ptr(), sums.data_ptr(), _stream()), "nb_tail_bwd")
    return g, sums


# ---- Discriminator head / adversarial loss (csrc/head.cu) ----------------------------------------------------
def linear1_fwd(x, w, b, act):
    n, k = x.shape
    y = torch.empty((n, 1), device=x.device, dtype=torch.float32)
    _lib.check(_lib.load().b200gan_linear1_fwd(x.data_ptr(), w.data_ptr(), _ptr(b), y.data_ptr(), n, k, act, _stream()),
               "linear1_fwd")
    return y


def linear1_bwd(x, w, y, dy, act, need_dx, need_db):
    n, k = x.shape
    dx = torch.empty_like(x) if need_dx else None
    dw = torch.empty((1, k), device=x.device, dtype=torch.float32)
    db = torch.empty(1, device=x.device, dtype=torch.float32) if need_db else None
    _lib.check(_lib.load().b200gan_linear1_bwd(x.data_ptr(), w.data_ptr(), y.data_ptr(), dy.data_ptr(), _ptr(dx),
                                               dw.data_ptr(), _ptr(db), n, k, act, _stream()), "linear1_bwd")
    return dx, dw, db


def bce_fwd(v, t):
    loss = torch.empty((), device=v.device, dtype=torch.float32)
    _lib.check(_lib.load().b200gan_bce_fwd(v.data_ptr(), t.data_ptr(), loss.data_ptr(), v.numel(), _stream()), "bce_fwd")
    return loss


def bce_bwd(v, t, gout):
    dv = torch.empty_like(v)
    _lib.check(_lib.load().b200gan_bce_bwd(v.data_ptr(), t.data_ptr(), gout.data_ptr(), dv.data_ptr(), v.numel(),
                                           _stream()), "bce_bwd")
    return dv


# ---- Auxiliary-classifier head and its loss: Linear(K, n) + Softmax, CrossEntropyLoss (csrc/head.cu) -------------------
def class_head_fwd(x, w, b):
    """softmax(x w^T + b) over the n = w.shape[0] outputs (2 <= n <= 32) of a contiguous [N, K] x; one launch."""
    n, k = x.shape
    y = torch.empty((n, w.shape[0]), device=x.device, dtype=torch.float32)
    _lib.check(_lib.load().b200gan_class_head_fwd(x.data_ptr(), w.data_ptr(), _ptr(b), y.data_ptr(), n, k, w.shape[0],
                                                  _stream()), "class_head_fwd")
    return y


def class_head_bwd(x, w, y, dy, need_dx, need_db):
    """(dx or None, dw, db or None) from the saved softmax output y and dy, both [N, n]; one launch."""
    n, k = x.shape
    nout = w.shape[0]
    dx = torch.empty_like(x) if need_dx else None
    dw = torch.empty((nout, k), device=x.device, dtype=torch.float32)
    db = torch.empty(nout, device=x.device, dtype=torch.float32) if need_db else None
    _lib.check(_lib.load().b200gan_class_head_bwd(x.data_ptr(), w.data_ptr(), y.data_ptr(), dy.data_ptr(), _ptr(dx),
                                                  dw.data_ptr(), _ptr(db), n, k, nout, _stream()), "class_head_bwd")
    return dx, dw, db


def cross_entropy_fwd(x, target, ignore_index):
    """[loss, count] (fp32, on the device) of CrossEntropyLoss(reduction='mean') of contiguous [N, C] logits and int64
    class indices [N]; one launch.  out[0] is the loss; the backward reads out[1]."""
    n, c = x.shape
    out = torch.empty(2, device=x.device, dtype=torch.float32)
    _lib.check(_lib.load().b200gan_cross_entropy_fwd(x.data_ptr(), target.data_ptr(), out.data_ptr(), n, c,
                                                     int(ignore_index), _stream()), "cross_entropy_fwd")
    return out


def cross_entropy_bwd(x, target, out, gout, ignore_index):
    """d loss / d x for the upstream gradient gout (0-dim, read on the device); one launch."""
    n, c = x.shape
    dx = torch.empty_like(x)
    _lib.check(_lib.load().b200gan_cross_entropy_bwd(x.data_ptr(), target.data_ptr(), out.data_ptr(), gout.data_ptr(),
                                                     dx.data_ptr(), n, c, int(ignore_index), _stream()),
               "cross_entropy_bwd")
    return dx


# ---- MSELoss / L1Loss, reduction 'mean' (csrc/pixel_loss/) --------------------------------------------------------------
def pixel_layout(t):
    """_lib.LAYOUT_NCHW for a contiguous tensor, LAYOUT_NHWC for a 4-D channels_last one, else None (not dense in either
    layout: a strided view, an expanded tensor)."""
    if t.is_contiguous():
        return _lib.LAYOUT_NCHW
    if t.dim() == 4 and t.is_contiguous(memory_format=CL):
        return _lib.LAYOUT_NHWC
    return None


def pixel_loss_desc(a, b, mode):
    """The kernel's description of loss(a, b): one shape of at most 4 dimensions (padded with leading 1s), 0 < n < 2^31,
    each operand in its own layout.  None if the pair is not one the kernels take."""
    if a.shape != b.shape or a.dim() > 4 or not 0 < a.numel() < 2 ** 31:
        return None
    la, lb = pixel_layout(a), pixel_layout(b)
    if la is None or lb is None:
        return None
    d = PixelLossDesc()
    d.mode, d.layout_a, d.layout_b, d.n = mode, la, lb, a.numel()
    d.N, d.C, d.H, d.W = (1,) * (4 - a.dim()) + tuple(a.shape)
    return d


_pixel_ws = {}


def _pixel_loss_workspace(device, nbytes):
    """The forward's workspace, zeroed once per device: every call leaves its completion ticket at zero again, so no
    fill kernel runs per loss.  One buffer per device suffices because loss calls never interleave on the stream."""
    t = _pixel_ws.get(device)
    if t is None or t.numel() < nbytes:
        t = torch.zeros(max(nbytes, 16 + 8 * 1024), device=device, dtype=torch.uint8)
        _pixel_ws[device] = t
    return t


def _pixel_loss_check(a, b, mode):
    _require_cuda(a, "loss input")
    _require_cuda(b, "loss target")
    d = pixel_loss_desc(a, b, mode)
    if d is None:
        raise RuntimeError(f"b200gan: pixel loss of {tuple(a.shape)} / {tuple(b.shape)} tensors: one shape of at most 4 "
                           "dimensions, each NCHW- or channels_last-contiguous, is required")
    return d


def pixel_loss_fwd(a, b, mode):
    """mean((a - b)^2) (mode PIXEL_LOSS_MSE) or mean(|a - b|) (PIXEL_LOSS_L1) as a 0-dim fp32 tensor; one launch."""
    d = _pixel_loss_check(a, b, mode)
    lib = _lib.load()
    ws = _pixel_loss_workspace(a.device, lib.b200gan_pixel_loss_workspace_bytes(ctypes.byref(d)))
    loss = torch.empty((), device=a.device, dtype=torch.float32)
    _lib.check(lib.b200gan_pixel_loss_fwd(ctypes.byref(d), a.data_ptr(), b.data_ptr(), loss.data_ptr(), ws.data_ptr(),
                                          _stream()), "pixel_loss_fwd")
    return loss


def pixel_loss_bwd(a, b, gout, mode, need_db):
    """(da, db) for the upstream gradient gout (0-dim, read on the device): da in a's layout, db = -da in b's layout or
    None; one launch."""
    d = _pixel_loss_check(a, b, mode)
    da = torch.empty_like(a)
    db = torch.empty_like(b) if need_db else None
    _lib.check(_lib.load().b200gan_pixel_loss_bwd(ctypes.byref(d), a.data_ptr(), b.data_ptr(), gout.data_ptr(),
                                                  da.data_ptr(), _ptr(db), _stream()), "pixel_loss_bwd")
    return da, db


# ---- MLP critic under autograd: Linear -> LeakyReLU -> Linear -> LeakyReLU -> Linear(-> 1) (csrc/mlp_critic.cu) ------
def _mlp_critic_desc(x, w1, w2, w3, slope):
    if x.dim() != 2 or w1.dim() != 2 or w2.dim() != 2:
        raise RuntimeError("b200gan mlp_critic: x, W1 and W2 must be matrices")
    d = MlpCriticDesc()
    d.N, d.Din, d.H1, d.H2, d.slope = x.shape[0], x.shape[1], w1.shape[0], w2.shape[0], float(slope)
    if w1.shape[1] != d.Din or w2.shape[1] != d.H1 or w3.numel() != d.H2 or min(d.N, d.Din, d.H1, d.H2) < 1:
        raise RuntimeError(f"b200gan mlp_critic: shapes do not chain: x {tuple(x.shape)}, W1 {tuple(w1.shape)}, "
                           f"W2 {tuple(w2.shape)}, W3 {tuple(w3.shape)}")
    return d


def _f32(name, *ts):
    for t_ in ts:
        if t_ is not None:
            _require_cuda(t_, name)
    return [None if t_ is None else t_.contiguous() for t_ in ts]


def mlp_critic_fwd(x, w1, b1, w2, b2, w3, b3, slope):
    """D(x) in one launch.  Returns (out [N, 1], m1, a1, m2, a2): the LeakyReLU masks and activations of both hidden
    layers, which the two backward passes read (see b200gan_mlp_critic_fwd in include/b200gan.h)."""
    x, w1, b1, w2, b2, w3, b3 = _f32("mlp_critic operand", x, w1, b1, w2, b2, w3, b3)
    d = _mlp_critic_desc(x, w1, w2, w3, slope)
    if b1.numel() != d.H1 or b2.numel() != d.H2 or b3.numel() != 1:
        raise RuntimeError("b200gan mlp_critic: bias sizes do not match the layers")
    dev, n = x.device, d.N
    out = torch.empty((n, 1), device=dev, dtype=torch.float32)
    m1, a1 = (torch.empty((n, d.H1), device=dev, dtype=torch.float32) for _ in range(2))
    m2, a2 = (torch.empty((n, d.H2), device=dev, dtype=torch.float32) for _ in range(2))
    _lib.check(_lib.load().b200gan_mlp_critic_fwd(ctypes.byref(d), x.data_ptr(), w1.data_ptr(), b1.data_ptr(),
                                                  w2.data_ptr(), b2.data_ptr(), w3.data_ptr(), b3.data_ptr(),
                                                  out.data_ptr(), m1.data_ptr(), a1.data_ptr(), m2.data_ptr(),
                                                  a2.data_ptr(), _stream()), "mlp_critic_fwd")
    return out, m1, a1, m2, a2


def mlp_critic_bwd(dout, x, w1, w2, w3, m1, a1, m2, a2, need, keep_u=False):
    """First-order backward for the output gradient dout [N, 1].  need: 7 flags for the gradients of
    (x, W1, b1, W2, b2, W3, b3); the others come back as None.  Returns (dx, dW1, db1, dW2, db2, dW3, db3, U1, U2), with
    U1 [N, H1] and U2 [N, H2] (the double backward's operands) only when keep_u."""
    dout, x, w1, w2, w3, m1, a1, m2, a2 = _f32("mlp_critic operand", dout, x, w1, w2, w3, m1, a1, m2, a2)
    d = _mlp_critic_desc(x, w1, w2, w3, 0.0)  # the masks carry the slope
    if dout.numel() != d.N or m1.shape != (d.N, d.H1) or m2.shape != (d.N, d.H2):
        raise RuntimeError("b200gan mlp_critic_bwd: dout / saved activations do not match the layers")
    lib, dev, f32 = _lib.load(), x.device, torch.float32
    shapes = ((d.N, d.Din), tuple(w1.shape), (d.H1,), tuple(w2.shape), (d.H2,), tuple(w3.shape), (1,))
    grads = [torch.empty(s_, device=dev, dtype=f32) if nd else None for s_, nd in zip(shapes, need)]
    u1 = torch.empty((d.N, d.H1), device=dev, dtype=f32) if keep_u else None
    u2 = torch.empty((d.N, d.H2), device=dev, dtype=f32) if keep_u else None
    ws = None if keep_u else torch.empty(lib.b200gan_mlp_critic_bwd_workspace_floats(ctypes.byref(d)), device=dev,
                                         dtype=f32)
    _lib.check(lib.b200gan_mlp_critic_bwd(ctypes.byref(d), dout.data_ptr(), x.data_ptr(), w1.data_ptr(), w2.data_ptr(),
                                          w3.data_ptr(), m1.data_ptr(), a1.data_ptr(), m2.data_ptr(), a2.data_ptr(),
                                          *[_ptr(g) for g in grads], _ptr(u1), _ptr(u2), _ptr(ws), _stream()),
               "mlp_critic_bwd")
    return (*grads, u1, u2)


def mlp_critic_dbwd(u, dout, u1, u2, m1, m2, w1, w2, w3, need):
    """Double backward of the input gradient dx = U1 W1 for the gradient u [N, Din] arriving at dx.  need: 4 flags for
    the gradients of (dout, W1, W2, W3).  Returns (ddout [N, 1], dW1, dW2, dW3), None where not needed; the gradients
    w.r.t. x and the biases are exactly zero."""
    u, dout, u1, u2, m1, m2, w1, w2, w3 = _f32("mlp_critic operand", u, dout, u1, u2, m1, m2, w1, w2, w3)
    d = _mlp_critic_desc(u, w1, w2, w3, 0.0)
    if dout.numel() != d.N or u1.shape != (d.N, d.H1) or u2.shape != (d.N, d.H2):
        raise RuntimeError("b200gan mlp_critic_dbwd: operands do not match the layers")
    lib, dev, f32 = _lib.load(), u.device, torch.float32
    shapes = ((d.N, 1), tuple(w1.shape), tuple(w2.shape), tuple(w3.shape))
    ddout, dw1, dw2, dw3 = [torch.empty(s_, device=dev, dtype=f32) if nd else None for s_, nd in zip(shapes, need)]
    ws = torch.empty(lib.b200gan_mlp_critic_dbwd_workspace_floats(ctypes.byref(d)), device=dev, dtype=f32)
    _lib.check(lib.b200gan_mlp_critic_dbwd(ctypes.byref(d), u.data_ptr(), dout.data_ptr(), u1.data_ptr(), u2.data_ptr(),
                                           m1.data_ptr(), m2.data_ptr(), w1.data_ptr(), w2.data_ptr(), w3.data_ptr(),
                                           _ptr(dw1), _ptr(dw2), _ptr(dw3), _ptr(ddout), ws.data_ptr(), _stream()),
               "mlp_critic_dbwd")
    return ddout, dw1, dw2, dw3


def mlp_disc_fwd(x, w1, b1, w2, b2, w3, b3, slope):
    """sigmoid(D(x)), the vanilla GAN discriminator, in one launch.  Returns (y [N, 1], m1, a1, m2, a2) as
    mlp_critic_fwd does (see b200gan_mlp_disc_fwd in include/b200gan.h)."""
    x, w1, b1, w2, b2, w3, b3 = _f32("mlp_disc operand", x, w1, b1, w2, b2, w3, b3)
    d = _mlp_critic_desc(x, w1, w2, w3, slope)
    if b1.numel() != d.H1 or b2.numel() != d.H2 or b3.numel() != 1:
        raise RuntimeError("b200gan mlp_disc: bias sizes do not match the layers")
    dev, n = x.device, d.N
    y = torch.empty((n, 1), device=dev, dtype=torch.float32)
    m1, a1 = (torch.empty((n, d.H1), device=dev, dtype=torch.float32) for _ in range(2))
    m2, a2 = (torch.empty((n, d.H2), device=dev, dtype=torch.float32) for _ in range(2))
    _lib.check(_lib.load().b200gan_mlp_disc_fwd(ctypes.byref(d), x.data_ptr(), w1.data_ptr(), b1.data_ptr(),
                                                w2.data_ptr(), b2.data_ptr(), w3.data_ptr(), b3.data_ptr(), y.data_ptr(),
                                                m1.data_ptr(), a1.data_ptr(), m2.data_ptr(), a2.data_ptr(), _stream()),
               "mlp_disc_fwd")
    return y, m1, a1, m2, a2


def mlp_disc_bwd(dout, y, x, w1, w2, w3, m1, a1, m2, a2, need):
    """Backward of mlp_disc_fwd for the output gradient dout [N, 1], y its output.  need: 7 flags for the gradients of
    (x, W1, b1, W2, b2, W3, b3); the others come back as None."""
    dout, y, x, w1, w2, w3, m1, a1, m2, a2 = _f32("mlp_disc operand", dout, y, x, w1, w2, w3, m1, a1, m2, a2)
    d = _mlp_critic_desc(x, w1, w2, w3, 0.0)  # the masks carry the slope
    if dout.numel() != d.N or y.numel() != d.N or m1.shape != (d.N, d.H1) or m2.shape != (d.N, d.H2):
        raise RuntimeError("b200gan mlp_disc_bwd: dout / saved activations do not match the layers")
    lib, dev, f32 = _lib.load(), x.device, torch.float32
    shapes = ((d.N, d.Din), tuple(w1.shape), (d.H1,), tuple(w2.shape), (d.H2,), tuple(w3.shape), (1,))
    grads = [torch.empty(s_, device=dev, dtype=f32) if nd else None for s_, nd in zip(shapes, need)]
    ws = torch.empty(lib.b200gan_mlp_disc_bwd_workspace_floats(ctypes.byref(d)), device=dev, dtype=f32)
    _lib.check(lib.b200gan_mlp_disc_bwd(ctypes.byref(d), dout.data_ptr(), y.data_ptr(), x.data_ptr(), w1.data_ptr(),
                                        w2.data_ptr(), w3.data_ptr(), m1.data_ptr(), a1.data_ptr(), m2.data_ptr(),
                                        a2.data_ptr(), *[_ptr(g) for g in grads], ws.data_ptr(), _stream()),
               "mlp_disc_bwd")
    return tuple(grads)


def critic_step_mlp(real, fake, alpha, w1, b1, w2, b2, w3, b3, slope, lambda_gp):
    """wgan_gp.py:164-173 for the MLP critic in one kernel.  Returns (losses[2], dW1, db1, dW2, db2, dW3, db3)."""
    real, fake, alpha, w1, b1, w2, b2, w3, b3 = _f32("critic_step operand", real, fake, alpha, w1, b1, w2, b2, w3, b3)
    n = real.shape[0]
    real, fake, alpha = real.view(n, -1), fake.view(n, -1), alpha.view(-1)
    d = _mlp_critic_desc(real, w1, w2, w3, slope)
    if fake.shape != real.shape or alpha.numel() != n or b1.numel() != d.H1 or b2.numel() != d.H2 or b3.numel() != 1:
        raise RuntimeError("b200gan critic_step_mlp: fake, alpha or the biases do not match real and the layers")
    lib, dev = _lib.load(), real.device
    ws = torch.empty(lib.b200gan_critic_step_workspace_floats(ctypes.byref(d)), device=dev, dtype=torch.float32)
    losses = torch.empty(2, device=dev, dtype=torch.float32)
    grads = [torch.empty_like(t_) for t_ in (w1, b1, w2, b2, w3, b3)]
    _lib.check(lib.b200gan_critic_step_mlp(ctypes.byref(d), float(lambda_gp), real.data_ptr(), fake.data_ptr(),
                                           alpha.data_ptr(), w1.data_ptr(), b1.data_ptr(), w2.data_ptr(), b2.data_ptr(),
                                           w3.data_ptr(), b3.data_ptr(), losses.data_ptr(),
                                           *[g.data_ptr() for g in grads], ws.data_ptr(), _stream()), "critic_step_mlp")
    return (losses, *grads)


# ---- MLP generator: [Linear -> (BatchNorm1d)? -> LeakyReLU] x (L - 1), Linear -> Tanh (csrc/mlp_generator) ----------
def _mlp_gen_desc(z, layers, slope, eps, momentum):
    """layers: [(W, b, norm)] with norm = (gamma, beta, running_mean, running_var, num_batches_tracked) or None; the
    running statistics may be None (not tracked)."""
    if z.dim() != 2 or not 1 <= len(layers) <= _lib.MLP_GEN_MAX_LAYERS:
        raise RuntimeError(f"b200gan mlp_gen: z must be a matrix and 1 <= layers <= {_lib.MLP_GEN_MAX_LAYERS}")
    d = MlpGenDesc()
    d.L, d.N = len(layers), z.shape[0]
    d.width[0] = z.shape[1]
    d.slope, d.eps, d.momentum = float(slope), float(eps), float(momentum)
    for l, (w, b, norm) in enumerate(layers):
        if w.dim() != 2 or w.shape[1] != d.width[l] or (b is not None and b.numel() != w.shape[0]):
            raise RuntimeError(f"b200gan mlp_gen: layer {l}: W {tuple(w.shape)} does not chain from width {d.width[l]}")
        d.width[l + 1] = w.shape[0]
        d.W[l], d.b[l] = w.data_ptr(), _ptr(b)
        if norm is not None:
            d.has_norm[l] = 1
            for name, t_ in zip(("gamma", "beta", "running_mean", "running_var", "num_batches_tracked"), norm):
                getattr(d, name)[l] = _ptr(t_)
    return d


def mlp_gen_fwd(z, layers, slope, eps, momentum, keep):
    """The generator's forward in one launch; updates the running statistics in place.  Returns (out [N, width[L]],
    saved): saved is what mlp_gen_bwd reads (see b200gan_mlp_gen_saved_floats in include/b200gan.h) when keep, else
    None."""
    z = _f32("mlp_gen operand", z)[0]
    layers = [(*_f32("mlp_gen operand", w, b), None if n is None else (*_f32("mlp_gen operand", *n[:4]), n[4]))
              for w, b, n in layers]
    d = _mlp_gen_desc(z, layers, slope, eps, momentum)
    lib, dev = _lib.load(), z.device
    out = torch.empty((d.N, d.width[d.L]), device=dev, dtype=torch.float32)
    saved = torch.empty(lib.b200gan_mlp_gen_saved_floats(ctypes.byref(d)), device=dev, dtype=torch.float32) if keep \
        else None
    ws = torch.empty(lib.b200gan_mlp_gen_workspace_floats(ctypes.byref(d)), device=dev, dtype=torch.float32)
    _lib.check(lib.b200gan_mlp_gen_fwd(ctypes.byref(d), z.data_ptr(), out.data_ptr(), _ptr(saved), ws.data_ptr(),
                                       _stream()), "mlp_gen_fwd")
    return out, saved


def mlp_gen_bwd(dout, z, out, saved, layers, slope, eps, momentum, need_dz, need):
    """Backward of mlp_gen_fwd for the output gradient dout.  need: per layer 4 flags for (dW, db, dgamma, dbeta).
    Returns (dz or None, [(dW, db, dgamma, dbeta)] with None where not needed or where the layer has no norm)."""
    dout, z, out = _f32("mlp_gen operand", dout, z, out)
    layers = [(*_f32("mlp_gen operand", w), None, None if n is None else (*_f32("mlp_gen operand", *n[:2]),
                                                                          None, None, None))
              for w, _, n in layers]
    d = _mlp_gen_desc(z, layers, slope, eps, momentum)
    if dout.shape != (d.N, d.width[d.L]) or out.shape != dout.shape:
        raise RuntimeError("b200gan mlp_gen_bwd: dout / out do not match the layers")
    lib, dev, f32 = _lib.load(), z.device, torch.float32
    gr = MlpGenGrads()
    grads = []
    for l, ((w, _, norm), flags) in enumerate(zip(layers, need)):
        shapes = (tuple(w.shape), (w.shape[0],), (w.shape[0],), (w.shape[0],))
        row = [torch.empty(s_, device=dev, dtype=f32) if f and (k < 2 or norm is not None) else None
               for k, (s_, f) in enumerate(zip(shapes, flags))]
        for name, t_ in zip(("dW", "db", "dgamma", "dbeta"), row):
            getattr(gr, name)[l] = _ptr(t_)
        grads.append(tuple(row))
    dz = torch.empty_like(z) if need_dz else None
    ws = torch.empty(lib.b200gan_mlp_gen_workspace_floats(ctypes.byref(d)), device=dev, dtype=f32)
    _lib.check(lib.b200gan_mlp_gen_bwd(ctypes.byref(d), dout.data_ptr(), z.data_ptr(), out.data_ptr(), _ptr(saved),
                                       _ptr(dz), ctypes.byref(gr), ws.data_ptr(), _stream()), "mlp_gen_bwd")
    return dz, grads
