"""Autograd nodes of the b200gan hot path.  Every forward/backward here is one or more calls into
libb200gan.so; torch only provides the tensors and the autograd tape.

Reference behaviour mirrored (file:line under implementations/):
  conv blocks        dcgan/dcgan.py:52-64, 77-88   pix2pix/models.py:20-52   cyclegan/models.py:22-87
  training-mode BN   dcgan/dcgan.py:53,56,60,80 (eps = 0.8)    InstanceNorm  pix2pix/models.py:25,40
"""
import weakref
from dataclasses import dataclass
from typing import Optional, Tuple

import torch

from . import ops
from ._lib import ConvGeom
from ._lib import (ACT_LRELU, ACT_NONE, ACT_RELU, ACT_SIGMOID, ACT_TANH, ALGO_SIMT,  # noqa: F401 (re-exported)
                   PACK_SIMT_DGRAD, PACK_SIMT_FPROP, PAD_ZERO, PIXEL_LOSS_MSE)


@dataclass(frozen=True)
class ConvSpec:
    stride: int = 1
    pads: Tuple[int, int, int, int] = (0, 0, 0, 0)  # top, left, bottom, right of the virtual input
    pad_mode: int = PAD_ZERO
    up: int = 1
    transposed: bool = False
    act: int = ACT_NONE
    slope: float = 0.0
    stats: Optional[bool] = None  # None: no fused statistics; False: per channel (BN); True: per sample (IN)
    rtf_out: bool = False         # round the output to TF32 (it feeds a wgmma conv)
    rtf_dz: bool = False          # round the epilogue-backward output (feeds wgmma dgrad/wgrad)


@dataclass(frozen=True)
class NormSpec:
    per_sample: bool = False
    eps: float = 1e-5
    momentum: float = 0.1
    act: int = ACT_NONE
    slope: float = 0.0
    rtf_out: bool = False
    rtf_dx: bool = False


class PackCache:
    """Derived packed copies of one weight Parameter, invalidated by the tensor version counter.  Caches register
    themselves per parameter so that an optimizer can refresh every packed copy of its weights in ONE launch right
    after the update (refresh_packs) instead of one pack launch per copy at the next forward."""

    registry = weakref.WeakValueDictionary()  # id(parameter storage) -> PackCache

    def __init__(self):
        self._d = {}

    def get(self, g, w, kind):
        key = (kind, g.C, g.K, g.R, g.S, g.transposed)
        ver = (w._version, w.data_ptr())
        hit = self._d.get(key)
        if ops.Config.weight_cache and hit is not None and hit[0] == ver:
            return hit[1]
        if hit is not None and hit[1].device == w.device:
            packed = hit[1]          # same buffer: a CUDA graph that captured it stays valid
            ops.pack_weights(g, w, kind, out=packed)
        else:
            packed = ops.pack_weights(g, w, kind)
        g_copy = ConvGeom.from_buffer_copy(g)
        self._d[key] = (ver, packed, g_copy)
        PackCache.registry[w.data_ptr()] = self
        return packed

    def jobs(self, w):
        """(geometry, kind, packed buffer) of every live copy, for ops.pack_weights_multi."""
        return [(e[2], key[0], e[1]) for key, e in self._d.items() if e[1].device == w.device]

    def mark_fresh(self, w):
        ver = (w._version, w.data_ptr())
        for key, e in list(self._d.items()):
            self._d[key] = (ver, e[1], e[2])


def refresh_packs(params):
    """Re-pack, in one launch, every cached packed copy of the given (just updated) weight tensors."""
    jobs, touched = [], []
    for w in params:
        cache = PackCache.registry.get(w.data_ptr())
        if cache is None:
            continue
        js = cache.jobs(w)
        if js:
            jobs.extend((g, kind, w, packed) for g, kind, packed in js)
            touched.append((cache, w))
    if jobs:
        ops.pack_weights_multi(jobs)
        for cache, w in touched:
            cache.mark_fresh(w)


def _as_cl(t):
    return t if ops.is_cl(t) else ops.to_cl(t)


def _conv_forward(x, weight, bias, chan_scale, spec: ConvSpec, cache: PackCache):
    """(geometry, output, fused statistics or None) of the conv block `spec` on the channels_last input x"""
    g, _ = ops.make_geom(tuple(x.shape), tuple(weight.shape), spec.stride, spec.pads, spec.pad_mode, spec.up,
                         spec.transposed)
    algo, kind = ops.conv_plan(g, 0, chan_scale)
    packed = cache.get(g, weight.detach(), kind)
    stats = None
    if spec.stats is not None:
        stats = ops.zero_scratch(x.device, 2 * (g.N * g.K if spec.stats else g.K))
    y = ops.conv_fprop(g, x, packed, algo, bias=None if bias is None else bias.detach(), act=spec.act,
                       slope=spec.slope, chan_scale=chan_scale, stats=stats, stats_per_sample=bool(spec.stats),
                       round_tf32=spec.rtf_out)
    return g, y, stats


def _with_stats(ctx, y, stats):
    """The outputs of a node whose conv may also produce the statistics of the norm after it"""
    if stats is None:
        return y
    ctx.mark_non_differentiable(stats)
    ctx.set_materialize_grads(False)  # no zero-filled gradient is launched for the statistics output
    return y, stats


def _conv_dz(dy, y, chan_scale, spec: ConvSpec):
    """The gradient w.r.t. the conv's raw output: the backward of its fused activation and Dropout2d scale"""
    if spec.act != ACT_NONE or chan_scale is not None:
        return ops.epilogue_bwd(dy, y, chan_scale, spec.act, spec.slope, spec.rtf_dz)
    return dy


def _conv_param_grads(g, x, dz, dy, y, chan_scale, spec: ConvSpec, wshape, need_dw, need_db):
    """(dw, db) of a conv block from dz = _conv_dz(dy, ...); the bias gradient comes out of the weight-gradient kernel"""
    db = None
    if need_db and dz is not dy and spec.rtf_dz:
        # dz was rounded to TF32 for the tensor-core passes; a bias gradient is a sum with heavy cancellation
        # and must come from the unrounded values
        db = ops.bias_grad(dy, y, chan_scale, spec.act, spec.slope)
        need_db = False
    dw = None
    if need_dw or need_db:
        dw, db2 = ops.conv_wgrad(g, x, dz, wshape, need_db, ops.conv_plan(g, 2)[0])
        db = db2 if need_db else db
        if not need_dw:
            dw = None
    return dw, db


class ConvFn(torch.autograd.Function):
    """[Upsample x2] [pad] Conv2d/ConvTranspose2d [+bias] [act] [* Dropout2d scale] (+ BN/IN partial sums)."""

    @staticmethod
    def forward(ctx, x, weight, bias, chan_scale, spec: ConvSpec, cache: PackCache):
        ops._require_cuda(x, "conv input")
        ops._require_cuda(weight, "conv weight")
        x = _as_cl(x)
        g, y, stats = _conv_forward(x, weight, bias, chan_scale, spec, cache)
        ctx.spec, ctx.cache, ctx.g = spec, cache, g
        ctx.has_bias = bias is not None
        need_y = spec.act != ACT_NONE
        ctx.save_for_backward(x, weight, y if need_y else None, chan_scale)
        return _with_stats(ctx, y, stats)

    @staticmethod
    def backward(ctx, dy, *unused):
        x, weight, y, chan_scale = ctx.saved_tensors
        spec, g, nig = ctx.spec, ctx.g, ctx.needs_input_grad
        if torch.is_grad_enabled():
            # autograd.grad(..., create_graph=True): the gradient penalty of a conv critic (stargan.py:142-161,
            # dragan.py:144-167) differentiates THROUGH this backward -- build it from differentiable nodes
            dx, dw, db, _, _ = _conv_backward_differentiable(dy, x, weight, y, chan_scale, spec.act, spec.slope, g,
                                                             nig[0], nig[1], ctx.has_bias and nig[2])
            return dx, dw, db, None, None, None
        dy = _as_cl(dy)
        dz = _conv_dz(dy, y, chan_scale, spec)
        dx = None
        if nig[0]:
            algo, kind = ops.conv_plan(g, 1)
            dx = ops.conv_dgrad(g, dz, ctx.cache.get(g, weight.detach(), kind), algo)
        dw, db = _conv_param_grads(g, x, dz, dy, y, chan_scale, spec, tuple(weight.shape), nig[1],
                                   ctx.has_bias and nig[2])
        return dx, dw, db, None, None, None


# ---- double backward through convolutions (SURVEY.md 8f N2: conv-critic gradient penalties) ---------------------------
# conv is bilinear in (x, w): the backward of its backward needs no new kernels.  With F = fprop(x, w):
#   D = dgrad(dz, w)  (= dF/dx applied to dz):   dD/d(dz) applied to u = fprop(u, w),   dD/dw applied to u = wgrad(u, dz)
#   W = wgrad(x, dz)  (= dF/dw applied to dz):   dW/dx applied to v  = dgrad(dz, v),    dW/d(dz) applied to v = fprop(x, v)
# simt=True: the fp32 SIMT kernels whatever the geometry -- the double backward of a fused chain with BatchNorm2d, whose
# own kernels are fp32 (csrc/narrow_block.cu); a norm-free chain keeps the routing of ConvFn
def _plain_fprop(g, x, w, simt=False):
    algo, kind = (ALGO_SIMT, PACK_SIMT_FPROP) if simt else ops.conv_plan(g, 0)
    return ops.conv_fprop(g, x, ops.pack_weights(g, w, kind), algo)


def _plain_dgrad(g, dz, w, simt=False):
    algo, kind = (ALGO_SIMT, PACK_SIMT_DGRAD) if simt else ops.conv_plan(g, 1)
    return ops.conv_dgrad(g, dz, ops.pack_weights(g, w, kind), algo)


def _plain_wgrad(g, x, dz, wshape, simt=False):
    return ops.conv_wgrad(g, x, dz, wshape, False, ALGO_SIMT if simt else ops.conv_plan(g, 2)[0])[0]


class ConvDgradFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, dz, weight, g, simt=False):
        ctx.g, ctx.simt = g, simt
        ctx.save_for_backward(dz, weight)
        return _plain_dgrad(g, _as_cl(dz.detach()), weight.detach(), simt)

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, u):
        dz, weight = ctx.saved_tensors
        g, u, simt = ctx.g, _as_cl(u), ctx.simt
        ddz = _plain_fprop(g, u, weight.detach(), simt) if ctx.needs_input_grad[0] else None
        dw = _plain_wgrad(g, u, _as_cl(dz.detach()), tuple(weight.shape), simt) if ctx.needs_input_grad[1] else None
        return ddz, dw, None, None


class ConvWgradFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, dz, g, wshape, simt=False):
        ctx.g, ctx.simt = g, simt
        ctx.save_for_backward(x, dz)
        return _plain_wgrad(g, _as_cl(x.detach()), _as_cl(dz.detach()), wshape, simt)

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, v):
        x, dz = ctx.saved_tensors
        g, v, simt = ctx.g, v.contiguous(), ctx.simt
        dx = _plain_dgrad(g, _as_cl(dz.detach()), v, simt) if ctx.needs_input_grad[0] else None
        ddz = _plain_fprop(g, _as_cl(x.detach()), v, simt) if ctx.needs_input_grad[1] else None
        return dx, ddz, None, None, None


def _conv_backward_differentiable(dy, x, weight, y, chan_scale, act, slope, g, need_dx, need_dw, need_db, norm=None,
                                  simt=False):
    """(dx, dw, db, dgamma, dbeta) of a [training-mode norm ->] conv block [+bias] [act] [* Dropout2d scale] from
    differentiable nodes, for a backward under autograd.grad(..., create_graph=True).  x is the block's input; dz is
    rebuilt from (y, act, slope, chan_scale).  norm: None, or (gamma, beta, NormSpec, need_params) of the norm between
    x and the conv, whose output no node kept: it is recomputed from x as a differentiable NormFn output (no
    running-statistics update) and its backward is NormBwdFn."""
    if g.up != 1 or g.pad_mode != PAD_ZERO:
        raise NotImplementedError("b200gan: double backward through a conv with a folded upsample / reflection "
                                  "padding")
    xin = x
    if norm is not None:
        gamma, beta, nspec, need_params = norm
        _refuse_second_order_act(nspec.act, "a normalisation")
        xin, mr, ss = _norm_recompute(x, gamma, beta, nspec)
        need_dx = need_dx or need_params
    if chan_scale is not None and act in (ACT_TANH, ACT_SIGMOID):
        raise NotImplementedError("b200gan: double backward through Dropout2d fused with tanh / sigmoid")
    dz = dy
    if act == ACT_LRELU:
        dz = dz * torch.where(y > 0, 1.0, slope)           # piecewise constant mask: no second-order term
    elif act == ACT_RELU:
        dz = dz * (y > 0).to(dy.dtype)
    elif act == ACT_TANH:
        dz = dz * (1 - y * y)                              # y is this node's (differentiable) output
    elif act == ACT_SIGMOID:
        dz = dz * (y * (1 - y))
    if chan_scale is not None:
        dz = dz * chan_scale.view(chan_scale.shape[0], chan_scale.shape[1], 1, 1)
    dx = ConvDgradFn.apply(dz, weight, g, simt) if need_dx else None
    dw = ConvWgradFn.apply(xin, dz, g, tuple(weight.shape), simt) if need_dw else None
    db = dz.sum((0, 2, 3)) if need_db else None
    dgamma = dbeta = None
    if norm is not None and dx is not None:
        dx, dgamma, dbeta = NormBwdFn.apply(dx, x, gamma, mr, ss, nspec, need_params)
    return dx, dw, db, dgamma, dbeta


# ---- double backward through training-mode norms (SURVEY.md 8f N2: penalties on normalised conv critics) --------------
def _refuse_second_order_act(act, what):
    if act in (ACT_TANH, ACT_SIGMOID):
        raise NotImplementedError(f"b200gan: double backward through {what} fused with tanh / sigmoid (its activation "
                                  "has a second-order term of its own)")


def _norm_params_grads(dgb, shape, per_sample=False):
    """(dgamma, dbeta) per channel from the [dgamma; dbeta] per-group output of a norm backward on a tensor of `shape`
    (None: not computed)"""
    if dgb is None:
        return None, None
    groups = dgb.numel() // 2
    dgamma, dbeta = dgb[:groups], dgb[groups:]
    if per_sample:  # affine InstanceNorm2d: parameters are shared across samples
        n, c = shape[0], shape[1]
        dgamma, dbeta = dgamma.view(n, c).sum(0), dbeta.view(n, c).sum(0)
    return dgamma, dbeta


class NormBwdFn(torch.autograd.Function):
    """The first-order backward of NormFn, (dy, x, gamma) -> (dx, dgamma, dbeta), as a node that can be differentiated
    once more (autograd.grad(..., create_graph=True) through a training-mode norm).  mean_rstd / scale_shift are the
    batch statistics of x and its affine transform; the double backward (ops.norm_double_backward) includes their
    dependence on x.  Activation none / LeakyReLU / ReLU, the mask recomputed from x."""

    @staticmethod
    def forward(ctx, dy, x, gamma, mean_rstd, scale_shift, spec, need_params):
        ctx.set_materialize_grads(False)
        dy = _as_cl(dy.detach())
        dx, dgb = ops.norm_backward(dy, x.detach(), None, mean_rstd, None if gamma is None else gamma.detach(),
                                    spec.per_sample, spec.eps, spec.act, spec.slope, need_params, spec.rtf_dx,
                                    scale_shift)
        ctx.spec, ctx.dy = spec, dy
        ctx.save_for_backward(x, gamma, mean_rstd, scale_shift)
        return (dx,) + _norm_params_grads(dgb, x.shape, spec.per_sample)

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, u, ugamma, ubeta):
        x, gamma, mean_rstd, scale_shift = ctx.saved_tensors
        spec, nig = ctx.spec, ctx.needs_input_grad
        need_ggamma = gamma is not None and nig[2]
        if (u is None and ugamma is None and ubeta is None) or not (nig[0] or nig[1] or need_ggamma):
            return (None,) * 7
        u = torch.zeros_like(x, memory_format=torch.channels_last) if u is None else _as_cl(u)
        ugb = None
        if gamma is not None and (ugamma is not None or ubeta is not None):
            zero = torch.zeros_like(gamma)
            ugb = torch.cat([zero if ugamma is None else ugamma, zero if ubeta is None else ubeta]).contiguous()
        gx, gdy, gg = ops.norm_double_backward(ctx.dy, x.detach(), mean_rstd, scale_shift,
                                               None if gamma is None else gamma.detach(), u, ugb, spec.per_sample,
                                               spec.act, spec.slope, nig[1], nig[0], need_ggamma)
        if gg is not None and spec.per_sample:
            gg = gg.view(x.shape[0], x.shape[1]).sum(0)
        return gdy, gx, gg, None, None, None, None


def _norm_recompute(x, gamma, beta, spec):
    """(NormFn output, mean_rstd, scale_shift) of x with batch statistics and no running-statistics update: the
    normalised tensor a fused node never kept, recomputed as a differentiable function of (x, gamma, beta)."""
    box = []
    y = NormFn.apply(x, gamma, beta, None, None, None, None, spec, box)
    return (y,) + box[0]


def _bn_consts(a, gamma, beta, eps):
    """(mean_rstd, scale_shift) of a BatchNorm2d of `a` with batch statistics, without a running-statistics update"""
    return ops.norm_finalize(a.shape, ops.norm_stats(a, False), gamma, beta, None, None, None, False, eps, 0.0,
                             a.device)



def _norm_forward(x, gamma, beta, stats, running_mean, running_var, nbt, spec: NormSpec):
    """(y, mean_rstd, scale_shift) of the training-mode norm `spec` on the channels_last input x"""
    return ops.norm_forward(x, None if gamma is None else gamma.detach(), None if beta is None else beta.detach(),
                            running_mean, running_var, nbt, spec.per_sample, spec.eps, spec.momentum, spec.act,
                            spec.slope, stats, spec.rtf_out, return_scale_shift=True)


class NormFn(torch.autograd.Function):
    """Training-mode BatchNorm2d / InstanceNorm2d with an optional fused activation."""

    @staticmethod
    def forward(ctx, x, gamma, beta, stats, running_mean, running_var, nbt, spec: NormSpec, box=None):
        """box: None, or a list that receives (mean_rstd, scale_shift) (_norm_recompute)"""
        ops._require_cuda(x, "norm input")
        x = _as_cl(x)
        y, mean_rstd, scale_shift = _norm_forward(x, gamma, beta, stats, running_mean, running_var, nbt, spec)
        if box is not None:
            box.append((mean_rstd, scale_shift))
        ctx.spec = spec
        # LeakyReLU / ReLU masks are recomputed from x in backward (sign of x * scale + shift): y need not be kept
        mask_from_x = spec.act in (ACT_LRELU, ACT_RELU)
        need_y = spec.act != ACT_NONE and not mask_from_x
        ctx.save_for_backward(x, y if need_y else None, mean_rstd, gamma, scale_shift if mask_from_x else None)
        return y

    @staticmethod
    def backward(ctx, dy):
        x, y, mean_rstd, gamma, scale_shift = ctx.saved_tensors
        spec = ctx.spec
        need_params = gamma is not None and (ctx.needs_input_grad[1] or ctx.needs_input_grad[2])
        if torch.is_grad_enabled():
            # autograd.grad(..., create_graph=True): a gradient penalty through this norm (dragan.py:144-167,
            # dualgan.py:116-135) differentiates THROUGH this backward
            _refuse_second_order_act(spec.act, "a normalisation")
            dx, dgamma, dbeta = NormBwdFn.apply(dy, x, gamma, mean_rstd, scale_shift, spec, need_params)
            return dx, dgamma, dbeta, None, None, None, None, None, None
        x, dy = x.detach(), _as_cl(dy.detach())
        dx, dgb = ops.norm_backward(dy, x, y, mean_rstd, None if gamma is None else gamma.detach(), spec.per_sample,
                                    spec.eps, spec.act, spec.slope, need_params, spec.rtf_dx, scale_shift)
        return (dx,) + _norm_params_grads(dgb, x.shape, spec.per_sample) + (None,) * 6


class NormConvFn(torch.autograd.Function):
    """Training-mode BatchNorm2d [-> LeakyReLU/ReLU] [-> Upsample x2] -> Conv2d (dcgan.py:53-55, 56-59): the forward
    is NormFn's and ConvFn's, the backward reads no tensor twice for the norm -- its sums come out of the conv's
    data-gradient epilogue (ops.conv_dgrad_norm) -- and takes the bias gradient from the weight-gradient kernel.
    Only for geometries with ops.conv_dgrad_norm_supported (nn.Sequential checks)."""

    @staticmethod
    def forward(ctx, x, gamma, beta, stats, running_mean, running_var, nbt, weight, bias, chan_scale, nspec: NormSpec,
                cspec: ConvSpec, cache: PackCache):
        ops._require_cuda(x, "norm input")
        ops._require_cuda(weight, "conv weight")
        x = _as_cl(x)
        a, mean_rstd, scale_shift = _norm_forward(x, gamma, beta, stats, running_mean, running_var, nbt, nspec)
        g, y, out_stats = _conv_forward(a, weight, bias, chan_scale, cspec, cache)
        ctx.nspec, ctx.cspec, ctx.cache, ctx.g = nspec, cspec, cache, g
        ctx.has_bias = bias is not None
        # the norm output `a` is the conv's weight-gradient operand; the conv's output is kept only for its activation
        ctx.save_for_backward(x, mean_rstd, scale_shift, gamma, a, weight, y if cspec.act != ACT_NONE else None,
                              chan_scale, beta)
        return _with_stats(ctx, y, out_stats)

    @staticmethod
    def backward(ctx, dy, *unused):
        x, mean_rstd, scale_shift, gamma, a, weight, y, chan_scale, beta = ctx.saved_tensors
        nspec, cspec, g = ctx.nspec, ctx.cspec, ctx.g
        nig = ctx.needs_input_grad
        need_params = gamma is not None and (nig[1] or nig[2])
        if torch.is_grad_enabled():
            dx, dw, db, dgamma, dbeta = _conv_backward_differentiable(
                dy, x, weight, y, chan_scale, cspec.act, cspec.slope, g, nig[0], nig[7], ctx.has_bias and nig[8],
                norm=(gamma, beta, nspec, need_params))
            return dx, dgamma, dbeta, None, None, None, None, dw, db, None, None, None, None
        x, a, y, dy = x.detach(), a.detach(), None if y is None else y.detach(), _as_cl(dy.detach())
        dz = _conv_dz(dy, y, chan_scale, cspec)
        dx = dgamma = dbeta = None
        if nig[0] or need_params:
            algo, kind = ops.conv_plan(g, 1)
            da, sums = ops.conv_dgrad_norm(g, dz, ctx.cache.get(g, weight.detach(), kind), x, mean_rstd, scale_shift,
                                           nspec.act, nspec.slope)
            dx, dgb = ops.norm_backward_from_sums(da, x, mean_rstd, None if gamma is None else gamma.detach(), sums,
                                                  nspec.eps, nspec.act, nspec.slope, need_params, nspec.rtf_dx,
                                                  scale_shift)
            dgamma, dbeta = _norm_params_grads(dgb, x.shape)
            if not nig[0]:
                dx = None
        dw, db = _conv_param_grads(g, a, dz, dy, y, chan_scale, cspec, tuple(weight.shape), nig[7],
                                   ctx.has_bias and nig[8])
        return dx, dgamma, dbeta, None, None, None, None, dw, db, None, None, None, None


@dataclass(frozen=True)
class TailSpec:
    eps: float = 1e-5
    momentum: float = 0.0
    act_mid: int = ACT_NONE
    slope: float = 0.0
    act_out: int = ACT_NONE
    rtf_dx: bool = False


class TailFn(torch.autograd.Function):
    """Training-mode BatchNorm2d -> LeakyReLU/ReLU -> Conv2d(C, K<=3, 3, 1, 1) [-> Tanh] on the raw output `a` of
    the preceding conv (dcgan.py:60-63), without materialising the normalised tensor or any gradient of it."""

    @staticmethod
    def forward(ctx, a, stats, gamma, beta, running_mean, running_var, nbt, weight, bias, spec: TailSpec):
        ops._require_cuda(a, "tail input")
        a = _as_cl(a)
        if stats is None:
            stats = ops.norm_stats(a, False)
        mean_rstd, scale_shift = ops.norm_finalize(
            tuple(a.shape), stats, None if gamma is None else gamma.detach(), None if beta is None else beta.detach(),
            running_mean, running_var, nbt, False, spec.eps, spec.momentum, a.device)
        d = ops.tail_desc(tuple(a.shape), weight.shape[0], spec.act_mid, spec.slope, spec.act_out)
        w = weight.detach().contiguous()
        out = ops.tail_fprop(d, a, scale_shift, w, None if bias is None else bias.detach())
        ctx.spec, ctx.d = spec, d
        ctx.has_affine, ctx.has_bias = gamma is not None, bias is not None
        ctx.save_for_backward(a, mean_rstd, scale_shift, weight, out if spec.act_out != ACT_NONE else None)
        return out

    @staticmethod
    def backward(ctx, dout):
        if torch.is_grad_enabled():
            raise NotImplementedError("b200gan: double backward (create_graph=True) through the fused generator tail "
                                      "(BatchNorm2d -> activation -> Conv2d(C, K<=3, 3, 1, 1))")
        a, mean_rstd, scale_shift, weight, out = ctx.saved_tensors
        spec = ctx.spec
        a, out, dout = a.detach(), None if out is None else out.detach(), _as_cl(dout.detach())
        g = ops.epilogue_bwd(dout, out, None, spec.act_out, 0.0) if spec.act_out != ACT_NONE else dout
        need_affine = ctx.has_affine and (ctx.needs_input_grad[2] or ctx.needs_input_grad[3])
        need_bias = ctx.has_bias and ctx.needs_input_grad[8]
        da, dgb, dw, db = ops.tail_bwd(ctx.d, a, mean_rstd, scale_shift, weight.detach().contiguous(), g, need_affine,
                                       need_bias, spec.rtf_dx)
        dgamma, dbeta = _norm_params_grads(dgb, a.shape)
        return da, None, dgamma, dbeta, None, None, None, dw, db, None


class AffineActFn(torch.autograd.Function):
    """y = act(x * scale[c] + shift[c]) with constant scale/shift: eval-mode BatchNorm2d."""

    @staticmethod
    def forward(ctx, x, scale_shift, act, slope):
        x = _as_cl(x)
        y = ops.norm_apply_affine(x, scale_shift, False, act, slope)
        ctx.act, ctx.slope = act, slope
        ctx.save_for_backward(y, scale_shift)
        return y

    @staticmethod
    def backward(ctx, dy):
        y, scale_shift = ctx.saved_tensors
        c = y.shape[1]
        if torch.is_grad_enabled():
            # create_graph=True: linear in x apart from the piecewise-constant mask, so differentiable torch ops suffice
            _refuse_second_order_act(ctx.act, "an eval-mode BatchNorm2d")
            if ctx.act == ACT_LRELU:
                dy = dy * torch.where(y > 0, 1.0, ctx.slope)
            elif ctx.act == ACT_RELU:
                dy = dy * (y > 0).to(dy.dtype)
            return dy * scale_shift[:c].view(1, c, 1, 1), None, None, None
        y, dy = y.detach(), _as_cl(dy.detach())
        dz = ops.epilogue_bwd(dy, y, None, ctx.act, ctx.slope) if ctx.act != ACT_NONE else dy
        zero = torch.zeros_like(scale_shift)
        zero[:c] = scale_shift[:c]
        # dx = dz * scale: an affine apply with shift = 0
        return ops.norm_apply_affine(dz, zero, False), None, None, None


class ToChannelsLastFn(torch.autograd.Function):
    """Layout change NCHW -> NHWC.  Linear, so under create_graph=True (gradient penalties, SURVEY.md 8f N2) the
    backward is the opposite layout node rather than a detached copy."""

    @staticmethod
    def forward(ctx, x):
        return ops.to_cl(x)

    @staticmethod
    def backward(ctx, dy):
        if torch.is_grad_enabled() and dy.requires_grad:
            return ToContiguousFn.apply(dy)
        return ops.to_nchw(dy.detach())


class ToContiguousFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x):
        return ops.to_nchw(x)

    @staticmethod
    def backward(ctx, dy):
        if torch.is_grad_enabled() and dy.requires_grad:
            return dy if ops.is_cl(dy) else ToChannelsLastFn.apply(dy)
        return _as_cl(dy.detach())


class UpsampleFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x):
        return ops.upsample2x(_as_cl(x))

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, dy):
        return ops.upsample2x_bwd(_as_cl(dy))


class PadFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, pads, mode, round_tf32=False):
        ctx.pads, ctx.mode = pads, mode
        return ops.pad2d(_as_cl(x), pads, mode, round_tf32)

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, dy):
        return ops.pad2d_bwd(_as_cl(dy), ctx.pads, ctx.mode), None, None, None


class ActFn(torch.autograd.Function):
    """y = mask * act(x).  mask: None, per-(n,c) [N,C] (Dropout2d) or element-wise (Dropout)."""

    @staticmethod
    def forward(ctx, x, act, slope, mask, mask_per_channel):
        x = _as_cl(x)
        y = ops.act_forward(x, act, slope, mask, mask_per_channel)
        ctx.act, ctx.slope, ctx.mpc = act, slope, mask_per_channel
        ctx.save_for_backward(y if act != ACT_NONE else None, mask)
        return y

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, dy):
        y, mask = ctx.saved_tensors
        dy = _as_cl(dy)
        if mask is not None and not ctx.mpc:
            if ctx.act in (ACT_TANH, ACT_SIGMOID):
                raise NotImplementedError("b200gan: element-wise mask fused with tanh/sigmoid")
            dy = ops.act_forward(dy, ACT_NONE, 0.0, mask, False)
            mask = None
        if ctx.act == ACT_NONE and mask is None:
            return dy, None, None, None, None
        return ops.epilogue_bwd(dy, y, mask, ctx.act, ctx.slope), None, None, None, None


@dataclass(frozen=True)
class NbSpec:
    stride: int = 1
    pad: int = 0
    act: int = ACT_NONE
    slope: float = 0.0
    momentum: float = 0.0     # of the BatchNorm on the INPUT edge (its running statistics are updated by this conv)
    want_stats: bool = False  # a training-mode BatchNorm follows: produce the batch sums of the output
    groups: int = 1           # statistics groups of the batch (ops.bn_groups)


class ChainPass:
    """Shared by the nodes of one forward of a fused chain.  Once a backward under create_graph=True has run through the
    chain, its grad-mode nodes feed TRUE gradients (w.r.t. the stored raw outputs a_l) back into the chain's forward
    nodes, which the virtual-gradient protocol would add to virtual ones.  So from then on (true_grads) every first-order
    backward of these nodes takes and returns true gradients: each node finishes the backward of its own input
    BatchNorm and calls nb_dz without an output edge."""

    def __init__(self):
        self.true_grads = False


def _finish_bn(g, a, edge, sums, need_gamma, need_beta):
    """(da, dgamma, dbeta): the backward of the chain BatchNorm `edge` on its raw input a, given the gradient g w.r.t.
    its (virtual) output and sums = (sum g, sum g * ahat) from nb_dgrad / nb_tail_bwd; hands `sums` back zeroed"""
    mean_rstd, _ = _bn_consts(a, edge.gamma, edge.beta, edge.eps)
    need = edge.gamma is not None and (need_gamma or need_beta)
    da, dgb = ops.norm_backward_from_sums(g, a, mean_rstd, edge.gamma, sums, edge.eps, need_params=need)
    dgamma, dbeta = _norm_params_grads(dgb, a.shape)
    return da, (dgamma if need_gamma else None), (dbeta if need_beta else None)


def _chain_params_grads(sums, groups, c, need_gamma, need_beta):
    """(dgamma, dbeta) of a chain BatchNorm from the [groups][sum g; sum g * ahat] sums of the backward of its
    consumer, summed over the statistics groups: beta's gradient is the first half, gamma's the second"""
    if not (need_gamma or need_beta):
        return None, None
    # one conversion kernel for both parameter gradients
    dgb = sums.float() if groups == 1 else sums.view(groups, 2 * c).sum(0).float()
    return (dgb[c:] if need_gamma else None), (dgb[:c] if need_beta else None)


def _refuse_grouped_chain(groups):
    if groups > 1:
        raise NotImplementedError("b200gan: double backward (create_graph=True) through a fused chain under "
                                  "ops.bn_groups > 1")


class NbConvFn(torch.autograd.Function):
    """One layer of a fused narrow chain (csrc/narrow_block.cu): conv over the (virtually normalised) stored output of
    the previous layer, + bias, activation, Dropout2d scale, + the batch sums for the following BatchNorm.

    Chain protocol.  `in_edge` / `out_edge` are ops.BnEdge objects shared with the neighbouring layers.  In backward the
    incoming gradient is w.r.t. the VIRTUAL normalised output (the consumer could not finish the BatchNorm backward
    without the batch sums); by then the consumer has stored those sums in out_edge.sums.  This node finishes the norm
    backward (nb_dz), computes its parameter gradients, and hands ITS producer a virtual gradient plus in_edge.sums.
    Only valid when the stored output has exactly one consumer: the next node of the same chain.  After a backward under
    create_graph=True, true gradients instead (ChainPass)."""

    @staticmethod
    def forward(ctx, x, weight, bias, chan_scale, in_gamma, in_beta, in_rm, in_rv, in_nbt, in_edge, out_box, spec, cache,
                chain):
        ops._require_cuda(x, "conv input")
        x = _as_cl(x)
        g, _ = ops.make_geom(tuple(x.shape), tuple(weight.shape), spec.stride, (spec.pad,) * 4)
        w = weight.detach()
        packed = cache.get(g, w, PACK_SIMT_FPROP)
        y, stats = ops.nb_fprop(g, x, packed, None if bias is None else bias.detach(), spec.act, spec.slope, chan_scale,
                                in_edge, in_rm, in_rv, in_nbt, spec.momentum, spec.want_stats, spec.groups)
        ctx.g, ctx.spec, ctx.cache, ctx.in_edge, ctx.out_box, ctx.chain = g, spec, cache, in_edge, out_box, chain
        ctx.has_bias = bias is not None
        ctx.save_for_backward(x, weight, y, chan_scale, in_gamma, in_beta)
        if spec.want_stats:
            ctx.mark_non_differentiable(stats)
            return y, stats
        return y

    @staticmethod
    def backward(ctx, gy, *unused):
        x, weight, y, chan_scale, in_gamma, in_beta = ctx.saved_tensors
        g, spec, in_edge = ctx.g, ctx.spec, ctx.in_edge
        out_edge = ctx.out_box[0] if ctx.out_box else None
        nig = ctx.needs_input_grad
        if torch.is_grad_enabled():
            # autograd.grad(..., create_graph=True) through a chain: the gradient penalty of a conv critic (SURVEY.md 8f
            # N2: stargan.py:142-161 without norms, dragan.py:144-167 with BatchNorm2d).  gy and the returned gradient
            # are TRUE gradients w.r.t. the raw stored tensors: the input BatchNorm's output is recomputed as a
            # differentiable NormFn output, the conv runs the same differentiable nodes as ConvFn, and the norm's
            # backward is NormBwdFn.  edge.sums is neither read nor written.
            _refuse_grouped_chain(spec.groups)
            ctx.chain.true_grads = True
            norm = None
            if in_edge is not None:
                norm = (in_gamma, in_beta, NormSpec(eps=in_edge.eps), in_gamma is not None and (nig[4] or nig[5]))
            gx, dw, db, dgamma, dbeta = _conv_backward_differentiable(
                gy, x, weight, y, chan_scale, spec.act, spec.slope, g, nig[0], nig[1], ctx.has_bias and nig[2],
                norm=norm, simt=in_edge is not None or out_edge is not None)
            return gx, dw, db, None, dgamma, dbeta, None, None, None, None, None, None, None, None
        true_grads = ctx.chain.true_grads
        if true_grads:
            out_edge = None  # gy is w.r.t. the stored output itself
        gy, y, x = gy.detach(), y.detach(), x.detach()
        if out_edge is not None and out_edge.sums is None:
            raise RuntimeError("b200gan: fused conv chain: the consumer of this layer did not run its backward first")
        gy = _as_cl(gy)
        want_db = ctx.has_bias and ctx.needs_input_grad[2]
        dz, db = ops.nb_dz(gy, y, chan_scale, spec.act, spec.slope, out_edge, want_db)
        dw = None
        if ctx.needs_input_grad[1]:
            dw = ops.nb_wgrad(g, x, dz, in_edge, tuple(weight.shape))
        gx = dgamma = dbeta = None
        need_in = ctx.needs_input_grad[0] or (in_edge is not None and (ctx.needs_input_grad[4] or ctx.needs_input_grad[5]))
        if need_in:
            packed = ctx.cache.get(g, weight.detach(), PACK_SIMT_DGRAD)
            gx, sums = ops.nb_dgrad(g, dz, packed, in_edge, x)
            if in_edge is not None and true_grads:
                gx, dgamma, dbeta = _finish_bn(gx, x, in_edge, sums, ctx.needs_input_grad[4], ctx.needs_input_grad[5])
            elif in_edge is not None:
                in_edge.sums = sums
                dgamma, dbeta = _chain_params_grads(sums, in_edge.groups, g.C, ctx.needs_input_grad[4],
                                                    ctx.needs_input_grad[5])
        return gx, dw, db, None, dgamma, dbeta, None, None, None, None, None, None, None, None


class NbTailFn(torch.autograd.Function):
    """End of a fused narrow chain: the last BatchNorm's output as a real tensor (optionally NCHW-contiguous: the layout
    the script's `.view(N, -1)` needs, dcgan.py:96).  Returns a virtual gradient as NbConvFn does, or, under
    create_graph=True and after it (ChainPass), the true gradient w.r.t. `a`."""

    @staticmethod
    def forward(ctx, a, gamma, beta, rm, rv, nbt, edge, momentum, nchw, chain):
        a = _as_cl(a)
        out = ops.nb_tail_fwd(a, edge, rm, rv, nbt, momentum, nchw)
        ctx.edge, ctx.nchw, ctx.chain = edge, nchw, chain
        ctx.save_for_backward(a, gamma, beta)
        return out

    @staticmethod
    def backward(ctx, dout):
        a, gamma, beta = ctx.saved_tensors
        nig = ctx.needs_input_grad
        if torch.is_grad_enabled():
            _refuse_grouped_chain(ctx.edge.groups)
            ctx.chain.true_grads = True
            mr, ss = _bn_consts(a.detach(), ctx.edge.gamma, ctx.edge.beta, ctx.edge.eps)
            need_params = gamma is not None and (nig[1] or nig[2])
            da, dgamma, dbeta = NormBwdFn.apply(dout, a, gamma, mr, ss, NormSpec(eps=ctx.edge.eps), need_params)
            return da, dgamma, dbeta, None, None, None, None, None, None, None
        a, dout = a.detach(), dout.detach()
        dout = dout.contiguous() if ctx.nchw else _as_cl(dout)
        g, sums = ops.nb_tail_bwd(a, ctx.edge, dout, ctx.nchw)
        if ctx.chain.true_grads:
            return _finish_bn(g, a, ctx.edge, sums, nig[1], nig[2]) + (None,) * 7
        ctx.edge.sums = sums
        dgamma, dbeta = _chain_params_grads(sums, ctx.edge.groups, a.shape[1], nig[1], nig[2])
        return g, dgamma, dbeta, None, None, None, None, None, None, None


class _tf32_matmul:
    """cuBLAS TF32 for the GEMMs inside the block (a plain library GEMM: dcgan.py:50, Linear(100, 128 * 16 * 16))."""

    def __enter__(self):
        self.prev = torch.backends.cuda.matmul.allow_tf32
        torch.backends.cuda.matmul.allow_tf32 = True

    def __exit__(self, *exc):
        torch.backends.cuda.matmul.allow_tf32 = self.prev


class LinearWideFn(torch.autograd.Function):
    """nn.Linear with a wide output (the generator's first layer, dcgan.py:50: 0.84 GFLOP, 16.8 MB written) as TF32
    library GEMMs; torch's default for matmul is fp32 SIMT (30 us per GEMM here), while every convolution after it is
    TF32 anyway."""

    @staticmethod
    def forward(ctx, x, weight, bias):
        ctx.save_for_backward(x, weight)
        ctx.has_bias = bias is not None
        with _tf32_matmul():
            return torch.addmm(bias, x, weight.t()) if bias is not None else x @ weight.t()

    @staticmethod
    def backward(ctx, dy):
        x, weight = ctx.saved_tensors
        dx = dw = db = None
        with _tf32_matmul():
            if ctx.needs_input_grad[0]:
                dx = dy @ weight
            if ctx.needs_input_grad[1]:
                dw = dy.t() @ x
        if ctx.has_bias and ctx.needs_input_grad[2]:
            db = dy.sum(0)
        return dx, dw, db


class Linear1Fn(torch.autograd.Function):
    """nn.Linear(K, 1) [+ Sigmoid/Tanh/...] on a 2-D CUDA tensor: the discriminator head (dcgan.py:92)."""

    @staticmethod
    def forward(ctx, x, weight, bias, act):
        ops._require_cuda(x, "linear input")
        x = x.contiguous()
        y = ops.linear1_fwd(x, weight.detach().contiguous(), None if bias is None else bias.detach(), act)
        ctx.act, ctx.has_bias = act, bias is not None
        ctx.save_for_backward(x, weight, y)
        return y

    @staticmethod
    def backward(ctx, dy):
        x, weight, y = ctx.saved_tensors
        if torch.is_grad_enabled():  # create_graph=True: stay differentiable (plain torch ops on the saved tensors)
            if ctx.act == ACT_SIGMOID:
                dl = dy * y * (1 - y)
            elif ctx.act == ACT_TANH:
                dl = dy * (1 - y * y)
            else:
                dl = dy
            return dl @ weight, dl.t() @ x, (dl.sum(0) if ctx.has_bias else None), None
        dx, dw, db = ops.linear1_bwd(x, weight.detach().contiguous(), y, dy.contiguous(), ctx.act,
                                     ctx.needs_input_grad[0], ctx.has_bias and ctx.needs_input_grad[2])
        return dx, dw if ctx.needs_input_grad[1] else None, db, None


class BCEMeanFn(torch.autograd.Function):
    """torch.nn.BCELoss() (reduction 'mean') forward and backward as one kernel each (dcgan.py:103,166)."""

    @staticmethod
    def forward(ctx, v, t):
        v, t = v.contiguous(), t.contiguous()
        ctx.save_for_backward(v, t)
        return ops.bce_fwd(v, t)

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, gout):
        v, t = ctx.saved_tensors
        return ops.bce_bwd(v, t, gout.contiguous()), None


class ClassHeadFn(torch.autograd.Function):
    """nn.Linear(K, n) + nn.Softmax over the n outputs on a 2-D CUDA tensor, 2 <= n <= 32: the auxiliary-classifier head
    of acgan.py:100 / sgan.py:99 / infogan.py:111, one kernel per direction (csrc/head.cu).  dx, dW and db are each
    optional."""

    @staticmethod
    def forward(ctx, x, weight, bias):
        ops._require_cuda(x, "linear input")
        y = ops.class_head_fwd(x.contiguous(), weight.detach().contiguous(), None if bias is None else bias.detach())
        ctx.has_bias = bias is not None
        # the input itself, not a contiguous copy made here: a create_graph=True backward differentiates through it
        ctx.save_for_backward(x, weight, y)
        return y

    @staticmethod
    def backward(ctx, dy):
        x, weight, y = ctx.saved_tensors
        need_dx, need_dw = ctx.needs_input_grad[0], ctx.needs_input_grad[1]
        need_db = ctx.has_bias and ctx.needs_input_grad[2]
        if not (need_dx or need_dw or need_db):
            return None, None, None
        if torch.is_grad_enabled():  # create_graph=True: stay differentiable (plain torch ops on the saved tensors)
            dz = y * (dy - (dy * y).sum(1, keepdim=True))
            return (dz @ weight if need_dx else None), (dz.t() @ x if need_dw else None), \
                (dz.sum(0) if need_db else None)
        dx, dw, db = ops.class_head_bwd(x.detach().contiguous(), weight.detach().contiguous(), y, dy.contiguous(),
                                        need_dx, need_db)
        return dx, (dw if need_dw else None), db


class CrossEntropyMeanFn(torch.autograd.Function):
    """torch.nn.CrossEntropyLoss() (reduction 'mean', class-index targets, no class weights, no label smoothing) of
    [N, C] logits, forward and backward as one kernel each (csrc/head.cu): the auxiliary loss of acgan.py:113 /
    sgan.py:112 / infogan.py:126.  The gradient is with respect to the logits only."""

    @staticmethod
    def forward(ctx, x, target, ignore_index):
        target = target.contiguous()
        out = ops.cross_entropy_fwd(x.contiguous(), target, ignore_index)
        ctx.ignore_index = ignore_index
        # the input itself, not a contiguous copy made here: a create_graph=True backward differentiates through it
        ctx.save_for_backward(x, target, out)
        # out[0] would be a view, which autograd refuses to modify in place (`loss += reg`); alias the storage instead
        return out.new_empty(0).set_(out.untyped_storage(), out.storage_offset(), ())

    @staticmethod
    def backward(ctx, gout):
        x, target, out = ctx.saved_tensors
        if not ctx.needs_input_grad[0]:
            return None, None, None
        if torch.is_grad_enabled():  # create_graph=True: stay differentiable (plain torch ops on the saved tensors)
            hit = torch.arange(x.shape[1], device=x.device) == target[:, None]
            keep = (target != ctx.ignore_index)[:, None]
            d = (torch.softmax(x, 1) - hit.to(x.dtype)) * (gout / out[1])
            return torch.where(keep, d, torch.zeros_like(d)), None, None
        return ops.cross_entropy_bwd(x.detach().contiguous(), target, out, gout.detach().contiguous(),
                                     ctx.ignore_index), None, None


class PixelLossFn(torch.autograd.Function):
    """torch.nn.MSELoss() / torch.nn.L1Loss() (reduction 'mean') forward and backward as one kernel each
    (csrc/pixel_loss/): the adversarial, pixel, cycle and identity losses of the image translators
    (pix2pix.py:50-51, cyclegan.py:50-52).  Either gradient is optional."""

    @staticmethod
    def forward(ctx, input, target, mode):
        ctx.mode = mode
        ctx.save_for_backward(input, target)
        return ops.pixel_loss_fwd(input.detach(), target.detach(), mode)

    @staticmethod
    def backward(ctx, gout):
        a, b = ctx.saved_tensors
        need_a, need_b = ctx.needs_input_grad[0], ctx.needs_input_grad[1]
        if not (need_a or need_b):
            return None, None, None
        if torch.is_grad_enabled():  # create_graph=True: stay differentiable (plain torch ops on the saved tensors)
            diff = a - b
            if ctx.mode == PIXEL_LOSS_MSE:
                d = diff * (gout * (2.0 / a.numel()))
            else:
                d = torch.sign(diff) * (gout / a.numel())
            return (d if need_a else None), (-d if need_b else None), None
        da, db = ops.pixel_loss_bwd(a, b, gout.detach().contiguous(), ctx.mode, need_b)
        return (da if need_a else None), db, None


def conv_block(x, weight, bias, chan_scale, spec, cache):
    return ConvFn.apply(x, weight, bias, chan_scale, spec, cache)


def norm_block(x, gamma, beta, stats, running_mean, running_var, nbt, spec):
    return NormFn.apply(x, gamma, beta, stats, running_mean, running_var, nbt, spec)


class CriticStepMLPFn(torch.autograd.Function):
    """d_loss = -mean(D(real)) + mean(D(fake)) + lambda * gp(D, interpolates) of wgan_gp.py:164-171 for the MLP critic,
    with every parameter gradient produced by the same kernel (first-order backward + closed-form double backward)."""

    @staticmethod
    def forward(ctx, real, fake, alpha, w1, b1, w2, b2, w3, b3, slope, lambda_gp):
        out = ops.critic_step_mlp(real.detach(), fake.detach(), alpha, *[t.detach().contiguous() for t in
                                                                        (w1, b1, w2, b2, w3, b3)], slope, lambda_gp)
        losses, grads = out[0], out[1:]
        ctx.save_for_backward(*grads)
        ctx.mark_non_differentiable(losses[1:])
        return losses[0], losses[1]

    @staticmethod
    def backward(ctx, g, _g_gp):
        return (None, None, None) + tuple(g * t for t in ctx.saved_tensors) + (None, None)


def critic_step_mlp(critic_layers, real, fake, alpha, lambda_gp):
    """critic_layers: nn.Sequential(Linear, LeakyReLU, Linear, LeakyReLU, Linear(-> 1)) (wgan_gp.py:72-78), as
    nn.mlp_critic_layers accepts it (no hooks).  Returns (d_loss, lambda * gradient penalty); d_loss.backward() fills the
    gradients of all six parameters."""
    from .nn import mlp_critic_layers  # nn imports this module
    critic = mlp_critic_layers(list(critic_layers), real[0].numel())
    if critic is None:
        raise NotImplementedError("b200gan: fused critic step expects Linear-LReLU-Linear-LReLU-Linear(->1) with biases, "
                                  "one slope, no hooks, taking the flattened images")
    l1, l2, l3, slope = critic
    return CriticStepMLPFn.apply(real, fake, alpha, l1.weight, l1.bias, l2.weight, l2.bias, l3.weight, l3.bias, slope,
                                 float(lambda_gp))


# ---- the MLP critic under autograd (csrc/mlp_critic.cu) ------------------------------------------------------------
class MlpCriticFn(torch.autograd.Function):
    """D(x) = W3 lrelu(W2 lrelu(W1 x + b1) + b2) + b3 (wgan_gp.py:72-78, wgan_div.py:72-78): one launch forward, one
    launch backward.  Under autograd.grad(..., create_graph=True) -- a gradient penalty the script computes itself
    (wgan_gp.py:125-137, wgan_div.py:143-163) -- the backward is the differentiable node MlpCriticGradFn, whose own
    backward is one more launch, so the penalty's double backward never leaves the fused kernels."""

    @staticmethod
    def forward(ctx, x, w1, b1, w2, b2, w3, b3, slope):
        out, m1, a1, m2, a2 = ops.mlp_critic_fwd(x.detach(), *[t.detach() for t in (w1, b1, w2, b2, w3, b3)], slope)
        ctx.save_for_backward(x, w1, w2, w3, m1, a1, m2, a2)
        return out

    @staticmethod
    def backward(ctx, dout):
        x, w1, w2, w3, m1, a1, m2, a2 = ctx.saved_tensors
        need = tuple(ctx.needs_input_grad[:7])
        if torch.is_grad_enabled():
            return MlpCriticGradFn.apply(dout, x, w1, w2, w3, m1, a1, m2, a2, need) + (None,)
        grads = ops.mlp_critic_bwd(dout, x.detach(), w1.detach(), w2.detach(), w3.detach(), m1, a1, m2, a2, need)
        return (*grads[:7], None)


class MlpCriticGradFn(torch.autograd.Function):
    """The first-order backward of MlpCriticFn as a differentiable function of (dout, W1, W2, W3): outputs the
    gradients w.r.t. (x, W1, b1, W2, b2, W3, b3) that `need` asks for (None for the rest).  Only the input gradient
    dx = dD/dx may be differentiated again (a gradient penalty); its backward is the closed-form double backward, in
    which x and the biases get exactly zero."""

    @staticmethod
    def forward(ctx, dout, x, w1, w2, w3, m1, a1, m2, a2, need):
        ctx.set_materialize_grads(False)  # outputs nothing depends on arrive as None, not as zero-filled tensors
        grads = ops.mlp_critic_bwd(dout.detach(), x.detach(), w1.detach(), w2.detach(), w3.detach(), m1, a1, m2, a2,
                                   need, keep_u=True)
        ctx.save_for_backward(dout, w1, w2, w3, m1, m2, grads[7], grads[8])
        return grads[:7]

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, gx, *gparams):
        if any(g is not None for g in gparams):
            raise NotImplementedError("b200gan: the MLP critic's parameter gradients were differentiated (a penalty on "
                                      "parameter gradients); only its input gradient dD/dx is differentiable")
        none = (None,) * 10
        nig = ctx.needs_input_grad
        need = (nig[0], nig[2], nig[3], nig[4])
        if gx is None or not any(need):
            return none
        dout, w1, w2, w3, m1, m2, u1, u2 = ctx.saved_tensors
        ddout, dw1, dw2, dw3 = ops.mlp_critic_dbwd(gx, dout.detach(), u1, u2, m1, m2, w1.detach(), w2.detach(),
                                                   w3.detach(), need)
        if ddout is not None:
            ddout = ddout.view(dout.shape)
        return (ddout, None, dw1, dw2, dw3) + none[5:]


def mlp_critic(x, l1, l2, l3, slope):
    """Linear l1 -> LeakyReLU(slope) -> Linear l2 -> LeakyReLU(slope) -> Linear l3 (-> 1) on x [N, Din] as MlpCriticFn."""
    return MlpCriticFn.apply(x, l1.weight, l1.bias, l2.weight, l2.bias, l3.weight, l3.bias, float(slope))


# ---- the vanilla GAN discriminator: the MLP critic -> Sigmoid (csrc/mlp_critic.cu) ---------------------------------
class MlpDiscriminatorFn(torch.autograd.Function):
    """sigmoid(D(x)), D the MLP critic above (gan.py:64-80, bgan.py:66-80, aae.py:90-104): one launch forward, one
    launch backward, on the critic kernels in their Sigmoid mode.  A backward under grad mode (autograd.grad(...,
    create_graph=True): a penalty through the discriminator) recomputes the six modules from the saved inputs with
    torch ops, so its gradients stay differentiable in every input."""

    @staticmethod
    def forward(ctx, x, w1, b1, w2, b2, w3, b3, slope):
        y, m1, a1, m2, a2 = ops.mlp_disc_fwd(x.detach(), *[t.detach() for t in (w1, b1, w2, b2, w3, b3)], slope)
        ctx.slope = slope
        ctx.save_for_backward(x, w1, b1, w2, b2, w3, b3, y, m1, a1, m2, a2)
        return y

    @staticmethod
    def backward(ctx, dout):
        x, w1, b1, w2, b2, w3, b3, y, m1, a1, m2, a2 = ctx.saved_tensors
        need = tuple(ctx.needs_input_grad[:7])
        if torch.is_grad_enabled():
            inputs = (x, w1, b1, w2, b2, w3, b3)
            lrelu = torch.nn.functional.leaky_relu
            h = lrelu(torch.addmm(b1, x, w1.t()), ctx.slope)
            h = lrelu(torch.addmm(b2, h, w2.t()), ctx.slope)
            out = torch.sigmoid(torch.addmm(b3, h, w3.t()))
            grads = iter(torch.autograd.grad(out, [t for t, n in zip(inputs, need) if n], dout, create_graph=True))
            return tuple(next(grads) if n else None for n in need) + (None,)
        grads = ops.mlp_disc_bwd(dout, y, x.detach(), w1.detach(), w2.detach(), w3.detach(), m1, a1, m2, a2, need)
        return (*grads, None)


def mlp_discriminator(x, l1, l2, l3, slope):
    """Linear l1 -> LeakyReLU(slope) -> Linear l2 -> LeakyReLU(slope) -> Linear l3 (-> 1) -> Sigmoid on x [N, Din] as
    MlpDiscriminatorFn.  Without autograd (torch.no_grad(), nothing requiring grad) the forward records no node."""
    params = (l1.weight, l1.bias, l2.weight, l2.bias, l3.weight, l3.bias)
    if torch.is_grad_enabled() and (x.requires_grad or any(p.requires_grad for p in params)):
        return MlpDiscriminatorFn.apply(x, *params, float(slope))
    return ops.mlp_disc_fwd(x, *[p.detach() for p in params], float(slope))[0]


# ---- the MLP generator under autograd (csrc/mlp_generator) --------------------------------------------------------
class MlpGenSpec:
    """The non-tensor half of a generator call: per layer whether a BatchNorm1d follows its Linear and that norm's
    running-statistics buffers (updated in place by the forward), and the slope, eps and momentum shared by all."""

    def __init__(self, norms, slope, eps, momentum):
        self.norms = norms          # per layer: (running_mean, running_var, num_batches_tracked) or None
        self.slope, self.eps, self.momentum = float(slope), float(eps), float(momentum)

    def layers(self, params):
        """[(W, b, norm)] for ops.mlp_gen_*, from the flat parameter list W0, b0, [gamma0, beta0], W1, ..."""
        out, i = [], 0
        for norm in self.norms:
            w, b = params[i], params[i + 1]
            i += 2
            if norm is not None:
                out.append((w, b, (params[i], params[i + 1], *norm)))
                i += 2
            else:
                out.append((w, b, None))
        return out


class MlpGeneratorFn(torch.autograd.Function):
    """G(z) = tanh(W_L ... lrelu(BatchNorm1d(W_1 lrelu(W_0 z + b_0) + b_1)) ... + b_L) (wgan_gp.py:42-65, gan.py:38-61):
    one launch forward, one launch backward.  Inputs: z, the spec, then W, b (and gamma, beta after a norm) per layer."""

    @staticmethod
    def forward(ctx, z, spec, *params):
        out, saved = ops.mlp_gen_fwd(z.detach(), spec.layers([p.detach() for p in params]), spec.slope, spec.eps,
                                     spec.momentum, keep=True)
        ctx.spec = spec
        ctx.save_for_backward(z, out, saved, *params)
        return out

    @staticmethod
    def backward(ctx, dout):
        if torch.is_grad_enabled():
            raise NotImplementedError("b200gan: the fused MLP generator is not twice differentiable (create_graph=True)")
        z, out, saved, *params = ctx.saved_tensors
        spec = ctx.spec
        nig = ctx.needs_input_grad
        need, i = [], 2
        for norm in spec.norms:
            k = 4 if norm is not None else 2
            need.append(tuple(nig[i:i + k]) + (False,) * (4 - k))
            i += k
        dz, grads = ops.mlp_gen_bwd(dout.contiguous(), z.detach(), out, saved, spec.layers([p.detach() for p in params]),
                                    spec.slope, spec.eps, spec.momentum, nig[0], need)
        flat = []
        for norm, g in zip(spec.norms, grads):
            flat += list(g if norm is not None else g[:2])
        return (dz, None, *flat)


def mlp_generator(z, layers, slope):
    """layers: [(Linear, BatchNorm1d or None)] (nn.mlp_generator_layers) on z [N, width[0]]: Linear -> (norm) ->
    LeakyReLU(slope) blocks, the last Linear -> Tanh.  Without autograd (torch.no_grad(), nothing requiring grad) the
    forward keeps nothing for a backward."""
    params, norms, eps, momentum = [], [], 0.0, 0.0
    for lin, bn in layers:
        params += [lin.weight, lin.bias]
        if bn is not None:
            params += [bn.weight, bn.bias]
            norms.append((bn.running_mean, bn.running_var, bn.num_batches_tracked))
            eps, momentum = bn.eps, bn.momentum
        else:
            norms.append(None)
    spec = MlpGenSpec(norms, slope, eps, momentum)
    if torch.is_grad_enabled() and (z.requires_grad or any(p.requires_grad for p in params)):
        return MlpGeneratorFn.apply(z, spec, *params)
    return ops.mlp_gen_fwd(z, spec.layers([p.detach() for p in params]), spec.slope, spec.eps, spec.momentum,
                           keep=False)[0]
