"""Drop-in replacements for the torch.nn leaf modules the reference's Generator/Discriminator
classes instantiate (SURVEY.md section 8b).  Same constructor and forward signatures, same class
*names* (the reference's weights_init_normal dispatches on `__class__.__name__`, dcgan.py:36-42),
same Parameters / buffers / state_dict keys -- the arithmetic runs in libb200gan.so.

`Sequential` keeps the module tree the scripts build (dcgan.py:52-64, 83-88) and fuses at call
time: [Upsample][Pad] Conv [act][Dropout2d] (+ statistics for a following norm) and Norm [act]
become single fused nodes; anything unknown is executed leaf by leaf.

There is no CPU / cuDNN fallback for the conv and norm modules: CPU tensors raise.
"""
import torch
import torch.nn as tnn

from . import _lib
from . import functional as F
from . import ops
from ._lib import (ACT_LRELU, ACT_NONE, ACT_RELU, ACT_SIGMOID, ACT_TANH, PAD_REFLECT, PAD_ZERO, PIXEL_LOSS_L1,
                   PIXEL_LOSS_MSE)
from .functional import ConvSpec, NormSpec, PackCache

_T = {  # the stock classes, captured before any patching
    n: getattr(tnn, n) for n in (
        "Conv2d", "ConvTranspose2d", "BatchNorm2d", "InstanceNorm2d", "LeakyReLU", "ReLU", "Tanh", "Sigmoid",
        "Upsample", "ZeroPad2d", "ReflectionPad2d", "Dropout", "Dropout2d", "Sequential", "Linear", "BCELoss",
        "BatchNorm1d", "MSELoss", "L1Loss")
}


def _pair_same(v, what):
    if isinstance(v, (tuple, list)):
        if len(v) != 2 or v[0] != v[1]:
            raise NotImplementedError(f"b200gan: {what}={v} (h != w) is not supported")
        return int(v[0])
    return int(v)


def _act_of(m):
    if isinstance(m, _T["LeakyReLU"]):
        if m.negative_slope < 0:
            # the fused backward kernels recover the derivative from the sign of the output y, which a negative
            # slope makes positive on the negative side as well
            raise NotImplementedError(f"b200gan: {m} (negative_slope < 0)")
        return ACT_LRELU, float(m.negative_slope)
    if isinstance(m, _T["ReLU"]):
        return ACT_RELU, 0.0
    if isinstance(m, _T["Tanh"]):
        return ACT_TANH, 0.0
    if isinstance(m, _T["Sigmoid"]):
        return ACT_SIGMOID, 0.0
    return None


def _is_up2(m):
    if not isinstance(m, _T["Upsample"]):
        return False
    sf = m.scale_factor
    if isinstance(sf, (tuple, list)):
        sf = sf[0] if len(set(sf)) == 1 else None
    return m.size is None and sf is not None and float(sf) == 2.0 and m.mode == "nearest"


def _pads_of(m):
    """torch padding order (left, right, top, bottom) -> (top, left, bottom, right)."""
    p = m.padding
    if isinstance(p, int):
        p = (p, p, p, p)
    l, r, t, b = p
    return (int(t), int(l), int(b), int(r))


def _conv_ok(m):
    if isinstance(m.padding, str) or m.padding_mode != "zeros":
        return False
    if tuple(m.dilation) != (1, 1) or m.groups != 1:
        return False
    if len(set(m.stride)) != 1 or len(set(m.padding)) != 1:
        return False
    if isinstance(m, _T["ConvTranspose2d"]) and tuple(m.output_padding) != (0, 0):
        return False
    return True


def _tc_like(conv, up, full=False):
    """Static mirror of tc_supported() used to decide where TF32 rounding of operands pays.  full: every pass (forward,
    data gradient, weight gradient) is on the tensor cores, not just the forward."""
    if ops.Config.algo == "simt":
        return False
    if up == 2:
        return (not isinstance(conv, _T["ConvTranspose2d"]) and conv.stride[0] == 1 and conv.in_channels % 32 == 0
                and conv.out_channels % 64 == 0)
    if conv.stride[0] in (1, 2) and conv.in_channels % 32 == 0 and conv.out_channels % 32 == 0:
        return True
    # fewer than 32 output channels (cyclegan/models.py:82: Conv2d(64, 3, 7)): the FORWARD runs on wgmma (weight rows
    # zero-padded to 32 by TMA), the gradients on the fp32 kernels
    return (full is False and not isinstance(conv, _T["ConvTranspose2d"]) and conv.stride[0] == 1
            and conv.in_channels % 32 == 0 and conv.out_channels < 32)


def _no_groups(what):
    """ops.bn_groups is honoured by the fused chain only: anything else that depends on the batch composition refuses."""
    if ops.bn_groups.active > 1:
        raise RuntimeError(f"b200gan: ops.bn_groups({ops.bn_groups.active}) is active but {what} would treat the batch "
                           "as one pass; run the passes separately")


def _dropout2d_scale(x_shape, p, device):
    """Exactly the draw F.dropout2d makes (feature_dropout: noise [N,C,1,1] ~ Bernoulli(1-p) / (1-p)),
    so masks are bit-identical to the reference's under the same seed (dcgan.py:77)."""
    n, c = x_shape[0], x_shape[1]
    noise = torch.empty((n, c, 1, 1), device=device, dtype=torch.float32)
    if p >= 1.0:
        return noise.zero_().view(n, c)
    return noise.bernoulli_(1.0 - p).div_(1.0 - p).view(n, c)


def _conv_cache(conv):
    cache = conv.__dict__.get("_b200_cache")
    if cache is None:
        cache = PackCache()
        conv.__dict__["_b200_cache"] = cache
    return cache


def _run_conv(conv, x, up=1, extra_pads=(0, 0, 0, 0), pad_mode=PAD_ZERO, act=ACT_NONE, slope=0.0, chan_scale=None,
              stats=None, rtf_out=False, rtf_dz=False):
    if not _conv_ok(conv):
        raise NotImplementedError(f"b200gan: unsupported convolution configuration: {conv}")
    transposed = isinstance(conv, _T["ConvTranspose2d"])
    pad = int(conv.padding[0])
    if pad_mode == PAD_REFLECT and pad != 0:
        raise NotImplementedError("b200gan: reflection padding in front of a zero-padded conv")
    if pad_mode == PAD_REFLECT and up == 1 and _tc_like(conv, 1):
        # tensor-core path wants zero padding (TMA out-of-bounds fill): materialise the mirrored border once
        # (cyclegan/models.py:27-28: ReflectionPad2d(1) -> Conv2d(256, 256, 3)) and run the conv un-padded
        x = F.PadFn.apply(x, tuple(extra_pads), PAD_REFLECT, True)  # RN-round: operands of a TF32 MMA
        extra_pads, pad_mode = (0, 0, 0, 0), PAD_ZERO
    pads = tuple(e + pad for e in extra_pads)
    spec = ConvSpec(stride=int(conv.stride[0]), pads=pads, pad_mode=pad_mode, up=up, transposed=transposed, act=act,
                    slope=slope, stats=stats, rtf_out=rtf_out, rtf_dz=rtf_dz)
    return F.conv_block(x, conv.weight, conv.bias, chan_scale, spec, _conv_cache(conv))


def _batch_norm_spec(norm, per_sample, act, slope, rtf_out, rtf_dx):
    """(NormSpec, running_mean, running_var, num_batches_tracked) of a norm that normalises with batch statistics."""
    rm = rv = nbt = None
    momentum = 0.0
    if not per_sample and norm.training and norm.track_running_stats:
        if norm.momentum is None:
            raise NotImplementedError("b200gan: BatchNorm2d(momentum=None)")
        rm, rv, nbt, momentum = norm.running_mean, norm.running_var, norm.num_batches_tracked, float(norm.momentum)
    spec = NormSpec(per_sample=per_sample, eps=float(norm.eps), momentum=momentum, act=act, slope=slope,
                    rtf_out=rtf_out, rtf_dx=rtf_dx)
    return spec, rm, rv, nbt


def _run_norm(norm, x, act=ACT_NONE, slope=0.0, stats=None, rtf_out=False, rtf_dx=False):
    per_sample = isinstance(norm, _T["InstanceNorm2d"])
    if per_sample and norm.track_running_stats:
        raise NotImplementedError("b200gan: InstanceNorm2d(track_running_stats=True)")
    if x.dim() != 4:
        raise ValueError(f"expected 4D input (got {x.dim()}D input)")
    if per_sample and x.shape[2] * x.shape[3] == 1 and norm.training:
        raise ValueError(f"Expected more than 1 spatial element when training, got input size {tuple(x.shape)}")
    use_batch_stats = per_sample or norm.training or norm.running_mean is None
    if use_batch_stats and not per_sample:
        _no_groups("a stand-alone BatchNorm2d")
    if use_batch_stats:
        spec, rm, rv, nbt = _batch_norm_spec(norm, per_sample, act, slope, rtf_out, rtf_dx)
        return F.norm_block(x, norm.weight, norm.bias, stats, rm, rv, nbt, spec)
    # eval-mode BatchNorm2d: constant per-channel affine
    rstd = torch.rsqrt(norm.running_var + norm.eps)
    scale = rstd if norm.weight is None else norm.weight * rstd
    shift = -norm.running_mean * scale if norm.bias is None else norm.bias - norm.running_mean * scale
    return F.AffineActFn.apply(x, torch.cat([scale, shift]).detach(), act, slope)


def _on_device(x):
    """True for tensors the product path takes (CUDA).  A test hook: the CPU wiring tests replace it."""
    return x.is_cuda


def _gpu4d(x):
    return x.dim() == 4 and _on_device(x)


# ---- leaf modules ----------------------------------------------------------------------------------
class Conv2d(_T["Conv2d"]):
    def forward(self, x):
        return _run_conv(self, x)


class ConvTranspose2d(_T["ConvTranspose2d"]):
    def forward(self, x, output_size=None):
        if output_size is not None:
            raise NotImplementedError("b200gan: ConvTranspose2d(output_size=...)")
        return _run_conv(self, x)


class BatchNorm2d(_T["BatchNorm2d"]):
    def forward(self, x):
        return _run_norm(self, x)


class InstanceNorm2d(_T["InstanceNorm2d"]):
    def forward(self, x):
        return _run_norm(self, x)


class _Act:
    def forward(self, x):
        if not _gpu4d(x):
            return super().forward(x)  # MLP / CPU use of the same class (gan.py, wgan_gp.py): stock op
        act, slope = _act_of(self)
        return F.ActFn.apply(x, act, slope, None, False)


class LeakyReLU(_Act, _T["LeakyReLU"]):
    pass


class ReLU(_Act, _T["ReLU"]):
    pass


class Tanh(_Act, _T["Tanh"]):
    pass


class Sigmoid(_Act, _T["Sigmoid"]):
    pass


class Upsample(_T["Upsample"]):
    def forward(self, x):
        if _gpu4d(x) and _is_up2(self):
            return F.UpsampleFn.apply(x)
        if _gpu4d(x):
            raise NotImplementedError(f"b200gan: {self} (only nearest x2 is on the hot path)")
        return super().forward(x)


class ZeroPad2d(_T["ZeroPad2d"]):
    def forward(self, x):
        if not _gpu4d(x):
            return super().forward(x)
        return F.PadFn.apply(x, _pads_of(self), PAD_ZERO)


class ReflectionPad2d(_T["ReflectionPad2d"]):
    def forward(self, x):
        if not _gpu4d(x):
            return super().forward(x)
        return F.PadFn.apply(x, _pads_of(self), PAD_REFLECT)


class Dropout2d(_T["Dropout2d"]):
    def forward(self, x):
        if not _gpu4d(x):
            return super().forward(x)
        if not self.training or self.p == 0.0:
            return x
        _no_groups("a stand-alone Dropout2d")
        return F.ActFn.apply(x, ACT_NONE, 0.0, _dropout2d_scale(x.shape, self.p, x.device), True)


class Dropout(_T["Dropout"]):
    def forward(self, x):
        if not _gpu4d(x):
            return super().forward(x)
        if not self.training or self.p == 0.0:
            return x
        _no_groups("a stand-alone Dropout")
        xc = x if ops.is_cl(x) else ops.to_cl(x)
        mask = torch.empty_like(xc, memory_format=torch.channels_last)
        if self.p >= 1.0:
            mask.zero_()
        else:
            mask.bernoulli_(1.0 - self.p).div_(1.0 - self.p)
        return F.ActFn.apply(xc, ACT_NONE, 0.0, mask, False)


def _gpu2d_f32(x):
    return torch.is_tensor(x) and x.dim() == 2 and x.is_cuda and x.dtype == torch.float32


class Linear(_T["Linear"]):
    """nn.Linear.  Inside a Sequential (Sequential._forward_2d), two patterns run as b200gan kernels: Linear(K, 1) +
    Sigmoid/Tanh -- the head of a discriminator (dcgan.py:92) -- as one kernel per direction, and the whole MLP critic
    Linear -> LeakyReLU -> Linear -> LeakyReLU -> Linear(-> 1) of wgan_gp.py:72-78 / wgan_div.py:72-78 as one
    cooperative kernel per pass, double-differentiable for the script's own autograd.grad(create_graph=True)
    (functional.MlpCriticFn).  Anywhere else it is a plain library GEMM and stays on torch/cuBLAS (wgan_gp.py:46-60;
    dcgan.py:50).  A wide output (>= 8192 features: the generator's first layer, dcgan.py:50) uses the TF32 library
    GEMM like the convolutions behind it."""

    def forward(self, x):
        if _gpu2d_f32(x) and self.out_features >= 8192 and ops.Config.algo != "simt":
            return F.LinearWideFn.apply(x, self.weight, self.bias)
        return super().forward(x)


class BatchNorm1d(_T["BatchNorm1d"]):
    """nn.BatchNorm1d, same state_dict.  Inside the MLP generator pattern of a Sequential (mlp_generator_layers,
    wgan_gp.py:42-65, gan.py:38-61) it runs in the fused generator kernels; anywhere else, and on the CPU, it is the stock
    module."""


class BCELoss(_T["BCELoss"]):
    def forward(self, input, target):
        if (input.is_cuda and input.dtype == torch.float32 and self.reduction == "mean" and self.weight is None
                and target.shape == input.shape and target.dtype == torch.float32 and not target.requires_grad):
            return F.BCEMeanFn.apply(input, target)
        return super().forward(input, target)


def pixel_loss_routed(input, target, reduction):
    """True if MSELoss / L1Loss(input, target) runs on the pixel-loss kernels (functional.PixelLossFn): two CUDA fp32
    tensors of one shape (no broadcasting) on one device, each NCHW- or channels_last-contiguous, at most 4-D, with at
    least one element, and reduction 'mean'.  Everything else -- including the legacy size_average / reduce arguments,
    which the stock constructor maps onto `reduction` -- is the stock module.  No side effects."""
    if reduction != "mean" or not (torch.is_tensor(input) and torch.is_tensor(target)):
        return False
    if not (_on_device(input) and _on_device(target) and input.device == target.device):
        return False
    if input.dtype != torch.float32 or target.dtype != torch.float32:
        return False
    return ops.pixel_loss_desc(input, target, PIXEL_LOSS_MSE) is not None


class MSELoss(_T["MSELoss"]):
    """nn.MSELoss (lsgan.py:102, pix2pix.py:50, cyclegan.py:50); routing: pixel_loss_routed."""

    def forward(self, input, target):
        if pixel_loss_routed(input, target, self.reduction):
            return F.PixelLossFn.apply(input, target, PIXEL_LOSS_MSE)
        return super().forward(input, target)


class L1Loss(_T["L1Loss"]):
    """nn.L1Loss (pix2pix.py:51, cyclegan.py:51-52); routing: pixel_loss_routed."""

    def forward(self, input, target):
        if pixel_loss_routed(input, target, self.reduction):
            return F.PixelLossFn.apply(input, target, PIXEL_LOSS_L1)
        return super().forward(input, target)


# ---- fusion planner ------------------------------------------------------------------------------------
class _ConvStep:
    def __init__(self, conv, up, extra_pads, pad_mode, act, slope, dropout2d, stats):
        self.conv, self.up, self.extra_pads, self.pad_mode = conv, up, extra_pads, pad_mode
        self.act, self.slope, self.dropout2d, self.stats = act, slope, dropout2d, stats
        self.rtf_out = False
        self.rtf_dz = False
        self.next_norm = None

    def tc_like(self, full=False):
        if self.pad_mode == PAD_REFLECT and self.up != 1:
            return False
        return _tc_like(self.conv, self.up, full)


class _NormStep:
    def __init__(self, norm, act, slope, takes_stats):
        self.norm, self.act, self.slope, self.takes_stats = norm, act, slope, takes_stats
        self.rtf_out = False
        self.rtf_dx = False


class _LeafStep:
    def __init__(self, mod):
        self.mod = mod


class _TailStep:
    """BatchNorm2d [-> LeakyReLU/ReLU] -> Conv2d(C, K<=3, 3, 1, 1) [-> act]: the fused Generator tail (dcgan.py:60-63).
    Keeps the two steps it replaces for the cases the fused kernels do not take (eval mode, odd sizes)."""

    def __init__(self, norm_step, conv_step):
        self.norm_step, self.conv_step = norm_step, conv_step


def _no_hooks(m):
    return not (m._forward_hooks or m._forward_pre_hooks or m._backward_hooks)


def _norm_conv_fused(ns, cs, x_shape):
    """True if a norm step and the conv step after it run as functional.NormConvFn at this input shape: BatchNorm2d
    [-> LeakyReLU/ReLU] with batch statistics (training mode) [-> Upsample x2] -> Conv2d, stride 1, zero padding, no
    hooks, and a geometry whose data gradient can carry the norm's sums (dcgan.py:53-55, 56-59).  No side effects."""
    if not (isinstance(ns, _NormStep) and isinstance(cs, _ConvStep)):
        return False
    norm, conv = ns.norm, cs.conv
    if not isinstance(norm, _T["BatchNorm2d"]) or ns.act not in (ACT_NONE, ACT_LRELU, ACT_RELU):
        return False
    if isinstance(conv, _T["ConvTranspose2d"]) or cs.pad_mode != PAD_ZERO or tuple(conv.stride) != (1, 1):
        return False
    if not (_no_hooks(norm) and _no_hooks(conv) and norm.training and ops.bn_groups.active <= 1):
        return False
    if norm.track_running_stats and norm.momentum is None:
        return False
    if not (len(x_shape) == 4 and x_shape[1] == norm.num_features == conv.in_channels):
        return False
    pads = tuple(e + int(conv.padding[0]) for e in cs.extra_pads)
    g, _ = ops.make_geom(tuple(x_shape), tuple(conv.weight.shape), 1, pads, PAD_ZERO, cs.up)
    return ops.conv_dgrad_norm_supported(g)


def _chain_plan(chain, shape):
    """[(conv step, norm step, output shape)] if every layer of the chain qualifies for the fused kernels at this input
    shape (and under the active ops.bn_groups), else None.  No side effects."""
    plan = []
    for cs, ns in chain.layers:
        conv = cs.conv
        if shape[1] != conv.in_channels or not _conv_ok(conv):
            return None
        g, oshape = ops.make_geom(shape, tuple(conv.weight.shape), int(conv.stride[0]), (int(conv.padding[0]),) * 4)
        macs = float(oshape[0]) * oshape[2] * oshape[3] * conv.out_channels * conv.in_channels * g.R * g.S
        if macs > _ChainStep.MAX_MACS or not ops.nb_supported(g) or oshape[2] * oshape[3] < 1:
            return None
        if ns is not None:
            norm = ns.norm
            if not (norm.training and norm.num_features == conv.out_channels):
                return None
            if norm.track_running_stats and norm.momentum is None:
                return None
        plan.append((cs, ns, oshape))
        shape = oshape
    return plan


def groups_eligible(seq, x_shape, groups):
    """True if the drop-in Sequential `seq` would take a [N, C, H, W] fp32 CUDA batch of `groups` statistics groups
    entirely through fused chains (the only code that honours ops.bn_groups)."""
    if not isinstance(seq, Sequential) or not ops.Config.fuse_narrow_chain or x_shape[0] % groups != 0:
        return False
    steps = seq._plan()
    if not steps or not all(isinstance(st, _ChainStep) for st in steps):
        return False
    shape = tuple(x_shape)
    with ops.bn_groups(groups):
        for st in steps:
            plan = _chain_plan(st, shape)
            if plan is None:
                return False
            shape = plan[-1][2]
    return True


class _ChainStep:
    """A run of narrow [Conv2d -> act -> Dropout2d] (+ BatchNorm2d) blocks (dcgan.py:77-88) executed as the fused chain
    of csrc/narrow_block.cu when the runtime shapes qualify; `steps` are the ordinary steps it stands for."""

    MAX_MACS = 6.0e8   # per layer: above this the tensor-core path is the better choice

    def __init__(self, steps):
        self.steps = steps
        self.layers = []  # (conv step, norm step or None)
        i = 0
        while i < len(steps):
            ns = steps[i + 1] if i + 1 < len(steps) and isinstance(steps[i + 1], _NormStep) else None
            self.layers.append((steps[i], ns))
            i += 2 if ns is not None else 1


def _chain_conv_candidate(cs):
    if not isinstance(cs, _ConvStep):
        return False
    conv = cs.conv
    if isinstance(conv, _T["ConvTranspose2d"]) or cs.up != 1 or cs.extra_pads != (0, 0, 0, 0) or cs.pad_mode != PAD_ZERO:
        return False
    if cs.act not in (ACT_NONE, ACT_LRELU, ACT_RELU):
        return False
    k, c = conv.out_channels, conv.in_channels
    if not (4 <= k <= 128 and (k & (k - 1)) == 0 and 1 <= c <= 128 and (c == 1 or c % 4 == 0)):
        return False
    return tuple(conv.kernel_size) in ((3, 3), (4, 4)) and conv.stride[0] in (1, 2)


def _chain_norm_candidate(ns):
    return isinstance(ns, _NormStep) and isinstance(ns.norm, _T["BatchNorm2d"]) and ns.act == ACT_NONE


def _fuse_chains(steps):
    out, i, n = [], 0, len(steps)
    while i < n:
        j, convs = i, 0
        while j < n and _chain_conv_candidate(steps[j]):
            convs += 1
            j += 1
            if j < n and steps[j - 1].stats is False and _chain_norm_candidate(steps[j]):
                j += 1
            elif steps[j - 1].stats is not None:
                j -= 1          # a norm follows that the chain cannot take: the run ends before this conv
                convs -= 1
                break
        if convs >= 2:
            out.append(_ChainStep(steps[i:j]))
            i = j
        else:
            out.append(steps[i])
            i += 1
    return out


def _uses_batch_stats(norm):
    return isinstance(norm, _T["InstanceNorm2d"]) or norm.training or norm.running_mean is None


def _tail_candidate(ns, cs):
    if not (isinstance(ns, _NormStep) and isinstance(cs, _ConvStep)):
        return False
    norm, conv = ns.norm, cs.conv
    if not isinstance(norm, _T["BatchNorm2d"]) or ns.act not in (ACT_NONE, ACT_LRELU, ACT_RELU):
        return False
    if isinstance(conv, _T["ConvTranspose2d"]) or cs.up != 1 or cs.extra_pads != (0, 0, 0, 0) or cs.pad_mode != PAD_ZERO:
        return False
    if cs.dropout2d is not None or cs.stats is not None:
        return False
    return (tuple(conv.kernel_size) == (3, 3) and tuple(conv.stride) == (1, 1) and tuple(conv.padding) == (1, 1)
            and conv.out_channels <= 3 and conv.in_channels in (32, 64, 128))


def _is_norm(m):
    return isinstance(m, (_T["BatchNorm2d"], _T["InstanceNorm2d"]))


def _build_plan(mods):
    steps, i, n = [], 0, len(mods)
    while i < n:
        j, up, extra, mode = i, 1, (0, 0, 0, 0), PAD_ZERO
        if _is_up2(mods[j]):
            up, j = 2, j + 1
        if j < n and isinstance(mods[j], (_T["ZeroPad2d"], _T["ReflectionPad2d"])):
            extra = _pads_of(mods[j])
            mode = PAD_REFLECT if isinstance(mods[j], _T["ReflectionPad2d"]) else PAD_ZERO
            j += 1
        conv = mods[j] if j < n else None
        is_conv = isinstance(conv, (_T["Conv2d"], _T["ConvTranspose2d"])) and _conv_ok(conv)
        if is_conv and isinstance(conv, _T["ConvTranspose2d"]) and (up != 1 or j != i):
            is_conv = False
        if is_conv and mode == PAD_REFLECT and int(conv.padding[0]) != 0:
            is_conv = False
        if is_conv:
            j += 1
            act, slope, d2 = ACT_NONE, 0.0, None
            if j < n and _act_of(mods[j]) is not None:
                act, slope = _act_of(mods[j])
                j += 1
            if j < n and isinstance(mods[j], _T["Dropout2d"]):
                d2 = mods[j]
                j += 1
            stats = None
            if j < n and _is_norm(mods[j]):
                stats = isinstance(mods[j], _T["InstanceNorm2d"])
            steps.append(_ConvStep(conv, up, extra, mode, act, slope, d2, stats))
            steps[-1].next_norm = mods[j] if stats is not None else None
            i = j
            continue
        m = mods[i]
        if _is_norm(m):
            j = i + 1
            act, slope = ACT_NONE, 0.0
            if j < n and _act_of(mods[j]) is not None:
                act, slope = _act_of(mods[j])
                j += 1
            prev = steps[-1] if steps else None
            takes = isinstance(prev, _ConvStep) and prev.stats is not None
            steps.append(_NormStep(m, act, slope, takes))
            i = j
            continue
        steps.append(_LeafStep(m))
        i += 1
    # TF32 operand rounding: producers that feed a tensor-core conv store RN-rounded values
    for k, s in enumerate(steps):
        if isinstance(s, _ConvStep) and s.tc_like():
            if k > 0 and isinstance(steps[k - 1], (_ConvStep, _NormStep)):
                steps[k - 1].rtf_out = True
            if not s.tc_like(full=True):
                continue        # forward only: the gradients of this conv run in fp32
            s.rtf_dz = True
            # A conv with a fused epilogue (activation / Dropout2d) rounds its dz in epilogue_bwd and takes its bias
            # gradient from the unrounded values; only a conv WITHOUT epilogue consumes the norm's dx directly, and
            # only then does the norm backward store TF32-rounded values (that conv's bias gradient is exactly zero
            # anyway: it sits in front of the norm).
            if (k + 1 < len(steps) and isinstance(steps[k + 1], _NormStep) and s.act == ACT_NONE
                    and s.dropout2d is None):
                steps[k + 1].rtf_dx = True
    steps = _fuse_chains(steps)
    # the Generator tail: norm + narrow 3x3 conv as one fused node
    fused, k = [], 0
    while k < len(steps):
        if k + 1 < len(steps) and _tail_candidate(steps[k], steps[k + 1]):
            fused.append(_TailStep(steps[k], steps[k + 1]))
            k += 2
        else:
            fused.append(steps[k])
            k += 1
    return fused


def mlp_critic_layers(mods, in_features):
    """(Linear 1, Linear 2, Linear 3, slope) if the module list `mods` is exactly the MLP critic of wgan_gp.py:72-78 /
    wgan_div.py:72-78 -- Linear(in_features, H1) -> LeakyReLU(s) -> Linear(H1, H2) -> LeakyReLU(s) -> Linear(H2, 1), all
    with biases, one slope -- which runs as functional.MlpCriticFn; else None.  No side effects."""
    def plain(m, name):  # the stock class or its drop-in, with no hooks that calling the module would run
        return (type(m) in (_T[name], REPLACEMENTS[name]) and not m._forward_hooks and not m._forward_pre_hooks
                and not m._backward_hooks)

    if len(mods) != 5 or not all(plain(mods[i], "Linear") for i in (0, 2, 4)):
        return None
    if not all(plain(mods[i], "LeakyReLU") for i in (1, 3)):
        return None
    l1, l2, l3 = mods[0], mods[2], mods[4]
    if any(m.bias is None for m in (l1, l2, l3)) or mods[1].negative_slope != mods[3].negative_slope:
        return None
    if l1.in_features != in_features or l2.in_features != l1.out_features or l3.in_features != l2.out_features:
        return None
    if l3.out_features != 1:
        return None
    return l1, l2, l3, float(mods[1].negative_slope)


def mlp_discriminator_layers(mods, in_features):
    """(Linear 1, Linear 2, Linear 3, slope) if the module list `mods` is exactly the vanilla GAN discriminator of
    gan.py:64-80 / bgan.py:66-80 / aae.py:90-104 -- the critic mlp_critic_layers accepts, with a slope >= 0, followed by
    a Sigmoid -- which runs as functional.MlpDiscriminatorFn; else None.  Stock or drop-in classes only, without hooks.
    No side effects."""
    if len(mods) != 6:
        return None
    sig = mods[5]
    if (type(sig) not in (_T["Sigmoid"], REPLACEMENTS["Sigmoid"]) or sig._forward_hooks or sig._forward_pre_hooks
            or sig._backward_hooks):
        return None
    critic = mlp_critic_layers(mods[:5], in_features)
    if critic is None or critic[3] < 0:
        return None
    return critic


def mlp_generator_layers(mods, in_features):
    """([(Linear, BatchNorm1d or None)], slope) if the module list `mods` is the MLP generator of wgan_gp.py:42-65 /
    gan.py:38-61 -- [Linear -> (BatchNorm1d)? -> LeakyReLU(s)] x (L - 1), Linear -> Tanh, at most 8 Linears of at most
    8192 features, all with biases, chained widths from in_features, one slope >= 0 -- which runs as
    functional.MlpGeneratorFn; else None.  Every BatchNorm1d is in training mode, affine, with tracked running statistics and a momentum (not None), all with
    one eps and one momentum: what the kernels compute.  A last Linear with one output stays with the Linear(K, 1) + Tanh
    head kernel.  Stock or drop-in classes only, without hooks.  No side effects."""
    def plain(m, name):  # the stock class or its drop-in, with no hooks that calling the module would run
        return (type(m) in (_T[name], REPLACEMENTS[name]) and not m._forward_hooks and not m._forward_pre_hooks
                and not m._backward_hooks)

    layers, slopes, norms, i, width = [], set(), [], 0, in_features
    while i < len(mods):
        lin = mods[i]
        if not plain(lin, "Linear") or lin.bias is None or lin.in_features != width:
            return None
        width, i = lin.out_features, i + 1
        if i + 1 == len(mods):  # the output layer
            if not plain(mods[i], "Tanh") or width == 1:
                return None
            layers.append((lin, None))
            break
        bn = None
        if i < len(mods) and plain(mods[i], "BatchNorm1d"):
            bn = mods[i]
            if not (bn.training and bn.affine and bn.track_running_stats and bn.running_mean is not None
                    and bn.momentum is not None and bn.num_features == width):
                return None
            norms.append((bn.eps, bn.momentum))
            i += 1
        if i >= len(mods) or not plain(mods[i], "LeakyReLU"):
            return None
        slopes.add(mods[i].negative_slope)
        layers.append((lin, bn))
        i += 1
    else:
        return None
    widths = [in_features] + [lin.out_features for lin, _ in layers]
    if len(layers) > _lib.MLP_GEN_MAX_LAYERS or max(widths) > _lib.MLP_GEN_MAX_WIDTH:
        return None
    if len(slopes) > 1 or len(set(norms)) > 1:
        return None
    slope = slopes.pop() if slopes else 0.0
    if slope < 0:
        return None
    return layers, float(slope)


class Sequential(_T["Sequential"]):
    def _plan(self):
        mods = list(self._modules.values())
        key = tuple(id(m) for m in mods) + (ops.Config.algo,)
        cached = self.__dict__.get("_b200_plan")
        if cached is None or cached[0] != key:
            cached = (key, _build_plan(mods))
            self.__dict__["_b200_plan"] = cached
        return cached[1]

    def _run_chain(self, chain, x, nchw_out):
        """Execute a _ChainStep through the fused kernels, or return None if the runtime shapes do not qualify."""
        if not ops.Config.fuse_narrow_chain:
            return None
        shape = tuple(x.shape)
        plan = _chain_plan(chain, shape)
        if plan is None:
            return None
        groups = ops.bn_groups.active
        if groups > 1 and shape[0] % groups != 0:
            raise RuntimeError("b200gan: ops.bn_groups: the batch does not split evenly into the groups")
        # Dropout2d masks.  One pass: drawn layer by layer as F.dropout2d does.  G statistics groups = G forward passes of
        # the reference: pass 0 draws all its layers' masks, then pass 1, ... -- drawn up front in that order.
        scales = [None] * len(plan)
        for gq in range(groups):
            for li, (cs, ns, oshape) in enumerate(plan):
                if cs.dropout2d is not None and cs.dropout2d.training and cs.dropout2d.p > 0.0:
                    part = _dropout2d_scale((x.shape[0] // groups, cs.conv.out_channels), cs.dropout2d.p, x.device)
                    scales[li] = part if scales[li] is None else torch.cat([scales[li], part])
        edge, prev_norm = None, None
        chain = F.ChainPass()
        for li, (cs, ns, oshape) in enumerate(plan):
            conv = cs.conv
            scale = scales[li]
            gam = bet = rm = rv = nbt = None
            momentum = 0.0
            if prev_norm is not None:
                gam, bet = prev_norm.weight, prev_norm.bias
                if prev_norm.track_running_stats and prev_norm.running_mean is not None:
                    rm, rv, nbt = prev_norm.running_mean, prev_norm.running_var, prev_norm.num_batches_tracked
                    momentum = float(prev_norm.momentum)
            spec = F.NbSpec(stride=int(conv.stride[0]), pad=int(conv.padding[0]), act=cs.act, slope=cs.slope,
                            momentum=momentum, want_stats=ns is not None, groups=groups)
            cache = conv.__dict__.get("_b200_cache")
            if cache is None:
                cache = PackCache()
                conv.__dict__["_b200_cache"] = cache
            out_box = []
            res = F.NbConvFn.apply(x, conv.weight, conv.bias, scale, gam, bet, rm, rv, nbt, edge, out_box, spec, cache,
                                   chain)
            if ns is not None:
                x, stats = res
                norm = ns.norm
                edge = ops.BnEdge(stats, None if norm.weight is None else norm.weight.detach(),
                                  None if norm.bias is None else norm.bias.detach(), norm.eps,
                                  oshape[0] // groups * oshape[2] * oshape[3], groups)
                out_box.append(edge)
                prev_norm = norm
            else:
                x, edge, prev_norm = res, None, None
        if edge is not None:
            norm = prev_norm
            rm = rv = nbt = None
            momentum = 0.0
            if norm.track_running_stats and norm.running_mean is not None:
                rm, rv, nbt, momentum = norm.running_mean, norm.running_var, norm.num_batches_tracked, float(norm.momentum)
            x = F.NbTailFn.apply(x, norm.weight, norm.bias, rm, rv, nbt, edge, momentum, bool(nchw_out), chain)
        return x

    def _forward_2d(self, x):
        """Matrix input: the whole MLP critic (wgan_gp.py:72-78), the whole vanilla GAN discriminator (gan.py:64-80), the
        MLP generator, or Linear(K, 1) + activation (the adv_layer of a discriminator, dcgan.py:92) as one node."""
        mods = list(self._modules.values())
        critic = mlp_critic_layers(mods, x.shape[1])
        if critic is not None and x.shape[0] >= 1:
            return F.mlp_critic(x, *critic)
        disc = mlp_discriminator_layers(mods, x.shape[1])
        if disc is not None and x.shape[0] >= 1:
            return F.mlp_discriminator(x, *disc)
        gen = mlp_generator_layers(mods, x.shape[1])
        # one row with a norm: the stock BatchNorm1d raises torch's own ValueError on the leaf-by-leaf path below
        if gen is not None and (x.shape[0] >= 2 or all(bn is None for _, bn in gen[0])) \
                and x.shape[0] <= _lib.MLP_GEN_MAX_N:
            return F.mlp_generator(x, *gen)
        i = 0
        while i < len(mods):
            m = mods[i]
            if (isinstance(m, _T["Linear"]) and m.out_features == 1 and _gpu2d_f32(x) and x.shape[0] <= 4096
                    and i + 1 < len(mods) and _act_of(mods[i + 1]) is not None
                    and _act_of(mods[i + 1])[0] in (ACT_SIGMOID, ACT_TANH)):
                x = F.Linear1Fn.apply(x, m.weight, m.bias, _act_of(mods[i + 1])[0])
                i += 2
            else:
                x = m(x)
                i += 1
        return x

    def forward(self, x):
        if _gpu2d_f32(x):
            return self._forward_2d(x)
        if not (torch.is_tensor(x) and x.dim() == 4 and _on_device(x) and x.dtype == torch.float32):
            return super().forward(x)
        steps = self._plan()
        if all(isinstance(s, _LeafStep) for s in steps):
            return _T["Sequential"].forward(self, x)
        # Output memory format follows the input's -- the scripts .view() conv outputs only where they are small
        # (dcgan.py:96: [N,128,4,4] -> [N,2048]); large maps stay NHWC so that U-Net / ResNet blocks chain and
        # torch.cat (pix2pix/models.py:50) without a layout round trip per block.
        want_contiguous = x.is_contiguous()
        stats = None
        queue = list(steps)
        while queue:
            s = queue.pop(0)
            if isinstance(s, _ChainStep):
                at_end = not queue
                res = self._run_chain(s, x, want_contiguous and at_end)
                if res is None:
                    _no_groups("a conv chain that does not qualify for the fused kernels")
                    queue[0:0] = s.steps
                else:
                    x, stats = res, None
                    if at_end and want_contiguous and x.is_contiguous():
                        return x
                continue
            if isinstance(s, _TailStep):
                ns, cs = s.norm_step, s.conv_step
                norm, conv = ns.norm, cs.conv
                _no_groups("the fused generator tail")
                if (norm.training and x.shape[1] == conv.in_channels and x.shape[1] == norm.num_features
                        and ops.tail_supported(tuple(x.shape), conv.out_channels, ns.act, ns.slope, cs.act)):
                    rm = rv = nbt = None
                    momentum = 0.0
                    if norm.track_running_stats and norm.running_mean is not None:
                        if norm.momentum is None:
                            raise NotImplementedError("b200gan: BatchNorm2d(momentum=None)")
                        rm, rv, nbt, momentum = norm.running_mean, norm.running_var, norm.num_batches_tracked, float(norm.momentum)
                    spec = F.TailSpec(eps=float(norm.eps), momentum=momentum, act_mid=ns.act, slope=ns.slope,
                                      act_out=cs.act, rtf_dx=ns.rtf_dx)
                    x = F.TailFn.apply(x, stats if ns.takes_stats else None, norm.weight, norm.bias, rm, rv, nbt,
                                       conv.weight, conv.bias, spec)
                    stats = None
                else:
                    queue[0:0] = [ns, cs]
                continue
            if queue and _norm_conv_fused(s, queue[0], tuple(x.shape)):
                # one node whose backward takes the norm's sums from the conv's data-gradient epilogue
                ns, cs = s, queue.pop(0)
                scale = None
                if cs.dropout2d is not None and cs.dropout2d.training and cs.dropout2d.p > 0.0:
                    scale = _dropout2d_scale((x.shape[0], cs.conv.out_channels), cs.dropout2d.p, x.device)
                want = cs.stats if (cs.next_norm is not None and _uses_batch_stats(cs.next_norm)) else None
                norm, conv = ns.norm, cs.conv
                nspec, rm, rv, nbt = _batch_norm_spec(norm, False, ns.act, ns.slope, ns.rtf_out, ns.rtf_dx)
                cspec = ConvSpec(stride=1, pads=tuple(e + int(conv.padding[0]) for e in cs.extra_pads), up=cs.up,
                                 act=cs.act, slope=cs.slope, stats=want, rtf_out=cs.rtf_out, rtf_dz=cs.rtf_dz)
                out = F.NormConvFn.apply(x, norm.weight, norm.bias, stats if ns.takes_stats else None, rm, rv, nbt,
                                         conv.weight, conv.bias, scale, nspec, cspec, _conv_cache(conv))
                x, stats = out if want is not None else (out, None)
                continue
            if isinstance(s, _ConvStep):
                cs = None
                if s.dropout2d is not None and s.dropout2d.training and s.dropout2d.p > 0.0:
                    _no_groups("a Dropout2d outside a fused chain")
                    n = x.shape[0]
                    cs = _dropout2d_scale((n, s.conv.out_channels), s.dropout2d.p, x.device)
                # fused statistics only when the following norm really normalises with batch statistics (an eval-mode
                # BatchNorm2d never consumes -- and so never re-zeroes -- the shared accumulator)
                want = s.stats if (s.next_norm is not None and _uses_batch_stats(s.next_norm)) else None
                out = _run_conv(s.conv, x, s.up, s.extra_pads, s.pad_mode, s.act, s.slope, cs, want, s.rtf_out,
                                s.rtf_dz)
                if want is not None:
                    x, stats = out
                else:
                    x, stats = out, None
            elif isinstance(s, _NormStep):
                x = _run_norm(s.norm, x, s.act, s.slope, stats if s.takes_stats else None, s.rtf_out, s.rtf_dx)
                stats = None
            else:
                x = s.mod(x)
                stats = None
        if (want_contiguous and torch.is_tensor(x) and x.dim() == 4 and not x.is_contiguous()
                and x.shape[2] * x.shape[3] <= ops.Config.contiguous_hw_limit):
            x = F.ToContiguousFn.apply(x)
        return x


REPLACEMENTS = {
    "Conv2d": Conv2d, "ConvTranspose2d": ConvTranspose2d, "BatchNorm2d": BatchNorm2d,
    "InstanceNorm2d": InstanceNorm2d, "LeakyReLU": LeakyReLU, "ReLU": ReLU, "Tanh": Tanh, "Sigmoid": Sigmoid,
    "Upsample": Upsample, "ZeroPad2d": ZeroPad2d, "ReflectionPad2d": ReflectionPad2d, "Dropout": Dropout,
    "Dropout2d": Dropout2d, "Sequential": Sequential, "Linear": Linear, "BCELoss": BCELoss, "BatchNorm1d": BatchNorm1d,
    "MSELoss": MSELoss, "L1Loss": L1Loss,
}
for _n, _c in REPLACEMENTS.items():
    _c.__name__ = _n
    _c.__qualname__ = _n
