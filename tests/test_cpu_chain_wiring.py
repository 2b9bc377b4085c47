"""Host-side logic of the fused narrow conv chain WITHOUT a GPU: the planner (nn._ChainStep and its run) and the
autograd protocol of functional.NbConvFn / NbTailFn -- virtual gradients w.r.t. the never-materialised BatchNorm outputs,
the `sums` hand-over between neighbouring layers, dgamma / dbeta routing, frozen weights, two passes accumulating -- are
run on CPU with the six C entry points (b200gan_nb_*) replaced by torch restatements of what each kernel computes
(csrc/narrow_block.cu).  What this pins is the Python wiring and the algebra of the chain; the CUDA kernels themselves are
checked by tests/test_gpu_chain.py."""
import pytest
import torch
import torch.nn.functional as tf

from conftest import rel_err

CL = torch.channels_last


def _bn_consts(edge):
    c = edge.stats.numel() // 2
    mean = edge.stats[:c] / edge.count
    var = (edge.stats[c:] / edge.count - mean * mean).clamp_min(0)
    rstd = 1.0 / torch.sqrt(var + edge.eps)
    gamma = edge.gamma.double() if edge.gamma is not None else torch.ones(c, dtype=torch.float64)
    beta = edge.beta.double() if edge.beta is not None else torch.zeros(c, dtype=torch.float64)
    sc = gamma * rstd
    return mean, var, rstd, sc, beta - mean * sc


def _update_running(edge, rm, rv, nbt, momentum):
    if rm is None:
        return
    mean, var, _, _, _ = _bn_consts(edge)
    unbiased = var * edge.count / (edge.count - 1.0) if edge.count > 1 else var
    rm.mul_(1 - momentum).add_(momentum * mean.float())
    rv.mul_(1 - momentum).add_(momentum * unbiased.float())
    if nbt is not None:
        nbt.add_(1)


def _act(v, act, slope):
    return tf.leaky_relu(v, slope) if act == 1 else (torch.relu(v) if act == 2 else v)


@pytest.fixture
def emulated(monkeypatch):
    from b200gan import functional as F, nn as bnn, ops

    def nb_supported(g):
        return True

    def norm_in(x, edge):
        if edge is None:
            return x.double()
        _, _, _, sc, sh = _bn_consts(edge)
        return x.double() * sc.view(1, -1, 1, 1) + sh.view(1, -1, 1, 1)

    def nb_fprop(g, x, weight, bias, act, slope, chan_scale, in_edge, rm, rv, nbt, momentum, want_stats, groups=1):
        assert groups == 1   # the grouped pass is a GPU-kernel feature (tests/test_gpu_chain.py)
        if in_edge is not None:
            _update_running(in_edge, rm, rv, nbt, momentum)
        z = tf.conv2d(norm_in(x, in_edge), weight.double(), None if bias is None else bias.double(), g.stride, g.pad_t)
        y = _act(z, act, slope)
        if chan_scale is not None:
            y = y * chan_scale.double().view(y.shape[0], y.shape[1], 1, 1)
        stats = torch.cat([y.sum((0, 2, 3)), (y * y).sum((0, 2, 3))]) if want_stats else None
        return y.float().contiguous(memory_format=CL), stats

    def nb_dz(g_in, a, chan_scale, act, slope, out_edge, want_db):
        G, A = g_in.double(), a.double()
        dA = G
        if out_edge is not None:
            mean, _, rstd, sc, _ = _bn_consts(out_edge)
            k = mean.numel()
            m1 = (out_edge.sums[:k] / out_edge.count).view(1, -1, 1, 1)
            m2 = (out_edge.sums[k:] / out_edge.count).view(1, -1, 1, 1)
            ahat = (A - mean.view(1, -1, 1, 1)) * rstd.view(1, -1, 1, 1)
            dA = sc.view(1, -1, 1, 1) * (G - m1 - ahat * m2)
        grad = torch.where(A > 0, 1.0, slope) if act == 1 else ((A > 0).double() if act == 2 else torch.ones_like(A))
        dz = dA * grad
        if chan_scale is not None:
            dz = dz * chan_scale.double().view(A.shape[0], A.shape[1], 1, 1)
        return dz.float().contiguous(memory_format=CL), (dz.sum((0, 2, 3)).float() if want_db else None)

    def nb_wgrad(g, x, dz, in_edge, weight_shape):
        xin = norm_in(x, in_edge)
        return torch.nn.grad.conv2d_weight(xin, weight_shape, dz.double(), stride=g.stride, padding=g.pad_t).float()

    def nb_dgrad(g, dz, weight, in_edge, a_prev):
        gx = torch.nn.grad.conv2d_input((g.N, g.C, g.H, g.W), weight.double(), dz.double(), stride=g.stride, padding=g.pad_t)
        sums = None
        if in_edge is not None:
            mean, _, rstd, _, _ = _bn_consts(in_edge)
            ahat = (a_prev.double() - mean.view(1, -1, 1, 1)) * rstd.view(1, -1, 1, 1)
            sums = torch.cat([gx.sum((0, 2, 3)), (gx * ahat).sum((0, 2, 3))])
        return gx.float().contiguous(memory_format=CL), sums

    def nb_tail_fwd(a, edge, rm, rv, nbt, momentum, nchw):
        _update_running(edge, rm, rv, nbt, momentum)
        out = norm_in(a, edge).float()
        return out.contiguous() if nchw else out.contiguous(memory_format=CL)

    def nb_tail_bwd(a, edge, dout, nchw):
        mean, _, rstd, _, _ = _bn_consts(edge)
        ahat = (a.double() - mean.view(1, -1, 1, 1)) * rstd.view(1, -1, 1, 1)
        gd = dout.double()
        return dout.float().contiguous(memory_format=CL), torch.cat([gd.sum((0, 2, 3)), (gd * ahat).sum((0, 2, 3))])

    class RawCache:  # the emulation consumes the parameter itself, whatever layout a kernel would have wanted
        def get(self, g, w, kind):
            return w

    for name, fn in dict(nb_supported=nb_supported, nb_fprop=nb_fprop, nb_dz=nb_dz, nb_wgrad=nb_wgrad, nb_dgrad=nb_dgrad,
                         nb_tail_fwd=nb_tail_fwd, nb_tail_bwd=nb_tail_bwd).items():
        monkeypatch.setattr(ops, name, fn)
    monkeypatch.setattr(ops, "_require_cuda", lambda t, name="tensor": None)
    monkeypatch.setattr(ops, "to_cl", lambda x: x.contiguous(memory_format=CL))
    monkeypatch.setattr(ops, "to_nchw", lambda x: x.contiguous())
    monkeypatch.setattr(bnn, "_on_device", lambda x: True)
    monkeypatch.setattr(bnn, "PackCache", RawCache)
    monkeypatch.setattr(ops.Config, "fuse_narrow_chain", True)
    return bnn


def _disc(ns, chans, p):
    layers = []
    for i, (cin, cout) in enumerate(zip(chans[:-1], chans[1:])):
        layers += [ns.Conv2d(cin, cout, 3, 2, 1), ns.LeakyReLU(0.2, inplace=True), ns.Dropout2d(p)]
        if i > 0:
            layers.append(ns.BatchNorm2d(cout, 0.8))
    return ns.Sequential(*layers)


def _pair(chans, p):
    from b200gan import zoo
    torch.manual_seed(5)
    ref = _disc(zoo.namespace(stock=True), chans, p).train()
    ours = _disc(zoo.namespace(), chans, p).train()
    with torch.no_grad():
        for m in ref.modules():
            if isinstance(m, torch.nn.BatchNorm2d):
                m.weight.normal_(1.0, 0.2)
                m.bias.normal_(0.0, 0.2)
    ours.load_state_dict(ref.state_dict())
    return ref, ours


@pytest.mark.parametrize("p", [0.0, 0.25])
def test_chain_wiring_matches_stock_autograd(emulated, p):
    ref, ours = _pair((1, 16, 32, 64), p)
    assert [type(s).__name__ for s in ours._plan()] == ["_ChainStep"]
    for step in range(2):
        x = torch.randn(6, 1, 32, 32)
        xr, xo = x.clone().requires_grad_(True), x.clone().requires_grad_(True)
        torch.manual_seed(70 + step)
        yr = ref(xr)
        torch.manual_seed(70 + step)
        yo = ours(xo)
        assert yo.is_contiguous() and rel_err(yo, yr) < 1e-5          # NCHW out: the script .view()s it (dcgan.py:96)
        gy = torch.randn_like(yr)
        ref.zero_grad(); ours.zero_grad()
        yr.backward(gy)
        yo.backward(gy)
        assert rel_err(xo.grad, xr.grad) < 1e-5
        for (name, po), (_, pr) in zip(ours.named_parameters(), ref.named_parameters()):
            assert rel_err(po.grad, pr.grad) < 1e-5, name
        for (name, bo), (_, br) in zip(ours.named_buffers(), ref.named_buffers()):
            assert rel_err(bo.float(), br.float()) < 1e-5, name


def test_chain_wiring_frozen_weights_and_accumulation(emulated):
    from b200gan import train
    ref, ours = _pair((1, 16, 32, 64), 0.0)
    x = torch.randn(4, 1, 32, 32)
    xr, xo = x.clone().requires_grad_(True), x.clone().requires_grad_(True)
    with train.frozen(ref), train.frozen(ours):                       # generator step: input gradient only
        ref(xr).square().mean().backward()
        ours(xo).square().mean().backward()
    assert rel_err(xo.grad, xr.grad) < 1e-5 and all(q.grad is None for q in ours.parameters())
    a, b = torch.randn(4, 1, 32, 32), torch.randn(4, 1, 32, 32)       # d_loss = f(D(real)) + f(D(fake)): two passes
    for net in (ref, ours):
        (net(a).mean() + net(b).square().mean()).backward()
    for (name, po), (_, pr) in zip(ours.named_parameters(), ref.named_parameters()):
        assert rel_err(po.grad, pr.grad) < 1e-5, name


def test_chain_falls_back_when_a_norm_is_in_eval_mode(emulated, monkeypatch):
    """eval-mode BatchNorm inside the run: the chain must not be taken (the ordinary steps run; on CPU they raise the
    product path's 'no CPU fallback' error, which is the evidence that the fallback branch was chosen)."""
    from b200gan import ops
    monkeypatch.setattr(ops, "_require_cuda", lambda t, name="tensor": (_ for _ in ()).throw(RuntimeError("fell back")))
    _, ours = _pair((1, 16, 32, 64), 0.0)
    ours.eval()
    with pytest.raises(RuntimeError, match="fell back"):
        ours(torch.randn(2, 1, 32, 32))
