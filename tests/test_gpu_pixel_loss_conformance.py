"""MSELoss / L1Loss (reduction 'mean') on the pixel-loss kernels (csrc/pixel_loss/) element by element
against fp64, and the drop-in modules end to end against stock fp32.

For every case of tests/pixel_loss_cases.py, through ops: the loss within 1e-6 relative of fp64, each gradient element
within 4 units of 2^-24 relative of fp64, CUDA-graph replays bit-identical to the eager run, and exactly the table's
kernels and grids (tests/conformance.py's check_route)."""
import os

import pytest
import torch

from conformance import check_route
from conftest import rel_err
from pixel_loss_cases import CASES, GOUT, GRAD_TOL, KERNEL, MODES, fwd_grid, grad_ref, loss_ref, make

pytestmark = pytest.mark.gpu


def _run(case, a, b, gout):
    from b200gan import ops
    loss = ops.pixel_loss_fwd(a, b, MODES[case.mode])
    da, db = ops.pixel_loss_bwd(a, b, gout, MODES[case.mode], case.want_db)
    return loss, da, db


def _check_grad(got, want, what):
    got, want = got.double().cpu(), want.cpu()
    err = (got - want).abs()
    bad = err > GRAD_TOL * want.abs()
    assert not bad.any(), f"{what}: {int(bad.sum())} elements off, worst {float(err.max()):.3e}"


def _ticket(device):
    """the forward workspace's completion ticket (its first word), which every call leaves at zero"""
    from b200gan import ops
    return int(ops._pixel_ws[device][:4].view(torch.int32).item())


# ---- the case table --------------------------------------------------------------------------------------------------
def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.mark.parametrize("case", CASES, ids=lambda c: c.id)
def test_case_against_fp64(case):
    a, b = make(case)
    gout = torch.tensor(GOUT, device="cuda")
    loss, da, db = _run(case, a, b, gout)
    torch.cuda.synchronize()
    assert _ticket(a.device) == 0, "the forward left its completion ticket set"
    want = loss_ref(a.cpu(), b.cpu(), case.mode).item()
    if want == 0.0:
        assert loss.item() == 0.0
    else:
        assert abs(loss.item() - want) <= 1e-6 * abs(want), (loss.item(), want)
    g = grad_ref(a.cpu(), b.cpu(), GOUT, case.mode)
    assert da.stride() == a.stride() and da.shape == a.shape
    _check_grad(da, g, "d_input")
    if case.want_db:
        assert db.stride() == b.stride()
        _check_grad(db, -g, "d_target")
    else:
        assert db is None
    if case.equal:
        assert da.eq(0).all() and (db is None or db.eq(0).all())

    # CUDA-graph replay: bit-identical to the eager run, twice (the ticket is back at zero after each replay)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        _run(case, a, b, gout)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        static = _run(case, a, b, gout)
    for _ in range(2):
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(static[0], loss) and torch.equal(static[1], da)
        assert db is None or torch.equal(static[2], db)

    assert _ticket(a.device) == 0

    # the table's kernels and grids, nothing else of this family
    check_route(case.id, lambda: _run(case, a, b, gout), case.kernels(_sms()), family=tuple(KERNEL.values()))
    assert _ticket(a.device) == 0


def test_c_abi_refuses_bad_arguments():
    import ctypes
    from b200gan import _lib
    lib = _lib.load()
    a = torch.randn(64, device="cuda")
    b = torch.randn(64, device="cuda")
    loss = torch.empty((), device="cuda")
    ws = torch.zeros(16 + 8 * 1024, device="cuda", dtype=torch.uint8)
    gout = torch.ones((), device="cuda")
    da = torch.empty_like(a)
    s = torch.cuda.current_stream().cuda_stream

    def desc(**kw):
        d = _lib.PixelLossDesc()
        d.mode, d.layout_a, d.layout_b, d.n, d.N, d.C, d.H, d.W = 0, 0, 0, 64, 1, 1, 1, 64
        for k, v in kw.items():
            setattr(d, k, v)
        return d

    def fwd(d, a_=a.data_ptr(), b_=b.data_ptr(), l_=loss.data_ptr(), w_=ws.data_ptr()):
        return lib.b200gan_pixel_loss_fwd(ctypes.byref(d), a_, b_, l_, w_, s)

    def bwd(d, a_=a.data_ptr(), b_=b.data_ptr(), g_=gout.data_ptr(), da_=da.data_ptr()):
        return lib.b200gan_pixel_loss_bwd(ctypes.byref(d), a_, b_, g_, da_, None, s)

    BAD, UNSUPPORTED = -2, -1
    assert fwd(desc()) == 0 and bwd(desc()) == 0
    for what, d in {"n = 0": desc(n=0, W=0), "unknown mode": desc(mode=2), "unknown input layout": desc(layout_a=2),
                    "unknown target layout": desc(layout_b=-1), "shape does not hold n": desc(W=32),
                    "zero extent": desc(N=0)}.items():
        assert fwd(d) == BAD, what
        assert bwd(d) == BAD, what
        assert lib.b200gan_pixel_loss_workspace_bytes(ctypes.byref(d)) == 0, what
    assert fwd(desc(n=2 ** 31, N=2, C=1024, H=1024, W=1024)) == UNSUPPORTED
    for slot in ("a_", "b_", "l_", "w_"):
        assert fwd(desc(), **{slot: None}) == BAD, slot
    assert fwd(desc(), w_=ws.data_ptr() + 8) == BAD, "misaligned workspace"
    for slot in ("a_", "b_", "g_", "da_"):
        assert bwd(desc(), **{slot: None}) == BAD, slot
    assert lib.b200gan_pixel_loss_fwd(None, a.data_ptr(), b.data_ptr(), loss.data_ptr(), ws.data_ptr(), s) == BAD
    assert lib.b200gan_pixel_loss_workspace_bytes(ctypes.byref(desc())) == 16 + 8 * fwd_grid(64, _sms())[0]
    torch.cuda.synchronize()
    assert abs(loss.item() - loss_ref(a.cpu(), b.cpu(), "mse").item()) <= 1e-6 * loss.item()


# ---- end to end against stock fp32 -----------------------------------------------------------------------------------
def _set_tf32(on):
    torch.backends.cudnn.allow_tf32 = on
    torch.backends.cuda.matmul.allow_tf32 = on


def _pix2pix_g_loss(d, mse, l1, fake, real_a, real_b):
    """pix2pix.py:141-148: the generator's loss at a fake image (a leaf here, so that dx is its gradient)"""
    pred = d(fake, real_a)
    valid = torch.ones_like(pred)
    loss = mse(pred, valid) + 100.0 * l1(fake, real_b)
    loss.backward()
    return loss.detach(), fake.grad.detach().clone(), [(k, p.grad.detach().clone()) for k, p in d.named_parameters()]


def test_pix2pix_generator_loss_against_stock_fp32():
    """MSE(D(fake, a), valid) + 100 L1(fake, real): the loss, dx and every parameter gradient of D.  With the stock
    discriminator only the two losses differ (tight); with the drop-in discriminator its TF32 convolutions set the
    yardstick, as in test_gpu_baseline_configs."""
    import copy
    from b200gan import nn as bnn, zoo
    n, size = 4, 64
    gen = torch.Generator().manual_seed(3)
    real_a, real_b, fake0 = [torch.rand(n, 3, size, size, generator=gen).mul(2).sub(1).cuda() for _ in range(3)]
    fake0 = fake0.contiguous(memory_format=torch.channels_last)   # a drop-in generator's output layout
    torch.manual_seed(0)
    d_stock = zoo.Pix2PixDiscriminator(nn=zoo.namespace(stock=True)).cuda()
    d_stock.apply(zoo.weights_init_normal)
    _set_tf32(False)
    ref = _pix2pix_g_loss(copy.deepcopy(d_stock), torch.nn.MSELoss(), torch.nn.L1Loss(),
                          fake0.clone().requires_grad_(True), real_a, real_b)
    # stock D: only the losses change
    ours = _pix2pix_g_loss(copy.deepcopy(d_stock), bnn.MSELoss(), bnn.L1Loss(), fake0.clone().requires_grad_(True),
                           real_a, real_b)
    assert abs(ours[0].item() - ref[0].item()) <= 1e-6 * abs(ref[0].item())
    assert rel_err(ours[1], ref[1]) < 1e-6, "dx"
    for (k, go), (_, gr) in zip(ours[2], ref[2]):
        assert rel_err(go, gr) < 1e-5, k
    # drop-in D and losses against stock fp32, yardstick stock TF32
    _set_tf32(True)
    tf32 = _pix2pix_g_loss(copy.deepcopy(d_stock), torch.nn.MSELoss(), torch.nn.L1Loss(),
                           fake0.clone().requires_grad_(True), real_a, real_b)
    _set_tf32(False)
    d_ours = zoo.Pix2PixDiscriminator().cuda()
    d_ours.load_state_dict(d_stock.state_dict())
    full = _pix2pix_g_loss(d_ours, bnn.MSELoss(), bnn.L1Loss(), fake0.clone().requires_grad_(True), real_a, real_b)
    assert abs(full[0].item() - ref[0].item()) <= max(1e-3, 1.5 * abs(tf32[0].item() - ref[0].item())) * ref[0].item()
    top = max(r.double().norm().item() for _, r in ref[2])
    for what, o, r, t in [("dx", full[1], ref[1], tf32[1])] + [(k, o, r, t) for (k, o), (_, r), (_, t) in
                                                               zip(full[2], ref[2], tf32[2])]:
        if r.double().norm().item() < 1e-5 * top:  # conv bias in front of InstanceNorm2d: zero gradient, fp noise only
            continue
        assert rel_err(o, r) < max(2e-3, 1.5 * rel_err(t, r)), what


@pytest.mark.parametrize("mode", ["mse", "l1"])
def test_create_graph_backward_through_the_dropin_loss(mode):
    """a gradient penalty through the loss (autograd.grad(create_graph=True), then backward) matches stock fp32"""
    from b200gan import nn as bnn
    gen = torch.Generator().manual_seed(5)
    x0 = torch.randn(2, 3, 8, 8, generator=gen).cuda().contiguous(memory_format=torch.channels_last)
    t = torch.randn(2, 3, 8, 8, generator=gen).cuda()
    w = torch.randn(3, 3, 3, 3, generator=gen).cuda()

    def run(loss_mod):
        x = x0.clone().requires_grad_(True)
        wp = w.clone().requires_grad_(True)
        y = torch.nn.functional.conv2d(x, wp, padding=1).tanh()
        loss = loss_mod(y, t)
        gx, = torch.autograd.grad(loss, x, create_graph=True)
        total = loss + 10.0 * gx.pow(2).sum()
        total.backward()
        return total.detach(), x.grad, wp.grad

    stock = torch.nn.MSELoss() if mode == "mse" else torch.nn.L1Loss()
    ours = bnn.MSELoss() if mode == "mse" else bnn.L1Loss()
    assert bnn.pixel_loss_routed(x0, t, "mean")
    _set_tf32(False)
    r, o = run(stock), run(ours)
    assert abs(o[0].item() - r[0].item()) <= 1e-5 * abs(r[0].item())
    assert rel_err(o[1], r[1]) < 1e-5 and rel_err(o[2], r[2]) < 1e-5


def test_reference_idiom_lsgan_script_under_the_launcher_on_cuda(monkeypatch):
    """launch.run() of tests/scripts/mini_lsgan (conv critic, nn.MSELoss(), an nn.L1Loss pixel term) on the GPU: stock
    torch against the drop-ins, same seeds: the printed losses agree and the patched run used the pixel-loss kernels"""
    from b200gan import launch, ops
    calls = {"fwd": 0, "bwd": 0}
    fwd, bwd = ops.pixel_loss_fwd, ops.pixel_loss_bwd

    def count_fwd(*a, **k):
        calls["fwd"] += 1
        return fwd(*a, **k)

    def count_bwd(*a, **k):
        calls["bwd"] += 1
        return bwd(*a, **k)
    monkeypatch.setattr(ops, "pixel_loss_fwd", count_fwd)
    monkeypatch.setattr(ops, "pixel_loss_bwd", count_bwd)
    script = os.path.join(os.path.dirname(os.path.abspath(__file__)), "scripts", "mini_lsgan", "mini_lsgan.py")
    args = ["--epochs", "1", "--batch_size", "16"]
    ref = launch.run(script, args, iters=3, seed=0, stock=True, quiet=True)
    assert calls == {"fwd": 0, "bwd": 0}
    ours = launch.run(script, args, iters=3, seed=0, stock=False, quiet=True)
    # per iteration: G step MSE + L1, D step two MSEs -- four forwards, four backwards
    assert calls == {"fwd": 12, "bwd": 12}

    def losses(run):
        rows = [line for line in run["__b200_stdout__"].splitlines() if "[D " in line]
        return [(float(r.split("[D ")[1].split("]")[0]), float(r.split("[G ")[1].split("]")[0])) for r in rows]
    lr, lo = losses(ref), losses(ours)
    assert len(lr) == len(lo) == 3
    for (dr, gr), (do, go) in zip(lr, lo):
        assert abs(do - dr) < 2e-3 * max(abs(dr), 1.0) and abs(go - gr) < 2e-3 * max(abs(gr), 1.0), (lr, lo)
