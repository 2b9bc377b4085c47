"""MSELoss / L1Loss on the pixel-loss kernels (csrc/pixel_loss/, functional.PixelLossFn) without a GPU:
which calls the drop-in modules route to the kernels and which go to the stock forward, the class names and the patch,
the fp64 references of tests/pixel_loss_cases.py against torch float64 autograd, and the case table against the kernel
source and ptxas."""
import os
import re
import warnings

import pytest
import torch

import pixel_loss_cases as pl
from b200gan import nn as bnn
from conformance import CSRC, declared, functions, needs_nvcc, ptxas_report, source

PL_CU = os.path.join(CSRC, "pixel_loss", "pixel_loss.cu")
PL_CUH = os.path.join(CSRC, "pixel_loss", "pixel_loss_kernels.cuh")
CL = torch.channels_last


# ---- routing ---------------------------------------------------------------------------------------------------------
@pytest.fixture
def on_device(monkeypatch):
    """CPU tensors stand in for CUDA ones: the routing predicate is host logic"""
    monkeypatch.setattr(bnn, "_on_device", lambda t: True)


def _t(*shape, layout="nchw", dtype=torch.float32):
    t = torch.randn(shape, dtype=dtype)
    return t.contiguous(memory_format=CL) if layout == "nhwc" else t


def test_routes_dense_fp32_same_shape_mean(on_device):
    accept = {
        "0-d": (_t(), _t()),
        "1-d": (_t(7), _t(7)),
        "2-d": (_t(16, 1), _t(16, 1)),
        "3-d": (_t(3, 5, 7), _t(3, 5, 7)),
        "4-d nchw": (_t(2, 3, 8, 8), _t(2, 3, 8, 8)),
        "4-d nhwc": (_t(2, 3, 8, 8, layout="nhwc"), _t(2, 3, 8, 8, layout="nhwc")),
        "nhwc / nchw": (_t(2, 3, 8, 8, layout="nhwc"), _t(2, 3, 8, 8)),
        "nchw / nhwc": (_t(2, 3, 8, 8), _t(2, 3, 8, 8, layout="nhwc")),
        "target requires grad": (_t(2, 3, 8, 8), _t(2, 3, 8, 8).requires_grad_(True)),
        "storage offset": (torch.randn(101)[1:].view(4, 25), _t(4, 25)),
    }
    for what, (a, b) in accept.items():
        assert bnn.pixel_loss_routed(a, b, "mean"), what


def test_everything_else_goes_to_stock(on_device):
    x = _t(2, 3, 8, 8)
    reject = {
        "fp64 input": (_t(2, 3, 8, 8, dtype=torch.float64), x, "mean"),
        "fp64 target": (x, _t(2, 3, 8, 8, dtype=torch.float64), "mean"),
        "broadcast target": (x, _t(1, 3, 8, 8), "mean"),
        "broadcast scalar": (x, _t(), "mean"),
        "sum": (x, x, "sum"),
        "none": (x, x, "none"),
        "strided view": (_t(2, 3, 8, 16)[..., ::2], x, "mean"),
        "transposed": (_t(2, 3, 8, 8).transpose(2, 3), x, "mean"),
        "expanded target": (x, _t(1, 3, 8, 8).expand(2, 3, 8, 8), "mean"),
        "5-d": (_t(2, 3, 2, 4, 4), _t(2, 3, 2, 4, 4), "mean"),
        "empty": (_t(0, 3), _t(0, 3), "mean"),
        "not a tensor": (x, 1.0, "mean"),
    }
    for what, (a, b, red) in reject.items():
        assert not bnn.pixel_loss_routed(a, b, red), what


def test_cpu_tensors_go_to_stock():
    a, b = _t(2, 3, 8, 8), _t(2, 3, 8, 8)
    assert not bnn.pixel_loss_routed(a, b, "mean")


@pytest.mark.parametrize("name", ["MSELoss", "L1Loss"])
def test_forward_dispatch(name, on_device, monkeypatch):
    """routed calls go to PixelLossFn with the module's mode; the rest run the stock forward"""
    seen = []

    class Fake:
        @staticmethod
        def apply(a, b, mode):
            seen.append(mode)
            return torch.zeros(())
    monkeypatch.setattr(bnn.F, "PixelLossFn", Fake)
    a, b = _t(2, 3, 8, 8, layout="nhwc"), _t(2, 3, 8, 8)
    mod = getattr(bnn, name)()
    assert mod(a, b).item() == 0.0
    assert seen == [0 if name == "MSELoss" else 1]
    want = getattr(torch.nn, name)(reduction="sum")(a, b)
    assert torch.equal(getattr(bnn, name)(reduction="sum")(a, b), want) and len(seen) == 1


@pytest.mark.parametrize("name", ["MSELoss", "L1Loss"])
def test_stock_behaviour_off_the_kernels(name):
    """on the CPU the drop-in is the stock module bit for bit, with torch's broadcast warning and the legacy arguments"""
    ours, stock = getattr(bnn, name), getattr(torch.nn, name)
    a, b = _t(4, 3, 5, 5), _t(4, 3, 5, 5)
    for red in ("mean", "sum", "none"):
        assert torch.equal(ours(reduction=red)(a, b), stock(reduction=red)(a, b)), red
    with pytest.warns(UserWarning, match="broadcast"):
        ours()(a, _t(1, 3, 5, 5))
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        assert ours(size_average=False).reduction == "sum" and ours(reduce=False).reduction == "none"
    aa = a.clone().requires_grad_(True)
    ours()(aa, b).backward()
    ref = a.clone().requires_grad_(True)
    stock()(ref, b).backward()
    assert torch.equal(aa.grad, ref.grad)


def test_names_replacements_and_patch():
    import b200gan
    from b200gan import zoo
    for name in ("MSELoss", "L1Loss"):
        cls = bnn.REPLACEMENTS[name]
        assert cls is getattr(bnn, name) and cls.__name__ == name and cls.__qualname__ == name
        assert issubclass(cls, bnn._T[name]) and bnn._T[name] is not cls
        assert getattr(zoo.namespace(), name) is cls and getattr(zoo.namespace(stock=True), name) is bnn._T[name]
    stock = (torch.nn.MSELoss, torch.nn.L1Loss)
    b200gan.patch(optimizers=False)
    try:
        assert torch.nn.MSELoss is bnn.MSELoss and torch.nn.L1Loss is bnn.L1Loss
        assert type(torch.nn.MSELoss()).__name__ == "MSELoss"
    finally:
        b200gan.unpatch()
    assert (torch.nn.MSELoss, torch.nn.L1Loss) == stock


def test_train_steps_pick_the_losses_from_the_networks():
    from b200gan import train, zoo
    dropin = zoo.Pix2PixDiscriminator()
    stock = zoo.Pix2PixDiscriminator(nn=zoo.namespace(stock=True))
    mse, l1 = train._pixel_losses(dropin)
    assert type(mse) is bnn.MSELoss and type(l1) is bnn.L1Loss
    assert train._pixel_losses(stock) == (torch.nn.functional.mse_loss, torch.nn.functional.l1_loss)


# ---- the fp64 references ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", ["mse", "l1"])
@pytest.mark.parametrize("layouts", [("nchw", "nchw"), ("nhwc", "nchw")])
def test_references_are_torch_float64(mode, layouts):
    g = torch.Generator().manual_seed(1)
    a = torch.randn(2, 3, 5, 7, generator=g, dtype=torch.float64)
    b = torch.randn(2, 3, 5, 7, generator=g, dtype=torch.float64)
    b.view(-1)[::4] = a.view(-1)[::4]   # ties: sign(0) = 0
    if layouts[0] == "nhwc":
        a = a.contiguous(memory_format=CL)
    fn = torch.nn.functional.mse_loss if mode == "mse" else torch.nn.functional.l1_loss
    aa, bb = a.clone().requires_grad_(True), b.clone().requires_grad_(True)
    loss = fn(aa, bb)
    da, db = torch.autograd.grad(loss, (aa, bb), torch.tensor(1.7, dtype=torch.float64))
    torch.testing.assert_close(pl.loss_ref(a, b, mode), loss.detach(), rtol=1e-14, atol=0)
    want = pl.grad_ref(a, b, 1.7, mode)
    torch.testing.assert_close(want, da, rtol=1e-14, atol=0)
    torch.testing.assert_close(-want, db, rtol=1e-14, atol=0)
    if mode == "l1":
        assert want.reshape(-1)[::4].eq(0).all() and da.reshape(-1)[::4].eq(0).all()


def test_operands_of_the_table_have_their_layouts():
    for c in pl.CASES:
        a, b = pl.make(c, device="cpu")
        assert a.shape == b.shape == torch.Size(c.shape)
        from b200gan import ops
        d = ops.pixel_loss_desc(a, b, pl.MODES[c.mode])
        assert d is not None, c.id
        real_nhwc = len(c.shape) == 4 and c.shape[1] > 1 and c.shape[2] * c.shape[3] > 1
        assert (d.layout_a, d.layout_b) == (pl.LAYOUTS[c.la] if real_nhwc else 0, pl.LAYOUTS[c.lb] if real_nhwc else 0), \
            c.id
        assert (a.storage_offset() == 1) == c.offset and (b.storage_offset() == 1) == c.offset
        if c.equal:
            assert torch.equal(a, b)


# ---- the case table and the kernel source ----------------------------------------------------------------------------
def test_table_covers_its_edges():
    ids = [c.id for c in pl.CASES]
    assert len(ids) == len(set(ids)) and all(c.why for c in pl.CASES)
    for mode in ("mse", "l1"):
        cs = [c for c in pl.CASES if c.mode == mode]
        ns = {c.n for c in cs}
        assert {1, 7, 4096, 16 * 16 * 16, 8 * 3 * 256 * 256, 16 * 3 * 256 * 256} <= ns, mode
        assert any(c.n % 4 for c in cs if c.n > 8)
        assert {(c.la, c.lb) for c in cs if len(c.shape) == 4 and c.shape[1] > 1} >= {
            ("nchw", "nchw"), ("nhwc", "nhwc"), ("nhwc", "nchw"), ("nchw", "nhwc")}
        assert any(c.want_db for c in cs) and any(not c.want_db for c in cs)
        assert any(c.equal for c in cs) and any(c.offset for c in cs)
        # more elements than one pass of the forward grid (2 * SMs blocks of 256 x 8) on a 132-SM H100
        assert any(c.n > 2 * 132 * pl.THREADS * pl.PER_THREAD for c in cs)
    for c in pl.CASES:
        assert [k for k, _ in c.kernels()] == [pl.KERNEL["fwd"], pl.KERNEL["bwd"]]


def test_the_header_declares_the_two_kernels_and_the_entry_points_launch_only_them():
    assert declared(PL_CUH) == set(pl.KERNEL.values()) == {k for c in pl.CASES for k, _ in c.kernels()}
    assert declared(PL_CU) == set()
    assert '#include "pixel_loss_kernels.cuh"' in open(PL_CU).read()
    src = source(PL_CU)
    fns = functions(src)
    assert {"b200gan_pixel_loss_fwd", "b200gan_pixel_loss_bwd", "b200gan_pixel_loss_workspace_bytes"} <= set(fns)

    def launched(name, seen=()):
        body = fns[name]
        out = set(re.findall(r"(\w+)\s*<<<", body))
        for callee in set(re.findall(r"\b(\w+)\s*\(", body)) & set(fns):
            if callee != name and callee not in seen:
                out |= launched(callee, seen + (name,))
        return out
    assert launched("b200gan_pixel_loss_fwd") == {pl.KERNEL["fwd"]}
    assert launched("b200gan_pixel_loss_bwd") == {pl.KERNEL["bwd"]}
    assert launched("b200gan_pixel_loss_workspace_bytes") == set()
    assert len(re.findall(r"<<<", src)) == 2


def test_build_compiles_the_subdirectory():
    import build as b200_build
    assert os.path.join("pixel_loss", "pixel_loss.cu") in b200_build.sources()


@needs_nvcc
def test_kernels_do_not_spill_and_keep_their_registers():
    rep = ptxas_report(PL_CU)
    for name, r in rep.items():
        assert r["stack"] == r["spills"] == 0, f"{name}: {r}"
    regs = {k: r["registers"] for k, r in rep.items()}
    smem = {k: r["smem"] for k, r in rep.items()}
    assert regs == pl.REGISTERS, f"ptxas {regs}, table {pl.REGISTERS}"
    assert smem == pl.SMEM_BYTES, f"ptxas {smem}, table {pl.SMEM_BYTES}"
