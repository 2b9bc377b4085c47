"""The auxiliary-classifier head (Linear(K, n) + Softmax, functional.ClassHeadFn) and CrossEntropyLoss
(functional.CrossEntropyMeanFn) without a GPU: which calls route to the kernels and which go to the stock forward, the
Softmax dim=None warning, the class names and the patch, the fp64 references of tests/class_head_cases.py against torch
float64 autograd, the case table against csrc/head.cu and ptxas, and tests/scripts/mini_acgan under the launcher on the
CPU, patched against stock."""
import os
import re
import warnings

import pytest
import torch

import class_head_cases as hc
import stream_cases as sc
from b200gan import nn as bnn
from conformance import CSRC, declared, functions, needs_nvcc, ptxas_report, source

HEAD_CU = os.path.join(CSRC, "head.cu")


# ---- routing ---------------------------------------------------------------------------------------------------------
@pytest.fixture
def on_device(monkeypatch):
    """CPU tensors stand in for CUDA ones: the routing predicates are host logic"""
    monkeypatch.setattr(bnn, "_on_device", lambda t: True)


def _head(k=512, n=10, bias=True, dim=None, stock=False):
    ns = torch.nn if stock else bnn
    return ns.Linear(k, n, bias=bias), ns.Softmax(dim=dim)


def _snapshot(*mods):
    return [(k, v.clone()) for m in mods for k, v in m.state_dict().items()]


def test_class_head_routes_linear_softmax_over_dim_1(on_device):
    x = torch.randn(64, 512)
    accept = {
        "dim None": (*_head(), x),
        "dim 1": (*_head(dim=1), x),
        "dim -1": (*_head(dim=-1), x),
        "stock classes": (*_head(stock=True), x),
        "no bias": (*_head(bias=False), x),
        "n 2": (*_head(n=2), x),
        "n 32": (*_head(n=32), x),
        "one row": (*_head(), x[:1]),
        "K 1": (*_head(k=1), torch.randn(8, 1)),
        "at the bound": (*_head(n=4), torch.randn(3071, 512)),
    }
    for what, (lin, sm, xx) in accept.items():
        before = _snapshot(lin, sm)
        with warnings.catch_warnings():
            warnings.simplefilter("error")      # the predicate raises no warning, not even for dim=None
            assert bnn.class_head_routed(lin, sm, xx), what
        assert all(torch.equal(a, b) for (_, a), (_, b) in zip(before, _snapshot(lin, sm))), what


def test_class_head_rejects_everything_else(on_device):
    x = torch.randn(64, 512)
    lin, sm = _head()
    hooked = bnn.Softmax()
    hooked.register_forward_hook(lambda *a: None)
    hooked_lin = bnn.Linear(512, 10)
    hooked_lin.register_forward_pre_hook(lambda *a: None)

    class MySoftmax(torch.nn.Softmax):
        pass
    reject = {
        "dim 0": (lin, bnn.Softmax(dim=0), x),
        "dim 2": (lin, bnn.Softmax(dim=2), x),
        "dim -2": (lin, bnn.Softmax(dim=-2), x),
        "n 1": (*_head(n=1), x),
        "n 33": (*_head(n=33), x),
        "over the bound": (*_head(n=32), torch.randn(384, 512)),
        "no softmax": (lin, None, x),
        "LogSoftmax": (lin, torch.nn.LogSoftmax(dim=1), x),
        "Softmax subclass": (lin, MySoftmax(dim=1), x),
        "hooked softmax": (lin, hooked, x),
        "hooked linear": (hooked_lin, sm, x),
        "not a Linear": (torch.nn.Identity(), sm, x),
        "3-d input": (lin, sm, torch.randn(2, 64, 512)),
        "fp64 input": (lin, sm, x.double()),
        "fp64 weight": (bnn.Linear(512, 10).double(), sm, x),
        "wrong width": (lin, sm, torch.randn(64, 511)),
        "no rows": (lin, sm, torch.randn(0, 512)),
    }
    for what, (l, s, xx) in reject.items():
        assert not bnn.class_head_routed(l, s, xx), what


def test_class_head_stays_off_the_cpu():
    lin, sm = _head()
    assert not bnn.class_head_routed(lin, sm, torch.randn(4, 512))


def test_a_routed_sequential_raises_the_stock_softmax_warning(on_device, monkeypatch):
    """Sequential(Linear, Softmax()) on the class-head route warns about the implicit dim exactly as the stock module
    does: same category, message, file and line, once per call; an explicit dim warns on neither path"""
    seen = []

    class Fake:
        @staticmethod
        def apply(x, w, b):
            seen.append(tuple(w.shape))
            return torch.softmax(x @ w.t() + b, 1)
    monkeypatch.setattr(bnn.F, "ClassHeadFn", Fake)
    monkeypatch.setattr(bnn, "_gpu2d_f32", lambda x: True)
    torch.manual_seed(0)
    x = torch.randn(8, 512)

    def record(net):
        with warnings.catch_warnings(record=True) as w:
            warnings.simplefilter("always")
            y = net(x)
        return y, [(r.category, str(r.message), r.filename, r.lineno) for r in w]
    lin, sm = _head()
    ours = bnn.Sequential(lin, sm)
    stock = torch.nn.Sequential(*_head(stock=True))
    stock.load_state_dict(ours.state_dict())
    y, got = record(ours)
    y_ref, want = record(stock)
    assert seen == [(10, 512)] and len(want) == 1 and got == want
    assert "Implicit dimension choice for softmax" in want[0][1]
    torch.testing.assert_close(y, y_ref)
    ours[1].dim = stock[1].dim = 1
    assert record(ours)[1] == [] and record(stock)[1] == [] and seen == [(10, 512)] * 2


def test_head_routes_after_the_existing_patterns(on_device, monkeypatch):
    """Linear(K, 1) + Sigmoid still takes Linear1Fn; Linear(K, n) without a Softmax, and a Softmax alone, are stock"""
    taken = []

    class Fake:
        def __init__(self, name):
            self.name = name

        def apply(self, x, w, b, *rest):
            taken.append(self.name)
            return torch.zeros(x.shape[0], w.shape[0])
    monkeypatch.setattr(bnn.F, "ClassHeadFn", Fake("head"))
    monkeypatch.setattr(bnn.F, "Linear1Fn", Fake("linear1"))
    monkeypatch.setattr(bnn, "_gpu2d_f32", lambda x: True)
    x = torch.randn(4, 64)
    bnn.Sequential(bnn.Linear(64, 1), bnn.Sigmoid())._forward_2d(x)
    bnn.Sequential(bnn.Linear(64, 10))._forward_2d(x)
    bnn.Sequential(bnn.Linear(64, 10), bnn.LeakyReLU(0.2), bnn.Softmax(dim=1))._forward_2d(x)
    bnn.Sequential(bnn.Linear(64, 32), bnn.LeakyReLU(0.2), bnn.Linear(32, 10), bnn.Softmax(dim=1))._forward_2d(x)
    assert taken == ["linear1", "head"]


def test_cross_entropy_routes_class_indices_mean(on_device):
    x, t = torch.randn(64, 10), torch.randint(0, 10, (64,))
    accept = {
        "acgan": (x, t, None, "mean", 0.0),
        "C 1": (torch.randn(8, 1), torch.zeros(8, dtype=torch.long), None, "mean", 0.0),
        "C 1024": (torch.randn(4, 1024), torch.randint(0, 1024, (4,)), None, "mean", 0.0),
        "one row": (x[:1], t[:1], None, "mean", 0.0),
        "64 Ki logits": (torch.randn(64, 1024), torch.randint(0, 1024, (64,)), None, "mean", 0.0),
        "non-contiguous input": (torch.randn(10, 64).t(), t, None, "mean", 0.0),
        "input requires grad": (x.clone().requires_grad_(True), t, None, "mean", 0.0),
    }
    for what, args in accept.items():
        assert bnn.cross_entropy_routed(*args), what
    reject = {
        "probabilities": (x, torch.softmax(torch.randn(64, 10), 1), None, "mean", 0.0),
        "int32 target": (x, t.int(), None, "mean", 0.0),
        "K-dimensional": (torch.randn(4, 10, 3, 3), torch.randint(0, 10, (4, 3, 3)), None, "mean", 0.0),
        "unbatched": (torch.randn(10), torch.tensor(3), None, "mean", 0.0),
        "sum": (x, t, None, "sum", 0.0),
        "none": (x, t, None, "none", 0.0),
        "class weights": (x, t, torch.ones(10), "mean", 0.0),
        "label smoothing": (x, t, None, "mean", 0.1),
        "fp64": (x.double(), t, None, "mean", 0.0),
        "over 64 Ki logits": (torch.randn(6554, 10), torch.randint(0, 10, (6554,)), None, "mean", 0.0),
        "C 1025": (torch.randn(4, 1025), torch.randint(0, 1025, (4,)), None, "mean", 0.0),
        "C 0": (torch.randn(4, 0), torch.zeros(4, dtype=torch.long), None, "mean", 0.0),
        "no rows": (torch.randn(0, 10), torch.zeros(0, dtype=torch.long), None, "mean", 0.0),
        "length mismatch": (x, t[:63], None, "mean", 0.0),
        "not a tensor": (x, 3, None, "mean", 0.0),
    }
    for what, args in reject.items():
        assert not bnn.cross_entropy_routed(*args), what


def test_cross_entropy_stays_off_the_cpu_and_is_stock_there():
    x, t = torch.randn(16, 10), torch.randint(0, 10, (16,))
    t[3] = 3
    assert not bnn.cross_entropy_routed(x, t, None, "mean", 0.0)
    for kw in ({}, dict(reduction="sum"), dict(reduction="none"), dict(label_smoothing=0.2), dict(ignore_index=3),
               dict(weight=torch.rand(10))):
        ours, stock = bnn.CrossEntropyLoss(**kw), torch.nn.CrossEntropyLoss(**kw)
        a, b = x.clone().requires_grad_(True), x.clone().requires_grad_(True)
        la, lb = ours(a, t), stock(b, t)
        assert torch.equal(la, lb), kw
        la.sum().backward()
        lb.sum().backward()
        assert torch.equal(a.grad, b.grad), kw


def test_cross_entropy_dispatch(on_device, monkeypatch):
    seen = []

    class Fake:
        @staticmethod
        def apply(x, t, ignore_index):
            seen.append(ignore_index)
            return torch.zeros(())
    monkeypatch.setattr(bnn.F, "CrossEntropyMeanFn", Fake)
    x, t = torch.randn(8, 10), torch.randint(0, 10, (8,))
    assert bnn.CrossEntropyLoss(ignore_index=7)(x, t).item() == 0.0 and seen == [7]
    assert torch.equal(bnn.CrossEntropyLoss(reduction="sum")(x, t), torch.nn.CrossEntropyLoss(reduction="sum")(x, t))
    assert seen == [7]


def test_names_replacements_and_patch():
    import b200gan
    from b200gan import zoo
    for name in ("Softmax", "CrossEntropyLoss"):
        cls = bnn.REPLACEMENTS[name]
        assert cls is getattr(bnn, name) and cls.__name__ == name and cls.__qualname__ == name
        assert issubclass(cls, bnn._T[name]) and bnn._T[name] is not cls
        assert getattr(zoo.namespace(), name) is cls and getattr(zoo.namespace(stock=True), name) is bnn._T[name]
    stock = (torch.nn.Softmax, torch.nn.CrossEntropyLoss)
    b200gan.patch(optimizers=False)
    try:
        assert torch.nn.Softmax is bnn.Softmax and torch.nn.CrossEntropyLoss is bnn.CrossEntropyLoss
    finally:
        b200gan.unpatch()
    assert (torch.nn.Softmax, torch.nn.CrossEntropyLoss) == stock


def test_acgan_modules_restate_the_script():
    from b200gan import zoo
    d = zoo.ACGANDiscriminator(32, 1, 10)
    g = zoo.ACGANGenerator(32, 100, 10, 1)
    assert [type(m).__name__ for m in d.aux_layer] == ["Linear", "Softmax"] and d.aux_layer[1].dim is None
    assert (d.aux_layer[0].in_features, d.aux_layer[0].out_features) == (512, 10)
    assert (d.adv_layer[0].in_features, d.adv_layer[0].out_features) == (512, 1)
    assert type(g.label_emb) is torch.nn.Embedding and g.label_emb.weight.shape == (10, 100)
    ds = zoo.ACGANDiscriminator(32, 1, 10, nn=zoo.namespace(stock=True))
    assert list(ds.state_dict()) == list(d.state_dict())


# ---- the fp64 references -----------------------------------------------------------------------------------------------
def test_head_references_are_torch_float64():
    g = torch.Generator().manual_seed(1)
    x, w, b = (torch.randn(*s, generator=g, dtype=torch.float64) for s in ((7, 33), (11, 33), (11,)))
    dy = torch.randn(7, 11, generator=g, dtype=torch.float64)
    xx, ww, bb = (t.clone().requires_grad_(True) for t in (x, w, b))
    y = torch.softmax(xx @ ww.t() + bb, 1)
    gx, gw, gb = torch.autograd.grad(y, (xx, ww, bb), dy)
    y_ref, _ = hc.head_ref(x, w, b)
    torch.testing.assert_close(y_ref, y.detach(), rtol=1e-14, atol=1e-16)
    dx, dw, db, _ = hc.head_grad_ref(x, w, y.detach(), dy)
    for got, want in ((dx, gx), (dw, gw), (db, gb)):
        torch.testing.assert_close(got, want, rtol=1e-12, atol=1e-15)


@pytest.mark.parametrize("ignore_index", [-100, 3])
def test_cross_entropy_references_are_torch_float64(ignore_index):
    g = torch.Generator().manual_seed(2)
    x = torch.randn(20, 10, generator=g, dtype=torch.float64) * 3
    t = torch.randint(0, 10, (20,), generator=g)
    t[::4] = ignore_index
    xx = x.clone().requires_grad_(True)
    loss = torch.nn.functional.cross_entropy(xx, t, ignore_index=ignore_index)
    gx, = torch.autograd.grad(loss, xx, torch.tensor(1.5, dtype=torch.float64))
    ref, _, count = hc.ce_ref(x, t, ignore_index)
    assert count == int((t != ignore_index).sum())
    torch.testing.assert_close(ref, loss.detach(), rtol=1e-14, atol=0)
    torch.testing.assert_close(hc.ce_grad_ref(x, t, ignore_index, 1.5, count), gx, rtol=1e-12, atol=1e-16)


@pytest.fixture
def stubbed(monkeypatch):
    """the launch wrappers replaced by the fp64 references, so that the autograd nodes run on the CPU"""
    from b200gan import ops
    monkeypatch.setattr(ops, "_require_cuda", lambda *a: None)
    monkeypatch.setattr(ops, "class_head_fwd", lambda x, w, b: hc.head_ref(x, w, b)[0])
    monkeypatch.setattr(ops, "cross_entropy_fwd", lambda x, t, ig: torch.stack(
        [hc.ce_ref(x, t, ig)[0], torch.tensor(float(hc.ce_ref(x, t, ig)[2]), dtype=torch.float64)]).to(x.dtype))

    def head_bwd(x, w, y, dy, need_dx, need_db):
        dx, dw, db, _ = hc.head_grad_ref(x, w, y, dy)
        return (dx if need_dx else None), dw, (db if need_db else None)
    monkeypatch.setattr(ops, "class_head_bwd", head_bwd)
    monkeypatch.setattr(ops, "cross_entropy_bwd",
                        lambda x, t, out, gout, ig: hc.ce_grad_ref(x, t, ig, gout, out[1]).to(x.dtype))


@pytest.mark.parametrize("layout", ["contiguous", "transposed"])
def test_create_graph_backward_formulas_are_torch_float64(stubbed, layout):
    """the torch-op backwards ClassHeadFn and CrossEntropyMeanFn take under create_graph=True: twice differentiable
    like stock torch, also for a non-contiguous input, whose graph must reach the saved tensor"""
    from b200gan import functional as F
    g = torch.Generator().manual_seed(3)
    x, w, b = (torch.randn(*s, generator=g, dtype=torch.float64) for s in ((6, 9), (5, 9), (5,)))
    t = torch.tensor([0, 4, -100, 2, 1, 3])

    def leaf(v):   # a leaf, and the input built from it: the leaf itself or a transposed view of its transpose
        if layout == "contiguous":
            v = v.clone().requires_grad_(True)
            return v, v
        v = v.t().contiguous().requires_grad_(True)
        return v, v.t()

    def penalty(head, loss):
        (xx, xin), ww, bb = leaf(x), w.clone().requires_grad_(True), b.clone().requires_grad_(True)
        out = loss(head(xin, ww, bb), t)
        gx, = torch.autograd.grad(out, xx, create_graph=True)
        gp = (gx * gx).sum()
        return [v.detach() for v in (out, gp, *torch.autograd.grad(gp, (xx, ww, bb)))]
    ours = penalty(F.ClassHeadFn.apply, lambda p, t: F.CrossEntropyMeanFn.apply(p, t, -100))
    stock = penalty(lambda xx, ww, bb: torch.softmax(xx @ ww.t() + bb, 1),
                    lambda p, t: torch.nn.functional.cross_entropy(p, t))
    for a, s in zip(ours, stock):
        torch.testing.assert_close(a, s, rtol=1e-12, atol=1e-14)

    def loss_penalty(loss):   # the loss alone on the logits
        xx, xin = leaf(torch.randn(6, 5, generator=torch.Generator().manual_seed(4), dtype=torch.float64))
        gx, = torch.autograd.grad(loss(xin, t), xx, create_graph=True)
        gp = (gx * gx).sum()
        assert gp.requires_grad
        return [gp.detach(), *torch.autograd.grad(gp, xx)]
    for a, s in zip(loss_penalty(lambda p, t: F.CrossEntropyMeanFn.apply(p, t, -100)),
                    loss_penalty(torch.nn.functional.cross_entropy)):
        torch.testing.assert_close(a, s, rtol=1e-12, atol=1e-14)


def test_routed_loss_takes_in_place_updates(stubbed, on_device):
    """the drop-in's loss is not a view of the kernel's [loss, count] buffer: `loss += reg` works as on stock torch"""
    x = torch.randn(6, 5)
    t = torch.tensor([0, 4, -100, 2, 1, 3])
    assert bnn.cross_entropy_routed(x, t, None, "mean", 0.0)
    got = []
    for crit in (bnn.CrossEntropyLoss(), torch.nn.CrossEntropyLoss()):
        xx = x.clone().requires_grad_(True)
        loss = crit(xx, t)
        assert loss._base is None and loss.dim() == 0
        assert ("CrossEntropyMeanFn" in type(loss.grad_fn).__name__) == (type(crit) is bnn.CrossEntropyLoss)
        loss += 0.5
        loss *= 2.0
        loss.backward()
        got.append((loss.detach(), xx.grad))
    for a, s in zip(*got):
        torch.testing.assert_close(a, s, rtol=1e-6, atol=1e-7)


# ---- the case table and the kernel source ----------------------------------------------------------------------------
def test_table_covers_its_edges():
    ids = [c.id for c in hc.CASES]
    assert len(ids) == len(set(ids)) and all(c.why for c in hc.CASES)
    head = [c for c in hc.CASES if c.op == "head" and not c.error]
    assert {2, 10, 11, 32} <= {c.dims[2] for c in head}
    ks = {c.dims[1] for c in head}
    assert {512, 2048, 1} <= ks and any(k % 4 for k in ks if k > 1)
    ns = {c.dims[0] for c in head}
    assert {1, 64} <= ns and any(c.dims[0] * c.dims[2] == hc.BWD_MAX_ELEMS for c in head)
    assert all(c.dims[0] * c.dims[2] <= hc.BWD_MAX_ELEMS for c in head)
    assert any(c.opt.get("offset") for c in head)
    for opt in ("b", "dx", "db"):
        assert any(c.opt.get(opt) is False for c in head), opt
    ce = [c for c in hc.CASES if c.op == "ce" and not c.error]
    assert {1, 10, 11, 1024} <= {c.dims[1] for c in ce}
    assert any(0 < c.opt.get("ignored", 0) < 1 for c in ce) and any(c.opt.get("ignored") == 1.0 for c in ce)
    assert any(c.opt.get("ignore", hc.IGNORE) != hc.IGNORE for c in ce) and any(c.opt.get("bad") for c in ce)
    assert any(c.opt.get("xscale", 1) >= 1e4 for c in ce) and any(c.opt.get("xshift", 0) <= -1e6 for c in ce)
    errors = [c for c in hc.CASES if c.error]
    assert {c.id for c in errors} >= {"head-nout1", "head-nout33", "head-over_limit", "head-n0", "ce-c0", "ce-c1025",
                                      "ce-n0"}
    assert all(c.opt.get("refused_by") for c in errors)
    for c in hc.CASES:
        if not c.error:
            want = ("linear1_fwd_kernel", "linear1_bwd_kernel") if c.op == "head" else ("bce_fwd_kernel",
                                                                                       "bce_bwd_kernel")
            assert c.kernels == want, c.id


def test_head_cu_keeps_its_four_kernels_and_the_entry_points_launch_only_theirs():
    assert declared(HEAD_CU) == {k for c in sc.CASES if c.op in ("linear1", "bce") for k in c.kernels} == \
        {k for c in hc.CASES for k in c.kernels}
    src = source(HEAD_CU)
    fns = functions(src)
    want = {"b200gan_class_head_fwd": "linear1_fwd_kernel", "b200gan_class_head_bwd": "linear1_bwd_kernel",
            "b200gan_cross_entropy_fwd": "bce_fwd_kernel", "b200gan_cross_entropy_bwd": "bce_bwd_kernel",
            "b200gan_linear1_fwd": "linear1_fwd_kernel", "b200gan_linear1_bwd": "linear1_bwd_kernel",
            "b200gan_bce_fwd": "bce_fwd_kernel", "b200gan_bce_bwd": "bce_bwd_kernel"}
    for fn, kernel in want.items():
        assert re.findall(r"(\w+)\s*<<<", fns[fn]) == [kernel], fn
    assert len(re.findall(r"<<<", src)) == len(want)
    assert "template" not in src, "head.cu's kernels stay non-template: the traced names are compared exactly"


@needs_nvcc
def test_head_kernels_do_not_spill():
    rep = ptxas_report(HEAD_CU)
    for name, r in rep.items():
        assert r["stack"] == r["spills"] == 0, f"{name}: {r}"
    assert set(rep) == declared(HEAD_CU)


# ---- the reference-idiom script on the CPU -----------------------------------------------------------------------------
def test_mini_acgan_under_the_launcher_on_the_cpu_matches_stock():
    """tests/scripts/mini_acgan patched with the drop-ins and stock, on the CPU, where every drop-in it uses falls back to
    the stock forward: the printed losses and accuracies are identical"""
    from b200gan import launch
    script = os.path.join(os.path.dirname(os.path.abspath(__file__)), "scripts", "mini_acgan", "mini_acgan.py")
    args = ["--epochs", "1", "--batch_size", "32"]
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        ours = launch.run(script, args, iters=3, seed=0, stock=False, quiet=True)
        stock = launch.run(script, args, iters=3, seed=0, stock=True, quiet=True)
    lines = [l for l in ours["__b200_stdout__"].splitlines() if "[D " in l]
    assert len(lines) == 3 and ours["__b200_stdout__"] == stock["__b200_stdout__"]
    assert type(ours["critic"].which_class[1]) is bnn.Softmax and type(ours["cls_criterion"]) is bnn.CrossEntropyLoss
    assert type(stock["critic"].which_class[1]) is torch.nn.Softmax
