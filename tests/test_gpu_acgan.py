"""ACGAN's auxiliary-classifier head and loss end to end on the GPU: the drop-in ACGAN discriminator (acgan.py:76-108)
against the stock modules in fp32, a create_graph=True penalty through the class head, train.acgan_step replayed from
a CUDA graph against an eager twin and against the stock modules, and tests/scripts/mini_acgan under the launcher.
Dropout2d is switched off where two runs are compared, so that both draw nothing."""
import copy
import os
import warnings

import pytest
import torch

from b200gan import functional as F
from b200gan import nn as bnn

pytestmark = pytest.mark.gpu


def rel_err(a, b):
    a, b = a.detach().double(), b.detach().double()
    return ((a - b).norm() / b.norm().clamp_min(1e-30)).item()


@pytest.fixture
def calls(monkeypatch):
    """counts of the class-head and cross-entropy kernel calls, forward and backward"""
    from b200gan import ops
    n = {"head_fwd": 0, "head_bwd": 0, "ce_fwd": 0, "ce_bwd": 0}
    for key, name in (("head_fwd", "class_head_fwd"), ("head_bwd", "class_head_bwd"), ("ce_fwd", "cross_entropy_fwd"),
                      ("ce_bwd", "cross_entropy_bwd")):
        fn = getattr(ops, name)

        def wrap(*a, _fn=fn, _key=key, **kw):
            n[_key] += 1
            return _fn(*a, **kw)
        monkeypatch.setattr(ops, name, wrap)
    return n


def _no_dropout(*nets):
    for net in nets:
        for m in net.modules():
            if isinstance(m, torch.nn.Dropout2d):
                m.p = 0.0


def _pair(seed, n_classes=10):
    from b200gan import zoo
    torch.manual_seed(seed)
    ref = zoo.ACGANDiscriminator(32, 1, n_classes, nn=zoo.namespace(stock=True)).cuda()
    ours = zoo.ACGANDiscriminator(32, 1, n_classes).cuda()
    ours.load_state_dict(ref.state_dict())
    _no_dropout(ref, ours)
    return ref, ours


def test_discriminator_and_losses_match_stock(calls):
    """validity, class posterior, both losses and every parameter gradient of the drop-in ACGAN discriminator against
    the stock modules, fp32; the heads and the losses run one kernel per direction each"""
    ref, ours = _pair(0)
    x = torch.rand(64, 1, 32, 32, device="cuda") * 2 - 1
    labels = torch.randint(0, 10, (64,), device="cuda")
    valid = torch.ones(64, 1, device="cuda")
    losses = []
    for net, ns in ((ref, torch.nn), (ours, bnn)):
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            v, p = net(x)
        loss_adv, loss_aux = ns.BCELoss()(v, valid), ns.CrossEntropyLoss()(p, labels)
        (0.5 * (loss_adv + loss_aux)).backward()
        losses.append((v.detach(), p.detach(), loss_adv.detach(), loss_aux.detach()))
    assert calls == {"head_fwd": 1, "head_bwd": 1, "ce_fwd": 1, "ce_bwd": 1}
    for a, b in zip(losses[1], losses[0]):
        assert rel_err(a, b) < 1e-4
    for (k, po), (_, pr) in zip(ours.named_parameters(), ref.named_parameters()):
        # the conv blocks' weight gradients carry the chain's usual fp32 reorderings through BatchNorm
        assert rel_err(po.grad, pr.grad) < (5e-3 if k.startswith("conv_blocks") else 1e-3), k


def test_no_grad_records_no_node(calls):
    _, ours = _pair(1)
    x = torch.rand(8, 1, 32, 32, device="cuda")
    with torch.no_grad(), warnings.catch_warnings():
        warnings.simplefilter("ignore")
        v, p = ours(x)
    assert p.grad_fn is None and calls["head_fwd"] == 1


def test_class_head_gradients_are_each_optional():
    torch.manual_seed(2)
    x = torch.randn(16, 512, device="cuda")
    w = torch.randn(10, 512, device="cuda") * 0.05
    b = torch.randn(10, device="cuda")
    dy = torch.randn(16, 10, device="cuda")
    full = [t.clone().requires_grad_(True) for t in (x, w, b)]
    y = F.ClassHeadFn.apply(*full)
    y_ref = torch.softmax(x.double() @ w.double().t() + b.double(), 1)
    assert rel_err(y, y_ref) < 1e-5
    y.backward(dy)
    ref = [t.double().requires_grad_(True) for t in (x, w, b)]
    torch.softmax(ref[0] @ ref[1].t() + ref[2], 1).backward(dy.double())
    for got, want in zip(full, ref):
        assert rel_err(got.grad, want.grad) < 1e-5
    for i in range(3):
        ins = [t.clone().requires_grad_(j == i) for j, t in enumerate((x, w, b))]
        F.ClassHeadFn.apply(*ins).backward(dy)
        assert torch.equal(ins[i].grad, full[i].grad), i
        assert all(t.grad is None for j, t in enumerate(ins) if j != i)


def test_create_graph_penalty_through_the_class_head(calls):
    """a gradient penalty on the class posterior's input gradient (autograd.grad(create_graph=True)): the double
    backward runs on torch ops, and the penalty and every head gradient match stock fp32"""
    torch.manual_seed(3)
    lin = torch.nn.Linear(512, 10).cuda()
    ref = torch.nn.Sequential(lin, torch.nn.Softmax(dim=1))
    ours = bnn.Sequential(copy.deepcopy(lin), bnn.Softmax(dim=1))
    x = torch.randn(64, 512, device="cuda")
    t = torch.randint(0, 10, (64,), device="cuda")
    out = []
    for net, ns in ((ref, torch.nn), (ours, bnn)):
        xi = x.clone().requires_grad_(True)
        p = net(xi)
        loss = ns.CrossEntropyLoss()(p, t)
        gx, = torch.autograd.grad(loss, xi, create_graph=True)
        gp = ((gx.norm(2, dim=1) - 1) ** 2).mean()
        (loss + 10.0 * gp).backward()
        out.append((gp.detach(), [q.grad.clone() for q in net.parameters()]))
    assert calls["head_fwd"] == 1 and calls["ce_fwd"] == 1
    assert rel_err(out[1][0], out[0][0]) < 1e-4
    for go, gr in zip(out[1][1], out[0][1]):
        assert rel_err(go, gr) < 1e-4


def test_create_graph_penalty_on_non_contiguous_logits(calls):
    """a penalty on the gradient of CrossEntropyLoss with respect to transposed (non-contiguous) logits and of the class
    head with respect to a transposed input: the double backward reaches the caller's tensors, as on stock torch"""
    torch.manual_seed(5)
    t = torch.randint(0, 10, (64,), device="cuda")
    b0 = torch.randn(10, 64, device="cuda")
    out = []
    for crit in (torch.nn.CrossEntropyLoss(), bnn.CrossEntropyLoss()):
        b = b0.clone().requires_grad_(True)
        gb, = torch.autograd.grad(crit(b.t(), t), b, create_graph=True)
        gp = (gb * gb).sum()
        assert gp.requires_grad
        out.append((gp.detach(), *torch.autograd.grad(gp, b)))
    assert calls["ce_fwd"] == 1
    for a, r in zip(out[1], out[0]):
        assert rel_err(a, r) < 1e-4
    lin = torch.nn.Linear(512, 10).cuda()
    x0 = torch.randn(512, 64, device="cuda")
    out = []
    for net in (torch.nn.Sequential(lin, torch.nn.Softmax(dim=1)),
                bnn.Sequential(copy.deepcopy(lin), bnn.Softmax(dim=1))):
        x = x0.clone().requires_grad_(True)
        gx, = torch.autograd.grad(torch.nn.functional.nll_loss(net(x.t()), t), x, create_graph=True)
        gp = (gx * gx).sum()
        out.append((gp.detach(), *torch.autograd.grad(gp, (x, *net.parameters()))))
    assert calls["head_fwd"] == 1
    for a, r in zip(out[1], out[0]):
        assert rel_err(a, r) < 1e-4


def test_routed_cross_entropy_takes_in_place_updates(calls):
    """the drop-in's loss is a tensor of its own, not a view of the kernel's [loss, count] buffer: `loss += reg` and
    `loss *= w` work and give stock torch's value and gradient"""
    torch.manual_seed(6)
    x0, t = torch.randn(64, 10, device="cuda"), torch.randint(0, 10, (64,), device="cuda")
    got = []
    for crit in (torch.nn.CrossEntropyLoss(), bnn.CrossEntropyLoss()):
        x = x0.clone().requires_grad_(True)
        loss = crit(x, t)
        loss += 0.25
        loss *= 2.0
        loss.backward()
        got.append((loss.detach(), x.grad))
    assert calls == {"head_fwd": 0, "head_bwd": 0, "ce_fwd": 1, "ce_bwd": 1}
    for a, r in zip(got[1], got[0]):
        assert rel_err(a, r) < 1e-5


def _acgan_nets(seed, stock=False):
    from b200gan import zoo
    torch.manual_seed(seed)
    ns = zoo.namespace(stock=stock)
    g = zoo.ACGANGenerator(32, 100, 10, 1, nn=ns).cuda()
    d = zoo.ACGANDiscriminator(32, 1, 10, nn=ns).cuda()
    g.apply(zoo.weights_init_normal)
    d.apply(zoo.weights_init_normal)
    _no_dropout(d)
    return g, d


def _acgan_inputs(seed):
    gen = torch.Generator("cuda").manual_seed(seed)
    return (torch.rand(64, 1, 32, 32, device="cuda", generator=gen) * 2 - 1,
            torch.randint(0, 10, (64,), device="cuda", generator=gen),
            torch.randn(64, 100, device="cuda", generator=gen),
            torch.randint(0, 10, (64,), device="cuda", generator=gen))


def test_acgan_step_graph_replays_match_an_eager_twin(calls):
    """train.acgan_step (acgan.py:184-223) at batch 64, 32 x 32, with the capturable Adam, captured with
    train.GraphedStep: the replays match an eager twin step for step"""
    from b200gan import optim, train
    g, d = _acgan_nets(0)
    g2, d2 = copy.deepcopy(g), copy.deepcopy(d)

    def make_step(g, d):
        og = optim.Adam(g.parameters(), lr=2e-4, betas=(0.5, 0.999))
        od = optim.Adam(d.parameters(), lr=2e-4, betas=(0.5, 0.999))

        def step(imgs, labels, z, gen_labels):
            gl, dl, _, _, _ = train.acgan_step(g, d, og, od, imgs, labels, z, gen_labels)
            return torch.stack([gl, dl])
        return step

    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        graphed = train.GraphedStep(make_step(g, d), _acgan_inputs(0))
        # three D passes and three losses per step, four steps
        assert calls == {"head_fwd": 12, "head_bwd": 12, "ce_fwd": 12, "ce_bwd": 12}
        eager = make_step(g2, d2)
        for _ in range(3):
            eager(*_acgan_inputs(0))
        for seed in (1, 2, 3):
            a = graphed(*_acgan_inputs(seed)).clone()
            b = eager(*_acgan_inputs(seed))
            assert rel_err(a, b) < 1e-5, seed
    torch.cuda.synchronize()
    for (k, x), (_, y) in zip(list(d.named_parameters()) + list(d.named_buffers()),
                              list(d2.named_parameters()) + list(d2.named_buffers())):
        assert rel_err(x, y) < 1e-3, k


def test_acgan_step_against_stock(calls):
    """three train.acgan_step steps on the drop-ins against the stock modules (torch Adam on both): the losses and the
    class posteriors agree"""
    from b200gan import train
    g_ref, d_ref = _acgan_nets(4, stock=True)
    g, d = _acgan_nets(4)
    g.load_state_dict(g_ref.state_dict())
    d.load_state_dict(d_ref.state_dict())
    opt = lambda ps: torch.optim.Adam(ps, lr=2e-4, betas=(0.5, 0.999))  # noqa: E731
    ogr, odr, og, od = opt(g_ref.parameters()), opt(d_ref.parameters()), opt(g.parameters()), opt(d.parameters())
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        for it in range(3):
            inputs = _acgan_inputs(10 + it)
            glr, dlr, _, rar, far = train.acgan_step(g_ref, d_ref, ogr, odr, *inputs)
            gl, dl, _, ra, fa = train.acgan_step(g, d, og, od, *inputs)
            assert abs(gl.item() - glr.item()) < 1e-3 * abs(glr.item()), it
            assert abs(dl.item() - dlr.item()) < 1e-3 * abs(dlr.item()), it
            assert rel_err(ra, rar) < 1e-3 and rel_err(fa, far) < 1e-3, it
    assert calls == {"head_fwd": 9, "head_bwd": 9, "ce_fwd": 9, "ce_bwd": 9}


def test_reference_idiom_acgan_script_under_the_launcher_on_cuda(calls):
    """launch.run() of tests/scripts/mini_acgan (label embedding, Softmax() class head, CrossEntropyLoss, numpy accuracy)
    on the GPU: stock torch and the drop-ins print losses within fp32 tolerance, and the drop-in run reaches the class
    head and the cross-entropy kernels on every pass"""
    from b200gan import launch
    script = os.path.join(os.path.dirname(os.path.abspath(__file__)), "scripts", "mini_acgan", "mini_acgan.py")
    args = ["--epochs", "1", "--batch_size", "32"]
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        ref = launch.run(script, args, iters=3, seed=0, stock=True, quiet=True)
        assert calls == {"head_fwd": 0, "head_bwd": 0, "ce_fwd": 0, "ce_bwd": 0}
        ours = launch.run(script, args, iters=3, seed=0, stock=False, quiet=True)
    assert calls == {"head_fwd": 9, "head_bwd": 9, "ce_fwd": 9, "ce_bwd": 9}

    def losses(out):
        rows = [l for l in out["__b200_stdout__"].splitlines() if "[D " in l]
        return [(float(l.split("[D ")[1].split(",")[0]), float(l.split("[G ")[1].rstrip("]"))) for l in rows]
    a, b = losses(ours), losses(ref)
    assert len(a) == len(b) == 3
    for (d1, g1), (d2, g2) in zip(a, b):
        assert abs(d1 - d2) < 1e-4 * abs(d2) and abs(g1 - g2) < 1e-4 * abs(g2)
