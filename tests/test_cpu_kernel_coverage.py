"""Every __global__ kernel of the library has an fp64 conformance case, and the references of the critic and stream
suites agree with stock torch float64.  Needs the built library (the case tables import it), not a GPU.

A kernel is covered when a case table of the registry (conformance.case_tables) names it; the few kernels a dedicated
test covers instead are listed in COVERED_BY_TEST with that test.  A new kernel without a case fails here.  The same
holds for the C ABI: every entry point of include/b200gan.h that launches work on a stream is named by one registered
family and called in that family's case table or GPU conformance test, or listed in ENTRY_POINTS_COVERED_BY_TEST.  An
entry point that is a run-time mode of an existing kernel (a fused epilogue, a from-sums pass) so needs cases of its own.
"""
import os
import re

import pytest
import torch
import torch.nn.functional as F

import critic_cases as cr
import stream_cases as sc
from conformance import CSRC, ROOT, case_tables, declared, declared_under_csrc, needs_nvcc, ptxas_report, \
    table_kernels

COVERED_BY_TEST = {
    "pack_multi_kernel": "tests/test_gpu_conv_conformance.py::test_pack_weights_multi_30_jobs (bit-exact, 30 jobs)",
}

ENTRY_POINTS_COVERED_BY_TEST = {
    "b200gan_pack_weights": "tests/test_gpu_conv_conformance.py::test_pack_weights_bit_exact",
    "b200gan_pack_weights_multi": "tests/test_gpu_conv_conformance.py::test_pack_weights_multi_30_jobs",
    "b200gan_norm_dbwd": "tests/test_gpu_norm_double_backward.py::test_norm_dbwd_case",
    "b200gan_mlp_disc_fwd": "tests/test_gpu_mlp_discriminator.py::test_disc_case",
    "b200gan_mlp_disc_bwd": "tests/test_gpu_mlp_discriminator.py::test_disc_case",
}
HEADER = os.path.join(ROOT, "include", "b200gan.h")


def test_every_kernel_has_a_case():
    """every __global__ under csrc/ -- in a .cu file or a .cuh header, at any depth -- is named by a registered case
    table or by COVERED_BY_TEST"""
    kernels = declared_under_csrc()
    assert len(kernels) > 30, f"parsed only {len(kernels)} __global__ kernels"
    for d in (e.name for e in os.scandir(CSRC) if e.is_dir()):
        assert any(f.startswith(d + os.sep) for f in kernels.values()), f"no kernel parsed under csrc/{d}"
    covered = set()
    for fam in case_tables().values():
        covered |= table_kernels(fam.cases, fam.names)
    missing = set(kernels) - covered - set(COVERED_BY_TEST)
    assert not missing, f"kernels without a conformance case: {sorted((kernels[k], k) for k in missing)}"
    stale = set(COVERED_BY_TEST) - set(kernels)
    assert not stale, f"COVERED_BY_TEST names kernels the sources do not declare: {sorted(stale)}"
    assert not set(COVERED_BY_TEST) & covered, "a kernel in COVERED_BY_TEST also has a case: drop it from the map"


def stream_entry_points(header):
    """the functions a C header declares with a `void *stream` parameter"""
    src = re.sub(r"/\*.*?\*/", "", header, flags=re.S)
    return {m.group(1) for m in re.finditer(r"\b(b200gan_\w+)\s*\(([^;{]*)\)\s*;", src)
            if re.search(r"\bvoid\s*\*\s*stream\b", m.group(2))}


def test_every_entry_point_has_a_case():
    """every entry point that takes a stream is named by one registered family and called in that family's case table
    or GPU conformance test, or listed in ENTRY_POINTS_COVERED_BY_TEST with the test that calls it"""
    with open(HEADER) as fh:
        entry = stream_entry_points(fh.read())
    assert len(entry) > 40, f"parsed only {len(entry)} entry points from {HEADER}"
    owner = {}
    for name, fam in case_tables().items():
        for e in fam.entry_points:
            assert e not in owner, f"{e} is named by the families {owner[e]!r} and {name!r}"
            owner[e] = name
            texts = []
            for m in fam.modules:
                with open(os.path.join(ROOT, "tests", m)) as fh:
                    texts.append(fh.read())
            assert any(re.search(r"\b" + e + r"\b", t) for t in texts), \
                f"family {name!r} names {e}, but none of {fam.modules} calls it"
    stale = (set(owner) | set(ENTRY_POINTS_COVERED_BY_TEST)) - entry
    assert not stale, f"entry points named in the registry or ENTRY_POINTS_COVERED_BY_TEST but not declared: {stale}"
    both = set(owner) & set(ENTRY_POINTS_COVERED_BY_TEST)
    assert not both, f"an entry point with a family is also in ENTRY_POINTS_COVERED_BY_TEST: drop it from the map: {both}"
    for e, test in ENTRY_POINTS_COVERED_BY_TEST.items():
        path, _, fn = test.partition("::")
        with open(os.path.join(ROOT, path)) as fh:
            text = fh.read()
        assert re.search(r"\b" + e + r"\b", text) and re.search(r"\bdef " + fn + r"\(", text), \
            f"{e}: {test} does not exist or does not call it"
    missing = entry - set(owner) - set(ENTRY_POINTS_COVERED_BY_TEST)
    assert not missing, f"entry points without a case: {sorted(missing)}"


def test_critic_and_stream_tables_match_their_sources():
    mc = declared(os.path.join(CSRC, "mlp_critic.cu"))
    assert mc == set(cr.KERNEL.values()) == table_kernels(cr.CASES), (mc, table_kernels(cr.CASES))
    streams = declared(os.path.join(CSRC, "head.cu")) | declared(os.path.join(CSRC, "index_ops.cu"))
    assert streams == table_kernels(sc.CASES), \
        f"declared but no case: {sorted(streams - table_kernels(sc.CASES))}; " \
        f"in the table but not declared: {sorted(table_kernels(sc.CASES) - streams)}"
    for cases in (cr.CASES, sc.CASES):
        ids = [c.id for c in cases]
        assert len(ids) == len(set(ids)), sorted(i for i in ids if ids.count(i) > 1)
        assert all(c.why for c in cases)


def cc_tiles(rows, cols):
    return -(-rows // 32) * -(-cols // 32)


def test_critic_edges_are_in_the_table():
    rows = {c.id: c for c in cr.CASES}
    for op in ("fwd", "bwd", "dbwd", "step"):
        ok = [c for c in cr.CASES if c.op == op and not c.error]
        assert any((c.N, c.Din, c.H1, c.H2) == (64, 1024, 512, 256) for c in ok), op
        assert any(c.Din == 784 for c in ok) and any(c.N == 1 for c in ok) and any(c.H2 == 1 for c in ok), op
        assert {0.0, 0.2, 1.0} <= {c.slope for c in ok}, op
        nrows = lambda c: 3 * c.N if op == "step" else c.N
        assert any(cc_tiles(nrows(c), max(c.H1, c.Din)) > 2 * cr.GRID[0] for c in ok), f"{op}: no case with many tiles"
    for out in cr.OUTPUTS["bwd"][:7]:
        assert f"bwd-{out}_only" in rows
    for out in cr.OUTPUTS["dbwd"]:
        assert f"dbwd-{out}_only" in rows
    step = [c for c in cr.CASES if c.op == "step"]
    assert {0.0, 10.0} <= {c.lam for c in step} and {"zero", "one"} <= {c.alpha for c in step}
    assert any(c.zero_w3 for c in step) and any(c.zero_row >= 0 for c in step)


@needs_nvcc
def test_critic_grid_follows_from_the_registers():
    """the cooperative grid is num_sms * min(2, blocks per SM); the blocks per SM follow from ptxas's registers"""
    rep = ptxas_report(os.path.join(CSRC, "mlp_critic.cu"))
    regs = {k: r["registers"] for k, r in rep.items()}
    assert regs == cr.REGISTERS, f"ptxas {regs}, table {cr.REGISTERS}"
    assert [r["smem"] for r in rep.values()] == [cr.SMEM_BYTES] * 4
    per_sm = min(cr.blocks_per_sm(v) for v in regs.values())
    assert cr.GRID == (cr.NUM_SMS * min(2, per_sm), 1, 1)
    assert all(c.grid == cr.GRID for c in cr.CASES if not c.error)


# ---- the critic references against nn.Sequential autograd --------------------------------------------------------------
def _critic(N=5, Din=7, H1=6, H2=4, slope=0.2, seed=0):
    g = torch.Generator().manual_seed(seed)
    net = torch.nn.Sequential(torch.nn.Linear(Din, H1), torch.nn.LeakyReLU(slope), torch.nn.Linear(H1, H2),
                              torch.nn.LeakyReLU(slope), torch.nn.Linear(H2, 1)).double()
    with torch.no_grad():
        for p in net.parameters():
            p.copy_(torch.randn(p.shape, generator=g, dtype=torch.float64) * 0.5)
    W = [net[0].weight, net[0].bias, net[2].weight, net[2].bias, net[4].weight, net[4].bias]
    return net, W, g


@pytest.mark.parametrize("slope", [0.2, 0.0, 1.0])
def test_critic_references_are_sequential_autograd(slope):
    net, W, g = _critic(slope=slope)
    Wd = [w.detach() for w in W]
    x = torch.randn(5, 7, generator=g, dtype=torch.float64, requires_grad=True)
    out = net(x).reshape(-1)
    f = cr.critic_fwd_ref(x.detach(), *Wd, slope)
    torch.testing.assert_close(f["out"], out.detach(), rtol=1e-12, atol=1e-12)
    dout = torch.randn(5, generator=g, dtype=torch.float64, requires_grad=True)
    gx, = torch.autograd.grad(out, x, dout, create_graph=True)
    grads = torch.autograd.grad(out, [x] + W, dout, retain_graph=True)
    b = cr.critic_bwd_ref(dout.detach(), x.detach(), Wd[0], Wd[2], Wd[4].reshape(-1), f["m1"], f["a1"], f["m2"],
                            f["a2"])
    for name, want in zip(("dx", "dW1", "db1", "dW2", "db2", "dW3", "db3"), grads):
        torch.testing.assert_close(b[name][0].reshape(want.shape), want, rtol=1e-10, atol=1e-12, msg=name)
    u = torch.randn(5, 7, generator=g, dtype=torch.float64)
    dd = torch.autograd.grad(gx, [W[0], W[2], W[4], dout], u, allow_unused=True)
    r = cr.critic_dbwd_ref(u, dout.detach(), b["U1"][0], b["U2"][0], f["m1"], f["m2"], Wd[0], Wd[2],
                             Wd[4].reshape(-1))
    for name, want in zip(("dW1", "dW2", "dW3", "ddout"), dd):
        want = torch.zeros_like(r[name][0]) if want is None else want
        torch.testing.assert_close(r[name][0].reshape(want.shape), want, rtol=1e-10, atol=1e-12, msg=name)


def compute_gradient_penalty(D, real_samples, fake_samples, alpha):
    """the WGAN-GP reference's penalty (wgan_gp.py:119-138), with its random alpha passed in"""
    interpolates = (alpha * real_samples + ((1 - alpha) * fake_samples)).requires_grad_(True)
    d_interpolates = D(interpolates)
    fake = torch.ones(real_samples.shape[0], 1, dtype=real_samples.dtype)
    gradients = torch.autograd.grad(outputs=d_interpolates, inputs=interpolates, grad_outputs=fake,
                                    create_graph=True, retain_graph=True, only_inputs=True)[0]
    gradients = gradients.view(gradients.size(0), -1)
    return ((gradients.norm(2, dim=1) - 1) ** 2).mean()


@pytest.mark.parametrize("kind", ["plain", "zero_w3", "zero_row", "alpha01"])
def test_critic_step_reference_is_the_wgan_gp_iteration(kind):
    lam, slope = 10.0, 0.0 if kind == "zero_row" else 0.2
    net, W, g = _critic(N=6, slope=slope, seed=1)
    real = torch.randn(6, 7, generator=g, dtype=torch.float64)
    fake = torch.randn(6, 7, generator=g, dtype=torch.float64)
    alpha = torch.rand(6, 1, generator=g, dtype=torch.float64)
    with torch.no_grad():
        if kind == "zero_w3":
            W[4].zero_()
        if kind == "zero_row":   # the critic_cases zero_row case: b1 < 0 at slope 0, one sample all zeros
            W[1].copy_(-0.5 - 0.1 * W[1].abs())
            real[2].zero_()
            fake[2].zero_()
    if kind == "alpha01":
        alpha[:3], alpha[3:] = 0.0, 1.0
    gp = compute_gradient_penalty(net, real, fake, alpha)
    d_loss = -torch.mean(net(real)) + torch.mean(net(fake)) + lam * gp
    want = torch.autograd.grad(d_loss, W, retain_graph=True)
    Wd = [w.detach() for w in W]
    r = cr.critic_step_ref(real, fake, alpha.reshape(-1), *Wd, slope, lam)
    # the reference weighs the real / fake rows by the kernel's fp32 -1/N and 1/N: relative differences of ~2^-24
    torch.testing.assert_close(r["losses"][0], torch.stack([d_loss, lam * gp]).detach(), rtol=1e-6, atol=1e-12)
    for name, w in zip(("dW1", "db1", "dW2", "db2", "dW3", "db3"), want):
        torch.testing.assert_close(r[name][0].reshape(w.shape), w, rtol=1e-6, atol=1e-7, msg=name)
    if kind in ("zero_w3", "zero_row"):
        pen = torch.autograd.grad(lam * gp, W, allow_unused=True)
        r0 = cr.critic_step_ref(real, fake, alpha.reshape(-1), *Wd, slope, 0.0)
        assert r["coef"].eq(0).sum() >= (6 if kind == "zero_w3" else 1)
        for name, p in zip(("dW1", "db1", "dW2", "db2", "dW3", "db3"), pen):
            # torch's norm backward passes 0 at a zero norm: the penalty contributes no gradient through that sample
            if kind == "zero_w3":
                assert p is None or p.eq(0).all(), name
                assert torch.equal(r[name][0], r0[name][0]), name
        if kind == "zero_w3":
            assert abs(gp.item() - 1.0) < 1e-15


# ---- the stream references against stock torch --------------------------------------------------------------------------
@pytest.mark.parametrize("step0", [0, 7])
@pytest.mark.parametrize("gscale", [1.0, 0.25])
def test_adam_reference_is_torch_adam(step0, gscale):
    g = torch.Generator().manual_seed(3)
    p0 = torch.randn(1000, generator=g, dtype=torch.float64)
    grad = torch.randn(1000, generator=g, dtype=torch.float64)
    m0 = torch.randn(1000, generator=g, dtype=torch.float64) * 0.1
    v0 = torch.rand(1000, generator=g, dtype=torch.float64) * 0.01
    p = torch.nn.Parameter(p0.clone())
    opt = torch.optim.Adam([p], lr=sc.ADAM["lr"], betas=(sc.ADAM["b1"], sc.ADAM["b2"]), eps=sc.ADAM["eps"],
                           foreach=False)
    if step0:
        opt.state[p] = {"step": torch.tensor(float(step0)), "exp_avg": m0.clone(), "exp_avg_sq": v0.clone()}
    else:
        m0, v0 = torch.zeros_like(m0), torch.zeros_like(v0)
    p.grad = grad * gscale
    opt.step()
    (p1, _), (m1, _), (v1, _) = sc.adam_ref(p0, grad, m0, v0, step0, gscale)
    st = opt.state[p]
    # the reference keeps the kernel's fp32 casts of the hyper-parameter terms: relative differences of ~2^-24
    torch.testing.assert_close(m1, st["exp_avg"], rtol=1e-6, atol=0)
    torch.testing.assert_close(v1, st["exp_avg_sq"], rtol=1e-6, atol=0)
    torch.testing.assert_close(p1 - p0, p.detach() - p0, rtol=1e-6, atol=0)


def test_bce_reference_is_binary_cross_entropy():
    g = torch.Generator().manual_seed(4)
    v = 0.02 + 0.96 * torch.rand(64, generator=g, dtype=torch.float64)
    v[0::4], v[1::4] = 0.0, 1.0
    t = torch.tensor([0.0, 1.0, 0.3], dtype=torch.float64)[torch.randint(0, 3, (64,), generator=g)]
    vv = v.clone().requires_grad_(True)
    loss = F.binary_cross_entropy(vv, t)
    (dv,) = torch.autograd.grad(loss * 1.5, vv)
    torch.testing.assert_close(sc.bce_ref(v, t)[0], loss.detach(), rtol=1e-12, atol=0)
    torch.testing.assert_close(sc.bce_grad_ref(v, t, 1.5), dv, rtol=1e-6, atol=0)   # the clamp is 1e-12 in fp32


@pytest.mark.parametrize("pads,mode", [((1, 1, 0, 0), "zero"), ((1, 1, 1, 1), "reflect"), ((3, 3, 3, 3), "reflect"),
                                       ((4, 5, 4, 5), "reflect"), ((2, 0, 1, 3), "reflect")])
def test_pad_reference_is_the_stock_module(pads, mode):
    t, l, b, r = pads
    m = torch.nn.ReflectionPad2d((l, r, t, b)) if mode == "reflect" else torch.nn.ZeroPad2d((l, r, t, b))
    g = torch.Generator().manual_seed(5)
    x = torch.randn(2, 5, 6, 3, generator=g, dtype=torch.float64, requires_grad=True)
    y = m(x.permute(0, 3, 1, 2)).permute(0, 2, 3, 1)
    torch.testing.assert_close(sc.pad_ref(x.detach(), pads, mode), y.detach(), rtol=0, atol=0)
    dy = torch.randn(y.shape, generator=g, dtype=torch.float64)
    (dx,) = torch.autograd.grad(y, x, dy)
    torch.testing.assert_close(sc.pad_grad_ref(dy, x.shape, pads, mode), dx, rtol=1e-15, atol=1e-15)


def test_upsample_reference_is_interpolate():
    g = torch.Generator().manual_seed(6)
    x = torch.randn(2, 5, 7, 3, generator=g, dtype=torch.float64, requires_grad=True)
    y = F.interpolate(x.permute(0, 3, 1, 2), scale_factor=2, mode="nearest").permute(0, 2, 3, 1)
    torch.testing.assert_close(sc.upsample_ref(x.detach()), y.detach(), rtol=0, atol=0)
    dy = torch.randn(y.shape, generator=g, dtype=torch.float64)
    (dx,) = torch.autograd.grad(y, x, dy)
    torch.testing.assert_close(sc.upsample_grad_ref(dy), dx, rtol=1e-15, atol=1e-15)
