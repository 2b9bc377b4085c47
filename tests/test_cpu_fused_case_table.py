"""The fused-path case tables (tests/chain_cases.py, tests/tail_cases.py) against the library's eligibility predicates
and the kernels csrc/narrow_block.cu and csrc/tail.cu declare and launch, and the tables' fp64 references against stock
torch float64.  Needs the built library, not a GPU: the predicates are host logic (num_sms() is 132 without a device)."""
import ctypes
import os
import re

import pytest
import torch
import torch.nn.functional as F

import chain_cases as ch
import conv_cases as cc
import tail_cases as tl
from b200gan import _lib
from conformance import CSRC, declared, source

NB_CU = os.path.join(CSRC, "narrow_block.cu")
TAIL_CU = os.path.join(CSRC, "tail.cu")


def test_case_ids_unique_and_explained():
    for cases in (ch.CASES, tl.CASES):
        ids = [c.id for c in cases]
        assert len(ids) == len(set(ids)), sorted(i for i in ids if ids.count(i) > 1)
        for c in cases:
            assert c.why, f"{c.id}: every case names the edge it exists for"
    for c in ch.CASES:
        assert c.op in ch.OPS and c.edge in ch.EDGES, c.id
        assert c.error or c.kernels, f"{c.id}: a case that runs names its kernels"


@pytest.mark.parametrize("case", [c for c in ch.CASES if c.op in ("fprop", "wgrad", "dgrad", "plain_dgrad")],
                         ids=lambda c: c.id)
def test_chain_rows_against_the_predicates(case):
    lib = _lib.load()
    g = ch.chain_geom(case)
    if case.op == "plain_dgrad":
        # a staged data gradient through the conv entry: not a chain layer, no tensor-core route
        assert lib.b200gan_nb_supported(ctypes.byref(g)) == 0
        assert lib.b200gan_conv2d_supported(ctypes.byref(g), cc.DGRAD, _lib.ALGO_SIMT) == 1
        return
    assert lib.b200gan_nb_supported(ctypes.byref(g)) == 1, f"{case.id}: not a chain geometry"
    assert lib.b200gan_nb_groups_supported(ctypes.byref(g), case.groups) == 1, \
        f"{case.id}: no tile plan keeps tiles inside one of {case.groups} groups"
    if case.groups > 1:
        # the smallest batch the table uses for 3 and 4 groups is the smallest the planner allows
        assert case.N % case.groups == 0


def test_grouped_minimum_batches():
    lib = _lib.load()
    for c in ch.CASES:
        if c.groups in (3, 4) and c.op in ("fprop", "dgrad") and not c.error:
            smaller = [n for n in range(c.groups, c.N, c.groups)
                       if lib.b200gan_nb_groups_supported(ctypes.byref(ch.chain_geom(
                           ch.Case(c.name, c.op, n, c.C, c.K, c.H, c.W, c.R, c.stride))), c.groups)]
            assert not smaller, f"{c.id}: N = {smaller[0]} also runs with {c.groups} groups"


@pytest.mark.parametrize("case", tl.CASES, ids=lambda c: c.id)
def test_tail_rows_against_the_predicate(case):
    lib = _lib.load()
    d = _lib.TailDesc(case.N, case.H, case.W, case.C, case.K, ch.ACT_CODE[case.act_mid], ch.SLOPE,
                      ch.ACT_CODE[case.act_out])
    assert lib.b200gan_tail_supported(ctypes.byref(d)) == (0 if case.error else 1), case.id


def test_every_fused_kernel_has_a_case():
    tail = declared(TAIL_CU)
    assert tail == {"tail_fprop_tc_kernel", "tail_bwd_reduce_kernel", "tail_bwd_apply_kernel"}, tail
    covered = {cc.base_name(k) for c in tl.CASES for k in c.kernels if not c.error}
    assert tail <= covered, f"tail.cu kernels without a case: {sorted(tail - covered)}"
    nb = declared(NB_CU) - set(cc.NARROW_BLOCK_KERNELS)
    assert nb == {"nbk_dz_kernel", "nbk_tail_fwd_kernel", "nbk_tail_bwd_kernel"}, nb
    covered = {cc.base_name(k) for c in ch.CASES for k in c.kernels}
    assert nb <= covered, f"narrow_block.cu kernels without a case: {sorted(nb - covered)}"


def _launch_cases(macro):
    """the (KT, PT) list of an NB_*_INSTANCES X-macro, which both the launch and the refusal check expand"""
    src = source(NB_CU)
    m = re.search(r"#define " + macro + r"\(X\)((?:[^\n]*\\\n)*[^\n]*)", src)
    assert m, f"no {macro} in narrow_block.cu"
    assert f"{macro}(NB_IS_INSTANCE)" in src and re.search(macro + r"\(NB_\w+_CASE\)", src), \
        f"{macro} must drive both the refusal check and the launch"
    return {(int(a), int(b)) for a, b in re.findall(r"X\((\d+),\s*(\d+)\)", m.group(1))}


def test_every_planned_instance_is_covered_or_hook_only():
    covered = {k for c in ch.CASES if not c.error for k in c.kernels}
    for macro, fmt in (("NB_FPROP_INSTANCES", ch.fp), ("NB_DGRAD_INSTANCES", ch.dg)):
        launched = {fmt(*kp) for kp in _launch_cases(macro)}
        assert len(launched) >= 9, f"no {macro} lines parsed"
        missing = launched - covered - set(ch.HOOK_ONLY)
        assert not missing, f"instances without a case or a HOOK_ONLY reason: {sorted(missing)}"
        name = fmt(1, 1).split("<")[0]
        stale = {k for k in set(ch.HOOK_ONLY) | covered if k.startswith(name + "<")} - launched
        assert not stale, f"the table names instances narrow_block.cu does not launch: {sorted(stale)}"
    both = covered & set(ch.HOOK_ONLY)
    assert not both, f"HOOK_ONLY instances a case reaches: {sorted(both)}"
    assert all(ch.HOOK_ONLY.values())


def test_every_tail_instance_is_covered():
    src = source(TAIL_CU)
    fwd = {f"tail_fprop_tc_kernel<{a}, {b}>" for a, b in re.findall(r"launch_tail_fprop<(\d+),\s*(\d+)>\(p", src)}
    assert len(fwd) == 6, fwd
    ks = sorted({int(k) for k in re.findall(r"launch_tail_bwd<C4,\s*(\d+)>", src)})
    c4s = sorted({int(c) for c in re.findall(r"TAIL_BWD\((\d+)\)", src)})
    assert ks == [1, 2, 3] and c4s == [8, 16, 32], (ks, c4s)
    bwd = {f"tail_bwd_{p}_kernel<{c4}, {k}>" for p in ("reduce", "apply") for c4 in c4s for k in ks}
    covered = {k for c in tl.CASES if not c.error for k in c.kernels}
    missing = (fwd | bwd) - covered
    assert not missing, f"tail.cu instances without a case: {sorted(missing)}"
    assert covered <= fwd | bwd, sorted(covered - fwd - bwd)


def test_planner_candidates_are_launch_cases_or_refused():
    """nb_plan's candidates (its kts lists x PT in {1, 2, 4}) either have an instance or make the launcher refuse"""
    src = source(NB_CU)
    plan = src[src.index("static NbPlan nb_plan("):src.index("static NbPlan nb_plan_fprop")]
    kts = {int(v) for v in re.findall(r"kts\[\d\]\s*=\s*(\d+)", plan)}
    assert kts == {16, 8, 4, 1}, kts
    assert "kts[0] = nout" in plan and re.search(r"nout == 3 \|\| nout == 6", plan)
    kts |= {3, 6}
    cands = {(kt, pt) for kt in kts for pt in (1, 2, 4)}
    fprop, dgrad = _launch_cases("NB_FPROP_INSTANCES"), _launch_cases("NB_DGRAD_INSTANCES")
    # the forward plans nout = K, a power of two >= 4 (chain) or a multiple of 16 (staged conv entry)
    assert {c for c in cands if c[0] in (16, 8, 4)} <= fprop
    # the data gradient plans nout = C: every candidate but KT = 1 at PT > 1 (only the hook asks for those)
    assert cands - dgrad == {(1, 2), (1, 4)}, cands - dgrad
    for launcher, check in (("nb_fprop2_launch", "nb_fprop_instance(pl)"), ("nb_dgrad2_launch", "nb_dgrad_instance(pl)")):
        body = src[src.index(f"static int {launcher}("):]
        body = body[:body.index("\n}\n")]
        at = body.find(f"B2_CHECK_ARG({check},")
        assert at >= 0, f"{launcher} must refuse a plan without an instance"
        # before anything is written: the statistics memset and the launch come after the refusal
        assert at < body.index("cudaMemsetAsync") < body.index("<<<"), f"{launcher} writes before it refuses"


# ---- the fp64 references against stock torch float64 ------------------------------------------------------------------
def _bn_case(G, N=6, C=5, H=3, W=4, seed=0):
    gen = torch.Generator().manual_seed(seed)
    a = torch.randn(N, H, W, C, generator=gen, dtype=torch.float64) * 1.5 + 0.3
    gamma = 1 + 0.5 * torch.randn(C, generator=gen, dtype=torch.float64)
    beta = 0.3 * torch.randn(C, generator=gen, dtype=torch.float64)
    return a, gamma, beta, float(N // G * H * W)


@pytest.mark.parametrize("G", [1, 2, 3])
def test_grouped_batchnorm_reference_is_separate_batch_norm_calls(G):
    a, gamma, beta, count = _bn_case(G)
    N, C = a.shape[0], a.shape[-1]
    mean, var, rstd, sc, sh = ch.bn_consts(ch.group_sums(a, G), gamma, beta, count, G, C)
    x = a * ch.per_image(sc, N) + ch.per_image(sh, N)
    rm0, rv0 = torch.linspace(-0.2, 0.3, C, dtype=torch.float64), torch.linspace(0.5, 1.5, C, dtype=torch.float64)
    rm, rv = ch.running_ref(rm0, rv0, mean, var, count)
    trm, trv = rm0.clone(), rv0.clone()
    outs = []
    for g in range(G):   # the reference's separate forward passes, in batch order
        part = ch.nchw(a[g * (N // G):(g + 1) * (N // G)])
        outs.append(ch.nhwc(F.batch_norm(part, trm, trv, gamma, beta, True, ch.MOMENTUM, ch.BN_EPS)))
    torch.testing.assert_close(x, torch.cat(outs), rtol=1e-12, atol=1e-12)
    torch.testing.assert_close(rm, trm, rtol=1e-12, atol=1e-12)
    torch.testing.assert_close(rv, trv, rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize("G", [1, 2])
def test_dz_reference_is_batchnorm_backward(G):
    a, gamma, beta, count = _bn_case(G, seed=1)
    N, C = a.shape[0], a.shape[-1]
    gen = torch.Generator().manual_seed(2)
    G_ = torch.randn(a.shape, generator=gen, dtype=torch.float64)
    cs = torch.rand(N, 1, 1, C, generator=gen, dtype=torch.float64) * 2 - 0.5
    mean, var, rstd, sc, sh = ch.bn_consts(ch.group_sums(a, G), gamma, beta, count, G, C)
    xh = (a - ch.per_image(mean, N)) * ch.per_image(rstd, N)
    sums = torch.stack([G_.reshape(G, -1, C).sum(1), (G_ * xh).reshape(G, -1, C).sum(1)], 1)
    dz = ch.bn_bwd_ref(G_, a, mean, rstd, sc, sums, count, cs, "lrelu")
    av = a.clone().requires_grad_(True)
    parts = [F.batch_norm(ch.nchw(av[g * (N // G):(g + 1) * (N // G)]), None, None, gamma, beta, True, 0.0,
                          ch.BN_EPS) for g in range(G)]
    (da,) = torch.autograd.grad(ch.nhwc(torch.cat(parts)), av, G_)
    torch.testing.assert_close(dz, da * cs * torch.where(a > 0, 1.0, ch.SLOPE).double(), rtol=1e-10, atol=1e-12)


def test_conv_references_are_autograd_of_conv2d():
    gen = torch.Generator().manual_seed(3)
    x = torch.randn(2, 9, 9, 4, generator=gen, dtype=torch.float64)
    w = torch.randn(8, 4, 3, 3, generator=gen, dtype=torch.float64)
    xv, wv = ch.nchw(x).clone().requires_grad_(True), w.clone().requires_grad_(True)
    y = F.conv2d(xv, wv, stride=2, padding=1)
    torch.testing.assert_close(ch.conv_fwd(x, w, 2, 1), ch.nhwc(y), rtol=1e-12, atol=1e-12)
    dz = torch.randn(y.shape, generator=gen, dtype=torch.float64)
    gx, gw = torch.autograd.grad(y, (xv, wv), dz)
    torch.testing.assert_close(ch.conv_dgrad(ch.nhwc(dz), w, x.shape, 2, 1), ch.nhwc(gx), rtol=1e-12, atol=1e-12)
    torch.testing.assert_close(ch.conv_wgrad(x, ch.nhwc(dz), w.shape, 2, 1), gw, rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize("act_mid", ["none", "lrelu", "relu"])
def test_tail_references_are_the_stock_module(act_mid):
    """BatchNorm2d (batch statistics) -> act_mid -> Conv2d(C, K, 3, 1, 1), forward and backward, in float64"""
    gen = torch.Generator().manual_seed(4)
    N, H, W, C, K = 2, 5, 4, 8, 3
    a = torch.randn(N, H, W, C, generator=gen, dtype=torch.float64) * 1.5 + 0.3
    gamma = 1 + 0.3 * torch.randn(C, generator=gen, dtype=torch.float64)
    beta = 0.3 * torch.randn(C, generator=gen, dtype=torch.float64)
    w = torch.randn(K, C, 3, 3, generator=gen, dtype=torch.float64) / 6
    bias = torch.randn(K, generator=gen, dtype=torch.float64)
    g = torch.randn(N, H, W, K, generator=gen, dtype=torch.float64)
    a2 = a.reshape(-1, C)
    mean, var = a2.mean(0), a2.var(0, unbiased=False)
    rstd = 1 / torch.sqrt(var + 1e-5)
    sc = gamma * rstd
    mr, ss = torch.cat([mean, rstd]), torch.cat([sc, beta - mean * sc])
    av, gv, bv, wv, biv = (t.clone().requires_grad_(True) for t in (a, gamma, beta, w, bias))
    x = F.batch_norm(ch.nchw(av), None, None, gv, bv, True, 0.0, 1e-5)
    x = {"none": x, "lrelu": F.leaky_relu(x, ch.SLOPE), "relu": F.relu(x)}[act_mid]
    y = F.conv2d(x, wv, biv, padding=1)
    da, dgamma, dbeta, dw, db = torch.autograd.grad(y, (av, gv, bv, wv, biv), ch.nchw(g))
    r = tl.tail_bwd_ref(a, mr, ss, w, g, act_mid, (a * ss[:C] + ss[C:]) <= 0)
    for got, want in ((r["da"], da), (r["s2"], dgamma), (r["s1"], dbeta), (r["dw"], dw),
                      (r["db"], db)):
        torch.testing.assert_close(got, want, rtol=1e-9, atol=1e-11)
    # forward: the wgmma operand rounding is the kernel's, the rest is the module's
    out = ch.conv_fwd(ch.nhwc(x.detach()), w, 1, 1) + bias
    want, *_ = tl.tail_fwd_ref(a.float(), ss.float(), w.float(), bias.float(), act_mid, "tanh")
    torch.testing.assert_close(want, torch.tanh(out), rtol=0, atol=5e-3)


# ---- nb_plan restated: the instance and grid of every row, and which instances legal calls can reach -----------------
def _pow2ceil(v):
    r = 1
    while r < v:
        r *= 2
    return r


def _cdiv(a, b):
    return -(-a // b)


def nb_plan(nout, wrow, cin, N, Ho, Wo, ncls, allow_pt, groups, patch, sms=ch.NUM_SMS, red=256):
    """nb_plan of narrow_block.cu without its tuning hook: (KT, PT, KG, TN, TR, TQ) or None; red: the floats of the
    cross-warp sums (the forward keeps them in fp64)"""
    kts = [16, 8, 4] if nout % 16 == 0 else [8, 4] if nout % 8 == 0 else [4] if nout % 4 == 0 else \
        [nout] if nout in (3, 6) else [1]
    best, best_cost = None, 1e30
    for KT in kts:
        for PT in ((4, 2, 1) if allow_pt else (1,)):
            for KG in (8, 4, 2, 1):
                KB = KG * KT
                if KB > nout or nout % KB:
                    continue
                TP = PT * (256 // KG)
                TQ = min(_pow2ceil(Wo), 32, TP)
                TR = min(_pow2ceil(Ho), TP // TQ)
                TN = TP // (TQ * TR)
                if (TN > 1 and TN // 2 >= N) or (groups > 1 and (N // groups) % TN):
                    continue
                floats = ((wrow * KB + 3) & ~3) + ((patch(TN, TR, TQ) + 3) & ~3) + 2 * ((cin + 3) & ~3) + red
                if floats * 4 > 200 * 1024:
                    continue
                blocks = _cdiv(N, TN) * _cdiv(Ho, TR) * _cdiv(Wo, TQ) * (nout // KB) * ncls
                cost = max(0.25, (PT + KT) / (PT * KT)) / min(blocks, sms)
                if floats * 4 > 110 * 1024 or blocks < 256:
                    cost *= 1.4
                if cost < best_cost:
                    best_cost, best = cost, (KT, PT, KG, TN, TR, TQ)
    return best


def plan_fprop(N, C, K, H, W, R, stride, pad=1, groups=1):
    """(instance, grid) of nb_fprop2_launch, or None"""
    P, Q = (H + 2 * pad - R) // stride + 1, (W + 2 * pad - R) // stride + 1
    CP = C + 4 if C % 4 == 0 else C
    b = nb_plan(K, R * R * C, C, N, P, Q, 1, R * R * C >= 16, groups,
                lambda TN, TR, TQ: TN * ((TR - 1) * stride + R) * ((TQ - 1) * stride + R) * CP, red=512)
    if b is None:
        return None
    KT, PT, KG, TN, TR, TQ = b
    return ch.fp(KT, PT), (_cdiv(N, TN) * _cdiv(P, TR) * _cdiv(Q, TQ), K // (KG * KT), 1)


def plan_dgrad(N, C, K, H, W, R, stride, groups=1):
    """(instance, grid) of nb_dgrad2_launch, or None"""
    Rm = _cdiv(R, stride)
    Ho, Wo = _cdiv(H, stride), _cdiv(W, stride)
    b = nb_plan(C, Rm * Rm * K, C, N, Ho, Wo, stride * stride, C >= 4, groups,
                lambda TN, TR, TQ: TN * (TR + Rm - 1) * (TQ + Rm - 1) * (K + 4))
    if b is None:
        return None
    KT, PT, KG, TN, TR, TQ = b
    return ch.dg(KT, PT), (_cdiv(N, TN) * _cdiv(Ho, TR) * _cdiv(Wo, TQ), C // (KG * KT), stride * stride)


def wgrad_grid(c, sms=ch.NUM_SMS):
    """(gx, set chunks, 1) of nb_wgrad_plan"""
    P, Q = c.P, c.Q
    nsets = c.C * _cdiv(c.K, 4)
    spb = 256 if nsets >= 256 else _pow2ceil(nsets)
    nchunks = _cdiv(nsets, spb)
    TQ = min(Q, 32)
    TR = min(128 // TQ, P)
    TN = max(1, min(128 // (P * Q), c.N)) if (TR == P and TQ == Q) else 1

    def tile_bytes(TN, TR, TQ):
        PR, PC = (TR - 1) * c.stride + c.R, (TQ - 1) * c.stride + c.R
        return (((2 * spb + TN * TR * TQ + 3) & ~3) + ((TN * PR * PC * c.C + 3) & ~3) + TN * TR * TQ * _cdiv(c.K, 4) * 4
                + 2 * 4 * ((c.C + 3) & ~3)) * 4
    while TN > 1 and tile_bytes(TN, TR, TQ) > 96 * 1024:
        TN = (TN + 1) // 2
    while TR > 1 and tile_bytes(TN, TR, TQ) > 96 * 1024:
        TR = (TR + 1) // 2
    while TQ > 1 and tile_bytes(TN, TR, TQ) > 96 * 1024:
        TQ = (TQ + 1) // 2
    ntiles = _cdiv(c.N, TN) * _cdiv(P, TR) * _cdiv(Q, TQ)
    return (max(1, min(max(8, 2 * sms // nchunks), ntiles)), nchunks, 1)


@pytest.mark.parametrize("case", [c for c in ch.CASES if c.op in ("fprop", "dgrad", "plain_dgrad", "wgrad")
                                  and not c.error], ids=lambda c: c.id)
def test_rows_are_what_the_planner_picks(case):
    """the restated planner gives each row's instance and grid (the GPU test holds the rows to the library's trace)"""
    if case.op == "fprop":
        got = plan_fprop(case.N, case.C, case.K, case.H, case.W, case.R, case.stride, groups=case.groups)
    elif case.op == "wgrad":
        got = None, wgrad_grid(case)
        lib = _lib.load()
        nws = lib.b200gan_nb_wgrad_workspace_floats(ctypes.byref(ch.chain_geom(case)))
        # the library sizes the slabs from the same plan: gx slabs of K * C * R * S floats
        if case.ws or ch.WG_RED in case.kernels:   # a NULL workspace (ws False) takes the atomics whatever the plan
            assert (nws > 0) == (ch.WG_RED in case.kernels), f"{case.id}: workspace floats {nws}"
        if nws:
            assert nws == got[1][0] * case.K * case.C * case.R * case.R, f"{case.id}: {nws} workspace floats"
        assert case.grid == got[1], f"{case.id}: nb_wgrad_plan gives grid {got[1]}, the table {case.grid}"
        return
    else:
        got = plan_dgrad(case.N, case.C, case.K, case.H, case.W, case.R, case.stride,
                         groups=case.groups if case.edge != "none" else 1)
    assert got == (case.kernels[0], case.grid), f"{case.id}: nb_plan gives {got}, the table {case.kernels[0]} " \
                                                f"{case.grid}"


def _reachable():
    """instances nb_plan picks over legal calls: chain layers (groups 1 - 4, batches that split evenly, odd group
    sizes included) and the staged forward / data gradient of the conv entry (few input channels)"""
    fprop, dgrad = set(), set()
    sizes = (2, 3, 4, 5, 8, 9, 13, 16, 17, 32, 33, 64)
    per_group = (1, 2, 3, 4, 5, 7, 8, 15, 16, 30, 31, 32, 64, 128)
    for C in (1, 4, 16, 32, 64, 128):
        for K in (4, 8, 16, 32, 64, 128):
            for R in (3, 4):
                if R * R * C * K * 4 > 512 * 1024:
                    continue
                for stride in (1, 2):
                    for H in sizes:
                        if (H + 2 - R) // stride + 1 < 1:
                            continue
                        for groups in (1, 2, 3, 4):
                            for ng in per_group:
                                N = ng * groups
                                if N > 256:
                                    continue
                                if plan_fprop(N, C, K, H, H, R, stride) is None or \
                                        plan_dgrad(N, C, K, H, H, R, stride) is None:
                                    continue   # not a chain geometry (b200gan_nb_supported)
                                f = plan_fprop(N, C, K, H, H, R, stride, groups=groups)
                                d = plan_dgrad(N, C, K, H, H, R, stride, groups=groups)
                                if f and d:
                                    fprop.add(f[0])
                                    dgrad.add(d[0])
    for N in (1, 2, 3, 4, 8, 16, 64, 256):
        for H in (4, 8, 16, 32, 64, 128, 256):
            for R, pad in ((3, 1), (4, 1), (7, 3)):
                for stride in (1, 2):
                    for C in range(1, 9):
                        for K in (16, 32, 64, 128):
                            f = plan_fprop(N, C, K, H, H, R, stride, pad)
                            if f:
                                fprop.add(f[0])
                        if (C in (1, 3, 6) or C % 4 == 0) and (R != 7 or stride == 1):
                            for K in (4, 8, 16, 32, 64, 128):
                                d = plan_dgrad(N, C, K, H, H, R, stride)
                                if d:
                                    dgrad.add(d[0])
    return fprop | dgrad


def test_hook_only_is_exactly_the_unreachable_set():
    launched = {ch.fp(*kp) for kp in _launch_cases("NB_FPROP_INSTANCES")} | \
        {ch.dg(*kp) for kp in _launch_cases("NB_DGRAD_INSTANCES")}
    reached = _reachable()
    assert reached <= launched, f"the planner picks instances that are not launched: {sorted(reached - launched)}"
    assert set(ch.HOOK_ONLY) == launched - reached, \
        f"reached by legal calls but listed HOOK_ONLY: {sorted(set(ch.HOOK_ONLY) & reached)}; " \
        f"never reached but not listed: {sorted(launched - reached - set(ch.HOOK_ONLY))}"
