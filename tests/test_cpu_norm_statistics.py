"""The bounds of tests/stats_cases.py separate a pivoted fp32 summation from an unpivoted one.  No GPU needed.

Each kernel's statistics chain is emulated in numpy, with fp32 rounding at every step it rounds in fp32: the unpivoted
chain (fp32 sums of x and x^2 from zero, as the kernels summed before they took a pivot) and the pivoted chain (fp32
sums of x - p and (x - p)^2 around a value p of the group, then n p + a and b + 2 p a + n p^2 in fp64).  On every case's
group size, chain length and ladder of channels, the pivoted emulation meets stats_cases.bounds, and the unpivoted one
breaks it at least tenfold on the channel at R = |mean| / std = 10^4 and on the constant one.  (At R = 10^2 and 10^3
the unpivoted error of a random ladder channel stays near the worst case the bound allows for a pivoted chain: the
bound holds any pivot within max |x - mean| of the mean.)  A loosened bound fails here.
"""
import numpy as np
import pytest

import norm_cases as nc
import stats_cases as sc
from conformance import CSRC, declared_under_csrc

F32 = np.float32


def serial(v, axis):
    """fp32 sum along `axis`, one rounding per addition"""
    v = np.moveaxis(v, axis, 0)
    acc = np.zeros(v.shape[1:], F32)
    for t in v:
        acc = (acc + t).astype(F32)
    return acc


def serial_sq(v, axis):
    """fp32 fmaf(v, v, acc) along `axis`"""
    v = np.moveaxis(v, axis, 0)
    acc = np.zeros(v.shape[1:], F32)
    for t in v:
        acc = (t.astype(np.float64) * t + acc).astype(F32)
    return acc


def tree(v):
    """fp32 butterfly sum over the last axis (32 lanes)"""
    while v.shape[-1] > 1:
        h = v.shape[-1] // 2
        v = (v[..., :h] + v[..., h:]).astype(F32)
    return v[..., 0]


def padded(x, n):
    """x padded with zeros to n elements, and the mask of the real ones"""
    out, valid = np.zeros(n, F32), np.zeros(n, bool)
    out[:x.size], valid[:x.size] = x, True
    return out, valid


def centred(x, valid, unit_axes, pivot):
    """(x - p) inside the output, 0 outside, with p the first element of each unit (the leading axes); p and the unit's
    count of valid elements, as float64"""
    if not pivot:
        return np.where(valid, x, F32(0)), None, None
    lead = x.shape[:unit_axes]
    p = x.reshape(*lead, -1)[..., 0]
    pb = p.reshape(*lead, *([1] * (x.ndim - unit_axes)))
    d = np.where(valid, (x - pb).astype(F32), F32(0))
    return d, p.astype(np.float64), valid.reshape(*lead, -1).sum(-1).astype(np.float64)


def unpivot(a, b, p, n):
    a, b = a.astype(np.float64), b.astype(np.float64)
    return (n * p + a).sum(), (b + 2 * p * a + n * p * p).sum()


def emulate(x, ch, pivot):
    """(sum x, sum x^2) of one group as the kernel of chain `ch` forms them"""
    kind = ch.shape[0]
    if kind == "norm_stats":                      # blocks of rpb rows; thread t sums rows t, t + 8, ...
        _, yb, rpb = ch.shape
        nt = -(-rpb // 8)
        xs, valid = padded(x, yb * rpb)
        xs = np.concatenate([xs.reshape(yb, rpb), np.zeros((yb, nt * 8 - rpb), F32)], 1).reshape(yb, nt, 8)
        valid = np.concatenate([valid.reshape(yb, rpb), np.zeros((yb, nt * 8 - rpb), bool)], 1).reshape(yb, nt, 8)
        d, p, n = centred(xs, valid, 1, pivot)
        a, b = serial(d, 1), serial_sq(d, 1)   # [yb, 8]
        if not pivot:
            return a.astype(np.float64).sum(), b.astype(np.float64).sum()
        return unpivot(a.astype(np.float64).sum(1), b.astype(np.float64).sum(1), p, n)
    if kind == "conv":                            # warps of 32 pixels, `phases` per lane; four warps per tile
        phases = ch.shape[1]
        per = 4 * phases * 32
        xs, valid = padded(x, -(-x.size // per) * per)
        xs, valid = xs.reshape(-1, 4, phases, 32), valid.reshape(-1, 4, phases, 32)
        d, p, n = centred(xs, valid, 2, pivot)
        a = serial(tree(d), 2)                    # [tiles, 4]
        b = serial(tree((d * d).astype(F32)), 2)
        if not pivot:
            return serial(a, 1).astype(np.float64).sum(), serial(b, 1).astype(np.float64).sum()
        return unpivot(a, b, p, n)
    pt = ch.shape[1]                              # chain: pt pixels per lane, 32 lanes, 8 warps per channel group
    per = 8 * 32 * pt
    xs, valid = padded(x, -(-x.size // per) * per)
    xs, valid = xs.reshape(-1, 8, 32, pt), valid.reshape(-1, 8, 32, pt)
    d, p, n = centred(xs, valid, 2, pivot)
    a, b = tree(serial(d, 3)), tree(serial_sq(d, 3))   # [blocks, 8]
    if not pivot:
        return serial(a, 1).astype(np.float64).sum(), serial(b, 1).astype(np.float64).sum()
    return unpivot(a, b, p, n)


def ratios(x, ch, pivot):
    """|err| / bound of the mean and the variance"""
    x64 = x.astype(np.float64)
    m = x.size
    mean = x64.mean()
    var = ((x64 - mean) ** 2).mean()
    dev = np.abs(x64 - mean).max()
    mb, vb = sc.bounds(ch.K, ch.P, mean, var, dev)
    s1, s2 = emulate(x, ch, pivot)
    mk = s1 / m
    vk = max(s2 / m - mk * mk, 0.0)
    return abs(mk - mean) / mb, abs(vk - var) / vb


@pytest.mark.parametrize("case", sc.CASES, ids=lambda c: c.id)
def test_bounds_separate_pivoted_from_unpivoted_sums(case):
    ch = sc.chain(case)
    loc, sd = sc.ladder(len(sc.LADDER))
    rng = np.random.default_rng(0)
    for i in range(len(sc.LADDER)):
        x = (loc[i] + sd[i] * rng.standard_normal(case.m)).astype(F32)
        pm, pv = ratios(x, ch, True)
        assert pm <= 1 and pv <= 1, f"{case.id} channel {sc.LADDER[i]}: pivoted |err|/bound mean {pm:.3g} var {pv:.3g}"
        um, uv = ratios(x, ch, False)
        if loc[i] >= 1e4 * sd[i]:   # R >= 10^4, or constant
            assert max(um, uv) >= 10, f"{case.id} channel {sc.LADDER[i]}: unpivoted sums within {max(um, uv):.3g}x " \
                                      "of the bound: the bound does not tell them apart"


def test_table():
    ids = [c.id for c in sc.CASES]
    assert len(ids) == len(set(ids)) and all(c.why for c in sc.CASES)
    declared = declared_under_csrc()
    for c in sc.CASES:
        for k in c.kernels:
            assert k.split("<")[0] in declared, f"{c.id}: {k} is not declared under {CSRC}"
    paths = {(c.path, c.kernels[0].split("<")[0], c.deferred, c.per_sample) for c in sc.CASES}
    for want in [("norm", "norm_stats_kernel", True, False), ("norm", "norm_stats_kernel", True, True),
                 ("conv", "conv_tc_kernel", False, False), ("conv", "conv_tc_kernel", False, True),
                 ("conv", "conv_tc_up2_allphase_kernel", False, False),
                 ("conv", "conv_tc_up2_allphase_kernel", False, True), ("conv", "conv_tc_kernel", True, True),
                 ("chain", "nbk_fprop2_kernel", False, False)]:
        assert want in paths, f"no case of {want}"
    assert any(c.splitk for c in sc.CASES) and any(c.groups == 2 for c in sc.CASES)
    assert {c.kernels[3] for c in sc.CASES if c.path == "norm"} == {"norm_apply_kernel<4>", "norm_apply_kernel<1>"}
    # the large and offset geometries stay out of norm_cases.GEOMS, whose bounds the norm-conv suite shares
    assert not {g.name for g in sc.NORM_GEOMS} & {g.name for g in nc.GEOMS}
