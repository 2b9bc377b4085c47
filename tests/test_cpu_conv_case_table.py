"""The convolution route table (tests/conv_cases.py) against the library's eligibility predicate and the kernels the
sources declare.  Needs the built library, not a GPU: b200gan_conv2d_supported is host logic."""
import ctypes
import os

import pytest

import conv_cases as cc
from b200gan import _lib
from conformance import CSRC, declared


def geom(c):
    t, l, b, r = c.pads
    return _lib.ConvGeom(c.N, c.H, c.W, c.C, c.K, c.R, c.S, c.stride, t, l, b, r, c.pad_mode, c.up, int(c.transposed),
                         c.P, c.Q)


def test_case_ids_unique():
    ids = [c.id for c in cc.CASES]
    assert len(ids) == len(set(ids)), sorted(i for i in ids if ids.count(i) > 1)


@pytest.mark.parametrize("case", cc.CASES, ids=lambda c: c.id)
def test_tc_support_matches_table(case):
    lib = _lib.load()
    g = geom(case)
    assert lib.b200gan_conv2d_supported(ctypes.byref(g), case.pas, _lib.ALGO_SIMT) == 1, "invalid geometry"
    tc = lib.b200gan_conv2d_supported(ctypes.byref(g), case.pas, _lib.ALGO_TC) == 1
    if case.algo == "SIMT":
        assert not case.tc
        # forcing SIMT is only worth a case where the tensor-core path would otherwise run (or is not offered at all
        # for the pass: the weight gradient of a TC-eligible geometry forced onto the staged kernel)
        assert tc, f"{case.id}: SIMT forced on a geometry the tensor-core path does not take anyway"
    elif not case.error:
        assert tc == case.tc, f"{case.id}: b200gan_conv2d_supported(TC) = {tc}, the table expects a " \
                              f"{'wgmma' if case.tc else 'SIMT'} kernel {case.kernels}"
    assert case.why, f"{case.id}: every case names the edge it exists for"
    assert set(case.epi) <= set(cc.EPI_OPTIONS)
    assert case.pas == cc.FPROP or not case.epi


def test_table_covers_every_conv_kernel():
    kernels = set()
    for f in cc.COVERED_SOURCES:
        kernels |= declared(os.path.join(CSRC, f))
    nb = declared(os.path.join(CSRC, "narrow_block.cu")) & set(cc.NARROW_BLOCK_KERNELS)
    assert nb == set(cc.NARROW_BLOCK_KERNELS), "narrow_block.cu no longer declares " + \
        str(set(cc.NARROW_BLOCK_KERNELS) - nb)
    kernels |= nb
    assert len(kernels) == 18, f"source parse found {sorted(kernels)}"
    covered = {cc.base_name(k) for c in cc.CASES for k in c.kernels}
    missing = kernels - covered
    assert not missing, f"convolution kernels without a conformance case: {sorted(missing)}"
    unknown = covered - kernels - cc.HELPER_KERNELS
    assert not unknown, f"the table names kernels the sources do not declare: {sorted(unknown)}"
