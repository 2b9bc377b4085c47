"""The fused norm-conv case table (tests/norm_conv_cases.py) against the library's predicate
b200gan_conv2d_dgrad_norm_supported.  Needs the built library, not a GPU: the predicate is host logic, and without a
device num_sms() takes the 132 SMs of an H100 SXM."""
import ctypes

from b200gan import _lib
import norm_cases as nc
import norm_conv_cases as ncc


def geom(c):
    t, l, b, r = c.pads
    return _lib.ConvGeom(c.N, c.H, c.W, c.C, c.K, c.R, c.S, c.stride, t, l, b, r, c.pad_mode, c.up, int(c.transposed),
                         c.P, c.Q)


def supported(c):
    return _lib.load().b200gan_conv2d_dgrad_norm_supported(ctypes.byref(geom(c)))


def tiles(c):
    """128-pixel tiles of the data gradient's output grid (tc_tiles)"""
    bwl = min(max(0, (c.W - 1).bit_length()), 7)
    bhl = min(max(0, (c.H - 1).bit_length()), 7 - bwl)
    return -(-c.W // (1 << bwl)) * -(-c.H // (1 << bhl)) * -(-c.N // (128 >> (bwl + bhl)))


def block_n(C, t):
    """tc_block_n for the data gradient's C produced channels"""
    if C % 256 == 0 and t * (C // 256) >= ncc.NUM_SMS:
        return 256
    return 128 if C % 128 == 0 else 64 if C % 64 == 0 else 32


def test_ids_unique_and_every_case_says_why():
    ids = [c.id for c in ncc.CASES]
    assert len(ids) == len(set(ids)), sorted(i for i in ids if ids.count(i) > 1)
    assert all(c.why for c in ncc.CASES)


def test_predicate_matches_the_table():
    for c in ncc.FUSED:
        want = 0 if c.refuse == "geometry" else 1
        assert supported(c) == want, f"{c.id}: b200gan_conv2d_dgrad_norm_supported = {supported(c)}, table {want}"
        assert (c.code == 0) == (c.bn != 0), c.id
        if c.refuse == "geometry":
            assert c.code == -1, c.id


def test_block_n_and_grid_follow_from_c_and_the_tiles():
    for c in ncc.ACCEPTED:
        assert c.tiles == tiles(c), f"{c.id}: {tiles(c)} tiles, table {c.tiles}"
        assert c.bn == block_n(c.C, c.tiles) <= 128, c.id
        assert c.grid == (c.tiles, c.C // c.bn, 1)
        assert c.kernels[0] == f"conv_tc_kernel<{c.bn}, {ncc.STAGES[c.bn]}>"


def _has(cases, N, C, K, H, W, **kw):
    return any((c.N, c.C, c.K, c.H, c.W) == (N, C, K, H, W) and all(getattr(c, k) == v for k, v in kw.items())
               for c in cases)


def test_table_holds_each_edge_on_both_sides():
    acc, ref = ncc.ACCEPTED, [c for c in ncc.REFUSED if c.refuse == "geometry"]
    # the two DCGAN blocks at batch 128
    assert _has(acc, 128, 128, 128, 16, 16, up=2) and _has(acc, 128, 128, 64, 32, 32, up=2)
    # two n-tiles at BN = 128; BN = 256 refused
    assert _has(acc, 64, 256, 64, 16, 16) and _has(ref, 66, 256, 64, 16, 16)
    # three n-tiles at BN 32 / 64 / 128
    for C in (96, 192, 384):
        assert any(c.C == C and c.C // c.bn == 3 for c in acc), C
    assert {c.bn for c in acc if c.C // c.bn == 3} == {32, 64, 128}
    # just inside / outside the split-K rule
    assert _has(acc, 8, 64, 32, 16, 16) and _has(ref, 8, 64, 64, 16, 16)
    # several images per tile, the last tile past N
    for N, H in ((33, 4), (5, 2), (7, 1)):
        assert _has(acc, N, 64, 32, H, H), (N, H)
    assert _has(acc, 64, 64, 64, 16, 16, R=1, S=1)
    assert _has(acc, 96, 64, 32, 12, 12) and _has(acc, 80, 64, 64, 10, 10, up=2)
    # filters other than 3x3 p1: refused at batch 64 on 16x16 maps, accepted where the tiles fill the machine
    for kw in (dict(R=5, S=5), dict(R=3, S=3, pads=ncc.P0, K=64), dict(R=4, S=4, pads=ncc.ASYM), dict(R=7, S=7)):
        K = kw.pop("K", 32)
        assert _has(ref, 64, 64, K, 16, 16, **kw), kw
        if K == 32:
            assert any((c.R, c.S) == (kw["R"], kw["S"]) and c.pads == kw.get("pads", c.pads) for c in acc), kw
    # refusals other than the geometry
    kinds = {c.refuse for c in ncc.REFUSED}
    assert {"geometry", "per_sample", "act", "desc_N", "desc_C", "desc_HW", "x_offset"} <= kinds
    assert {c.act for c in ncc.REFUSED if c.refuse == "act"} == {"tanh", "sigmoid"}
    assert any(c.pad_mode == 1 for c in ref) and any(c.stride == 2 and not c.transposed for c in ref)
    assert any(c.transposed for c in ref)


def test_activations_are_spread_over_the_geometries():
    acc = ncc.ACCEPTED
    assert {c.act for c in acc} == {"none", "lrelu", "relu"}
    assert {c.slope for c in acc if c.act == "lrelu"} >= {0.2, 0.01}
    assert any(c.act == "relu" and c.beta0 for c in acc), "a ReLU case that masks about half of the pixels"
    assert {c.rtf for c in acc} == {False, True}


def test_from_sums_cases_cover_every_norm_geometry():
    for g in nc.GEOMS:
        for a in nc.ACTS:
            assert sum(c.geom == g and c.act == a for c in ncc.FROM_SUMS) == 1, (g.name, a)
    ok = [c for c in ncc.FROM_SUMS if not c.code]
    assert {c.geom.vec for c in ok} == {1, 4} and any(c.geom.slices > 1 for c in ok)
    assert any(c.geom.per_sample for c in ok) and any(not c.geom.affine for c in ok)
    assert {c.rtf for c in ok} == {False, True}
    assert {c.act for c in ncc.FROM_SUMS if c.code} == {"tanh", "sigmoid"}
