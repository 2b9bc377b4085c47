"""GPU parity of b200gan.optim.Adam (b200gan_adam_multi) against torch.optim.Adam with the reference's hyper-parameters
(dcgan.py:134-135: lr 2e-4, betas (0.5, 0.999), eps 1e-8, no weight decay, no amsgrad)."""
import itertools

import pytest
import torch

from conftest import rel_err

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("n", [1, 1000, 100003])
def test_one_tensor_adam_matches_torch_adam(n):
    """one parameter tensor of n elements through optim.Adam, five steps"""
    from b200gan import optim
    torch.manual_seed(5)
    p0 = torch.randn(n, device="cuda")
    grads = [torch.randn(n, device="cuda") * (0.1 + i) for i in range(5)]

    pr = torch.nn.Parameter(p0.clone())
    opt = torch.optim.Adam([pr], lr=2e-4, betas=(0.5, 0.999))
    for g in grads:
        pr.grad = g.clone()
        opt.step()

    p = torch.nn.Parameter(p0.clone())
    ours = optim.Adam([p], lr=2e-4, betas=(0.5, 0.999), eps=1e-8)
    for g in grads:
        p.grad = g.clone()
        ours.step()
    so, st = ours.state[p], opt.state[pr]
    assert so["step"].item() == 5.0  # the step count lives on the device (CUDA-graph capturable)
    assert rel_err(so["exp_avg"], st["exp_avg"]) < 1e-6
    assert rel_err(so["exp_avg_sq"], st["exp_avg_sq"]) < 1e-6
    # parameters: within 5 fp32 ulps / 1e-8 of torch's after five steps (the two differ only in FMA contraction of the
    # moment updates, i.e. by at most one rounding of p per step)
    assert torch.allclose(p.detach(), pr.detach(), rtol=6e-7, atol=1e-8)
    # and the accumulated update itself (~1e-3 of |p|, so one ulp of p is ~1e-4 of it): 4 significant digits over
    # the whole vector; an fp32 CPU emulation of the kernel's arithmetic sits at 2.5e-6
    if n >= 1000:
        assert rel_err(p.detach() - p0, pr.detach() - p0) < 2e-4


def test_adam_grad_scale_is_the_all_reduce_average():
    """grad_scale = 1/world_size folds the averaging of an all-reduce(sum) into the update (b200gan/ddp.py)."""
    from b200gan import optim
    torch.manual_seed(6)
    n = 4097
    p0, g = torch.randn(n, device="cuda"), torch.randn(n, device="cuda")
    outs = []
    for grad, scale in ((g * 4.0, 0.25), (g, 1.0)):
        p = torch.nn.Parameter(p0.clone())
        ours = optim.Adam([p], lr=2e-4, betas=(0.5, 0.999))
        ours.grad_scale = scale
        p.grad = grad.clone()
        ours.step()
        outs.append((p.detach(), ours.state[p]["exp_avg"], ours.state[p]["exp_avg_sq"]))
    for a, b in zip(*outs):
        assert torch.equal(a, b)  # x4 and x0.25 are exact in binary floating point


def test_multi_tensor_adam_optimizer_matches_torch_adam():
    """b200gan.optim.Adam: one launch for all parameters (b200gan_adam_multi), torch.optim.Adam's constructor and state
    layout; five steps on tensors of awkward sizes (several blocks per tensor, a 1-element tensor)."""
    from b200gan import optim
    torch.manual_seed(7)
    shapes = [(64, 128, 3, 3), (64,), (1,), (5000,), (1, 2048), (33, 7)]
    ref_p = [torch.nn.Parameter(torch.randn(s, device="cuda")) for s in shapes]
    our_p = [torch.nn.Parameter(p.detach().clone()) for p in ref_p]
    ref = torch.optim.Adam(ref_p, lr=2e-4, betas=(0.5, 0.999))
    ours = optim.Adam(our_p, lr=2e-4, betas=(0.5, 0.999))
    for it in range(5):
        for pr, po in zip(ref_p, our_p):
            g = torch.randn_like(pr) * (0.1 + it)
            pr.grad, po.grad = g.clone(), g.clone()
        ref.step()
        ours.step()
    for pr, po in zip(ref_p, our_p):
        assert torch.allclose(po, pr, rtol=6e-7, atol=1e-8)
        assert rel_err(ours.state[po]["exp_avg"], ref.state[pr]["exp_avg"]) < 1e-6
        assert rel_err(ours.state[po]["exp_avg_sq"], ref.state[pr]["exp_avg_sq"]) < 1e-6
        assert ours.state[po]["step"].item() == 5.0
    sd = ours.state_dict()
    assert len(sd["state"]) == len(shapes) and "_b200" not in sd["param_groups"][0]


def test_multi_tensor_adam_in_a_cuda_graph():
    from b200gan import optim
    torch.manual_seed(8)
    p = torch.nn.Parameter(torch.randn(10000, device="cuda"))
    q = torch.nn.Parameter(p.detach().clone())
    ref = torch.optim.Adam([p], lr=2e-4, betas=(0.5, 0.999))
    ours = optim.Adam([q], lr=2e-4, betas=(0.5, 0.999))
    g_static = torch.randn(10000, device="cuda")
    q.grad = g_static
    ours.step()  # warm-up outside the graph (allocates the state)
    p.grad = g_static.clone()
    ref.step()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        ours.step()
    for i in range(3):
        g_static.copy_(torch.randn(10000, device="cuda") * (i + 1))
        graph.replay()
        p.grad = g_static.clone()
        ref.step()
    torch.cuda.synchronize()
    # the capture itself does not execute; warm-up + 3 replays = 4 steps
    assert ours.state[q]["step"].item() == 4.0
    assert torch.allclose(q, p, rtol=6e-7, atol=1e-8)


def test_adam_step_invalidates_the_packed_weight_caches():
    """The optimizer kernel writes parameters through raw pointers; the conv modules' packed (wgmma / SIMT) weight
    copies are keyed on the tensor version counter, which optim.Adam bumps.  Forward after a step must use the NEW
    weights (fprop and dgrad read packed copies)."""
    from b200gan import nn as bnn, optim
    torch.manual_seed(9)
    for cin, cout in ((64, 64), (3, 8)):      # wgmma path and SIMT path
        ours = bnn.Conv2d(cin, cout, 3, 1, 1).cuda()
        ref = torch.nn.Conv2d(cin, cout, 3, 1, 1).cuda()
        ref.load_state_dict(ours.state_dict())
        oo = optim.Adam(ours.parameters(), lr=1e-2, betas=(0.5, 0.999))
        orf = torch.optim.Adam(ref.parameters(), lr=1e-2, betas=(0.5, 0.999))
        x = torch.randn(2, cin, 16, 16, device="cuda")
        y_prev = None
        for it in range(3):
            xo, xr = x.clone().requires_grad_(True), x.clone().requires_grad_(True)
            yo, yr = ours(xo), ref(xr)
            # Adam's m/sqrt(v) turns TF32-level gradient noise on near-zero gradient elements into O(lr) parameter
            # differences, so after a step the bound is 2e-2; a STALE packed copy would be off by the whole update
            # (lr 1e-2 on weights of ~4e-2: > 1e-1), which the second assert pins down directly
            assert rel_err(yo, yr) < (2e-3 if it == 0 else 2e-2)
            if y_prev is not None:
                assert rel_err(yo, y_prev) > 5e-2
            y_prev = yo.detach().clone()
            oo.zero_grad(); orf.zero_grad()
            yo.square().mean().backward(); yr.square().mean().backward()
            assert rel_err(xo.grad, xr.grad) < (5e-3 if it == 0 else 3e-2)
            oo.step(); orf.step()
        assert rel_err(ours.weight, ref.weight) < 2e-2


def _reference_pack(w, kind, transposed):
    """The packed layout of include/b200gan.h restated in torch: taps outermost, then [ci][co] or [co][ci]; the x2-upsample
    kinds sum the 3x3 taps of each phase tap in fp32, r-major then s, from 0; the TC kinds round to TF32 as
    cvt.rna.tf32.f32 does (to nearest, ties away from zero)."""
    from b200gan import _lib
    wk = w.transpose(0, 1) if transposed else w          # [co][ci][r][s]; ConvTranspose2d stores [ci][co][r][s]
    if kind in (_lib.PACK_TC_FPROP_UP2, _lib.PACK_TC_DGRAD_UP2):
        rset = {(0, 0): (0,), (0, 1): (1, 2), (1, 0): (0, 1), (1, 1): (2,)}   # 3x3 taps behind phase a, tap d
        taps = []
        for a, b, dr, ds in itertools.product((0, 1), repeat=4):            # t = (2a + b) * 4 + 2dr + ds
            v = torch.zeros_like(wk[:, :, 0, 0])
            for r in rset[a, dr]:
                for s in rset[b, ds]:
                    v = v + wk[:, :, r, s]
            taps.append(v)
        packed = torch.stack(taps)                                           # [16][co][ci]
    else:
        packed = wk.permute(2, 3, 0, 1).flatten(0, 1)                        # [r*S + s][co][ci]
    if kind in (_lib.PACK_SIMT_FPROP, _lib.PACK_TC_DGRAD, _lib.PACK_TC_DGRAD_UP2):
        packed = packed.transpose(1, 2)                                      # [tap][ci][co]
    packed = packed.contiguous()
    if kind != _lib.PACK_SIMT_FPROP and kind != _lib.PACK_SIMT_DGRAD:
        packed = ((packed.view(torch.int32) + 0x1000) & ~0x1FFF).view(torch.float32)
    return packed.flatten()


def test_multi_pack_is_bit_identical_to_the_per_layer_pack():
    """b200gan_pack_weights (one copy) and b200gan_pack_weights_multi (one launch per optimizer step) against the packed
    layout restated in torch: every layout, Conv2d and ConvTranspose2d parameters, ragged channel counts, a layer too
    narrow for the shared-memory tiles (element-wise mode), the folded x2-upsample layouts -- index arithmetic only, so
    bit-exact."""
    from b200gan import ops
    from b200gan import _lib
    torch.manual_seed(11)
    cases = []   # (x shape, weight shape, stride, pads, up, transposed, kinds)
    plain = (_lib.PACK_SIMT_FPROP, _lib.PACK_SIMT_DGRAD, _lib.PACK_TC_FPROP, _lib.PACK_TC_DGRAD)
    cases.append(((2, 64, 16, 16), (128, 64, 4, 4), 2, (1, 1, 1, 1), 1, False, plain))
    cases.append(((2, 40, 16, 16), (72, 40, 3, 3), 1, (1, 1, 1, 1), 1, False, plain))        # ragged tiles
    cases.append(((2, 128, 8, 8), (128, 64, 4, 4), 2, (1, 1, 1, 1), 1, True, plain))         # ConvTranspose2d [Cin][Cout][R][S]
    cases.append(((2, 3, 16, 16), (64, 3, 4, 4), 2, (1, 1, 1, 1), 1, False, plain))          # too narrow for tiles
    cases.append(((2, 128, 16, 16), (64, 128, 3, 3), 1, (1, 1, 1, 1), 2, False,
                  (_lib.PACK_TC_FPROP_UP2, _lib.PACK_TC_DGRAD_UP2)))
    jobs, refs = [], []
    for xs, ws, st, pads, up, tr, kinds in cases:
        w = torch.randn(*ws, device="cuda")
        g, _ = ops.make_geom(xs, ws, st, pads, 0, up, tr)
        for kind in kinds:
            ref = _reference_pack(w, kind, tr)
            assert torch.equal(ops.pack_weights(g, w, kind), ref), (tuple(w.shape), kind)
            jobs.append((g, kind, w, torch.full_like(ref, float("nan"))))
            refs.append(ref)
    ops.pack_weights_multi(jobs)
    for (g, kind, w, buf), ref in zip(jobs, refs):
        assert torch.equal(buf, ref), (tuple(w.shape), kind)
