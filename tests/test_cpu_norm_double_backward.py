"""The double backward of a training-mode BatchNorm2d / InstanceNorm2d with a fused LeakyReLU / ReLU, without a GPU:
the closed form b200gan_norm_dbwd computes (include/b200gan.h, csrc/norm.cu), written in fp64 and held to torch float64
double backward; and what ptxas makes of norm.cu now that its backward kernels carry a double-backward mode.

Notation (one normalisation group of m elements: a channel over N*H*W, or a (sample, channel) over H*W):
r = 1/sqrt(biased var + eps), xhat = (x - mean) r, a' = the activation's mask at x*scale + shift, g = dy a'.
First backward: dx = gamma r (g - A - xhat B), S1 = sum g, S2 = sum g xhat, A = S1/m, B = S2/m; dgamma = S2, dbeta = S1.
Incoming u = dL/d(dx), ugamma, ubeta; U = sum u, T = sum u xhat, Q = sum u g:
  dL/d(dy)    = a' (gamma r (u - U/m - xhat T/m) + ugamma xhat + ubeta)
  dL/d(gamma) = r (Q - A U - B T)   per group (summed over samples for InstanceNorm)
  dL/dx       = ugamma r (g - A - xhat B) - (gamma r^2/m) (xhat (Q - A U - 3 B T) + T (g - A) + B (m u - U))
Nothing assumes sum xhat^2 = m, which fails for DCGAN's eps = 0.8.
"""
import os

import pytest
import torch
import torch.nn.functional as tf

from conformance import CSRC, declared, needs_nvcc, ptxas_report
from norm_cases import KERNELS, SLOPE, closed_form

NORM_CU = os.path.join(CSRC, "norm.cu")


def torch_double_backward(x, dy, gamma, beta, u, ugamma, ubeta, eps, act, per_sample):
    x, dy = x.clone().requires_grad_(True), dy.clone().requires_grad_(True)
    params = [] if gamma is None else [gamma.clone().requires_grad_(True), beta.clone().requires_grad_(True)]
    ga, be = (params + [None, None])[:2]
    if per_sample:
        z = tf.instance_norm(x, weight=ga, bias=be, eps=eps)
    else:
        z = tf.batch_norm(x, None, None, ga, be, training=True, eps=eps)
    y = {"none": lambda: z, "lrelu": lambda: tf.leaky_relu(z, SLOPE), "relu": lambda: torch.relu(z)}[act]()
    first = torch.autograd.grad(y, [x] + params, dy, create_graph=True)
    loss = (first[0] * u).sum()
    if params and ugamma is not None:
        loss = loss + (first[1] * ugamma).sum() + (first[2] * ubeta).sum()
    second = torch.autograd.grad(loss, [dy, x] + params[:1], allow_unused=True)
    return second[0], second[1], (second[2] if params else None)


def rel(a, b):
    return ((a - b).abs().max() / b.abs().max().clamp_min(1e-300)).item()


@pytest.mark.parametrize("per_sample", [False, True], ids=["bn", "in"])
@pytest.mark.parametrize("affine", [True, False], ids=["affine", "plain"])
@pytest.mark.parametrize("eps", [0.8, 1e-5])
@pytest.mark.parametrize("act", ["none", "lrelu", "relu"])
@pytest.mark.parametrize("incoming", ["u_gamma_beta", "u_only"])
def test_closed_form_matches_torch_float64_double_backward(per_sample, affine, eps, act, incoming):
    gen = torch.Generator().manual_seed(3)
    n, c, h, w = 4, 6, 5, 3
    f64 = torch.float64
    x = torch.randn(n, c, h, w, generator=gen, dtype=f64) * 2 + 0.5
    dy = torch.randn(n, c, h, w, generator=gen, dtype=f64)
    u = torch.randn(n, c, h, w, generator=gen, dtype=f64)
    gamma = 1 + 0.5 * torch.randn(c, generator=gen, dtype=f64) if affine else None
    beta = 0.3 * torch.randn(c, generator=gen, dtype=f64) if affine else None
    ug = ub = None
    if affine and incoming == "u_gamma_beta":
        ug, ub = torch.randn(c, generator=gen, dtype=f64), torch.randn(c, generator=gen, dtype=f64)
    got = closed_form(x, dy, gamma, beta, u, ug, ub, eps, act, per_sample)
    ref = torch_double_backward(x, dy, gamma, beta, u, ug, ub, eps, act, per_sample)
    for name, a, b in zip(("dL/d(dy)", "dL/dx", "dL/dgamma"), got, ref):
        if b is None:
            assert a is None or not affine, name
            continue
        assert rel(a, b) < 1e-10, f"{name}: {rel(a, b):.3e}"


def test_norm_cu_still_declares_exactly_the_six_kernels():
    assert declared(NORM_CU) == KERNELS


@needs_nvcc
def test_norm_backward_kernels_keep_their_register_and_shared_memory_budgets():
    """Every norm.cu instance: no stack frame, no spills.  The VEC 4 backward instances stay at or below 80 registers
    (3 blocks of 256 threads per SM); the reduce instances keep their 2048 / 8192 B of shared memory."""
    rep = ptxas_report(NORM_CU)
    for name, r in rep.items():
        assert r["stack"] == r["spills"] == 0, f"{name}: {r}"
    regs = {k: r["registers"] for k, r in rep.items()}
    smem = {k: r["smem"] for k, r in rep.items()}
    assert regs["norm_bwd_reduce_kernel<4>"] <= 80 and regs["norm_bwd_apply_kernel<4>"] <= 80, regs
    assert smem["norm_bwd_reduce_kernel<1>"] == 2048 and smem["norm_bwd_reduce_kernel<4>"] == 8192, smem
    assert smem["norm_bwd_apply_kernel<1>"] == smem["norm_bwd_apply_kernel<4>"] == 0, smem
