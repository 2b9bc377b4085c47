"""Time MSELoss and L1Loss, forward + backward, on the pixel-loss kernels (csrc/pixel_loss) against stock ATen, at the
sizes the Pix2Pix and CycleGAN steps use them:

    pix2pix  L1  [16, 3, 256, 256]  generator output (channels_last) against the NCHW target   pix2pix.py:145
             MSE [16, 1, 16, 16]    PatchGAN output against ones                               pix2pix.py:143
    cyclegan L1  [8, 3, 256, 256]   cycle / identity: generator output (channels_last) vs NCHW cyclegan.py:180-197
             MSE [8, 1, 16, 16]     PatchGAN output against ones                               cyclegan.py:187-189

    python tools/pixel_loss_bench.py [--rounds 7] [--iters 100] [--out DIR]

One iteration is `loss = mod(x, t); torch.autograd.grad(loss, x)` with x a leaf that requires grad.  Every round traces
`iters` iterations of the library module, then of the stock module (alternating, so drift hits both), with
torch.profiler, and sums the durations of their CUDA kernels: GPU kernel time per iteration, without the Python
overhead that dominates an eager loop at these sizes.  The median, minimum and maximum over rounds are reported, with the
launches of one iteration.  Prints one JSON line per workload and the card's name and power limit.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "pytorch-gan_b200"))

import torch  # noqa: E402


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip().splitlines()[0]
    except Exception as e:  # the numbers are still useful without it; say so
        return f"power limit unknown: {type(e).__name__}"


WORKLOADS = [
    ("pix2pix L1 pixel", "L1Loss", (16, 3, 256, 256), "nhwc", "nchw"),
    ("pix2pix MSE adversarial", "MSELoss", (16, 1, 16, 16), "nchw", "nchw"),
    ("cyclegan L1 cycle/identity", "L1Loss", (8, 3, 256, 256), "nhwc", "nchw"),
    ("cyclegan MSE adversarial", "MSELoss", (8, 1, 16, 16), "nchw", "nchw"),
]


def operands(shape, la, lb, seed=0):
    g = torch.Generator().manual_seed(seed)
    x = torch.rand(shape, generator=g).mul(2).sub(1).cuda()
    t = torch.rand(shape, generator=g).mul(2).sub(1).cuda()
    if la == "nhwc":
        x = x.contiguous(memory_format=torch.channels_last)
    if lb == "nhwc":
        t = t.contiguous(memory_format=torch.channels_last)
    return x.requires_grad_(True), t


def one(mod, x, t):
    loss = mod(x, t)
    return loss, torch.autograd.grad(loss, x)[0]


def kernel_ms(mod, x, t, iters):
    """GPU kernel time of one iteration: the durations of the CUDA kernels of `iters` iterations, from a torch.profiler
    trace, over iters.  Times the kernels themselves, not the Python and autograd overhead of an eager loop (which hides
    them at these sizes) nor the gaps between launches."""
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(iters):
            one(mod, x, t)
        torch.cuda.synchronize()
    us = sum(e.device_time for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA
             and not e.name.startswith(("Memcpy", "Memset")))
    return us / 1e3 / iters


def launches(mod, x, t):
    """kernels of one iteration; a sacrificial kernel goes first, because the first record of a session can be lost"""
    from torch.profiler import ProfilerActivity, profile
    marker = torch.ones(1, device="cuda")
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        marker.neg_()  # a kernel neither loss launches
        torch.cuda.synchronize()
        one(mod, x, t)
        torch.cuda.synchronize()
    names = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA
             and not e.name.startswith(("Memcpy", "Memset")) and "neg_kernel" not in e.name]
    return len(names), sorted(set(names))


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--iters", type=int, default=100)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "pixel_loss_bench.py needs a GPU"
    import b200gan
    from b200gan import nn as bnn
    b200gan.load_library()
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    info = card()
    print(json.dumps({"card": info, "torch": torch.__version__}), flush=True)
    rows = []
    for name, cls, shape, la, lb in WORKLOADS:
        x, t = operands(shape, la, lb)
        ours, stock = getattr(bnn, cls)(), getattr(torch.nn, cls)()
        # same numbers first: the loss and the gradient against stock fp32
        lo, go = one(ours, x, t)
        ls, gs = one(stock, x, t)
        torch.cuda.synchronize()
        loss_rel = abs(lo.item() - ls.item()) / abs(ls.item())
        grad_rel = ((go.double() - gs.double()).norm() / gs.double().norm()).item()
        for mod in (ours, stock):
            for _ in range(20):
                one(mod, x, t)
        t_ours, t_stock = [], []
        for _ in range(a.rounds):
            t_ours.append(kernel_ms(ours, x, t, a.iters))
            t_stock.append(kernel_ms(stock, x, t, a.iters))
        n_ours, k_ours = launches(ours, x, t)
        n_stock, k_stock = launches(stock, x, t)
        row = {"workload": name, "module": cls, "shape": list(shape), "layouts": [la, lb],
               "ours_kernel_ms": statistics.median(t_ours), "ours_kernel_ms_min": min(t_ours), "ours_kernel_ms_max": max(t_ours),
               "aten_kernel_ms": statistics.median(t_stock), "aten_kernel_ms_min": min(t_stock), "aten_kernel_ms_max": max(t_stock),
               "ours_launches": n_ours, "aten_launches": n_stock, "ours_kernels": k_ours, "aten_kernels": k_stock,
               "loss_rel_diff": loss_rel, "grad_rel_diff": grad_rel, "card": info}
        rows.append(row)
        print(json.dumps(row), flush=True)
        del x, t
        torch.cuda.empty_cache()
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "pixel_loss_bench.json"), "w") as fh:
            json.dump(rows, fh, indent=1)


if __name__ == "__main__":
    main()
