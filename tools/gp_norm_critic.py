"""Time the DRAGAN critic iteration (dragan.py:144-190: D(real), D(fake), the penalty on perturbed interpolates with its
double backward through BatchNorm2d(.8), d_loss.backward(), Adam) on the DCGAN discriminator at the DCGAN bench size,
b200gan drop-ins against stock torch fp32, alternating the two in one process: eager iterations between CUDA events
(the stock iteration cannot be replayed from a CUDA graph here); the launch count comes from one iteration under
torch.profiler.

    python tools/gp_norm_critic.py [--img 64] [--batch 128] [--iters 50] [--rounds 5] [--out FILE]
"""
import argparse
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "pytorch-gan_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)


def build(stock, img, batch):
    from b200gan import optim as bopt, zoo
    torch.manual_seed(0)
    d = zoo.DCGANDiscriminator(img, 1, nn=zoo.namespace(stock=stock)).cuda().train()
    opt = (torch.optim.Adam if stock else bopt.Adam)(d.parameters(), lr=2e-4, betas=(0.5, 0.999))
    real = torch.rand(batch, 1, img, img, device="cuda") * 2 - 1
    fake = torch.rand(batch, 1, img, img, device="cuda") * 2 - 1
    bce = torch.nn.BCELoss() if stock else zoo.namespace().BCELoss()
    ones, zeros = torch.ones(batch, 1, device="cuda"), torch.zeros(batch, 1, device="cuda")

    def iteration():
        opt.zero_grad(set_to_none=False)
        alpha = torch.rand(real.shape, device="cuda")
        xh = (alpha * real + (1 - alpha) * (real + 0.5 * real.std() * torch.rand(real.shape, device="cuda")))
        xh.requires_grad_(True)
        out = d(xh)
        g = torch.autograd.grad(out, xh, torch.ones_like(out), create_graph=True, retain_graph=True)[0]
        gp = 10.0 * ((g.norm(2, dim=1) - 1) ** 2).mean()
        loss = (bce(d(real), ones) + bce(d(fake), zeros)) / 2 + gp
        loss.backward()
        opt.step()
    return iteration


def launches(fn):
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return sum(1 for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--img", type=int, default=64)
    ap.add_argument("--batch", type=int, default=128)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    lines = [f"device: {torch.cuda.get_device_name()}", f"DRAGAN critic iteration, DCGAN discriminator, "
             f"{a.img}x{a.img}, batch {a.batch}; stock torch fp32 (cudnn.allow_tf32=False) vs b200gan drop-ins"]
    runs = {}
    for name, stock in (("stock", True), ("b200gan", False)):
        fn = build(stock, a.img, a.batch)
        for _ in range(3):
            fn()
        n = launches(fn)
        runs[name] = (fn, n)
        lines.append(f"{name}: {n} kernel launches per iteration (eager, torch.profiler)")
    times = {k: [] for k in runs}
    for _ in range(a.rounds):
        for name, (fn, _) in runs.items():
            fn()
            torch.cuda.synchronize()
            t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            t0.record()
            for _ in range(a.iters):
                fn()
            t1.record()
            torch.cuda.synchronize()
            times[name].append(t0.elapsed_time(t1) / a.iters)
    for name, ts in times.items():
        lines.append(f"{name}: {sum(ts) / len(ts):.3f} ms per iteration (eager, mean of {a.rounds} "
                     f"alternating rounds of {a.iters}; min {min(ts):.3f}, max {max(ts):.3f})")
    text = "\n".join(lines)
    print(text)
    if a.out:
        with open(a.out, "w") as fh:
            fh.write(text + "\n")


if __name__ == "__main__":
    main()
