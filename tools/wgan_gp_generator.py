"""Time the WGAN-GP generator (wgan_gp.py:42-65) on its two paths in one process, at BASELINE config-2 size:

    torch    G built from a namespace whose BatchNorm1d and Sequential are the stock classes (a drop-in Sequential
             routes stock leaf classes too): the generator runs leaf by leaf on cuBLAS / ATen, the path before the
             fused generator kernels
    fused    G built from the drop-in namespace (zoo.namespace()): one launch forward, one launch backward

in two workloads:

    critic   bench.py --config wgan_gp's step: G(z) under torch.no_grad(), then the one-kernel critic iteration
             (train.wgan_gp_critic_step(..., fused_gp="step")) and the fused Adam
    gstep    the generator step (train.wgan_gp_generator_step): G forward and backward, D frozen, the fused Adam on G

    python tools/wgan_gp_generator.py [--batch 64] [--img 32] [--rounds 10] [--iters 50] [--out FILE]

Each (workload, arm) is captured once into a CUDA graph (train.GraphedStep) and replayed; the arms alternate round by
round and every round times `iters` replays with CUDA events.  Launches per iteration, attributed by kernel name, come
from a separate torch.profiler run of eager iterations.  Prints the card's name and power limit with the numbers.
"""
import argparse
import collections
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "pytorch-gan_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)
import torch  # noqa: E402

ARMS = ("torch", "fused")
WORKLOADS = ("critic", "gstep")


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip().splitlines()[0]
    except Exception as e:  # the numbers are still useful without it; say so
        return f"{torch.cuda.get_device_name()} (power limit unknown: {type(e).__name__})"


def build(workload, arm, batch, img):
    from b200gan import optim, train, zoo
    ns = zoo.namespace()
    if arm == "torch":
        ns.BatchNorm1d, ns.Sequential = torch.nn.BatchNorm1d, torch.nn.Sequential
    torch.manual_seed(0)
    g = zoo.WGANGPGenerator((1, img, img), nn=ns).cuda()
    d = zoo.WGANGPDiscriminator((1, img, img), nn=zoo.namespace()).cuda()
    gen = torch.Generator().manual_seed(1)
    if workload == "critic":
        od = optim.Adam(d.parameters(), lr=2e-4, betas=(0.5, 0.999))

        def step(real, z, alpha):
            dl, gp = train.wgan_gp_critic_step(g, d, od, real, z, alpha, 10.0, fused_gp="step")
            return torch.stack([dl, gp])
        inputs = (torch.rand(batch, 1, img, img, generator=gen).cuda() * 2 - 1,
                  torch.randn(batch, 100, generator=gen).cuda(), torch.rand(batch, 1, 1, 1, generator=gen).cuda())
    else:
        og = optim.Adam(g.parameters(), lr=2e-4, betas=(0.5, 0.999))

        def step(z):
            return train.wgan_gp_generator_step(g, d, og, z).reshape(1)
        inputs = (torch.randn(batch, 100, generator=gen).cuda(),)
    return step, inputs


def launches(step, inputs, iters=5):
    from torch.profiler import ProfilerActivity, profile
    step(*inputs)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(iters):
            step(*inputs)
        torch.cuda.synchronize()
    names = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA
             and not e.name.startswith(("Memcpy", "Memset"))]
    return len(names) / iters, {k: n / iters for k, n in collections.Counter(names).most_common()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--img", type=int, default=32)
    ap.add_argument("--rounds", type=int, default=10)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    torch.backends.cuda.matmul.allow_tf32 = False
    from b200gan import train
    lines = [f"# GPU: {card()}  (name, power limit, max SM clock)",
             f"# WGAN-GP generator, batch {a.batch}, {a.img}x{a.img}; CUDA-graph replay, {a.rounds} alternating rounds x "
             f"{a.iters} replays per arm"]
    runs, first, kinds = {}, {}, {}
    for wl in WORKLOADS:
        for arm in ARMS:
            step, inputs = build(wl, arm, a.batch, a.img)
            first[wl, arm] = step(*inputs).tolist()     # from the same initial weights and inputs
            n_launch, kinds[wl, arm] = launches(step, inputs)
            runs[wl, arm] = (train.GraphedStep(step, inputs), n_launch)
    for g, _ in runs.values():                          # warm-up replays
        for _ in range(20):
            g.graph.replay()
    torch.cuda.synchronize()
    times = {k: [] for k in runs}
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(a.rounds):
        for k, (g, _) in runs.items():
            e0.record()
            for _ in range(a.iters):
                g.graph.replay()
            e1.record()
            e1.synchronize()
            times[k].append(e0.elapsed_time(e1) / a.iters)
    lines.append(f"{'workload':9s} {'arm':6s} {'ms/iter median':>15s} {'min':>8s} {'max':>8s} {'launches/iter':>14s}  "
                 "first losses")
    for k, t in times.items():
        lines.append(f"{k[0]:9s} {k[1]:6s} {statistics.median(t):15.4f} {min(t):8.4f} {max(t):8.4f} "
                     f"{runs[k][1]:14.1f}  {', '.join(f'{v:.6f}' for v in first[k])}")
    for k, c in kinds.items():
        lines.append(f"# launches per iteration, {k[0]} / {k[1]}:")
        for name, n in c.items():
            lines.append(f"#   {n:5.1f}  {name[:140]}")
    text = "\n".join(lines)
    print(text)
    if a.out:
        with open(a.out, "w") as fh:
            fh.write(text + "\n")


if __name__ == "__main__":
    main()
