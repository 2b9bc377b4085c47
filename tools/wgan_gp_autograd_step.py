"""Time the reference-form WGAN-GP critic iteration (wgan_gp.py:155-174: the penalty built with
autograd.grad(create_graph=True), then d_loss.backward()) at BASELINE config-2 size, three arms:

    stock    stock torch.nn modules, train.wgan_gp_critic_step(..., fused_gp=False)
    dropin   the b200gan drop-in modules, same call: the critic runs through functional.MlpCriticFn (three critic
             forwards, three first-order backwards, one double backward), torch keeps the penalty arithmetic and the
             gradient accumulation
    step     the drop-ins with fused_gp="step": the whole iteration in one kernel (a floor, not the same program)

    python tools/wgan_gp_autograd_step.py [--batch 64] [--img 32] [--rounds 10] [--iters 50] [--out FILE]

Each arm is captured once into a CUDA graph (train.GraphedStep) and replayed; the arms alternate round by round and
every round times `iters` replays with CUDA events.  Launches per iteration come from a separate torch.profiler run of
eager iterations.  Prints the card's name and power limit with the numbers.
"""
import argparse
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "pytorch-gan_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)
import torch  # noqa: E402

ARMS = ("stock", "dropin", "step")


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip().splitlines()[0]
    except Exception as e:  # the numbers are still useful without it; say so
        return f"{torch.cuda.get_device_name()} (power limit unknown: {type(e).__name__})"


def build(arm, batch, img):
    from b200gan import optim, train, zoo
    ns = zoo.namespace(stock=arm == "stock")
    torch.manual_seed(0)
    g = zoo.WGANGPGenerator((1, img, img), nn=ns).cuda()
    d = zoo.WGANGPDiscriminator((1, img, img), nn=ns).cuda()
    if arm == "stock":
        od = torch.optim.Adam(d.parameters(), lr=2e-4, betas=(0.5, 0.999), capturable=True)
    else:
        od = optim.Adam(d.parameters(), lr=2e-4, betas=(0.5, 0.999))
    fused = {"stock": False, "dropin": False, "step": "step"}[arm]

    def step(real, z, alpha):
        dl, gp = train.wgan_gp_critic_step(g, d, od, real, z, alpha, 10.0, fused_gp=fused)
        return torch.stack([dl, gp])
    gen = torch.Generator().manual_seed(1)
    inputs = (torch.rand(batch, 1, img, img, generator=gen).cuda() * 2 - 1, torch.randn(batch, 100, generator=gen).cuda(),
              torch.rand(batch, 1, 1, 1, generator=gen).cuda())
    return step, inputs


def launches(step, inputs, iters=5):
    from torch.profiler import ProfilerActivity, profile
    step(*inputs)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(iters):
            step(*inputs)
        torch.cuda.synchronize()
    kernels = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA
               and not e.name.startswith(("Memcpy", "Memset"))]
    return len(kernels) / iters


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
             f"# WGAN-GP critic iteration, batch {a.batch}, {a.img}x{a.img}; CUDA-graph replay, {a.rounds} alternating "
             f"rounds x {a.iters} replays per arm"]
    arms, first = {}, {}
    for arm in ARMS:
        step, inputs = build(arm, a.batch, a.img)
        first[arm] = step(*inputs).tolist()     # from the same initial weights and inputs
        n_launch = launches(step, inputs)
        arms[arm] = (train.GraphedStep(step, inputs), inputs, n_launch)
    times = {arm: [] for arm in ARMS}
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for arm in ARMS:                              # warm-up replays
        graphed, inputs, _ = arms[arm]
        for _ in range(20):
            graphed.graph.replay()
    torch.cuda.synchronize()
    for _ in range(a.rounds):
        for arm in ARMS:
            graphed = arms[arm][0]
            e0.record()
            for _ in range(a.iters):
                graphed.graph.replay()
            e1.record()
            e1.synchronize()
            times[arm].append(e0.elapsed_time(e1) / a.iters)
    lines.append(f"{'arm':8s} {'ms/iter median':>15s} {'min':>8s} {'max':>8s} {'launches/iter':>14s}  first d_loss, gp")
    for arm in ARMS:
        t = times[arm]
        lines.append(f"{arm:8s} {statistics.median(t):15.4f} {min(t):8.4f} {max(t):8.4f} {arms[arm][2]:14.1f}  "
                     f"{first[arm][0]:.6f}, {first[arm][1]:.6f}")
    text = "\n".join(lines)
    print(text)
    if a.out:
        with open(a.out, "w") as fh:
            fh.write(text + "\n")


if __name__ == "__main__":
    main()
