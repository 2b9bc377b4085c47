"""Per-kernel device time of one training step of a bench.py config, replayed from a CUDA graph, under torch.profiler
with CUDA activities (kernel names, launches per step, us per step, share of the step), as a text table.

    python tools/profile_step.py [--config dcgan] [--steps 20] [--out FILE]

Run it on its own: tracing slows the host, so step times come from bench.py, not from this.
"""
import argparse
import collections
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "pytorch-gan_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)
import torch  # noqa: E402


def gpu_name_and_power_limit():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip().splitlines()[0]
    except Exception as e:  # the table is still useful without it; say so
        return f"unknown ({type(e).__name__})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="dcgan")
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import bench
    import b200gan
    from b200gan import train
    from torch.profiler import ProfilerActivity, profile

    b200gan.load_library()
    torch.backends.cudnn.allow_tf32 = True
    dev = torch.device("cuda", 0)
    step, pools, _, _ = bench.build_job(torch, a.config, False, dev, 1, 0)
    dev_pools = [[t.to(dev) for t in p] for p in pools]
    n = len(dev_pools[0])
    runner = train.GraphedStep(step, [p[0] for p in dev_pools], warmup=3)
    for i in range(5):
        runner(*[p[i % n] for p in dev_pools])
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for i in range(a.steps):
            runner(*[p[i % n] for p in dev_pools])
        torch.cuda.synchronize()
    tot = collections.defaultdict(float)
    cnt = collections.Counter()
    for ev in prof.events():
        if ev.device_type == torch.autograd.DeviceType.CUDA:
            tot[ev.name] += ev.time_range.elapsed_us()
            cnt[ev.name] += 1
    busy = sum(tot.values()) / a.steps
    lines = [f"# {a.config} step, graph-replayed, {a.steps} steps under torch.profiler (CUDA activities)",
             f"# GPU: {gpu_name_and_power_limit()}  (name, power limit, max SM clock)",
             f"# kernel + copy time per step: {busy:.1f} us (sum of device activity; gaps not included)",
             f"{'us/step':>9s} {'share':>6s} {'launches/step':>13s}  kernel"]
    for name, t in sorted(tot.items(), key=lambda kv: -kv[1]):
        lines.append(f"{t / a.steps:9.1f} {t / a.steps / busy * 100:5.1f}% {cnt[name] / a.steps:13.1f}  {name[:160]}")
    text = "\n".join(lines) + "\n"
    sys.stdout.write(text)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fh:
            fh.write(text)


if __name__ == "__main__":
    main()
