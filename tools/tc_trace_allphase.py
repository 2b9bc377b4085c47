"""Per-CTA clock64 timeline of conv_tc_up2_allphase_kernel (same slot layout as tools/tc_trace.py) at the DCGAN conv2
shape (128 -> 64, 32x32 -> 64x64, batch 128): alone without an epilogue, alone with the step's epilogue (bias +
BatchNorm sums, as ConvFn.forward passes them), and inside the CUDA-graph-captured DCGAN training step.

    python tools/tc_trace_allphase.py
"""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "pytorch-gan_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)
import torch  # noqa: E402

from b200gan import ops  # noqa: E402
from b200gan._lib import ALGO_TC, PACK_TC_FPROP_UP2  # noqa: E402

NCTA = 4096


def gpu_clocks():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, timeout=30)
    return r.stdout.strip()


def traced(buf, fn):
    """runs fn with the trace pointer set: every launch fn makes (or captures) writes its timeline into buf"""
    os.environ["B200GAN_TC_TRACE"] = str(buf.data_ptr())
    try:
        return fn()
    finally:
        os.environ.pop("B200GAN_TC_TRACE", None)


def report(name, buf):
    t = buf.view(NCTA, 64).cpu()
    used = (t[:, 0] != 0).nonzero().flatten()
    f = lambda a, b: (t[used, a] - t[used, b]).float()  # noqa: E731
    print(f"== {name}: {len(used)} CTAs")
    for nm, v in [("lifetime", f(42, 0)), ("start -> epilogue start (main loop)", f(40, 0)),
                  ("first 15 producer intervals /15", f(17, 2) / 15),
                  ("epilogue start -> phase 0 store issued", f(50, 40)),
                  ("phase 0 -> phase 3 store issued", f(59, 50)),
                  ("phase 3 issued -> stores read", f(41, 59)),
                  ("stores read -> exit (statistics atomics)", f(42, 41))]:
        print(f"   {nm:42s} mean {v.mean():8.0f}  min {v.min():8.0f}  max {v.max():8.0f}")


def alone(epilogue):
    x = torch.randn(128, 128, 32, 32, device="cuda").contiguous(memory_format=torch.channels_last)
    wt = torch.randn(64, 128, 3, 3, device="cuda") * 0.02
    g, _ = ops.make_geom(tuple(x.shape), tuple(wt.shape), 1, (1, 1, 1, 1), 0, 2, False)
    packed = ops.pack_weights(g, wt, PACK_TC_FPROP_UP2)
    bias = torch.randn(64, device="cuda")
    stats = torch.zeros(128, device="cuda", dtype=torch.float64)
    kw = {"bias": bias, "stats": stats} if epilogue else {}
    fn = lambda: ops.conv_fprop(g, x, packed, ALGO_TC, **kw)  # noqa: E731
    for _ in range(3):
        fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(20):
        fn()
    e1.record()
    torch.cuda.synchronize()
    buf = torch.zeros(NCTA * 64, device="cuda", dtype=torch.int64)
    traced(buf, fn)
    torch.cuda.synchronize()
    report(f"alone, {'bias + BatchNorm sums' if epilogue else 'no epilogue'}: "
           f"{e0.elapsed_time(e1) / 20 * 1e3:.1f} us per launch", buf)


def in_step(steps=10):
    """The trace pointer is read when the launch is captured, so it is set only around the all-phase conv_fprop call
    (the step's other tensor-core launches would overwrite the same slots)."""
    import bench
    from b200gan import train
    buf = torch.zeros(NCTA * 64, device="cuda", dtype=torch.int64)
    orig = ops.conv_fprop
    seen = {}

    def conv_fprop(g, x, packed, algo, **kw):
        if algo == ALGO_TC and g.up == 2 and g.K % 128 != 0:
            seen.update({k: tuple(v.shape) if torch.is_tensor(v) else v for k, v in kw.items()})
            return traced(buf, lambda: orig(g, x, packed, algo, **kw))
        return orig(g, x, packed, algo, **kw)

    ops.conv_fprop = conv_fprop
    try:
        torch.backends.cudnn.allow_tf32 = True
        dev = torch.device("cuda", 0)
        step, pools, _, _ = bench.build_job(torch, "dcgan", False, dev, 1, 0)
        dev_pools = [[t.to(dev) for t in p] for p in pools]
        runner = train.GraphedStep(step, [p[0] for p in dev_pools], warmup=3)
    finally:
        ops.conv_fprop = orig
    print("   epilogue arguments in the step:", seen)
    for i in range(steps):
        runner(*[p[i % len(p)] for p in dev_pools])
    torch.cuda.synchronize()
    report(f"inside the graphed DCGAN step (last of {steps} replays)", buf)


if __name__ == "__main__":
    print("GPU:", gpu_clocks())
    alone(False)
    alone(True)
    in_step()
    print("GPU:", gpu_clocks())
