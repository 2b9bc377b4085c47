"""Device time of ops.norm_forward and ops.norm_backward (BatchNorm2d and InstanceNorm2d + LeakyReLU) at channel
counts no reference model has, where the plan differs from the reference layers: C = 5 (scalar channel groups),
96 and 768 (a block's rows do not use all 256 threads) and 1280 (two channel slices).  One JSON line per shape.

    python tools/norm_shapes.py [--iters 50]

CUDA events around `iters` back-to-back calls after a warm-up; prints the card's name and power limit first.
The backward is timed with the saved output y and without scale_shift, as bench.py times it.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "pytorch-gan_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)
import torch  # noqa: E402

# (N, C, H, W): 5 M to 21 M elements, sizes a user of the library would normalise
SHAPES = ((16, 5, 256, 256), (16, 96, 128, 64), (16, 768, 32, 32), (16, 1280, 32, 32))


def event_ms(fn, iters):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    a = ap.parse_args()
    from b200gan import _lib, ops
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    print(json.dumps({"gpu": r.stdout.strip()}))
    for n, c, h, w in SHAPES:
        x = torch.randn(n, c, h, w, device="cuda").contiguous(memory_format=torch.channels_last)
        dy = torch.randn_like(x)
        gamma, beta = torch.ones(c, device="cuda"), torch.zeros(c, device="cuda")
        for per_sample in (False, True):
            g, b = (None, None) if per_sample else (gamma, beta)
            eps = 1e-5 if per_sample else 0.8

            def fwd():
                return ops.norm_forward(x, g, b, None, None, None, per_sample, eps, 0.1, _lib.ACT_LRELU, 0.2)

            y, mr = fwd()
            f_ms = event_ms(fwd, a.iters)
            b_ms = event_ms(lambda: ops.norm_backward(dy, x, y, mr, g, per_sample, eps, _lib.ACT_LRELU, 0.2,
                                                      not per_sample), a.iters)
            print(json.dumps({"norm": "instance" if per_sample else "batch", "shape": [n, c, h, w],
                              "forward_ms": round(f_ms, 4), "backward_ms": round(b_ms, 4)}))


if __name__ == "__main__":
    main()
