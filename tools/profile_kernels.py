"""Run each hot kernel of the DCGAN step a few times in isolation (for `ncu --set full -k regex:...`), and
print CUDA-event timings + achieved TFLOP/s / GB/s for every one of them.

    python tools/profile_kernels.py [--iters 10]
"""
import argparse
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "pytorch-gan_b200"))
import torch  # noqa: E402

from b200gan import ops  # noqa: E402

CL = torch.channels_last


def timeit(fn, iters):
    for _ in range(2):
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
    ap.add_argument("--iters", type=int, default=10)
    a = ap.parse_args()
    n = 128
    rows = []
    # (name, cin, cout, k, stride, pad, h, w, up)  -- every conv of the DCGAN G and D at batch 128 / 64x64
    layers = [
        ("G conv1 up2 128->128 @16", 128, 128, 3, 1, 1, 16, 16, 2),
        ("G conv2 up2 128->64  @32", 128, 64, 3, 1, 1, 32, 32, 2),
        ("G conv3 64->1 @64", 64, 1, 3, 1, 1, 64, 64, 1),
        ("D conv1 1->16 s2 @64", 1, 16, 3, 2, 1, 64, 64, 1),
        ("D conv2 16->32 s2 @32", 16, 32, 3, 2, 1, 32, 32, 1),
        ("D conv3 32->64 s2 @16", 32, 64, 3, 2, 1, 16, 16, 1),
        ("D conv4 64->128 s2 @8", 64, 128, 3, 2, 1, 8, 8, 1),
        # CycleGAN / Pix2Pix interior layers (batch 8 / 16)
        ("CG res 256->256 @64 (bs8)", 256, 256, 3, 1, 1, 64, 64, 1, 8),
        ("CG down 128->256 s2 @128 (bs8)", 128, 256, 3, 2, 1, 128, 128, 1, 8),
        ("CG up2 256->128 @64 (bs8)", 256, 128, 3, 1, 1, 64, 64, 2, 8),
        ("P2P down 128->256 k4s2 @64 (bs16)", 128, 256, 4, 2, 1, 64, 64, 1, 16),
        ("P2P down 256->512 k4s2 @32 (bs16)", 256, 512, 4, 2, 1, 32, 32, 1, 16),
    ]
    for entry in layers:
        name, cin, cout, k, s, p, h, w, up = entry[:9]
        n = entry[9] if len(entry) > 9 else 128
        x = torch.randn(n, cin, h, w, device="cuda").contiguous(memory_format=CL)
        wt = torch.randn(cout, cin, k, k, device="cuda") * 0.02
        g, oshape = ops.make_geom(tuple(x.shape), tuple(wt.shape), s, (p, p, p, p), 0, up, False)
        dy = torch.randn(oshape, device="cuda").contiguous(memory_format=CL)
        flops_ref = 2.0 * oshape[0] * oshape[2] * oshape[3] * cout * cin * k * k
        flops_exec = flops_ref * (4.0 / 9.0 if up == 2 else 1.0)
        act_bytes = (x.numel() + dy.numel()) * 4
        for pas, pname in ((0, "fprop"), (1, "dgrad"), (2, "wgrad")):
            tc = ops.tc_supported(g, pas)
            algo, kind = ops.conv_plan(g, pas)
            if pas == 0:
                packed = ops.pack_weights(g, wt, kind)
                fn = lambda: ops.conv_fprop(g, x, packed, algo)  # noqa: E731
            elif pas == 1:
                packed = ops.pack_weights(g, wt, kind)
                fn = lambda: ops.conv_dgrad(g, dy, packed, algo)  # noqa: E731
            else:
                fn = lambda: ops.conv_wgrad(g, x, dy, tuple(wt.shape), True, algo)  # noqa: E731
            ms = timeit(fn, a.iters)
            fl = flops_exec if tc else flops_ref
            rows.append((name, pname, "wgmma" if tc else "simt", ms * 1e3, fl / ms / 1e9, act_bytes / ms / 1e6))
    print(f"{'layer':28s} {'pass':6s} {'path':8s} {'us':>9s} {'TFLOP/s':>9s} {'GB/s(act)':>10s}")
    for r in rows:
        print(f"{r[0]:28s} {r[1]:6s} {r[2]:8s} {r[3]:9.1f} {r[4]:9.2f} {r[5]:10.0f}")
    # normalisation / element-wise passes on the largest tensor of the step ([128,64,64,64] = 134 MB)
    n = 128
    x = torch.randn(n, 64, 64, 64, device="cuda").contiguous(memory_format=CL)
    gamma = torch.ones(64, device="cuda")
    beta = torch.zeros(64, device="cuda")
    y, mr = ops.norm_forward(x, gamma, beta, None, None, None, False, 0.8, 0.1, 1, 0.2)
    dyy = torch.randn_like(x)
    for nm, fn, nbytes in (
        ("BN fwd (stats+apply) 134MB", lambda: ops.norm_forward(x, gamma, beta, None, None, None, False, 0.8, 0.1, 1, 0.2), 3 * x.numel() * 4),
        ("BN bwd (reduce+apply) 134MB", lambda: ops.norm_backward(dyy, x, y, mr, gamma, False, 0.8, 1, 0.2, True), 7 * x.numel() * 4),
    ):
        ms = timeit(fn, a.iters)
        print(f"{nm:44s} {ms * 1e3:9.1f} us {nbytes / ms / 1e6:10.0f} GB/s")


if __name__ == "__main__":
    main()
