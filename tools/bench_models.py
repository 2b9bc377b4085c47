"""Step throughput of BASELINE configs 2-4 (WGAN-GP 32x32 bs64, Pix2Pix 256x256 bs16, CycleGAN 256x256 bs8) on one
H100 with the drop-in modules, next to the same step on stock torch (cuDNN, TF32 default = the reference's own GPU
path).  Eager loops (no CUDA graph), CUDA-event timing.  Prints one JSON line per config.

    python tools/bench_models.py [--steps 10] [--only pix2pix|cyclegan|wgan_gp]
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "pytorch-gan_b200"))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

from b200gan import train, zoo  # noqa: E402

CL = torch.channels_last


def adam(params):
    return torch.optim.Adam(params, lr=2e-4, betas=(0.5, 0.999))


def timeit(fn, steps, warmup=3):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def build(kind, stock):
    ns = zoo.namespace(stock=stock)
    torch.manual_seed(0)
    if kind == "pix2pix":
        g, d = zoo.GeneratorUNet(nn=ns).cuda(), zoo.Pix2PixDiscriminator(nn=ns).cuda()
        g.apply(zoo.weights_init_normal); d.apply(zoo.weights_init_normal)
        return g, d
    if kind == "cyclegan":
        shape = (3, 256, 256)
        nets = [zoo.GeneratorResNet(shape, 9, nn=ns), zoo.GeneratorResNet(shape, 9, nn=ns),
                zoo.CycleGANDiscriminator(shape, nn=ns), zoo.CycleGANDiscriminator(shape, nn=ns)]
        for m in nets:
            m.cuda().apply(zoo.weights_init_normal_cyclegan)
        return nets
    g, d = zoo.WGANGPGenerator((1, 32, 32), nn=ns).cuda(), zoo.WGANGPDiscriminator((1, 32, 32), nn=ns).cuda()
    return g, d


def run(kind, steps):
    out = {}
    for stock in (True, False):
        tag = "stock_torch_tf32" if stock else "b200gan"
        if kind == "pix2pix":
            n = 16
            g, d = build(kind, stock)
            og, od = adam(g.parameters()), adam(d.parameters())
            a = (torch.rand(n, 3, 256, 256, device="cuda") * 2 - 1).contiguous(memory_format=CL)
            b = (torch.rand(n, 3, 256, 256, device="cuda") * 2 - 1).contiguous(memory_format=CL)
            ms = timeit(lambda: train.pix2pix_step(g, d, og, od, a, b), steps)
            out[tag] = {"ms_per_step": ms, "images_per_s": n / ms * 1e3}
        elif kind == "cyclegan":
            n = 8
            g_ab, g_ba, d_a, d_b = build(kind, stock)
            import itertools
            og = adam(itertools.chain(g_ab.parameters(), g_ba.parameters()))
            oa, ob = adam(d_a.parameters()), adam(d_b.parameters())
            a = (torch.rand(n, 3, 256, 256, device="cuda") * 2 - 1).contiguous(memory_format=CL)
            b = (torch.rand(n, 3, 256, 256, device="cuda") * 2 - 1).contiguous(memory_format=CL)
            ba, bb = train.ReplayBuffer(), train.ReplayBuffer()
            ms = timeit(lambda: train.cyclegan_step(g_ab, g_ba, d_a, d_b, og, oa, ob, a, b, ba, bb), steps)
            out[tag] = {"ms_per_step": ms, "image_pairs_per_s": n / ms * 1e3}
        else:
            n = 64
            g, d = build(kind, stock)
            od = adam(d.parameters())
            real = torch.rand(n, 1, 32, 32, device="cuda") * 2 - 1
            z = torch.randn(n, 100, device="cuda")
            alpha = torch.rand(n, 1, 1, 1, device="cuda")
            ms = timeit(lambda: train.wgan_gp_critic_step(g, d, od, real, z, alpha, 10.0, fused_gp=not stock), steps * 10)
            out[tag] = {"us_per_critic_iter": ms * 1e3}
        torch.cuda.empty_cache()
    key = "ms_per_step" if kind != "wgan_gp" else "us_per_critic_iter"
    out["speedup_vs_stock_torch"] = out["stock_torch_tf32"][key] / out["b200gan"][key]
    print(json.dumps({"config": kind, **out}), flush=True)


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--only", default=None)
    a = ap.parse_args()
    torch.backends.cudnn.allow_tf32 = True
    torch.backends.cuda.matmul.allow_tf32 = True
    for kind in ("wgan_gp", "pix2pix", "cyclegan"):
        if a.only in (None, kind):
            run(kind, a.steps)
