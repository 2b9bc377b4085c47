"""Which Python lines launch the small torch kernels of the DCGAN step?

The DCGAN step launches torch kernels (fills, element-wise ops, multi-tensor Adam, RNG) next to the libb200gan
kernels.  This tool runs a few EAGER
steps (no CUDA graph) under torch.profiler with Python stacks and prints, per kernel name, how often it runs per step and
the innermost frames of this repository that caused it.  GPU only:

    python tools/attribute_torch_kernels.py > torch_kernels.txt
"""
import collections
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "pytorch-gan_b200"))

import torch  # noqa: E402
from torch.profiler import ProfilerActivity, profile  # noqa: E402


def main(steps=3, img=64, batch=128):
    import b200gan
    from b200gan import train, zoo
    assert torch.cuda.is_available(), "needs a GPU"
    dev = torch.device("cuda", 0)
    b200gan.load_library()
    torch.manual_seed(0)
    g, d = zoo.DCGANGenerator(img).to(dev), zoo.DCGANDiscriminator(img).to(dev)
    g.apply(zoo.weights_init_normal)
    d.apply(zoo.weights_init_normal)
    opt_g = torch.optim.Adam(g.parameters(), lr=2e-4, betas=(0.5, 0.999), capturable=True)
    opt_d = torch.optim.Adam(d.parameters(), lr=2e-4, betas=(0.5, 0.999), capturable=True)
    loss = torch.nn.BCELoss()
    valid, fake = torch.ones(batch, 1, device=dev), torch.zeros(batch, 1, device=dev)
    imgs = torch.rand(batch, 1, img, img, device=dev) * 2 - 1
    z = torch.randn(batch, 100, device=dev)

    def step():
        return train.dcgan_step(g, d, opt_g, opt_d, imgs, z, loss, valid, fake)

    for _ in range(3):
        step()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA], with_stack=True) as prof:
        for _ in range(steps):
            step()
        torch.cuda.synchronize()

    # CPU-side op events that launched kernels, keyed by the op and the innermost repository frames of its stack
    by_site = collections.defaultdict(lambda: [0, 0.0])
    for ev in prof.events():
        if ev.device_type != torch.autograd.DeviceType.CPU or not ev.kernels:
            continue
        frames = [f for f in (ev.stack or []) if ROOT in f or "b200gan" in f or "bench.py" in f]
        site = (" <- ".join(f.replace(ROOT + os.sep, "") for f in frames[:3])
                or "(no repository frame: autograd engine / optimizer)")
        for k in ev.kernels:
            if "b200gan::" in k.name:
                continue
            key = (k.name[:90], ev.name, site)
            by_site[key][0] += 1
            by_site[key][1] += k.duration
    total = sum(v[1] for v in by_site.values())
    print(f"torch kernels per step: {sum(v[0] for v in by_site.values()) / steps:.0f}, {total / steps:.0f} us of device time")
    for (kname, op, site), (n, us) in sorted(by_site.items(), key=lambda kv: -kv[1][1]):
        print(f"{us / steps:8.1f} us  n/step {n / steps:5.1f}  {op:32s} {kname}\n            {site}")


if __name__ == "__main__":
    main()
