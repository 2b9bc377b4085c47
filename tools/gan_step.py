"""Time gan.py's training step (gan.py:124-161) and its discriminator's forward + backward, on the drop-in modules of one
source tree, at gan.py's defaults (batch 64, 28 x 28, Adam lr 2e-4, betas (0.5, 0.999)):

    step     the whole G + D step: G(z), D(G(z)) with D frozen, BCE, G backward and Adam; D(real), D(fake), BCE,
             D backward and Adam -- the body of train.gan_step, restated here so that a tree without it runs the
             same code
    d        D(real) -> BCE -> backward alone (the parameters' gradients accumulate, as in a D step)

    python tools/gan_step.py [--tree DIR] [--label NAME] [--batch 64] [--rounds 5] [--iters 100] [--steps 20]

Each workload is captured once into a CUDA graph (train.GraphedStep) and replayed; every round times `iters` replays
with CUDA events, and the median and minimum over rounds are reported.  Launches per iteration come from a
torch.profiler trace of one eager iteration.  Before any timing, `steps` seeded eager steps from a seeded start give
the final losses and the norms of D's parameters, so that two trees can be checked to compute the same thing.
Prints one JSON line, with the card's name and power limit.  To compare two trees, run it on each in turn, alternating.
"""
import argparse
import collections
import json
import os
import statistics
import subprocess
import sys
import tempfile


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip().splitlines()[0]
    except Exception as e:  # the numbers are still useful without it; say so
        return f"power limit unknown: {type(e).__name__}"


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--tree", default=os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    ap.add_argument("--label", default="")
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--iters", type=int, default=100)
    ap.add_argument("--steps", type=int, default=20)
    a = ap.parse_args()
    tree = os.path.abspath(a.tree)
    sys.path[:0] = [tree, os.path.join(tree, "pytorch-gan_b200")]
    import torch
    import b200gan
    from b200gan import optim, train, zoo
    assert os.path.abspath(b200gan.__file__) == os.path.join(tree, "pytorch-gan_b200", "b200gan", "__init__.py")
    assert torch.cuda.is_available(), "tools/gan_step.py times the GPU; there is no CPU measurement"
    ns, n, dev = zoo.namespace(), a.batch, "cuda"

    class Discriminator(torch.nn.Module):  # gan.py:64-80
        def __init__(self):
            super().__init__()
            self.model = ns.Sequential(ns.Linear(784, 512), ns.LeakyReLU(0.2, inplace=True), ns.Linear(512, 256),
                                       ns.LeakyReLU(0.2, inplace=True), ns.Linear(256, 1), ns.Sigmoid())

        def forward(self, img):
            return self.model(img.view(img.shape[0], -1))

    def build(seed):
        torch.manual_seed(seed)
        g, d = zoo.WGANGPGenerator((1, 28, 28), nn=ns).to(dev), Discriminator().to(dev)  # gan.py:38-61 is WGAN-GP's G
        og = optim.Adam(g.parameters(), lr=2e-4, betas=(0.5, 0.999))
        od = optim.Adam(d.parameters(), lr=2e-4, betas=(0.5, 0.999))
        bce = ns.BCELoss()

        def step(real, z):
            valid = torch.ones(n, 1, device=dev)
            fake = torch.zeros(n, 1, device=dev)
            og.zero_grad()
            gen_imgs = g(z)
            with train.frozen(d):
                g_loss = bce(d(gen_imgs), valid)
                g_loss.backward()
            og.step()
            od.zero_grad()
            d_loss = (bce(d(real), valid) + bce(d(gen_imgs.detach()), fake)) / 2
            d_loss.backward()
            od.step()
            return torch.stack([g_loss.detach(), d_loss.detach()])

        def d_pass(real):
            loss = bce(d(real), torch.ones(n, 1, device=dev))
            loss.backward()
            return loss.detach()
        return g, d, step, d_pass

    def inputs(seed):
        gen = torch.Generator(dev).manual_seed(seed)
        return (torch.rand(n, 1, 28, 28, device=dev, generator=gen) * 2 - 1,
                torch.randn(n, 100, device=dev, generator=gen))

    # what the tree computes: seeded eager steps from a seeded start
    g, d, step, d_pass = build(0)
    for s in range(a.steps):
        losses = step(*inputs(100 + s))
    torch.cuda.synchronize()
    result = {"label": a.label, "card": card(), "batch": n, "losses_after": [round(v, 7) for v in losses.tolist()],
              "d_param_norms": [round(p.norm().item(), 6) for p in d.parameters()]}

    def launches(fn, *args):
        from torch.profiler import ProfilerActivity, profile
        for _ in range(3):
            fn(*args)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            fn(*args)
            torch.cuda.synchronize()
        with tempfile.TemporaryDirectory() as tmp:
            path = os.path.join(tmp, "trace.json")
            prof.export_chrome_trace(path)
            with open(path) as fh:
                names = [e["name"] for e in json.load(fh).get("traceEvents", []) if e.get("cat") == "kernel"]
        return len(names), collections.Counter(names)

    def timed(graphed, args):
        start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        for _ in range(10):
            graphed(*args)
        per_round = []
        for _ in range(a.rounds):
            torch.cuda.synchronize()
            start.record()
            for _ in range(a.iters):
                graphed(*args)
            stop.record()
            stop.synchronize()
            per_round.append(start.elapsed_time(stop) / a.iters)
        return round(statistics.median(per_round), 4), round(min(per_round), 4)

    g, d, step, d_pass = build(1)
    real, z = inputs(1)
    result["launches_step"], _ = launches(step, real, z)
    result["launches_d"], kernels_d = launches(d_pass, real)
    result["ms_step_median"], result["ms_step_min"] = timed(train.GraphedStep(step, (real, z)), (real, z))
    result["ms_d_median"], result["ms_d_min"] = timed(train.GraphedStep(d_pass, (real,)), (real,))
    result["kernels_d"] = {k[:100]: v for k, v in kernels_d.most_common()}
    print(json.dumps(result))


if __name__ == "__main__":
    main()
