"""Time acgan.py's training step (acgan.py:184-223) and its discriminator's two heads with their losses, on the drop-in
modules of one source tree, at acgan.py's defaults (batch 64, 32 x 32, 10 classes, Adam lr 2e-4, betas (0.5, 0.999)):

    step     the whole G + D step: G(z, labels), D(G(z)) with D frozen, BCE + CrossEntropy, G backward and Adam;
             D(real), D(fake), the four losses, D backward and Adam -- the body of train.acgan_step, restated here so
             that a tree without it runs the same code
    head     the heads alone on [64, 512] features: Sequential(Linear(512, 1), Sigmoid) -> BCELoss and
             Sequential(Linear(512, 10), Softmax()) -> CrossEntropyLoss, 0.5 (sum), backward to the features and the
             heads' parameters

    python tools/acgan_step.py [--tree DIR] [--label NAME] [--batch 64] [--rounds 5] [--iters 100] [--steps 20]

Each workload is captured once into a CUDA graph (train.GraphedStep) and replayed; every round times `iters` replays
with CUDA events, and the median and minimum over rounds are reported.  Launches per iteration, and the kernels of the
head workload by name, come from a torch.profiler trace of one eager iteration.  Before any timing, `steps` seeded
eager steps from a seeded start give the final losses and the norms of D's parameters, so that two trees can be checked
to compute the same thing.  Prints one JSON line, with the card's name and power limit.  To compare two trees, run it
on each in turn, alternating.
"""
import argparse
import collections
import json
import os
import statistics
import subprocess
import sys
import tempfile
import warnings


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
    assert torch.cuda.is_available(), "tools/acgan_step.py times the GPU; there is no CPU measurement"
    warnings.simplefilter("ignore")   # Softmax() without a dim warns on every call, as in the script
    ns, n, dev, n_classes, latent = zoo.namespace(), a.batch, "cuda", 10, 100

    class Generator(torch.nn.Module):  # acgan.py:46-73
        def __init__(self):
            super().__init__()
            self.label_emb = ns.Embedding(n_classes, latent)
            self.l1 = ns.Sequential(ns.Linear(latent, 128 * 8 * 8))
            self.conv_blocks = zoo.DCGANGenerator(32, latent, 1, nn=ns).conv_blocks

        def forward(self, noise, labels):
            out = self.l1(torch.mul(self.label_emb(labels), noise))
            return self.conv_blocks(out.view(out.shape[0], 128, 8, 8))

    class Discriminator(torch.nn.Module):  # acgan.py:76-108
        def __init__(self):
            super().__init__()
            self.conv_blocks = zoo.DCGANDiscriminator(32, 1, nn=ns).model
            self.adv_layer = ns.Sequential(ns.Linear(512, 1), ns.Sigmoid())
            self.aux_layer = ns.Sequential(ns.Linear(512, n_classes), ns.Softmax())

        def forward(self, img):
            out = self.conv_blocks(img)
            out = out.view(out.shape[0], -1)
            return self.adv_layer(out), self.aux_layer(out)

    def build(seed):
        torch.manual_seed(seed)
        g, d = Generator().to(dev), Discriminator().to(dev)
        g.apply(zoo.weights_init_normal)
        d.apply(zoo.weights_init_normal)
        og = optim.Adam(g.parameters(), lr=2e-4, betas=(0.5, 0.999))
        od = optim.Adam(d.parameters(), lr=2e-4, betas=(0.5, 0.999))
        bce, ce = ns.BCELoss(), ns.CrossEntropyLoss()

        def step(real, labels, z, gen_labels):
            valid = torch.ones(n, 1, device=dev)
            fake = torch.zeros(n, 1, device=dev)
            og.zero_grad()
            gen_imgs = g(z, gen_labels)
            with train.frozen(d):
                validity, pred_label = d(gen_imgs)
                g_loss = 0.5 * (bce(validity, valid) + ce(pred_label, gen_labels))
                g_loss.backward()
            og.step()
            od.zero_grad()
            real_pred, real_aux = d(real)
            d_real_loss = (bce(real_pred, valid) + ce(real_aux, labels)) / 2
            fake_pred, fake_aux = d(gen_imgs.detach())
            d_fake_loss = (bce(fake_pred, fake) + ce(fake_aux, gen_labels)) / 2
            d_loss = (d_real_loss + d_fake_loss) / 2
            d_loss.backward()
            od.step()
            return torch.stack([g_loss.detach(), d_loss.detach()])

        def head(feat, labels):
            x = feat.detach().requires_grad_(True)
            loss = 0.5 * (bce(d.adv_layer(x), torch.ones(n, 1, device=dev)) + ce(d.aux_layer(x), labels))
            loss.backward()
            return loss.detach()
        return g, d, step, head

    def inputs(seed):
        gen = torch.Generator(dev).manual_seed(seed)
        return (torch.rand(n, 1, 32, 32, device=dev, generator=gen) * 2 - 1,
                torch.randint(0, n_classes, (n,), device=dev, generator=gen),
                torch.randn(n, latent, device=dev, generator=gen),
                torch.randint(0, n_classes, (n,), device=dev, generator=gen))

    # what the tree computes: seeded eager steps from a seeded start
    g, d, step, head = build(0)
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

    g, d, step, head = build(1)
    args = inputs(1)
    feat = torch.randn(n, 512, device=dev)
    result["launches_step"], _ = launches(step, *args)
    result["launches_head"], kernels_head = launches(head, feat.clone(), args[1])
    result["ms_step_median"], result["ms_step_min"] = timed(train.GraphedStep(step, args), args)
    result["ms_head_median"], result["ms_head_min"] = timed(train.GraphedStep(head, (feat, args[1])), (feat, args[1]))
    result["kernels_head"] = {k[:100]: v for k, v in kernels_head.most_common()}
    print(json.dumps(result))


if __name__ == "__main__":
    main()
