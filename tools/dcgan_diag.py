"""Where does DCGAN gradient error come from?  Per-parameter relative error of
  (a) b200gan auto (wgmma TF32 for the big convs)     vs stock torch fp32 (cuDNN, TF32 off)
  (b) b200gan simt (pure fp32 kernels)                vs stock torch fp32
  (c) stock torch with TF32 ON (the reference's default GPU path) vs stock torch fp32
on identical inputs/parameters.  (c) is the yardstick: it is "the reference's own PyTorch/cuDNN path"."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "pytorch-gan_b200"))
import torch  # noqa: E402

import b200gan  # noqa: E402
from b200gan import zoo  # noqa: E402
from oracle import ref_models  # noqa: E402


def rel(a, b):
    a, b = a.detach().double(), b.detach().double()
    return ((a - b).norm() / b.norm().clamp_min(1e-30)).item()


def run(img, batch):
    g_ref, d_ref = ref_models.build_dcgan(img, seed=0)
    z = ref_models.synthetic_z(batch, seed=1).cuda()
    imgs = ref_models.synthetic_images(batch, 1, img, img, seed=1).cuda()
    ones = torch.ones(batch, 1, device="cuda")
    bce = torch.nn.BCELoss()

    def fwd_bwd(g, d):
        for m in d.modules():
            if isinstance(m, torch.nn.Dropout2d):
                m.p = 0.0
        g.zero_grad(); d.zero_grad()
        gen = g(z)
        loss = bce(d(gen), ones) + bce(d(imgs), ones * 0.9)
        loss.backward()
        return gen.detach(), {k: p.grad.clone() for k, p in list(g.named_parameters()) + list(d.named_parameters())}

    import copy
    results = {}
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    results["torch_fp32"] = fwd_bwd(copy.deepcopy(g_ref).cuda(), copy.deepcopy(d_ref).cuda())
    torch.backends.cudnn.allow_tf32 = True
    torch.backends.cuda.matmul.allow_tf32 = True
    results["torch_tf32"] = fwd_bwd(copy.deepcopy(g_ref).cuda(), copy.deepcopy(d_ref).cuda())
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    for algo in ("auto", "simt"):
        b200gan.Config.algo = algo
        g, d = zoo.DCGANGenerator(img), zoo.DCGANDiscriminator(img)
        g.load_state_dict(g_ref.state_dict()); d.load_state_dict(d_ref.state_dict())
        results["ours_" + algo] = fwd_bwd(g.cuda(), d.cuda())
    b200gan.Config.algo = "auto"
    base_gen, base = results["torch_fp32"]
    print(f"== DCGAN {img}x{img} bs {batch}: rel err vs stock torch fp32")
    print(f"{'tensor':28s} {'torch_tf32':>11s} {'ours_auto':>11s} {'ours_simt':>11s}")
    print(f"{'gen_imgs':28s} " + " ".join(f"{rel(results[k][0], base_gen):11.2e}" for k in ("torch_tf32", "ours_auto", "ours_simt")))
    for name in base:
        if base[name].double().norm().item() < 1e-7:
            continue
        print(f"{name:28s} " + " ".join(f"{rel(results[k][1][name], base[name]):11.2e}" for k in ("torch_tf32", "ours_auto", "ours_simt")))


if __name__ == "__main__":
    run(32, 8)
    run(64, 128)
