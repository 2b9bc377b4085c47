"""Pin the oracle against the reference itself and write the golden fixtures.

Needs a checkout of the reference (no GPU), its path in B200GAN_REFERENCE:

    B200GAN_REFERENCE=/path/to/PyTorch-GAN python oracle/make_golden.py

For each model family it (1) executes the reference's own Python (runpy for the flat scripts,
import for models.py files) under fixed seeds, (2) builds the oracle restatement under the same
seeds, (3) asserts parameters / outputs / gradients are IDENTICAL (both are stock torch on CPU),
and (4) stores seeded inputs + the reference's outputs as small fixtures in tests/golden/.
TEST INFRASTRUCTURE ONLY.
"""
import contextlib
import io
import os
import runpy
import sys
import tempfile

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
REF = os.environ.get("B200GAN_REFERENCE")
if __name__ == "__main__" and not REF:
    sys.exit("oracle/make_golden.py: set B200GAN_REFERENCE to a checkout of eriklindernoren/PyTorch-GAN")
GOLD = os.path.join(ROOT, "tests", "golden")
sys.path.insert(0, ROOT)

from oracle import ref_models  # noqa: E402


class _FakeMNIST(torch.utils.data.Dataset):
    """Stand-in for torchvision.datasets.MNIST (dcgan.py:121 asks for download=True; no network)."""

    def __init__(self, *a, **k):
        pass

    def __len__(self):
        return 1  # DataLoader(shuffle=True) refuses an empty dataset; --n_epochs 0 never iterates it

    def __getitem__(self, i):
        return torch.zeros(1, 8, 8), 0


@contextlib.contextmanager
def _script_env(argv):
    import torchvision.datasets as tvd
    old_argv, old_cwd, old_mnist = sys.argv, os.getcwd(), tvd.MNIST
    tmp = tempfile.mkdtemp(prefix="b200gan_ref_")
    work = os.path.join(tmp, "a", "b")
    os.makedirs(work)
    tvd.MNIST = _FakeMNIST
    sys.argv = argv
    os.chdir(work)
    try:
        with contextlib.redirect_stdout(io.StringIO()):
            yield
    finally:
        sys.argv = old_argv
        os.chdir(old_cwd)
        tvd.MNIST = old_mnist


def run_reference_script(rel, args, seed):
    """Execute an unmodified reference script with n_epochs=0: builds + initialises its models."""
    path = os.path.join(REF, "implementations", rel)
    torch.manual_seed(seed)
    with _script_env([path] + args):
        return runpy.run_path(path, run_name="__main__")


def _assert_same_state(a, b, what):
    sa, sb = a.state_dict(), b.state_dict()
    assert list(sa.keys()) == list(sb.keys()), f"{what}: state_dict keys differ"
    for k in sa:
        assert torch.equal(sa[k], sb[k]), f"{what}: parameter {k} differs from the reference"


def _grad_digest(model):
    return {k: p.grad.detach().clone() for k, p in model.named_parameters() if p.grad is not None}


def golden_dcgan(img_size, batch, seed=0):
    ref = run_reference_script("dcgan/dcgan.py", ["--n_epochs", "0", "--img_size", str(img_size), "--batch_size",
                                                  str(batch)], seed)
    g_ref, d_ref = ref["generator"], ref["discriminator"]
    g_or, d_or = ref_models.build_dcgan(img_size, seed=seed)
    _assert_same_state(g_ref, g_or, "dcgan G")
    _assert_same_state(d_ref, d_or, "dcgan D")

    z = ref_models.synthetic_z(batch, seed=seed)
    imgs = ref_models.synthetic_images(batch, 1, img_size, img_size, seed=seed)
    out = {}
    for tag, (g, d) in {"ref": (g_ref, d_ref), "oracle": (g_or, d_or)}.items():
        for m in d.modules():
            if isinstance(m, torch.nn.Dropout2d):
                m.p = 0.0  # masks come from a different RNG on the GPU; mask application is tested separately
        g.train()
        d.train()
        g.zero_grad()
        d.zero_grad()
        gen = g(z)
        validity = d(gen)
        loss = torch.nn.BCELoss()(validity, torch.ones(batch, 1))
        loss.backward()
        g_grads = _grad_digest(g)
        d.zero_grad()
        real_v = d(imgs)
        d_loss = (torch.nn.BCELoss()(real_v, torch.ones(batch, 1)) +
                  torch.nn.BCELoss()(d(gen.detach()), torch.zeros(batch, 1))) / 2
        d_loss.backward()
        out[tag] = dict(gen=gen.detach(), validity=validity.detach(), g_loss=loss.detach(), d_loss=d_loss.detach(),
                        real_v=real_v.detach(), g_grads=g_grads, d_grads=_grad_digest(d),
                        bn_running={k: v.clone() for k, v in g.state_dict().items() if "running" in k})
    r, o = out["ref"], out["oracle"]
    for k in ("gen", "validity", "g_loss", "d_loss", "real_v"):
        assert torch.equal(r[k], o[k]), f"dcgan {k}: oracle != reference"
    for k in r["g_grads"]:
        assert torch.equal(r["g_grads"][k], o["g_grads"][k]), f"dcgan G grad {k}"
    for k in r["d_grads"]:
        assert torch.equal(r["d_grads"][k], o["d_grads"][k]), f"dcgan D grad {k}"

    # fixture: inputs + reference outputs; big gradients are stored as (norm, first 64 values)
    def slim(gr):
        return {k: dict(norm=v.double().norm().item(), head=v.flatten()[:64].clone(), shape=tuple(v.shape))
                for k, v in gr.items()}

    fix = dict(img_size=img_size, batch=batch, seed=seed, z=z, imgs=imgs, gen=r["gen"], validity=r["validity"],
               real_v=r["real_v"], g_loss=r["g_loss"], d_loss=r["d_loss"], g_grads=slim(r["g_grads"]),
               d_grads=slim(r["d_grads"]), bn_running=r["bn_running"],
               torch_version=torch.__version__, reference="dcgan/dcgan.py@36d3c77")
    path = os.path.join(GOLD, f"dcgan_{img_size}_b{batch}.pt")
    torch.save(fix, path)
    print(f"dcgan img {img_size} batch {batch}: oracle == reference (bit-exact); wrote {path} "
          f"({os.path.getsize(path) / 1024:.0f} KiB)")


def golden_ops(seed=0):
    """Operator-level fixtures from stock torch CPU for every conv geometry on the hot path
    (SURVEY.md section 0.6), small sizes.  Checked against oracle/np_ops.py in the CPU tests."""
    torch.manual_seed(seed)
    cases = []
    specs = [  # (name, cin, cout, k, stride, pad, h, w, transposed)
        ("k3s1p1", 8, 6, 3, 1, 1, 9, 7, False),
        ("k3s2p1", 5, 7, 3, 2, 1, 10, 8, False),
        ("k3s1p0", 4, 4, 3, 1, 0, 8, 8, False),
        ("k4s2p1", 3, 8, 4, 2, 1, 12, 12, False),
        ("k4s1p1", 6, 2, 4, 1, 1, 9, 9, False),
        ("k7s1p0", 3, 5, 7, 1, 0, 14, 14, False),
        ("t4s2p1", 6, 4, 4, 2, 1, 5, 6, True),
    ]
    for name, cin, cout, k, s, p, h, w, tr in specs:
        x = torch.randn(2, cin, h, w, requires_grad=True)
        mod = (torch.nn.ConvTranspose2d if tr else torch.nn.Conv2d)(cin, cout, k, s, p)
        y = mod(x)
        gy = torch.randn_like(y)
        y.backward(gy)
        cases.append(dict(name=name, transposed=tr, stride=s, pad=p, x=x.detach(), w=mod.weight.detach().clone(),
                          b=mod.bias.detach().clone(), y=y.detach(), gy=gy, gx=x.grad.clone(),
                          gw=mod.weight.grad.clone(), gb=mod.bias.grad.clone()))
    path = os.path.join(GOLD, "ops_conv.pt")
    torch.save(cases, path)
    print(f"wrote {path} ({os.path.getsize(path) / 1024:.0f} KiB)")


def golden_wgan_gp(img_size=32, batch=64, seed=0):
    """wgan_gp.py: the reference's own compute_gradient_penalty (+ the double backward) on seeded inputs."""
    ref = run_reference_script("wgan_gp/wgan_gp.py", ["--n_epochs", "0", "--img_size", str(img_size), "--batch_size",
                                                      str(batch)], seed)
    g_ref, d_ref, cgp = ref["generator"], ref["discriminator"], ref["compute_gradient_penalty"]
    g_or, d_or = ref_models.build_wgan_gp(img_size, seed=seed)
    _assert_same_state(g_ref, g_or, "wgan_gp G")
    _assert_same_state(d_ref, d_or, "wgan_gp D")
    real = ref_models.synthetic_images(batch, 1, img_size, img_size, seed=seed)
    z = ref_models.synthetic_z(batch, seed=seed)
    g_ref.train()
    with torch.no_grad():
        fake = g_ref(z)
    lam = ref["lambda_gp"]
    np.random.seed(seed + 5)
    d_ref.zero_grad()
    gp_ref = cgp(d_ref, real, fake)           # draws alpha from numpy inside (wgan_gp.py:122)
    (lam * gp_ref).backward()
    alpha = ref_models.synthetic_alpha(batch, seed=seed + 5)
    d_or.zero_grad()
    gp_or = ref_models.compute_gradient_penalty(d_or, real, fake, alpha)
    (lam * gp_or).backward()
    assert torch.equal(gp_ref, gp_or), "wgan_gp gradient penalty: oracle != reference"
    for (k, pr), (_, po) in zip(d_ref.named_parameters(), d_or.named_parameters()):
        if pr.grad is None:
            assert po.grad is None or float(po.grad.abs().max()) == 0.0, k
        else:
            assert torch.equal(pr.grad, po.grad), f"wgan_gp D grad {k}"
    grads = {k: (None if p.grad is None else p.grad.clone()) for k, p in d_ref.named_parameters()}
    fix = dict(img_size=img_size, batch=batch, seed=seed, real=real, fake=fake, alpha=alpha, lambda_gp=lam,
               gp=gp_ref.detach(),
               dW1_head=grads["model.0.weight"][:4].clone(), dW1_norm=grads["model.0.weight"].double().norm().item(),
               dW2_head=grads["model.2.weight"][:8].clone(), dW2_norm=grads["model.2.weight"].double().norm().item(),
               dW3=grads["model.4.weight"].clone(),
               bias_grads_zero=all(grads[k] is None or float(grads[k].abs().max()) == 0.0
                                   for k in ("model.0.bias", "model.2.bias", "model.4.bias")),
               torch_version=torch.__version__, reference="wgan_gp/wgan_gp.py@36d3c77")
    path = os.path.join(GOLD, f"wgan_gp_{img_size}_b{batch}.pt")
    torch.save(fix, path)
    print(f"wgan_gp img {img_size} batch {batch}: oracle == reference (bit-exact), gp = {gp_ref.item():.6f}; "
          f"bias grads zero: {fix['bias_grads_zero']}; wrote {path} ({os.path.getsize(path) / 1024:.0f} KiB)")


def _import_reference_module(rel, name):
    """Import implementations/<rel> (pix2pix/models.py, cyclegan/models.py are side-effect free) under a unique name."""
    import importlib.util
    spec = importlib.util.spec_from_file_location(name, os.path.join(REF, "implementations", rel))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _slim(t, step=8):
    return t[..., ::step, ::step].clone() if t.dim() == 4 else t.clone()


def _grad_norms(model):
    return {k: p.grad.double().norm().item() for k, p in model.named_parameters() if p.grad is not None}


def golden_pix2pix(seed=0, size=256, batch=1):
    """pix2pix/models.py: GeneratorUNet + Discriminator, forward + backward of the script's G loss
    (pix2pix.py:141-150: MSE(D(fake_B, real_A), valid) + 100 * L1(fake_B, real_B)); dropout off (eval)."""
    ref = _import_reference_module("pix2pix/models.py", "ref_pix2pix_models")
    torch.manual_seed(seed)
    g_ref, d_ref = ref.GeneratorUNet(), ref.Discriminator()
    g_ref.apply(ref.weights_init_normal)
    d_ref.apply(ref.weights_init_normal)
    g_or, d_or = ref_models.build_pix2pix(seed)
    _assert_same_state(g_ref, g_or, "pix2pix G")
    _assert_same_state(d_ref, d_or, "pix2pix D")
    real_a = ref_models.synthetic_images(batch, 3, size, size, seed=seed + 1)
    real_b = ref_models.synthetic_images(batch, 3, size, size, seed=seed + 2)
    out = {}
    for tag, (g, d) in {"ref": (g_ref, d_ref), "oracle": (g_or, d_or)}.items():
        g.eval()  # Dropout(0.5) off; InstanceNorm keeps instance statistics in eval mode (no running stats)
        d.train()
        g.zero_grad(); d.zero_grad()
        fake_b = g(real_a)
        pred = d(fake_b, real_a)
        loss = torch.nn.MSELoss()(pred, torch.ones_like(pred)) + 100 * torch.nn.L1Loss()(fake_b, real_b)
        loss.backward()
        out[tag] = dict(fake_b=fake_b.detach(), pred=pred.detach(), loss=loss.detach(), gn=_grad_norms(g), dn=_grad_norms(d))
    r, o = out["ref"], out["oracle"]
    assert torch.equal(r["fake_b"], o["fake_b"]) and torch.equal(r["pred"], o["pred"]) and torch.equal(r["loss"], o["loss"])
    assert r["gn"] == o["gn"] and r["dn"] == o["dn"]
    fix = dict(seed=seed, size=size, batch=batch, fake_b=_slim(r["fake_b"]), pred=r["pred"], loss=r["loss"],
               g_grad_norms=r["gn"], d_grad_norms=r["dn"], torch_version=torch.__version__,
               reference="pix2pix/models.py@36d3c77")
    path = os.path.join(GOLD, f"pix2pix_{size}_b{batch}.pt")
    torch.save(fix, path)
    print(f"pix2pix {size}x{size} b{batch}: oracle == reference (bit-exact); wrote {path} ({os.path.getsize(path) / 1024:.0f} KiB)")


def golden_cyclegan(seed=0, size=64, batch=2, blocks=9):
    """cyclegan/models.py: GeneratorResNet + Discriminator; generator-side losses of cyclegan.py:177-204
    (identity, GAN, cycle) on seeded images."""
    ref = _import_reference_module("cyclegan/models.py", "ref_cyclegan_models")
    shape = (3, size, size)
    torch.manual_seed(seed)
    nets_ref = [ref.GeneratorResNet(shape, blocks), ref.GeneratorResNet(shape, blocks), ref.Discriminator(shape),
                ref.Discriminator(shape)]
    for m in nets_ref:
        m.apply(ref.weights_init_normal)
    nets_or = list(ref_models.build_cyclegan(shape, blocks, seed))
    for a, b, nm in zip(nets_ref, nets_or, ("G_AB", "G_BA", "D_A", "D_B")):
        _assert_same_state(a, b, "cyclegan " + nm)
    real_a = ref_models.synthetic_images(batch, 3, size, size, seed=seed + 1)
    real_b = ref_models.synthetic_images(batch, 3, size, size, seed=seed + 2)
    mse, l1 = torch.nn.MSELoss(), torch.nn.L1Loss()
    out = {}
    for tag, (g_ab, g_ba, d_a, d_b) in {"ref": nets_ref, "oracle": nets_or}.items():
        for m in (g_ab, g_ba, d_a, d_b):
            m.train()
            m.zero_grad()
        valid = torch.ones(batch, *d_a.output_shape)
        loss_id = (l1(g_ba(real_a), real_a) + l1(g_ab(real_b), real_b)) / 2          # cyclegan.py:180-183
        fake_b = g_ab(real_a)
        fake_a = g_ba(real_b)
        loss_gan = (mse(d_b(fake_b), valid) + mse(d_a(fake_a), valid)) / 2            # :186-191
        loss_cyc = (l1(g_ba(fake_b), real_a) + l1(g_ab(fake_a), real_b)) / 2          # :194-199
        loss_g = loss_gan + 10.0 * loss_cyc + 5.0 * loss_id                           # :202
        loss_g.backward()
        out[tag] = dict(fake_b=fake_b.detach(), fake_a=fake_a.detach(), loss_g=loss_g.detach(),
                        parts=(loss_id.item(), loss_gan.item(), loss_cyc.item()), gn=_grad_norms(g_ab), gn2=_grad_norms(g_ba))
    r, o = out["ref"], out["oracle"]
    assert torch.equal(r["fake_b"], o["fake_b"]) and torch.equal(r["loss_g"], o["loss_g"]) and r["gn"] == o["gn"]
    fix = dict(seed=seed, size=size, batch=batch, blocks=blocks, fake_b=_slim(r["fake_b"], 4), fake_a=_slim(r["fake_a"], 4),
               loss_g=r["loss_g"], parts=r["parts"], g_ab_grad_norms=r["gn"], g_ba_grad_norms=r["gn2"],
               torch_version=torch.__version__, reference="cyclegan/models.py@36d3c77")
    path = os.path.join(GOLD, f"cyclegan_{size}_b{batch}.pt")
    torch.save(fix, path)
    print(f"cyclegan {size}x{size} b{batch}: oracle == reference (bit-exact); wrote {path} ({os.path.getsize(path) / 1024:.0f} KiB)")


if __name__ == "__main__":
    os.makedirs(GOLD, exist_ok=True)
    golden_dcgan(32, 8)
    golden_ops()
    golden_wgan_gp()
    golden_pix2pix()
    golden_cyclegan()
