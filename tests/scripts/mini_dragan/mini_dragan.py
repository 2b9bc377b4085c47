"""A small DRAGAN-style training script in the API idiom of the reference's scripts (torch.nn looked up by attribute,
`nn.Sequential(*layers)`, name-based init through `.apply`, `Variable`, torchvision's MNIST loader), for exercising the
launcher end to end on a gradient penalty through a BatchNorm2d critic.  It is not a copy of any reference script: its
own generator, a three-block critic, its own option names; the interpolation and its perturbation are drawn on the
device."""
import argparse

import torch
import torch.autograd as autograd
import torch.nn as nn
import torchvision.transforms as transforms
from torch.autograd import Variable
from torch.utils.data import DataLoader
from torchvision import datasets

ap = argparse.ArgumentParser()
ap.add_argument("--img_size", type=int, default=32)
ap.add_argument("--batch_size", type=int, default=16)
ap.add_argument("--zdim", type=int, default=32)
ap.add_argument("--penalty", type=float, default=10.0)
cfg = ap.parse_args()
device = torch.device("cuda" if torch.cuda.is_available() else "cpu")


def init_by_name(m):
    name = m.__class__.__name__
    if "Conv" in name:
        torch.nn.init.normal_(m.weight.data, 0.0, 0.05)
    elif "BatchNorm2d" in name:
        torch.nn.init.normal_(m.weight.data, 1.0, 0.1)
        torch.nn.init.constant_(m.bias.data, 0.0)


class Gen(nn.Module):
    def __init__(self):
        super().__init__()
        self.s0 = cfg.img_size // 4
        self.fc = nn.Sequential(nn.Linear(cfg.zdim, 32 * self.s0 ** 2))
        self.body = nn.Sequential(nn.BatchNorm2d(32), nn.Upsample(scale_factor=2), nn.Conv2d(32, 32, 3, 1, 1),
                                  nn.BatchNorm2d(32, 0.8), nn.LeakyReLU(0.2, inplace=True), nn.Upsample(scale_factor=2),
                                  nn.Conv2d(32, 1, 3, 1, 1), nn.Tanh())

    def forward(self, z):
        h = self.fc(z)
        return self.body(h.view(h.shape[0], 32, self.s0, self.s0))


class Critic(nn.Module):
    def __init__(self):
        super().__init__()
        layers = []
        for i, (cin, cout) in enumerate(((1, 16), (16, 32), (32, 64))):
            layers += [nn.Conv2d(cin, cout, 3, 2, 1), nn.LeakyReLU(0.2, inplace=True), nn.Dropout2d(0.25)]
            if i:
                layers.append(nn.BatchNorm2d(cout, 0.8))
        self.body = nn.Sequential(*layers)
        self.head = nn.Sequential(nn.Linear(64 * (cfg.img_size // 8) ** 2, 1), nn.Sigmoid())

    def forward(self, x):
        f = self.body(x)
        return self.head(f.view(f.shape[0], -1))


def perturbed_penalty(critic, real):
    alpha = torch.rand(real.shape, device=real.device)
    noisy = real + 0.5 * real.std() * torch.rand(real.shape, device=real.device)
    mixed = Variable(alpha * real + (1 - alpha) * noisy, requires_grad=True)
    out = critic(mixed)
    grads = autograd.grad(outputs=out, inputs=mixed, grad_outputs=torch.ones_like(out), create_graph=True,
                          retain_graph=True, only_inputs=True)[0]
    return cfg.penalty * ((grads.norm(2, dim=1) - 1) ** 2).mean()


bce = torch.nn.BCELoss()
G, D = Gen().to(device), Critic().to(device)
G.apply(init_by_name)
D.apply(init_by_name)
data = DataLoader(datasets.MNIST("../../data/mnist", train=True, download=True,
                                 transform=transforms.Compose([transforms.Resize(cfg.img_size), transforms.ToTensor(),
                                                               transforms.Normalize([0.5], [0.5])])),
                  batch_size=cfg.batch_size, shuffle=False)
opt_g = torch.optim.Adam(G.parameters(), lr=2e-4, betas=(0.5, 0.999))
opt_d = torch.optim.Adam(D.parameters(), lr=2e-4, betas=(0.5, 0.999))
losses = []
for it, (imgs, _) in enumerate(data):
    real = imgs.to(device)
    ones = torch.ones(imgs.shape[0], 1, device=device)
    zeros = torch.zeros(imgs.shape[0], 1, device=device)
    opt_g.zero_grad()
    fakes = G(torch.randn(imgs.shape[0], cfg.zdim, device=device))
    loss_g = bce(D(fakes), ones)
    loss_g.backward()
    opt_g.step()
    opt_d.zero_grad()
    gp = perturbed_penalty(D, real)
    loss_d = (bce(D(real), ones) + bce(D(fakes.detach()), zeros)) / 2 + gp
    loss_d.backward()
    opt_d.step()
    losses.append({"d": loss_d.item(), "g": loss_g.item(), "gp": gp.item()})
    print("[it %d] [D %f] [G %f] [GP %f]" % (it, loss_d.item(), loss_g.item(), gp.item()))
