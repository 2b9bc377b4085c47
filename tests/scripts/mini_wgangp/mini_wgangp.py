"""A small stand-alone Wasserstein GAN training script with a gradient penalty, written in the API idiom of the reference's
scripts -- torch.nn classes looked up by attribute on `nn`, `nn.Sequential(*layers)`, `torch.cuda.FloatTensor(numpy)`,
`Variable`, the penalty built with `autograd.grad(create_graph=True)` on interpolates of `.data`, `n_critic` critic
iterations per generator step, torchvision's MNIST loader -- so that the launcher (b200gan/launch.py) can run the
MLP critic's double backward END TO END without the reference checkout.  It is not a copy of any reference script: its
own widths, option names and loop.  --penalty gp: lambda * (||dD/dx|| - 1)^2 on interpolates (WGAN-GP); --penalty div:
k/2 * (||dD/dx||^p on real + on fake) with real images requiring grad and the fakes attached to G (WGAN-div)."""
import argparse

import numpy as np
import torch
import torch.autograd as autograd
import torch.nn as nn
import torchvision.transforms as transforms
from torch.autograd import Variable
from torch.utils.data import DataLoader
from torchvision import datasets

ap = argparse.ArgumentParser()
ap.add_argument("--epochs", type=int, default=1)
ap.add_argument("--batch_size", type=int, default=16)
ap.add_argument("--side", type=int, default=16)
ap.add_argument("--zdim", type=int, default=20)
ap.add_argument("--critic_every", type=int, default=2, help="critic iterations per generator step")
ap.add_argument("--penalty", choices=("gp", "div"), default="gp")
ap.add_argument("--weight", type=float, default=10.0, help="lambda (gp) or k (div)")
ap.add_argument("--power", type=float, default=6.0, help="p of the div penalty")
cfg = ap.parse_args()
on_gpu = torch.cuda.is_available()
Tensor = torch.cuda.FloatTensor if on_gpu else torch.FloatTensor
pixels = cfg.side * cfg.side


class Gen(nn.Module):
    def __init__(self):
        super().__init__()
        self.net = nn.Sequential(nn.Linear(cfg.zdim, 96), nn.LeakyReLU(0.2, inplace=True), nn.Linear(96, pixels),
                                 nn.Tanh())

    def forward(self, z):
        return self.net(z).view(z.shape[0], 1, cfg.side, cfg.side)


class Critic(nn.Module):
    def __init__(self):
        super().__init__()
        self.net = nn.Sequential(nn.Linear(pixels, 160), nn.LeakyReLU(0.2, inplace=True), nn.Linear(160, 72),
                                 nn.LeakyReLU(0.2, inplace=True), nn.Linear(72, 1))

    def forward(self, img):
        return self.net(img.view(img.shape[0], -1))


def input_grad(score, inp):
    ones = Variable(Tensor(inp.shape[0], 1).fill_(1.0), requires_grad=False)
    g = autograd.grad(outputs=score, inputs=inp, grad_outputs=ones, create_graph=True, retain_graph=True,
                      only_inputs=True)[0]
    return g.view(g.shape[0], -1)


def gp_term(C, real, fake):
    mix = Tensor(np.random.random((real.shape[0], 1, 1, 1)))
    blend = (mix * real + (1 - mix) * fake).requires_grad_(True)
    return ((input_grad(C(blend), blend).norm(2, dim=1) - 1) ** 2).mean()


G, C = Gen(), Critic()
if on_gpu:
    G.cuda(); C.cuda()
data = DataLoader(datasets.MNIST("../../data/mnist", train=True, download=True,
                                 transform=transforms.Compose([transforms.Resize(cfg.side), transforms.ToTensor(),
                                                               transforms.Normalize([0.5], [0.5])])),
                  batch_size=cfg.batch_size, shuffle=False)
opt_g = torch.optim.Adam(G.parameters(), lr=2e-4, betas=(0.5, 0.999))
opt_c = torch.optim.Adam(C.parameters(), lr=2e-4, betas=(0.5, 0.999))
history = []
for epoch in range(cfg.epochs):
    for it, (imgs, _) in enumerate(data):
        real = Variable(imgs.type(Tensor), requires_grad=cfg.penalty == "div")
        opt_c.zero_grad()
        z = Variable(Tensor(np.random.normal(0, 1, (imgs.shape[0], cfg.zdim))))
        fakes = G(z)
        real_score, fake_score = C(real), C(fakes)
        if cfg.penalty == "gp":
            pen = cfg.weight * gp_term(C, real.data, fakes.data)
        else:
            real_norm = input_grad(real_score, real).pow(2).sum(1) ** (cfg.power / 2)
            fake_norm = input_grad(fake_score, fakes).pow(2).sum(1) ** (cfg.power / 2)
            pen = torch.mean(real_norm + fake_norm) * cfg.weight / 2
        loss_c = -torch.mean(real_score) + torch.mean(fake_score) + pen
        loss_c.backward()
        opt_c.step()
        opt_g.zero_grad()
        if it % cfg.critic_every == 0:
            fakes = G(z)
            loss_g = -torch.mean(C(fakes))
            loss_g.backward()
            opt_g.step()
            history.append((loss_c.item(), loss_g.item()))
            print("[epoch %d] [it %d] [C %f] [G %f]" % (epoch, it, loss_c.item(), loss_g.item()))
