"""A small stand-alone MLP GAN training script written in the API idiom of the reference's scripts -- torch.nn classes
looked up by attribute on `nn`, `nn.Sequential(*layers)` built from helper blocks, `Variable`, `Tensor(numpy_array)`,
`.type(Tensor)`, torchvision's MNIST loader, losses printed every iteration -- so that the launcher (b200gan/launch.py)
can run a whole training loop on the CPU without the reference checkout.  It is not a copy of any reference script:
its own layer widths, block helper and option names."""
import argparse

import numpy as np
import torch
import torch.nn as nn
import torchvision.transforms as transforms
from torch.autograd import Variable
from torch.utils.data import DataLoader
from torchvision import datasets

ap = argparse.ArgumentParser()
ap.add_argument("--epochs", type=int, default=1)
ap.add_argument("--batch_size", type=int, default=32)
ap.add_argument("--side", type=int, default=16)
ap.add_argument("--zdim", type=int, default=20)
cfg = ap.parse_args()
on_gpu = torch.cuda.is_available()
Tensor = torch.cuda.FloatTensor if on_gpu else torch.FloatTensor
npix = cfg.side * cfg.side


def dense(cin, cout, norm=True):
    layers = [nn.Linear(cin, cout)]
    if norm:
        layers.append(nn.BatchNorm1d(cout, 0.8))
    layers.append(nn.LeakyReLU(0.2, inplace=True))
    return layers


class Gen(nn.Module):
    def __init__(self):
        super().__init__()
        self.net = nn.Sequential(*dense(cfg.zdim, 64, norm=False), *dense(64, 128), nn.Linear(128, npix), nn.Tanh())

    def forward(self, z):
        return self.net(z).view(z.shape[0], 1, cfg.side, cfg.side)


class Disc(nn.Module):
    def __init__(self):
        super().__init__()
        self.net = nn.Sequential(nn.Linear(npix, 96), nn.LeakyReLU(0.2, inplace=True), nn.Linear(96, 1), nn.Sigmoid())

    def forward(self, img):
        return self.net(img.view(img.shape[0], -1))


bce = torch.nn.BCELoss()
G, D = Gen(), Disc()
if on_gpu:
    G.cuda(); D.cuda(); bce.cuda()
data = DataLoader(datasets.MNIST("../../data/mnist", train=True, download=True,
                                 transform=transforms.Compose([transforms.Resize(cfg.side), transforms.ToTensor(),
                                                               transforms.Normalize([0.5], [0.5])])),
                  batch_size=cfg.batch_size, shuffle=False)
opt_g = torch.optim.Adam(G.parameters(), lr=2e-4, betas=(0.5, 0.999))
opt_d = torch.optim.Adam(D.parameters(), lr=2e-4, betas=(0.5, 0.999))
for epoch in range(cfg.epochs):
    for it, (imgs, _) in enumerate(data):
        ones = Variable(Tensor(imgs.shape[0], 1).fill_(1.0), requires_grad=False)
        zeros = Variable(Tensor(imgs.shape[0], 1).fill_(0.0), requires_grad=False)
        real = Variable(imgs.type(Tensor))
        opt_g.zero_grad()
        z = Variable(Tensor(np.random.normal(0, 1, (imgs.shape[0], cfg.zdim))))
        fakes = G(z)
        loss_g = bce(D(fakes), ones)
        loss_g.backward()
        opt_g.step()
        opt_d.zero_grad()
        loss_d = (bce(D(real), ones) + bce(D(fakes.detach()), zeros)) / 2
        loss_d.backward()
        opt_d.step()
        print("[epoch %d] [it %d] [D %f] [G %f]" % (epoch, it, loss_d.item(), loss_g.item()))
