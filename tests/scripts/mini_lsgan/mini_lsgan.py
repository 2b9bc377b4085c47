"""A small stand-alone least-squares GAN training script in the API idiom of the reference's scripts -- torch.nn classes
looked up by attribute on `nn`, `nn.Sequential(*layers)`, name-based weight init through `.apply`,
`torch.cuda.FloatTensor(numpy_array)`, `Variable`, `.type(Tensor)`, `loss.cuda()`, torchvision's MNIST loader -- with an
`nn.MSELoss()` adversarial objective on a linear-output conv discriminator and an `nn.L1Loss()` pixel term, so that the
launcher (b200gan/launch.py) exercises both drop-in losses END TO END.  It is not a copy of any reference script."""
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
ap.add_argument("--batch_size", type=int, default=16)
ap.add_argument("--side", type=int, default=32)
ap.add_argument("--zdim", type=int, default=24)
ap.add_argument("--pixel_weight", type=float, default=0.5)
cfg = ap.parse_args()
on_gpu = torch.cuda.is_available()
Tensor = torch.cuda.FloatTensor if on_gpu else torch.FloatTensor


def init_by_name(m):
    name = m.__class__.__name__
    if "Conv" in name:
        torch.nn.init.normal_(m.weight.data, 0.0, 0.05)
    elif "BatchNorm2d" in name:
        torch.nn.init.normal_(m.weight.data, 1.0, 0.05)
        torch.nn.init.constant_(m.bias.data, 0.0)


class Gen(nn.Module):
    def __init__(self):
        super().__init__()
        self.s0 = cfg.side // 4
        self.fc = nn.Sequential(nn.Linear(cfg.zdim, 64 * self.s0 ** 2))
        stages = [nn.BatchNorm2d(64)]
        for cin, cout in ((64, 64), (64, 32)):
            stages += [nn.Upsample(scale_factor=2), nn.Conv2d(cin, cout, 3, stride=1, padding=1), nn.BatchNorm2d(cout, 0.8),
                       nn.LeakyReLU(0.2, inplace=True)]
        stages += [nn.Conv2d(32, 1, 3, stride=1, padding=1), nn.Tanh()]
        self.body = nn.Sequential(*stages)

    def forward(self, z):
        h = self.fc(z)
        return self.body(h.view(h.shape[0], 64, self.s0, self.s0))


class Critic(nn.Module):
    """conv blocks and a linear output: the least-squares objective scores raw values, no Sigmoid"""

    def __init__(self):
        super().__init__()
        layers = []
        for i, (cin, cout) in enumerate(((1, 16), (16, 32), (32, 64))):
            layers += [nn.Conv2d(cin, cout, 3, 2, 1), nn.LeakyReLU(0.2, inplace=True)]
            if i:
                layers.append(nn.BatchNorm2d(cout, 0.8))
        self.body = nn.Sequential(*layers)
        self.head = nn.Linear(64 * (cfg.side // 8) ** 2, 1)

    def forward(self, x):
        f = self.body(x)
        return self.head(f.view(f.shape[0], -1))


least_squares = torch.nn.MSELoss()
pixel = torch.nn.L1Loss()
G, D = Gen(), Critic()
if on_gpu:
    G.cuda(); D.cuda(); least_squares.cuda(); pixel.cuda()
G.apply(init_by_name)
D.apply(init_by_name)
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
        loss_g = least_squares(D(fakes), ones) + cfg.pixel_weight * pixel(fakes, real)
        loss_g.backward()
        opt_g.step()
        opt_d.zero_grad()
        loss_d = 0.5 * (least_squares(D(real), ones) + least_squares(D(fakes.detach()), zeros))
        loss_d.backward()
        opt_d.step()
        print("[epoch %d] [it %d] [D %f] [G %f]" % (epoch, it, loss_d.item(), loss_g.item()))
