"""A small stand-alone vanilla GAN training script in the API idiom of the reference's scripts -- torch.nn classes looked
up on `nn`, `nn.Sequential(...)` spelled out module by module, `Variable`, `Tensor(numpy_array)`, `.type(Tensor)`,
torchvision's MNIST loader, BCE losses printed every iteration -- whose discriminator is the three-Linear LeakyReLU MLP
with a Sigmoid output.  The launcher (b200gan/launch.py) runs it stock and on the drop-in modules.  It is not a copy of
any reference script: its own widths, option names and loop."""
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
ap.add_argument("--code", type=int, default=24)
ap.add_argument("--slope", type=float, default=0.2)
cfg = ap.parse_args()
use_cuda = torch.cuda.is_available()
Tensor = torch.cuda.FloatTensor if use_cuda else torch.FloatTensor
pixels = cfg.side * cfg.side


class Gen(nn.Module):
    def __init__(self):
        super().__init__()
        self.body = nn.Sequential(
            nn.Linear(cfg.code, 64), nn.LeakyReLU(cfg.slope, inplace=True),
            nn.Linear(64, 160), nn.BatchNorm1d(160, 0.8), nn.LeakyReLU(cfg.slope, inplace=True),
            nn.Linear(160, pixels), nn.Tanh())

    def forward(self, code):
        return self.body(code).view(code.size(0), 1, cfg.side, cfg.side)


class Critic(nn.Module):
    def __init__(self):
        super().__init__()
        self.body = nn.Sequential(
            nn.Linear(pixels, 192), nn.LeakyReLU(cfg.slope, inplace=True),
            nn.Linear(192, 80), nn.LeakyReLU(cfg.slope, inplace=True),
            nn.Linear(80, 1), nn.Sigmoid())

    def forward(self, img):
        return self.body(img.view(img.size(0), -1))


criterion = torch.nn.BCELoss()
gen, critic = Gen(), Critic()
if use_cuda:
    gen.cuda()
    critic.cuda()
    criterion.cuda()
loader = DataLoader(datasets.MNIST("../../data/mnist", train=True, download=True,
                                   transform=transforms.Compose([transforms.Resize(cfg.side), transforms.ToTensor(),
                                                                 transforms.Normalize([0.5], [0.5])])),
                    batch_size=cfg.batch_size, shuffle=False)
opt_gen = torch.optim.Adam(gen.parameters(), lr=2e-4, betas=(0.5, 0.999))
opt_critic = torch.optim.Adam(critic.parameters(), lr=2e-4, betas=(0.5, 0.999))
for epoch in range(cfg.epochs):
    for step, (imgs, _) in enumerate(loader):
        real_lbl = Variable(Tensor(imgs.size(0), 1).fill_(1.0), requires_grad=False)
        fake_lbl = Variable(Tensor(imgs.size(0), 1).fill_(0.0), requires_grad=False)
        real = Variable(imgs.type(Tensor))
        opt_gen.zero_grad()
        code = Variable(Tensor(np.random.normal(0, 1, (imgs.size(0), cfg.code))))
        made = gen(code)
        loss_gen = criterion(critic(made), real_lbl)
        loss_gen.backward()
        opt_gen.step()
        opt_critic.zero_grad()
        loss_critic = 0.5 * (criterion(critic(real), real_lbl) + criterion(critic(made.detach()), fake_lbl))
        loss_critic.backward()
        opt_critic.step()
        print("[epoch %d] [step %d] [D %f] [G %f]" % (epoch, step, loss_critic.item(), loss_gen.item()))
