"""A small stand-alone auxiliary-classifier GAN training script in the API idiom of the reference's scripts -- torch.nn
classes looked up on `nn`, a label embedding multiplied into the noise (`nn.Embedding`, `torch.mul`), a discriminator
with a validity head and a class head `nn.Sequential(nn.Linear(...), nn.Softmax())` (no dim), BCE and cross-entropy
losses, `Variable`, `LongTensor(numpy_array)`, the numpy accuracy readback -- on MLP networks, so that every module it
uses also runs on the CPU.  The launcher (b200gan/launch.py) runs it stock and on the drop-in modules.  It is not a copy
of any reference script: its own widths, option names and loop."""
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
ap.add_argument("--classes", type=int, default=10)
cfg = ap.parse_args()
use_cuda = torch.cuda.is_available()
FloatTensor = torch.cuda.FloatTensor if use_cuda else torch.FloatTensor
LongTensor = torch.cuda.LongTensor if use_cuda else torch.LongTensor
pixels = cfg.side * cfg.side


class Gen(nn.Module):
    def __init__(self):
        super().__init__()
        self.embed = nn.Embedding(cfg.classes, cfg.code)
        self.body = nn.Sequential(
            nn.Linear(cfg.code, 64), nn.LeakyReLU(0.2, inplace=True),
            nn.Linear(64, 160), nn.BatchNorm1d(160, 0.8), nn.LeakyReLU(0.2, inplace=True),
            nn.Linear(160, pixels), nn.Tanh())

    def forward(self, code, cls):
        return self.body(torch.mul(self.embed(cls), code)).view(code.size(0), 1, cfg.side, cfg.side)


class Critic(nn.Module):
    def __init__(self):
        super().__init__()
        self.trunk = nn.Sequential(nn.Linear(pixels, 192), nn.LeakyReLU(0.2, inplace=True),
                                   nn.Linear(192, 96), nn.LeakyReLU(0.2, inplace=True))
        self.real_or_fake = nn.Sequential(nn.Linear(96, 1), nn.Sigmoid())
        self.which_class = nn.Sequential(nn.Linear(96, cfg.classes), nn.Softmax())

    def forward(self, img):
        h = self.trunk(img.view(img.size(0), -1))
        return self.real_or_fake(h), self.which_class(h)


adv_criterion = torch.nn.BCELoss()
cls_criterion = torch.nn.CrossEntropyLoss()
gen, critic = Gen(), Critic()
if use_cuda:
    gen.cuda()
    critic.cuda()
    adv_criterion.cuda()
    cls_criterion.cuda()
loader = DataLoader(datasets.MNIST("../../data/mnist", train=True, download=True,
                                   transform=transforms.Compose([transforms.Resize(cfg.side), transforms.ToTensor(),
                                                                 transforms.Normalize([0.5], [0.5])])),
                    batch_size=cfg.batch_size, shuffle=False)
opt_gen = torch.optim.Adam(gen.parameters(), lr=2e-4, betas=(0.5, 0.999))
opt_critic = torch.optim.Adam(critic.parameters(), lr=2e-4, betas=(0.5, 0.999))
for epoch in range(cfg.epochs):
    for step, (imgs, digits) in enumerate(loader):
        n = imgs.size(0)
        real_lbl = Variable(FloatTensor(n, 1).fill_(1.0), requires_grad=False)
        fake_lbl = Variable(FloatTensor(n, 1).fill_(0.0), requires_grad=False)
        real = Variable(imgs.type(FloatTensor))
        digits = Variable(digits.type(LongTensor))
        opt_gen.zero_grad()
        code = Variable(FloatTensor(np.random.normal(0, 1, (n, cfg.code))))
        wanted = Variable(LongTensor(np.random.randint(0, cfg.classes, n)))
        made = gen(code, wanted)
        judged, guessed = critic(made)
        loss_gen = 0.5 * (adv_criterion(judged, real_lbl) + cls_criterion(guessed, wanted))
        loss_gen.backward()
        opt_gen.step()
        opt_critic.zero_grad()
        judged_real, guessed_real = critic(real)
        loss_real = (adv_criterion(judged_real, real_lbl) + cls_criterion(guessed_real, digits)) / 2
        judged_fake, guessed_fake = critic(made.detach())
        loss_fake = (adv_criterion(judged_fake, fake_lbl) + cls_criterion(guessed_fake, wanted)) / 2
        loss_critic = (loss_real + loss_fake) / 2
        probs = np.concatenate([guessed_real.data.cpu().numpy(), guessed_fake.data.cpu().numpy()], axis=0)
        truth = np.concatenate([digits.data.cpu().numpy(), wanted.data.cpu().numpy()], axis=0)
        acc = np.mean(np.argmax(probs, axis=1) == truth)
        loss_critic.backward()
        opt_critic.step()
        print("[epoch %d] [step %d] [D %f, acc %d%%] [G %f]" % (epoch, step, loss_critic.item(), 100 * acc,
                                                               loss_gen.item()))
