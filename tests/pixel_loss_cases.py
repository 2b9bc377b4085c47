"""Case table of the pixel-loss kernels (pytorch-gan_b200/csrc/pixel_loss/): MSELoss / L1Loss with reduction 'mean',
one forward and one backward launch per case.

Sizes n = 1, 7, 4096, the Pix2Pix patch output 16x1x16x16, the image losses 8x3x256x256 and 16x3x256x256 (more elements
than one pass of the forward grid), sizes that are not a multiple of 4, the four layout pairs NCHW/NCHW, NHWC/NHWC,
NHWC/NCHW, NCHW/NHWC, both modes, with and without the target's gradient, an input equal to its target (L1 gradient
exactly 0) and operands at a storage offset that rules out float4 loads.  Each case names the kernels it launches and
their grids, which follow from the device's SM count.

tests/test_gpu_pixel_loss_conformance.py runs every case against fp64; tests/test_cpu_pixel_loss.py holds the fp64
references to torch float64 and the table to the kernel sources and ptxas.
"""
import math
from dataclasses import dataclass
from typing import Tuple

import torch

KERNEL = {"fwd": "pixel_loss_fwd_kernel", "bwd": "pixel_loss_bwd_kernel"}
# ptxas -v, sm_90a (tests/test_cpu_pixel_loss.py recompiles the file and holds these)
REGISTERS = {"pixel_loss_fwd_kernel": 32, "pixel_loss_bwd_kernel": 24}
SMEM_BYTES = {"pixel_loss_fwd_kernel": 8260, "pixel_loss_bwd_kernel": 0}
THREADS, PER_THREAD, MAX_BLOCKS = 256, 8, 1024
MODES = {"mse": 0, "l1": 1}
LAYOUTS = {"nchw": 0, "nhwc": 1}
GRAD_TOL = 4 * 2.0 ** -24
GOUT = 1.7


def fwd_grid(n, sms):
    return (min(-(-n // (THREADS * PER_THREAD)), min(2 * sms, MAX_BLOCKS)), 1, 1)


def bwd_grid(n, sms):
    return (min(-(-n // (THREADS * 4)), 4 * sms), 1, 1)


@dataclass(frozen=True)
class Case:
    id: str
    mode: str
    shape: Tuple[int, ...]
    la: str = "nchw"
    lb: str = "nchw"
    want_db: bool = True
    equal: bool = False     # target == input exactly
    offset: bool = False    # both operands start one float into their storage: no float4 loads
    why: str = ""

    @property
    def n(self):
        return math.prod(self.shape)

    def kernels(self, sms=132):
        return [(KERNEL["fwd"], fwd_grid(self.n, sms)), (KERNEL["bwd"], bwd_grid(self.n, sms))]


def _cases():
    out = []
    for mode in ("mse", "l1"):
        out += [
            Case(f"{mode}-n1", mode, (1,), why="one element: one block, one thread, the ticket wraps at once"),
            Case(f"{mode}-n7", mode, (7,), want_db=False, why="n not a multiple of 4: the float4 body is empty"),
            Case(f"{mode}-n4096", mode, (64, 64), why="two forward blocks, 2-D"),
            Case(f"{mode}-patch", mode, (16, 1, 16, 16), why="the Pix2Pix PatchGAN output (C = 1: both layouts agree)"),
            Case(f"{mode}-3d", mode, (3, 5, 7), why="3-D, odd size"),
            Case(f"{mode}-0d", mode, (), why="a 0-dim tensor: padded to [1, 1, 1, 1]"),
        ]
        for la in ("nchw", "nhwc"):
            for lb in ("nchw", "nhwc"):
                out.append(Case(f"{mode}-ragged-{la}-{lb}", mode, (2, 3, 5, 7), la, lb,
                                why="210 elements: not a multiple of 4, every layout pair"))
                out.append(Case(f"{mode}-many-{la}-{lb}", mode, (3, 5, 37, 41), la, lb, want_db=(la != lb),
                                why="22755 elements: twelve forward blocks, a ragged last block"))
        out += [
            Case(f"{mode}-img8-nhwc-nchw", mode, (8, 3, 256, 256), "nhwc", "nchw",
                 why="a drop-in generator's NHWC output against an NCHW target, beyond one grid pass"),
            Case(f"{mode}-img8-nhwc-nhwc", mode, (8, 3, 256, 256), "nhwc", "nhwc", want_db=False,
                 why="one layout: float4 loads, beyond one grid pass"),
            Case(f"{mode}-img16-nhwc-nchw", mode, (16, 3, 256, 256), "nhwc", "nchw", want_db=False,
                 why="pix2pix.py:145 exactly: the L1 pixel loss of the benchmark step"),
            Case(f"{mode}-img16-nchw-nhwc", mode, (16, 3, 256, 256), "nchw", "nhwc",
                 why="the mirrored layout pair at the largest size"),
            Case(f"{mode}-img16-nchw-nchw", mode, (16, 3, 256, 256), why="NCHW on both sides at the largest size"),
            Case(f"{mode}-equal-nhwc-nhwc", mode, (4, 3, 16, 16), "nhwc", "nhwc", equal=True,
                 why="target == input: loss 0, gradients exactly 0 (sign(0) = 0 for L1)"),
            Case(f"{mode}-equal-nchw-nhwc", mode, (4, 3, 16, 16), "nchw", "nhwc", equal=True,
                 why="target == input in another layout"),
            Case(f"{mode}-offset", mode, (5, 3, 8, 8), offset=True,
                 why="operands one float into their storage: one layout without float4 loads"),
            Case(f"{mode}-offset-nhwc", mode, (5, 3, 8, 8), "nhwc", "nhwc", offset=True, want_db=False,
                 why="the same in channels_last"),
        ]
    return out


CASES = _cases()


# ---- fp64 references -------------------------------------------------------------------------------------------------
def loss_ref(a, b, mode):
    """fp64 loss of fp32 operands (any layouts: logical elements)"""
    d = a.double() - b.double()
    return (d * d).mean() if mode == "mse" else d.abs().mean()


def grad_ref(a, b, gout, mode):
    """fp64 d loss / d a for the upstream gradient gout; d loss / d b is its negation"""
    d = a.double() - b.double()
    n = max(a.numel(), 1)
    return 2.0 * d * gout / n if mode == "mse" else torch.sign(d) * gout / n


# ---- operands --------------------------------------------------------------------------------------------------------
def make(case, device="cuda", seed=0):
    g = torch.Generator().manual_seed(seed)
    a = torch.randn(case.shape, generator=g)
    b = a.clone() if case.equal else torch.randn(case.shape, generator=g)
    if case.mode == "l1" and not case.equal and a.numel() > 4:
        flat_b = b.view(-1)
        flat_b[::5] = a.reshape(-1)[::5]  # exact ties: sign(0) = 0 inside a real case too
    return place(a, case.la, case.offset, device), place(b, case.lb, case.offset, device)


def place(t, layout, offset, device):
    if layout == "nhwc":
        t = t.to(memory_format=torch.channels_last)
    if offset:
        buf = torch.empty(t.numel() + 1, device=device)
        out = torch.as_strided(buf, t.shape, t.stride(), 1)
        out.copy_(t)
        return out
    return t.to(device)
