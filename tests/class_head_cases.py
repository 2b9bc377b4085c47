"""Case table of the auxiliary-classifier head and its loss: the class-head mode of linear1_{fwd,bwd}_kernel
(Linear(K, n) + Softmax, b200gan_class_head_{fwd,bwd}) and the cross-entropy mode of bce_{fwd,bwd}_kernel
(CrossEntropyLoss, b200gan_cross_entropy_{fwd,bwd}), all in pytorch-gan_b200/csrc/head.cu.

A case is one forward + backward call pair of the C ABI (`op` "head" or "ce"), its geometry (`dims`: (N, K, n) or
(N, C)) and options (`opt`), and the kernels it must launch, in order, with their grids:
  head: linear1_fwd_kernel on N blocks (one per row), linear1_bwd_kernel on ceil(K / 128) blocks (one thread per k);
  ce:   bce_fwd_kernel on 1 block, bce_bwd_kernel on ceil(N / 8) blocks of 256 threads (a warp per row).
An error case names the entry points (`opt["refused_by"]`) that must each refuse it.

tests/test_gpu_class_head_conformance.py runs every case against torch float64; tests/test_cpu_class_head.py holds the
table to the kernel source.
"""
from dataclasses import dataclass, field

import torch

MAX_CLASSES = 32
BWD_MAX_ELEMS = 12284       # N * n floats of dz beside the kernel's 16 bytes of static shared memory: 48 KB
CE_MAX_CLASSES = 1024
CE_ROWS_PER_BLOCK = 8       # 256 threads, a warp per row
IGNORE = -100               # torch's default ignore_index


def cdiv(a, b):
    return -(-a // b)


@dataclass(frozen=True)
class Case:
    name: str
    op: str          # head | ce
    dims: tuple
    opt: dict = field(default_factory=dict, hash=False, compare=False)
    error: bool = False
    why: str = ""

    @property
    def id(self):
        return f"{self.op}-{self.name}"

    @property
    def launches(self):
        """[(kernel, grid)] in launch order"""
        if self.error:
            return []
        if self.op == "head":
            N, K, n = self.dims
            return [("linear1_fwd_kernel", (N, 1, 1)), ("linear1_bwd_kernel", (cdiv(K, 128), 1, 1))]
        if self.op == "ce":
            N, C = self.dims
            return [("bce_fwd_kernel", (1, 1, 1)), ("bce_bwd_kernel", (cdiv(N, CE_ROWS_PER_BLOCK), 1, 1))]
        raise ValueError(self.op)

    @property
    def kernels(self):
        return tuple(k for k, _ in self.launches)


_c = Case
CASES = [
    # ---- Linear(K, n) + Softmax -------------------------------------------------------------------------------------------
    _c("acgan", "head", (64, 512, 10), why="acgan.py's aux_layer at the script defaults: batch 64, K = 128 * 2 * 2, n = 10"),
    _c("n2", "head", (64, 512, 2), why="n = 2, the fewest classes"),
    _c("sgan_n11", "head", (64, 512, 11), why="n = 11: sgan.py's n_classes + 1"),
    _c("n32", "head", (64, 2048, 32), why="n = 32, a full warp of classes; K = 2048"),
    _c("k1", "head", (16, 1, 10), why="K = 1: one thread of 128 has work; scalar path"),
    _c("k_ragged", "head", (7, 131, 11), why="K = 131: scalar path, a second backward block with 3 columns"),
    _c("k2049", "head", (5, 2049, 32), why="K = 2049: 17 backward blocks, the last with one column"),
    _c("n_row1", "head", (1, 512, 10), why="N = 1"),
    _c("limit_n10", "head", (BWD_MAX_ELEMS // 10, 64, 10), why="N = 1228, n = 10: N * n just below the 12284 bound"),
    _c("limit_n32", "head", (BWD_MAX_ELEMS // 32, 100, 32), why="N = 383, n = 32: the most rows of a full warp"),
    _c("limit_n4", "head", (BWD_MAX_ELEMS // 4, 100, 4), why="N * n = 12284 exactly: dz fills the 48 KB"),
    _c("limit_n2", "head", (BWD_MAX_ELEMS // 2, 36, 2), why="N = 6142, n = 2: the most rows"),
    _c("misaligned", "head", (5, 512, 10), dict(offset=1),
       why="K % 4 == 0 but x one float off 16-byte alignment: the scalar path"),
    _c("no_b", "head", (9, 100, 10), dict(b=False), why="b NULL"),
    _c("no_dx", "head", (9, 100, 10), dict(dx=False), why="dx NULL"),
    _c("no_db", "head", (9, 100, 10), dict(db=False), why="db NULL"),
    _c("saturated", "head", (32, 512, 10), dict(xscale=40.0),
       why="logits of a few hundred: the softmax saturates to 0 and 1"),
    _c("nout1", "head", (8, 64, 1), dict(refused_by=("fwd", "bwd")), error=True, why="n = 1 is the linear1 entry point"),
    _c("nout33", "head", (8, 64, 33), dict(refused_by=("fwd", "bwd")), error=True, why="n = 33 > one warp"),
    _c("n0", "head", (0, 64, 10), dict(refused_by=("fwd", "bwd")), error=True, why="N = 0"),
    _c("k0", "head", (8, 0, 10), dict(refused_by=("fwd", "bwd")), error=True, why="K = 0"),
    _c("over_limit", "head", (BWD_MAX_ELEMS // 10 + 1, 64, 10), dict(refused_by=("bwd",)), error=True,
       why="N * n = 12290 > 12284: refused by the backward"),
    _c("null_x", "head", (8, 64, 10), dict(refused_by=("fwd", "bwd"), null="x"), error=True, why="x NULL"),
    _c("null_w", "head", (8, 64, 10), dict(refused_by=("fwd", "bwd"), null="w"), error=True, why="w NULL"),
    _c("null_y", "head", (8, 64, 10), dict(refused_by=("fwd", "bwd"), null="y"), error=True, why="y NULL"),
    _c("null_dy", "head", (8, 64, 10), dict(refused_by=("bwd",), null="dy"), error=True, why="dy NULL"),
    _c("null_dw", "head", (8, 64, 10), dict(refused_by=("bwd",), null="dw"), error=True, why="dw NULL"),
    # ---- CrossEntropyLoss, reduction 'mean', class indices ----------------------------------------------------------------
    _c("acgan", "ce", (64, 10), why="acgan.py's auxiliary loss at the script defaults"),
    _c("c1", "ce", (8, 1), why="C = 1: the loss and the gradient are 0"),
    _c("c11", "ce", (33, 11), why="C = 11 (sgan.py), 33 rows: a ragged last backward block"),
    _c("c1024", "ce", (64, 1024), why="C = 1024, the most classes: 32 logits per lane"),
    _c("n1", "ce", (1, 10), why="N = 1"),
    _c("n5000", "ce", (5000, 10), why="N = 5000: 1250 rows per warp of the forward's block"),
    _c("ignore_some", "ce", (64, 10), dict(ignore=IGNORE, ignored=0.25), why="ignore_index -100 on a quarter of rows"),
    _c("ignore_class", "ce", (64, 10), dict(ignore=3, ignored=0.3),
       why="ignore_index 3, a valid class, on 30 % of the rows"),
    _c("ignore_all", "ce", (16, 10), dict(ignore=IGNORE, ignored=1.0),
       why="every row ignored: loss 0 / 0 = NaN, zero gradient"),
    _c("out_of_range", "ce", (16, 10), dict(bad=((3, 10), (7, -5), (11, 1 << 40))),
       why="targets 10, -5 and 2^40, not ignore_index: NaN loss and NaN rows, nothing read outside a row"),
    _c("large", "ce", (64, 10), dict(xscale=1e4), why="logits of 10^4: every row saturated"),
    _c("very_negative", "ce", (64, 10), dict(xshift=-1e6), why="logits around -10^6: logsumexp must subtract the max"),
    _c("huge", "ce", (32, 11), dict(xscale=1e30), why="logits of 10^30 both ways"),
    _c("c0", "ce", (8, 0), dict(refused_by=("fwd", "bwd")), error=True, why="C = 0"),
    _c("c1025", "ce", (8, 1025), dict(refused_by=("fwd", "bwd")), error=True, why="C = 1025 > 1024"),
    _c("n0", "ce", (0, 10), dict(refused_by=("fwd", "bwd")), error=True, why="N = 0"),
    _c("null_x", "ce", (8, 10), dict(refused_by=("fwd", "bwd"), null="x"), error=True, why="x NULL"),
    _c("null_target", "ce", (8, 10), dict(refused_by=("fwd", "bwd"), null="target"), error=True, why="target NULL"),
    _c("null_out", "ce", (8, 10), dict(refused_by=("fwd", "bwd"), null="out"), error=True, why="out2 NULL"),
    _c("null_gout", "ce", (8, 10), dict(refused_by=("bwd",), null="gout"), error=True, why="gout NULL"),
    _c("null_dx", "ce", (8, 10), dict(refused_by=("bwd",), null="dx"), error=True, why="dx NULL"),
]


# ---- fp64 references (device-agnostic: tests/test_cpu_class_head.py holds them to torch float64 autograd) ------------
def head_ref(x, w, b):
    """softmax(x w^T + b) over dim 1, and the logits"""
    z = x.double() @ w.double().t() + (0 if b is None else b.double())
    return torch.softmax(z, 1), z


def head_grad_ref(x, w, y, dy):
    """(dx, dw, db, dz) of Linear + Softmax from the saved output y: dz = y (dy - sum_i y_i dy_i)"""
    y, dy = y.double(), dy.double()
    dz = y * (dy - (y * dy).sum(1, keepdim=True))
    return dz @ w.double(), dz.t() @ x.double(), dz.sum(0), dz


def ce_ref(x, target, ignore_index):
    """CrossEntropyLoss(reduction='mean', ignore_index) over the in-range targets, and the count of rows not ignored"""
    x = x.double()
    keep = target != ignore_index
    lse = torch.logsumexp(x, 1)
    t = target.clamp(0, x.shape[1] - 1)
    terms = torch.where(keep, lse - x.gather(1, t[:, None])[:, 0], torch.zeros_like(lse))
    count = int(keep.sum().item())
    return terms.sum() / count if count else torch.tensor(float("nan"), dtype=torch.float64), terms, count


def ce_grad_ref(x, target, ignore_index, gout, count):
    """gout / count (softmax(x) - onehot(target)), zero rows where ignored"""
    x = x.double()
    p = torch.softmax(x, 1)
    hit = torch.arange(x.shape[1], device=x.device) == target[:, None]
    d = (p - hit.double()) * (gout / count)
    return torch.where((target != ignore_index)[:, None], d, torch.zeros_like(d))
