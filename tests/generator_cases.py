"""Case table of the MLP generator (pytorch-gan_b200/csrc/mlp_generator/mlp_generator.cu): one row per call of
b200gan_mlp_gen_fwd and b200gan_mlp_gen_bwd.

Every call is one cooperative launch of num_sms * min(2, blocks per SM) blocks of 256 threads.  The blocks per SM
follow from the kernels' registers (ptxas -v, sm_90a) and their 8448 bytes of shared memory: 65536 registers per SM
over 256 threads * (registers rounded up to 8) gives 5 (fwd, 48 registers) and 3 (bwd, 80), so every grid is
2 * 132 = 264 blocks on a 132-SM H100 SXM.  tests/test_cpu_mlp_generator.py recompiles the kernel file and holds
REGISTERS and GRID to ptxas, and the fp64 references to torch float64 autograd.

tests/test_gpu_mlp_generator_conformance.py runs every case against its fp64 reference.
"""
import math
from dataclasses import dataclass

import torch

NUM_SMS = 132
REGISTERS = {"mlp_gen_fwd_kernel": 48, "mlp_gen_bwd_kernel": 80}
SMEM_BYTES = 2 * 32 * 33 * 4   # the two 32 x 33 tiles of tile_gemm.cuh
MAX_WIDTH = 8192


def blocks_per_sm(regs, threads=256):
    """resident 256-thread blocks per SM of an H100 (65536 registers, 2048 threads, 228 KB shared memory)"""
    return min(65536 // (threads * -(-regs // 8) * 8), 2048 // threads, (228 * 1024) // (SMEM_BYTES + 1024))


GRID = (NUM_SMS * min(2, min(blocks_per_sm(r) for r in REGISTERS.values())), 1, 1)
KERNEL = {"fwd": "mlp_gen_fwd_kernel", "bwd": "mlp_gen_bwd_kernel"}


@dataclass(frozen=True)
class Case:
    name: str
    op: str                   # fwd | bwd
    N: int
    widths: tuple             # width[0] .. width[L]
    norms: tuple = ()         # per hidden layer (L - 1 entries): a BatchNorm1d follows its Linear
    slope: float = 0.2
    keep: bool = True         # fwd: saved for a backward (False: the forward of a torch.no_grad() pass)
    only: tuple = None        # bwd: the outputs asked for (None: every one)
    no_ws: bool = False       # refusal: no workspace
    error: bool = False
    why: str = ""

    @property
    def id(self):
        return f"{self.op}-{self.name}"

    @property
    def L(self):
        return len(self.widths) - 1

    @property
    def has_norm(self):
        return tuple(bool(v) for v in self.norms) + (False,) * (self.L - len(self.norms))

    @property
    def kernels(self):
        return () if self.error else (KERNEL[self.op],)

    @property
    def grid(self):
        return None if self.error else GRID

    def all_outputs(self):
        out = ["dz"]
        for l in range(self.L):
            out += [f"dW{l}", f"db{l}"] + ([f"dgamma{l}", f"dbeta{l}"] if self.has_norm[l] else [])
        return tuple(out)

    def outputs(self):
        if self.op == "fwd":
            return ("out", "saved") if self.keep else ("out",)
        return self.all_outputs() if self.only is None else tuple(self.only)


_c = Case
WGAN = (100, 128, 256, 512, 1024, 1024)   # wgan_gp.py at 32 x 32 (bench.py --config wgan_gp)
GAN = (100, 128, 256, 512, 1024, 784)     # gan.py at its default 28 x 28
NORMS = (0, 1, 1, 1)                      # the first block has no norm
SMALL = (31, 33, 65, 17)                  # every width ragged against the 32 x 32 tile

CASES = [
    # forward
    _c("bench", "fwd", 64, WGAN, NORMS, why="the WGAN-GP generator at the benchmark size, kept for a backward"),
    _c("bench_nograd", "fwd", 64, WGAN, NORMS, keep=False,
       why="the benchmark's critic iteration runs G under torch.no_grad(): only out and the running statistics"),
    _c("gan", "fwd", 64, GAN, NORMS, why="gan.py: 784 outputs, ragged against 32"),
    _c("ragged", "fwd", 33, SMALL, (1, 1), why="every dimension ragged against the tile; a norm in the first block"),
    _c("n2", "fwd", 2, WGAN, NORMS, why="N = 2: the smallest batch a training-mode norm takes; unbiased var / 1"),
    _c("l1", "fwd", 64, (100, 784), (), why="L = 1: Linear -> Tanh alone"),
    _c("l1_n1", "fwd", 1, (100, 784), (), why="N = 1 without a norm is allowed"),
    _c("slope0", "fwd", 33, SMALL, (0, 1), slope=0.0, why="slope 0 (ReLU), a block without a norm after the first"),
    _c("slope1", "fwd", 33, SMALL, (1, 0), slope=1.0, keep=False, why="slope 1 (identity), no-grad forward"),
    _c("many_tiles", "fwd", 600, (96, 1024, 512), (1,),
       why="600 x 1024: 608 layer-1 tiles, more than two per block of the persistent grid"),
    _c("n1", "fwd", 1, SMALL, (1, 1), error=True, why="N = 1 with a norm is refused, as torch refuses it"),
    _c("wide", "fwd", 8, (31, MAX_WIDTH + 1, 17), (1,), error=True, why="a width over the limit is refused"),
    _c("no_ws", "fwd", 33, SMALL, (1, 1), no_ws=True, error=True, why="no workspace is refused"),
    # backward
    _c("bench", "bwd", 64, WGAN, NORMS, why="every gradient at the benchmark size"),
    _c("bench_params", "bwd", 64, WGAN, NORMS, only=Case("", "bwd", 0, WGAN, NORMS).all_outputs()[1:],
       why="the generator step: every parameter gradient, no dz (z does not require grad)"),
    _c("gan", "bwd", 64, GAN, NORMS, why="gan.py's widths"),
    _c("ragged", "bwd", 33, SMALL, (1, 1), why="ragged tiles, norms in both hidden blocks"),
    _c("n2", "bwd", 2, WGAN, NORMS, why="N = 2"),
    _c("l1", "bwd", 64, (100, 784), (), why="L = 1: tanh' then one layer"),
    _c("slope0", "bwd", 33, SMALL, (0, 1), slope=0.0, why="slope 0: masked rows give exact zeros"),
    _c("slope1", "bwd", 33, SMALL, (1, 0), slope=1.0, why="slope 1"),
    _c("many_tiles", "bwd", 600, (96, 1024, 512), (1,), why="many tiles per block in every GEMM phase"),
    *[_c(f"{o}_only", "bwd", 33, SMALL, (1, 1), only=(o,), why=f"{o} alone: only what it depends on is formed")
      for o in Case("", "bwd", 0, SMALL, (1, 1)).all_outputs()],
    _c("n1", "bwd", 1, SMALL, (1, 1), error=True, why="N = 1 with a norm is refused"),
    _c("wide", "bwd", 8, (31, MAX_WIDTH + 1, 17), (1,), error=True, why="a width over the limit is refused"),
    _c("no_ws", "bwd", 33, SMALL, (1, 1), no_ws=True, error=True, why="no workspace is refused"),
]


# ---- inputs and fp64 references (device-agnostic: tests/test_cpu_mlp_generator.py holds them to autograd) ----------
U = 2.0 ** -23
EPS, MOMENTUM = 0.8, 0.1     # BatchNorm1d(o, 0.8) of wgan_gp.py:49 / gan.py:45, torch's default momentum
F32 = torch.float32


def f32(v):
    return torch.tensor(v, dtype=F32).item()


def make(c, seed=0):
    """the case's fp32 inputs on the CPU: z, W{l}, b{l}, and per norm layer gamma, beta, rm, rv, nbt; dout"""
    g = torch.Generator().manual_seed(seed)
    rn = lambda *s, scale=1.0: torch.randn(*s, generator=g) * scale  # noqa: E731
    N, w = max(c.N, 1), c.widths
    P = {"z": rn(N, w[0])}
    for l in range(c.L):
        P[f"W{l}"] = rn(w[l + 1], w[l], scale=1 / math.sqrt(w[l]))
        P[f"b{l}"] = rn(w[l + 1], scale=0.2)
        if c.has_norm[l]:
            P[f"gamma{l}"] = 1 + rn(w[l + 1], scale=0.2)
            P[f"beta{l}"] = rn(w[l + 1], scale=0.2)
            P[f"rm{l}"] = rn(w[l + 1], scale=0.1)
            P[f"rv{l}"] = 1 + torch.rand(w[l + 1], generator=g)
            P[f"nbt{l}"] = torch.tensor([7], dtype=torch.int64)
    P["dout"] = rn(N, w[-1])
    return P


def mask(a, slope):
    return torch.where(a > 0, torch.ones_like(a), torch.full_like(a, slope))


def gen_fwd_ref(P, c, acts=None):
    """fp64 forward of case c from its (fp32) inputs P.  Per layer: x (the layer's input), h, and for a norm layer mean,
    var, rstd, xhat, the updated running statistics; y, a; and out.  acts: the kernel's activations, each layer then
    starts from the kernel's previous layer."""
    D = {k: v.double() for k, v in P.items() if v.is_floating_point()}
    slope, N = f32(c.slope), D["z"].shape[0]
    x, layers = D["z"], []
    for l in range(c.L):
        r = {"x": x, "h": x @ D[f"W{l}"].t() + D[f"b{l}"]}
        if l == c.L - 1:
            r["out"] = torch.tanh(r["h"])
        else:
            y = r["h"]
            if c.has_norm[l]:
                mean = y.mean(0)
                var = ((y - mean) ** 2).mean(0)
                r.update(mean=mean, var=var, rstd=1 / torch.sqrt(var + f32(EPS)))
                r["xhat"] = (y - mean) * r["rstd"]
                y = r["xhat"] * D[f"gamma{l}"] + D[f"beta{l}"]
                m = f32(MOMENTUM)
                r["rm"] = (1 - m) * D[f"rm{l}"] + m * mean
                r["rv"] = (1 - m) * D[f"rv{l}"] + m * var * N / (N - 1)
            r["y"], r["a"] = y, y * mask(y, slope)
            x = r["a"] if acts is None or acts[l] is None else acts[l].double()
        layers.append(r)
    return layers


def saved_of(c, layers):
    """the saved region (include/b200gan.h: a_l, then xhat and rstd of each norm layer) from a forward's layers"""
    hid = [layers[l] for l in range(c.L - 1)]
    parts = [r["a"] for r in hid] + [r["xhat"] for r, n in zip(hid, c.has_norm) if n] + \
        [r["rstd"] for r, n in zip(hid, c.has_norm) if n]
    return torch.cat([p.reshape(-1) for p in parts]) if parts else torch.zeros(0, dtype=torch.float64)


def split_saved(c, saved, N):
    """saved -> (acts, xhats, rstds), per hidden layer (None for layers without a norm)"""
    w, o = c.widths, 0
    acts, xh, rs = [], [None] * (c.L - 1), [None] * (c.L - 1)
    for l in range(c.L - 1):
        acts.append(saved[o:o + N * w[l + 1]].view(N, w[l + 1]))
        o += N * w[l + 1]
    for l in range(c.L - 1):
        if c.has_norm[l]:
            xh[l] = saved[o:o + N * w[l + 1]].view(N, w[l + 1])
            o += N * w[l + 1]
    for l in range(c.L - 1):
        if c.has_norm[l]:
            rs[l] = saved[o:o + w[l + 1]]
            o += w[l + 1]
    return acts, xh, rs


def mmr(A, eA, B, n):
    """A @ B in fp64 for an operand A off by eA and an exact B: the bound of the fp32 GEMM's own rounding, plus the
    operand errors carried as independent ones (root-sum-square); and the mean magnitude of one term"""
    S = A.abs() @ B.abs()
    return A @ B, U * (n + 4) * S + torch.sqrt((eA * eA) @ (B * B)), S / max(A.shape[-1], 1)


def rss(e, dim=0):
    return torch.sqrt((e * e).sum(dim))


def gen_bwd_ref(c, dout, out, z_, W, gamma, acts, xhat, rstd):
    """fp64 backward for dout with bounds: name -> (value, bound[, mean magnitude of one term]) for dz, dW{l}, db{l},
    dgamma{l}, dbeta{l}; every operand but the gradient itself is exact (the kernel reads the same fp32 values).  The
    gradient's own error is carried from layer to layer as independent per-element errors (mmr, rss): the worst case of
    correlated errors grows by the row sums of |W| per layer and is vacuous after five layers.  Each carried bound is
    itself a worst case of its layer's rounding, far above the error a kernel makes."""
    slope, N = f32(c.slope), dout.shape[0]
    g = dout * (1 - out * out)
    eg = U * (3 * g.abs() + 2 * dout.abs() * out * out)
    r = {}
    for l in range(c.L - 1, -1, -1):
        ain = z_ if l == 0 else acts[l - 1]
        r[f"dW{l}"] = mmr(g.t(), eg.t(), ain, N)
        r[f"db{l}"] = (g.sum(0), U * (N + 4) * g.abs().sum(0) + rss(eg))
        da, eda, _ = mmr(g, eg, W[l], W[l].shape[0])
        if l == 0:
            r["dz"] = (da, eda)
            break
        mk = mask(ain, slope)
        dy, edy = da * mk, eda * mk.abs() + U * (da * mk).abs()
        if c.has_norm[l - 1]:
            xh, k = xhat[l - 1], gamma[l - 1] * rstd[l - 1]
            s1, s2 = dy.sum(0), (dy * xh).sum(0)
            es1 = U * (N + 4) * dy.abs().sum(0) + rss(edy)
            es2 = U * (N + 4) * (dy * xh).abs().sum(0) + rss(edy * xh)
            r[f"dbeta{l - 1}"], r[f"dgamma{l - 1}"] = (s1, es1), (s2, es2)
            inner = dy - s1 / N - xh * s2 / N
            g = k * inner
            eg = k.abs() * (edy + es1 / N + xh.abs() * es2 / N
                            + 6 * U * (dy.abs() + (s1 / N).abs() + (xh * s2 / N).abs())) + 2 * U * g.abs()
        else:
            g, eg = dy, edy
    return r
