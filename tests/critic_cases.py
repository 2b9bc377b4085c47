"""Case table of the MLP critic (pytorch-gan_b200/csrc/mlp_critic.cu): one row per call of b200gan_mlp_critic_fwd,
b200gan_mlp_critic_bwd, b200gan_mlp_critic_dbwd and b200gan_critic_step_mlp.

Every call is one cooperative launch of num_sms * min(2, blocks per SM) blocks of 256 threads.  The blocks per SM
follow from the kernels' registers (ptxas -v, sm_90a) and their 8448 bytes of shared memory: 65536 registers per SM
over 256 threads * (registers rounded up to 8) gives 6 (fwd, 39 registers), 5 (bwd, 48) and 4 (dbwd and critic_step,
64), so every grid is 2 * 132 = 264 blocks on a 132-SM H100 SXM.  tests/test_cpu_kernel_coverage.py recompiles
mlp_critic.cu and holds REGISTERS and GRID to ptxas.

tests/test_gpu_critic_conformance.py runs every case against torch float64.
"""
import math
from dataclasses import dataclass

import torch

NUM_SMS = 132
REGISTERS = {"mlp_critic_fwd_kernel": 39, "mlp_critic_bwd_kernel": 48, "mlp_critic_dbwd_kernel": 64,
             "critic_step_kernel": 64}
SMEM_BYTES = 2 * 32 * 33 * 4   # the two 32 x 33 tiles of tile_gemm.cuh


def blocks_per_sm(regs, threads=256):
    """resident 256-thread blocks per SM of an H100 (65536 registers, 2048 threads, 228 KB shared memory)"""
    return min(65536 // (threads * -(-regs // 8) * 8), 2048 // threads, (228 * 1024) // (SMEM_BYTES + 1024))


GRID = (NUM_SMS * min(2, min(blocks_per_sm(r) for r in REGISTERS.values())), 1, 1)

KERNEL = {"fwd": "mlp_critic_fwd_kernel", "bwd": "mlp_critic_bwd_kernel", "dbwd": "mlp_critic_dbwd_kernel",
          "step": "critic_step_kernel"}
OUTPUTS = {"fwd": ("out", "m1", "a1", "m2", "a2"),
           "bwd": ("dx", "dW1", "db1", "dW2", "db2", "dW3", "db3", "U1", "U2"),
           "dbwd": ("dW1", "dW2", "dW3", "ddout"),
           "step": ("losses", "dW1", "db1", "dW2", "db2", "dW3", "db3")}


@dataclass(frozen=True)
class Case:
    name: str
    op: str                  # fwd | bwd | dbwd | step
    N: int
    Din: int
    H1: int
    H2: int
    slope: float = 0.2
    null: tuple = ()         # outputs passed as NULL (bwd: "U1" / "U2" NULL means they live in the workspace)
    lam: float = 10.0        # step: lambda_gp
    alpha: str = "rand"      # step: rand | zero | one
    zero_w3: bool = False    # step: W3 = 0, so every input gradient is zero
    zero_row: int = -1       # step: real = fake = 0 for this sample and b1 < 0 at slope 0: its input gradient is zero
    no_ws: bool = False      # refusal: no workspace
    no_w1: bool = False      # refusal: dx without W1
    error: bool = False
    why: str = ""

    @property
    def id(self):
        return f"{self.op}-{self.name}"

    @property
    def kernels(self):
        return () if self.error else (KERNEL[self.op],)

    @property
    def grid(self):
        return None if self.error else GRID

    @property
    def deterministic(self):
        """every output repeats bit for bit; critic_step's losses are summed with atomics and are not listed"""
        return True

    def outputs(self):
        return tuple(o for o in OUTPUTS[self.op] if o not in self.null)


_c = Case
BENCH = dict(N=64, Din=1024, H1=512, H2=256)   # bench.py --config wgan_gp: 1 x 32 x 32 images, 512 -> 256 -> 1
MNIST = dict(N=64, Din=784, H1=512, H2=256)    # wgan_gp.py at its default 28 x 28
RAGGED = dict(N=33, Din=31, H1=33, H2=31)

CASES = [
    # forward
    _c("bench", "fwd", **BENCH, why="the WGAN-GP critic at the benchmark size"),
    _c("mnist", "fwd", **MNIST, why="Din = 784: K ragged against 32 in layer 1"),
    _c("ragged", "fwd", **RAGGED, why="every dimension ragged against the 32 x 32 tile"),
    _c("ones", "fwd", 1, 1, 1, 1, why="N = Din = H1 = H2 = 1: one partial tile per phase"),
    _c("h2_1", "fwd", 31, 33, 33, 1, slope=0.0, why="H2 = 1 and slope 0 (ReLU masks)"),
    _c("many_tiles", "fwd", 600, 96, 1024, 64, slope=1.0,
       why="600 x 1024: 608 layer-1 tiles, more than two per block of the persistent grid; slope 1"),
    # backward
    _c("bench", "bwd", **BENCH, why="every output at the benchmark size"),
    _c("mnist_ws", "bwd", **MNIST, null=("U1", "U2"), why="U1 / U2 in the workspace"),
    _c("ragged", "bwd", **RAGGED, slope=0.0, why="ragged tiles, slope 0"),
    _c("ones", "bwd", 1, 1, 1, 1, why="N = Din = H1 = H2 = 1"),
    _c("h2_1", "bwd", 33, 31, 33, 1, slope=1.0, why="H2 = 1, slope 1"),
    _c("many_tiles", "bwd", 600, 96, 1024, 64, why="many tiles per block in P2 and P3"),
    _c("none", "bwd", 33, 31, 33, 31, null=("dx", "dW1", "db1", "dW2", "db2", "dW3", "db3"),
       why="no parameter or input gradient at all: only U1 / U2"),
    _c("dx_only", "bwd", 33, 31, 33, 31, null=("dW1", "db1", "dW2", "db2", "dW3", "db3", "U1", "U2"),
       why="dx alone, U1 / U2 in the workspace (the input gradient of a gradient penalty)"),
    _c("dW1_only", "bwd", 33, 31, 33, 31, null=("dx", "db1", "dW2", "db2", "dW3", "db3"), why="dW1 alone"),
    _c("db1_only", "bwd", 33, 31, 33, 31, null=("dx", "dW1", "dW2", "db2", "dW3", "db3"), why="db1 alone"),
    _c("dW2_only", "bwd", 33, 31, 33, 31, null=("dx", "dW1", "db1", "db2", "dW3", "db3"), why="dW2 alone"),
    _c("db2_only", "bwd", 33, 31, 33, 31, null=("dx", "dW1", "db1", "dW2", "dW3", "db3"), why="db2 alone"),
    _c("dW3_only", "bwd", 33, 31, 33, 31, null=("dx", "dW1", "db1", "dW2", "db2", "db3"), why="dW3 alone"),
    _c("db3_only", "bwd", 33, 31, 33, 31, null=("dx", "dW1", "db1", "dW2", "db2", "dW3"), why="db3 alone"),
    _c("zero_dims", "bwd", 0, 31, 33, 31, error=True, why="N = 0 is refused"),
    _c("dx_no_w1", "bwd", 33, 31, 33, 31, no_w1=True, error=True, why="dx without W1 is refused"),
    _c("no_ws", "bwd", 33, 31, 33, 31, null=("U1", "U2"), no_ws=True, error=True,
       why="neither U1 / U2 nor a workspace is refused"),
    # double backward
    _c("bench", "dbwd", **BENCH, why="every output at the benchmark size"),
    _c("mnist", "dbwd", **MNIST, slope=0.0, why="Din = 784, slope 0"),
    _c("ragged", "dbwd", **RAGGED, slope=1.0, why="ragged tiles, slope 1"),
    _c("ones", "dbwd", 1, 1, 1, 1, why="N = Din = H1 = H2 = 1"),
    _c("h2_1", "dbwd", 31, 33, 31, 1, why="H2 = 1"),
    _c("many_tiles", "dbwd", 600, 96, 1024, 64, why="many tiles per block in P1 and P2"),
    _c("dW1_only", "dbwd", 33, 31, 33, 31, null=("dW2", "dW3", "ddout"), why="dW1 alone: neither t nor s is formed"),
    _c("dW2_only", "dbwd", 33, 31, 33, 31, null=("dW1", "dW3", "ddout"), why="dW2 alone: t without s"),
    _c("dW3_only", "dbwd", 33, 31, 33, 31, null=("dW1", "dW2", "ddout"), why="dW3 alone: t and s"),
    _c("ddout_only", "dbwd", 33, 31, 33, 31, null=("dW1", "dW2", "dW3"), why="ddout alone: t and s"),
    _c("zero_h1", "dbwd", 33, 31, 0, 31, error=True, why="H1 = 0 is refused"),
    _c("no_ws", "dbwd", 33, 31, 33, 31, no_ws=True, error=True, why="no workspace is refused"),
    # the whole critic iteration
    _c("bench", "step", **BENCH, why="the iteration bench.py --config wgan_gp times"),
    _c("mnist", "step", **MNIST, why="Din = 784"),
    _c("ragged", "step", **RAGGED, why="3N = 99 rows and every dimension ragged against the tile"),
    _c("ones", "step", 1, 1, 1, 1, why="N = Din = H1 = H2 = 1"),
    _c("h2_1", "step", 31, 33, 33, 1, slope=0.0, why="H2 = 1, slope 0"),
    _c("many_tiles", "step", 200, 96, 1024, 64, slope=1.0, why="3N = 600 rows: many tiles per block; slope 1"),
    _c("lambda0", "step", 33, 31, 33, 31, lam=0.0, why="lambda 0: the penalty rows contribute nothing"),
    _c("alpha0", "step", 33, 31, 33, 31, alpha="zero", why="alpha exactly 0: the interpolates are the fakes"),
    _c("alpha1", "step", 33, 31, 33, 31, alpha="one", why="alpha exactly 1: the interpolates are the reals"),
    _c("zero_w3", "step", 33, 31, 33, 31, zero_w3=True,
       why="W3 = 0: r = 0 in every row; the penalty is lambda and its gradient zero (torch's norm backward)"),
    _c("zero_w3_lambda0", "step", 33, 31, 33, 31, zero_w3=True, lam=0.0, why="r = 0 with lambda 0"),
    _c("zero_row", "step", 16, 31, 33, 31, slope=0.0, zero_row=5,
       why="one sample with a zero input gradient among non-zero ones"),
    _c("zero_dims", "step", 33, 0, 33, 31, error=True, why="Din = 0 is refused"),
    _c("no_ws", "step", 33, 31, 33, 31, no_ws=True, error=True, why="no workspace is refused"),
]



# ---- fp64 references with their bounds (device-agnostic: tests/test_cpu_kernel_coverage.py holds them to autograd) ---
U = 2.0 ** -23


def mm(A, eA, B, eB, n):
    """A @ B in fp64, the bound of an fp32 evaluation with chains of n terms from operands off by eA, eB, and the
    mean magnitude of one term of the sum"""
    S = A.abs() @ B.abs()
    return A @ B, U * (n + 4) * S + eA @ B.abs() + A.abs() @ eB, S / max(A.shape[-1], 1)


def mask(h, slope):
    return torch.where(h > 0, torch.ones_like(h), torch.full_like(h, slope))


def z(t):
    return torch.zeros_like(t)


def rowdot_n(K):
    return math.ceil(K / 32) + 5


def critic_fwd_ref(x, W1, b1, W2, b2, W3, b3, slope, m1=None, m2=None):
    """h1, m1, a1, h2, m2, a2, out; each layer from the previous layer's (given) masks; with bounds of h1, h2, out"""
    r = {}
    h1, e1, _ = mm(x, z(x), W1.t(), z(W1).t(), x.shape[1] + 1)
    r["h1"], r["eh1"] = h1 + b1, e1 + U * 5 * b1.abs()
    r["m1"] = mask(r["h1"], slope) if m1 is None else m1
    r["a1"] = r["h1"] * r["m1"]
    h2, e2, _ = mm(r["a1"], z(r["a1"]), W2.t(), z(W2).t(), W2.shape[1] + 1)
    r["h2"], r["eh2"] = h2 + b2, e2 + U * 5 * b2.abs()
    r["m2"] = mask(r["h2"], slope) if m2 is None else m2
    r["a2"] = r["h2"] * r["m2"]
    out, eo, _ = mm(r["a2"], z(r["a2"]), W3.t(), z(W3).t(), rowdot_n(W3.shape[1]) + 1)
    r["out"], r["eout"] = out.reshape(-1) + b3, eo.reshape(-1) + U * 5 * b3.abs()
    return r


def critic_bwd_ref(dout, x, W1, W2, W3, m1, a1, m2, a2):
    N = x.shape[0]
    d = dout.reshape(-1, 1)
    U2 = d * W3.reshape(1, -1) * m2
    eU2 = 2 * U * U2.abs()
    r = {"U2": (U2, eU2)}
    r["dW3"] = tuple(v.reshape(1, -1) for v in mm(a2.t(), z(a2).t(), d, z(d), N))
    r["db3"] = (d.sum().reshape(1), U * (N + 4) * d.abs().sum().reshape(1))
    r["dW2"] = mm(U2.t(), eU2.t(), a1, z(a1), N)
    v, e, _ = mm(U2, eU2, W2, z(W2), W2.shape[0])
    U1 = v * m1
    eU1 = e * m1.abs() + U * U1.abs()
    r["U1"] = (U1, eU1)
    r["db2"] = (U2.sum(0), U * (N + 4) * U2.abs().sum(0) + eU2.sum(0))
    r["dW1"] = mm(U1.t(), eU1.t(), x, z(x), N)
    r["dx"] = mm(U1, eU1, W1, z(W1), W1.shape[0])
    r["db1"] = (U1.sum(0), U * (N + 4) * U1.abs().sum(0) + eU1.sum(0))
    return r


def critic_dbwd_ref(u, dout, U1, U2, m1, m2, W1, W2, W3):
    N = u.shape[0]
    r = {"dW1": mm(U1.t(), z(U1).t(), u, z(u), N)}
    v, e, _ = mm(u, z(u), W1.t(), z(W1).t(), W1.shape[1])
    t, et = v * m1, e * m1.abs() + U * (v * m1).abs()
    r["dW2"] = mm(U2.t(), z(U2).t(), t, et, N)
    v, e, _ = mm(t, et, W2.t(), z(W2).t(), W2.shape[1])
    s, es = v * m2, e * m2.abs() + U * (v * m2).abs()
    d = dout.reshape(-1, 1)
    r["dW3"] = tuple(v.reshape(1, -1) for v in mm(s.t(), es.t(), d, z(d), N))
    r["ddout"] = tuple(v.reshape(-1) for v in mm(s, es, W3.reshape(-1, 1), z(W3).reshape(-1, 1), rowdot_n(s.shape[1])))
    r["t"], r["s"] = (t, et), (s, es)
    return r


def critic_step_ref(real, fake, alpha, W1, b1, W2, b2, W3, b3, slope, lam, M1=None, M2=None):
    """the critic iteration: losses [d_loss, lambda * gp] and the gradient of d_loss w.r.t. every parameter, each as
    (value, bound); M1 / M2 [3N][H]: the masks of the stacked rows (None: the fp64 signs)"""
    N, Din = real.shape
    R = 3 * N
    a = alpha.reshape(-1, 1)
    X = torch.cat([real, fake, a * real + (1 - a) * fake])
    eX = torch.cat([z(real), z(fake), 3 * U * (a.abs() * real.abs() + (1 - a).abs() * fake.abs())])
    f = critic_fwd_ref(X, W1, b1, W2, b2, W3, b3, slope, M1, M2)
    M1, M2 = f["m1"], f["m2"]
    eh1 = f["eh1"] + eX @ W1.abs().t()
    ea1 = eh1 * M1.abs() + U * f["a1"].abs()
    eh2 = f["eh2"] + ea1 @ W2.abs().t()
    ea2 = eh2 * M2.abs() + U * f["a2"].abs()
    eout = f["eout"] + (ea2 @ W3.abs().t()).reshape(-1)
    r = {"h1": (f["h1"], eh1), "h2": (f["h2"], eh2), "M1": M1, "M2": M2}
    # dout = (-1/N, +1/N, 1) per row group, as the kernel forms it in fp32
    dout = torch.cat([torch.full((N,), -1.0 / N), torch.full((N,), 1.0 / N), torch.ones(N)])
    dout = dout.float().double().to(real.device).reshape(-1, 1)
    out = f["out"][:2 * N]
    wterms = out * dout[:2 * N, 0]
    U2 = dout * W3.reshape(1, -1) * M2
    eU2 = 2 * U * U2.abs()
    v, e, _ = mm(U2, eU2, W2, z(W2), W2.shape[0])
    U1, eU1 = v * M1, e * M1.abs() + U * (v * M1).abs()
    g1, eg1 = U1[2 * N:], eU1[2 * N:]
    gx, egx, _ = mm(g1, eg1, W1, z(W1), W1.shape[0])
    s = (gx * gx).sum(1)
    es = U * (rowdot_n(Din) + 4) * s + 2 * (gx.abs() * egx).sum(1)
    rn = torch.sqrt(s)
    pos = rn > 0
    safe = torch.where(pos, rn, torch.ones_like(rn))
    er = torch.where(pos, es / (2 * safe) + U * rn, torch.zeros_like(rn))
    k = lam * 2.0 / N
    coef = torch.where(pos, k * (rn - 1) / safe, torch.zeros_like(rn))
    ecoef = torch.where(pos, abs(k) * er / (safe * safe) + 4 * U * coef.abs(), torch.zeros_like(rn))
    pterms = lam * (rn - 1) ** 2 / N
    epterms = abs(lam) / N * 2 * (rn - 1).abs() * er + 4 * U * pterms
    gp = pterms.sum()
    egp = epterms.sum() + U * (N + 4) * pterms.abs().sum()
    ew = (eout[:2 * N] * dout[:2 * N, 0].abs()).sum() + 2 * U * wterms.abs().sum()
    loss = wterms.sum() + gp
    eloss = ew + egp + U * (3 * N + 4) * (wterms.abs().sum() + pterms.abs().sum())
    r["losses"] = (torch.stack([loss, gp]), torch.stack([eloss, egp]))
    c = coef.reshape(-1, 1)
    ec = ecoef.reshape(-1, 1)
    g1s = c * g1
    eg1s = c.abs() * eg1 + ec * g1.abs() + U * g1s.abs()
    Ucat, eUcat = torch.cat([U1[:2 * N], g1s]), torch.cat([eU1[:2 * N], eg1s])
    Xcat, eXcat = torch.cat([X[:2 * N], gx]), torch.cat([z(X[:2 * N]), egx])
    r["dW1"] = mm(Ucat.t(), eUcat.t(), Xcat, eXcat, R)
    acc, eacc, _ = mm(gx, egx, W1.t(), z(W1).t(), Din)
    Mp = M1[2 * N:]
    t = acc * c * Mp
    et = (eacc * c.abs() + acc.abs() * ec) * Mp.abs() + 2 * U * t.abs()
    A1cat, eA1cat = torch.cat([f["a1"][:2 * N], t]), torch.cat([ea1[:2 * N], et])
    r["dW2"] = mm(U2.t(), eU2.t(), A1cat, eA1cat, R)
    v, e, _ = mm(t, et, W2.t(), z(W2).t(), W2.shape[1])
    sp, esp = v * M2[2 * N:], e * M2[2 * N:].abs() + U * (v * M2[2 * N:]).abs()
    A2cat, eA2cat = torch.cat([f["a2"][:2 * N], sp]), torch.cat([ea2[:2 * N], esp])
    r["dW3"] = tuple(v.reshape(1, -1) for v in mm(A2cat.t(), eA2cat.t(), dout, z(dout), R))
    r["db1"] = (U1[:2 * N].sum(0), U * (2 * N + 4) * U1[:2 * N].abs().sum(0) + eU1[:2 * N].sum(0))
    r["db2"] = (U2[:2 * N].sum(0), U * (2 * N + 4) * U2[:2 * N].abs().sum(0) + eU2[:2 * N].sum(0))
    r["db3"] = (dout[:2 * N].sum().reshape(1), U * (2 * N + 4) * dout[:2 * N].abs().sum().reshape(1))
    r["coef"], r["ecoef"] = coef, ecoef
    # the workspace rows the kernel's last GEMMs read: U1 (penalty rows scaled), X3 (penalty rows gx), U2, A1
    # (penalty rows t), A2 (penalty rows (t W2^T) * m2)
    r["ws"] = {"U1": (Ucat, eUcat), "X3": (Xcat, eXcat), "U2": (U2, eU2), "A1": (A1cat, eA1cat), "A2": (A2cat, eA2cat)}
    r["dout"] = dout
    return r


F32 = torch.float32


def check_mask(what, m, h, eh, slope):
    """the kernel's mask equals the fp64 sign of h wherever |h| exceeds its bound, and is 1 or slope everywhere"""
    m = m.double().view_as(h)
    ok = (m == 1) | (m == torch.tensor(slope, dtype=F32).item())
    assert ok.all(), f"{what}: mask value {m[~ok][0].item()} is neither 1 nor the slope"
    sure = h.abs() > eh
    bad = sure & (m != mask(h, torch.tensor(slope, dtype=F32).item()))
    assert not bad.any(), f"{what}: mask differs from the sign of h at {tuple(bad.nonzero()[0].tolist())}, " \
                          f"h {h[bad][0].item():.3e}, bound {eh[bad][0].item():.3e}"
