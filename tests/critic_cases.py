"""Case table of the MLP critic (pytorch-gan_b200/csrc/mlp_critic.cu): one row per call of b200gan_mlp_critic_fwd,
b200gan_mlp_critic_bwd, b200gan_mlp_critic_dbwd and b200gan_critic_step_mlp.

Every call is one cooperative launch of num_sms * min(2, blocks per SM) blocks of 256 threads.  The blocks per SM
follow from the kernels' registers (ptxas -v, sm_90a) and their 8448 bytes of shared memory: 65536 registers per SM
over 256 threads * (registers rounded up to 8) gives 6 (fwd, 39 registers), 5 (bwd, 48) and 4 (dbwd and critic_step,
64), so every grid is 2 * 132 = 264 blocks on a 132-SM H100 SXM.  tests/test_cpu_kernel_coverage.py recompiles
mlp_critic.cu and holds REGISTERS and GRID to ptxas.

tests/test_gpu_critic_conformance.py runs every case against torch float64.
"""
from dataclasses import dataclass

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
