"""Case table of the MLP generator (pytorch-gan_b200/csrc/mlp_generator/mlp_generator.cu): one row per call of
b200gan_mlp_gen_fwd and b200gan_mlp_gen_bwd.

Every call is one cooperative launch of num_sms * min(2, blocks per SM) blocks of 256 threads.  The blocks per SM
follow from the kernels' registers (ptxas -v, sm_90a) and their 8448 bytes of shared memory: 65536 registers per SM
over 256 threads * (registers rounded up to 8) gives 5 (fwd, 48 registers) and 3 (bwd, 80), so every grid is
2 * 132 = 264 blocks on a 132-SM H100 SXM.  tests/test_cpu_mlp_generator.py recompiles the kernel file and holds
REGISTERS and GRID to ptxas, and the fp64 references to torch float64 autograd.

tests/test_gpu_mlp_generator_conformance.py runs every case against its fp64 reference.
"""
from dataclasses import dataclass

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
