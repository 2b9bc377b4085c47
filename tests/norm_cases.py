"""Case table of the normalisation entry points (b200gan_norm_stats / finalize / apply / bwd).

One geometry per edge of the apply and backward kernels' plan, each run with every fused activation, together with
what the library must launch for it: the vector width VEC of the norm_apply / norm_bwd_reduce / norm_bwd_apply
instances (4 when C % 4 == 0 and the streamed tensors are 16-byte aligned, else 1) and the number of channel slices
of at most 256 groups in gridDim.z.  Written from the launchers in pytorch-gan_b200/csrc/norm.cu, not from a run.

tests/test_cpu_norm_case_table.py checks it against the kernels the source declares and launches;
tests/test_gpu_norm_conformance.py runs every case against torch float64.
"""
from dataclasses import dataclass

ACTS = ("none", "lrelu", "relu", "tanh", "sigmoid")


@dataclass(frozen=True)
class Geom:
    name: str
    N: int
    C: int
    H: int
    W: int
    per_sample: bool      # InstanceNorm2d (groups n*C + c) rather than BatchNorm2d (groups c)
    affine: bool
    vec: int              # expected VEC of the apply / backward instances
    slices: int = 1       # expected gridDim.z
    offset: int = 0       # floats between x's aligned allocation and x (1 misaligns every float4)
    why: str = ""


GEOMS = (
    Geom("c3", 4, 3, 16, 16, False, True, vec=1, why="C % 4 != 0: 85 rows of 3 groups per block, 1 thread left over"),
    Geom("c5", 3, 5, 12, 12, True, False, vec=1, why="InstanceNorm with N > 1 at VEC 1: 51 rows of 5, 1 left over"),
    Geom("c16", 8, 16, 8, 8, False, True, vec=4, why="reference layer width: 4 groups, 64 rows per block"),
    Geom("c64", 2, 64, 16, 16, True, False, vec=4, why="reference InstanceNorm(64)"),
    Geom("c128", 4, 128, 8, 8, False, True, vec=4, why="reference BatchNorm(128)"),
    Geom("c512", 2, 512, 4, 4, True, False, vec=4, why="reference InstanceNorm(512): 128 groups, 2 rows per block"),
    Geom("c96", 4, 96, 8, 8, False, True, vec=4, why="256 % 24 != 0: 10 rows per block, 16 threads left over"),
    Geom("c768", 2, 768, 4, 4, True, False, vec=4, why="192 groups: one row per block, 64 threads left over"),
    Geom("c1280", 2, 1280, 4, 4, False, True, vec=4, slices=2, why="320 groups: slices of 256 and 64 groups"),
    Geom("c258", 2, 258, 4, 4, True, True, vec=1, slices=2,
         why="affine InstanceNorm at VEC 1 with slices of 256 and 2 channels: gamma indexed by channel"),
    Geom("c64_off", 4, 64, 8, 8, False, True, vec=1, offset=1, why="x one float past 16-byte alignment: VEC 1"),
    Geom("bn_hw1", 64, 128, 1, 1, False, True, vec=4, why="BatchNorm over a 1x1 map: the batch is the whole group"),
)


@dataclass(frozen=True)
class Case:
    geom: Geom
    act: str
    rtf: bool             # round_tf32 on y and dx

    @property
    def kernels(self):
        """the kernel instances a forward (stats, finalize, apply) and a backward launch, in order"""
        v = self.geom.vec
        return ("norm_stats_kernel", "norm_finalize_kernel", f"norm_apply_kernel<{v}>",
                f"norm_bwd_reduce_kernel<{v}>", f"norm_bwd_apply_kernel<{v}>", "norm_bwd_params_kernel")

    @property
    def id(self):
        return f"{self.geom.name}-{self.act}{'-rtf' if self.rtf else ''}"


# every geometry with every activation; round_tf32 alternates so that each activation runs with it on and off
CASES = tuple(Case(g, a, (i + j) % 2 == 1) for i, g in enumerate(GEOMS) for j, a in enumerate(ACTS))
