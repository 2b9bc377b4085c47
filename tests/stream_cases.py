"""Case table of the streaming kernels: the discriminator head and BCE loss (pytorch-gan_b200/csrc/head.cu) and the
index, activation, epilogue-backward and Adam kernels (pytorch-gan_b200/csrc/index_ops.cu).

A case is one call sequence of the C ABI (`op`), its geometry (`dims`) and options (`opt`), and the kernels it must
launch, in order, with their grids on a 132-SM H100 SXM.  The grids restate the host code's launch arithmetic:
stream_blocks(n) = clamp(ceil(n / 256), 1, 16 * num_sms), the BCE backward's 1184-block cap, bias_grad's row split
and adam_multi's ADAM_CHUNK blocks per tensor in launches of at most ADAM_MAX_TENSORS tensors.

tests/test_cpu_kernel_coverage.py holds the kernel names to the sources; tests/test_gpu_stream_conformance.py runs
every case against torch float64 (bit for bit where the kernel only moves data).
"""
from dataclasses import dataclass, field

NUM_SMS = 132
ADAM_CHUNK = 256 * 16
ADAM_MAX_TENSORS = 48
BCE_MAX_BLOCKS = 1184
ACTS = ("none", "lrelu", "relu", "tanh", "sigmoid")


def cdiv(a, b):
    return -(-a // b)


def stream_blocks(n):
    return max(1, min(cdiv(n, 256), NUM_SMS * 16))


def bias_grad_grid(rows, K):
    yb = max(1, NUM_SMS * 8 // cdiv(K, 32))
    rpb = max(cdiv(rows, yb), 64)
    return (cdiv(K, 32), cdiv(rows, rpb), 1), rpb


@dataclass(frozen=True)
class Case:
    name: str
    op: str          # linear1 | bce | transpose | upsample | pad | act | epilogue | adam
    dims: tuple
    opt: dict = field(default_factory=dict, hash=False, compare=False)
    error: bool = False
    why: str = ""

    @property
    def id(self):
        return f"{self.op}-{self.name}"

    @property
    def deterministic(self):
        """outputs that must repeat bit for bit in a replay (bias_grad sums with atomics)"""
        return self.op != "epilogue"

    @property
    def launches(self):
        """[(kernel, grid)] in launch order"""
        if self.error:
            return []
        d, o = self.dims, self.opt
        if self.op == "linear1":
            N, K = d
            return [("linear1_fwd_kernel", (N, 1, 1)), ("linear1_bwd_kernel", (cdiv(K, 128), 1, 1))]
        if self.op == "bce":
            (n,) = d
            return [("bce_fwd_kernel", (1, 1, 1)), ("bce_bwd_kernel", (min(cdiv(n, 256), BCE_MAX_BLOCKS), 1, 1))]
        if self.op == "transpose":
            N, C, HW = d
            rows, cols = (C, HW) if o.get("to_nhwc", True) else (HW, C)
            if rows == 1 or cols == 1:
                return []          # a device-to-device copy, no kernel
            return [("transpose_kernel", (cdiv(cols, 32), cdiv(rows, 32), N))]
        if self.op == "upsample":
            N, H, W, C = d
            return [("upsample2x_fwd_kernel", (stream_blocks(4 * N * H * W * C), 1, 1)),
                    ("upsample2x_bwd_kernel", (stream_blocks(N * H * W * C), 1, 1))]
        if self.op == "pad":
            N, H, W, C = d
            t, l, b, r = o["pads"]
            nout, nin = N * (H + t + b) * (W + l + r) * C, N * H * W * C
            if C % 4 == 0 and not o.get("offset"):
                return [("pad2d_fwd_v4_kernel", (stream_blocks(nout // 4), 1, 1)),
                        ("pad2d_bwd_v4_kernel", (stream_blocks(nin // 4), 1, 1))]
            return [("pad2d_fwd_kernel", (stream_blocks(nout), 1, 1)), ("pad2d_bwd_kernel", (stream_blocks(nin), 1, 1))]
        if self.op == "act":
            N, HW, C = d
            return [("act_fwd_kernel", (stream_blocks(N * HW * C), 1, 1))]
        if self.op == "epilogue":
            N, PQ, K = d
            return [("epilogue_bwd_kernel", (stream_blocks(N * PQ * K), 1, 1)),
                    ("bias_grad_kernel", bias_grad_grid(N * PQ, K)[0])]
        if self.op == "adam":
            sizes = self.adam_sizes()
            if not sizes:
                return [("adam_step_inc_kernel", (1, 1, 1))]
            return [("adam_multi_kernel", (sum(cdiv(n, ADAM_CHUNK) for n in sizes[b:b + ADAM_MAX_TENSORS]), 1, 1))
                    for b in range(0, len(sizes), ADAM_MAX_TENSORS)]
        raise ValueError(self.op)

    @property
    def kernels(self):
        return tuple(k for k, _ in self.launches)

    def adam_sizes(self):
        (count,) = self.dims
        cycle = self.opt.get("sizes", (1, ADAM_CHUNK, ADAM_CHUNK + 1))
        return [cycle[i % len(cycle)] for i in range(max(count, 0))]


_c = Case
CASES = [
    # ---- head.cu: Linear(K -> 1) [+ Sigmoid], forward and backward -----------------------------------------------------
    _c("dcgan", "linear1", (128, 2048), dict(act="sigmoid"), why="the DCGAN head: Linear(128 * 4 * 4, 1) + Sigmoid"),
    _c("k1", "linear1", (128, 1), dict(act="sigmoid"), why="K = 1: one thread of 128 has work; scalar path"),
    _c("k3", "linear1", (7, 3), dict(act="none"), why="K = 3: scalar path, no activation"),
    _c("k129", "linear1", (33, 129), dict(act="sigmoid"), why="K = 129: two backward blocks, the second with one k"),
    _c("k4_offset", "linear1", (5, 4), dict(act="sigmoid", offset=1),
       why="K = 4 with x one float off 16-byte alignment: the scalar path of a K % 4 == 0 row"),
    _c("n1", "linear1", (1, 64), dict(act="sigmoid"), why="N = 1"),
    _c("n4096", "linear1", (4096, 129), dict(act="sigmoid", sparse=True),
       why="N = 4096: the backward's shared-memory limit; dy non-zero on every 64th row and the last"),
    _c("nulls", "linear1", (9, 100), dict(act="none", b=False, dx=False, db=False), why="b, dx and db NULL"),
    _c("n4097", "linear1", (4097, 4), dict(act="sigmoid"), error=True, why="N = 4097 is refused by the backward"),
    # ---- head.cu: BCELoss(reduction='mean') -------------------------------------------------------------------------------
    _c("n1", "bce", (1,), dict(t=1.0), why="n = 1, target 1"),
    _c("n128", "bce", (128,), dict(t=0.0), why="n = 128, target 0"),
    _c("n128_soft", "bce", (128,), dict(t=0.3), why="target 0.3"),
    _c("clamps", "bce", (256,), dict(t="mixed", edges=True),
       why="v exactly 0 and 1 with targets 0, 1, 0.3: the -100 log clamp and the 1e-12 denominator clamp"),
    _c("n1e6", "bce", (10 ** 6,), dict(t="mixed"), why="n = 10^6: beyond the backward's 1184-block grid"),
    _c("over_cap", "bce", (1184 * 256 + 4097,), dict(t="mixed"), why="n just above 1184 * 256: a second grid-stride pass"),
    # ---- index_ops.cu: layout transpose -------------------------------------------------------------------------------
    _c("ragged", "transpose", (2, 33, 45), dict(to_nhwc=True), why="NCHW -> NHWC ragged against 32 both ways"),
    _c("ragged_back", "transpose", (3, 65, 31), dict(to_nhwc=False), why="NHWC -> NCHW ragged against 32 both ways"),
    _c("c1", "transpose", (4, 1, 50), dict(to_nhwc=True), why="C = 1 (rows == 1): a copy, no kernel may run"),
    _c("hw1", "transpose", (4, 70, 1), dict(to_nhwc=False), why="HW = 1 (cols == 1): a copy, no kernel may run"),
    _c("n65536", "transpose", (65536, 2, 2), dict(to_nhwc=True), error=True, why="N = 65536 > the grid's z limit"),
    # ---- index_ops.cu: nearest x2 upsample -------------------------------------------------------------------------------
    _c("c1", "upsample", (2, 5, 7, 1), why="C = 1, odd H and W"),
    _c("c3", "upsample", (3, 7, 5, 3), why="C = 3, odd H and W"),
    _c("c64", "upsample", (2, 3, 9, 64), why="C = 64, odd H and W"),
    # ---- index_ops.cu: padding ----------------------------------------------------------------------------------------------
    _c("zero_pix2pix", "pad", (2, 8, 8, 64), dict(pads=(1, 1, 0, 0), mode="zero"),
       why="nn.ZeroPad2d((1, 0, 1, 0)) of pix2pix, C = 64: the float4 kernels"),
    _c("reflect1", "pad", (2, 8, 8, 64), dict(pads=(1, 1, 1, 1), mode="reflect"),
       why="nn.ReflectionPad2d(1) of the CycleGAN residual blocks: the float4 kernels"),
    _c("reflect3_c3", "pad", (1, 16, 16, 3), dict(pads=(3, 3, 3, 3), mode="reflect"),
       why="nn.ReflectionPad2d(3) in front of the CycleGAN generator, C = 3: the scalar kernels"),
    _c("reflect_h_1", "pad", (2, 5, 5, 4), dict(pads=(4, 4, 4, 4), mode="reflect"),
       why="a reflection pad of H - 1 on every side: every mirror row and column folds back"),
    _c("reflect_h_1_c3", "pad", (2, 5, 6, 3), dict(pads=(4, 5, 4, 5), mode="reflect"),
       why="reflection pads of H - 1 and W - 1, scalar kernels"),
    _c("reflect_asym", "pad", (1, 6, 7, 8), dict(pads=(2, 0, 1, 3), mode="reflect"), why="four different pads"),
    _c("zero_h1", "pad", (2, 1, 9, 4), dict(pads=(2, 1, 2, 1), mode="zero"), why="H = 1 with zero padding"),
    _c("zero_w1", "pad", (2, 9, 1, 3), dict(pads=(1, 2, 1, 2), mode="zero"), why="W = 1 with zero padding, C = 3"),
    _c("c3_zero", "pad", (2, 7, 5, 3), dict(pads=(1, 1, 1, 1), mode="zero"), why="C = 3: the scalar kernels"),
    _c("misaligned", "pad", (2, 6, 6, 8), dict(pads=(2, 2, 2, 2), mode="reflect", offset=1),
       why="C % 4 == 0 but x and dy one float off 16-byte alignment: the scalar kernels"),
    _c("rtf_v4", "pad", (2, 8, 8, 64), dict(pads=(1, 1, 1, 1), mode="reflect", rtf=True),
       why="round_tf32 on the float4 kernel"),
    _c("rtf_scalar", "pad", (1, 9, 9, 3), dict(pads=(3, 3, 3, 3), mode="reflect", rtf=True),
       why="round_tf32 on the scalar kernel"),
    _c("reflect_ge_h", "pad", (1, 3, 8, 4), dict(pads=(3, 1, 1, 1), mode="reflect"), error=True,
       why="a reflection pad of H is refused by the forward and the backward"),
    _c("reflect_ge_w", "pad", (1, 8, 3, 3), dict(pads=(1, 1, 1, 4), mode="reflect"), error=True,
       why="a reflection pad beyond W is refused by the forward and the backward"),
    # ---- index_ops.cu: activation (+ dropout mask) --------------------------------------------------------------------------
    *[_c(f"{a}_{m}_c{C}", "act", (3, 37, C), dict(act=a, mask=m), why=f"{a}, mask {m}, C = {C}")
      for a in ACTS for m, C in (("none", 3), ("elem", 1), ("chan", 3), ("chan", 1))],
    # ---- index_ops.cu: epilogue backward and bias gradient ------------------------------------------------------------------
    *[_c(f"{a}{'_cs' if cs else ''}", "epilogue", (4, 50, 33), dict(act=a, cs=cs),
         why=f"{a} {'with' if cs else 'without'} chan_scale (zeros included), K = 33")
      for a in ACTS for cs in (False, True)],
    _c("rtf_tanh_cs", "epilogue", (2, 40, 33), dict(act="tanh", cs=True, rtf=True), why="round_tf32, tanh, chan_scale"),
    _c("rtf_lrelu", "epilogue", (2, 40, 33), dict(act="lrelu", rtf=True), why="round_tf32, LeakyReLU"),
    _c("k1", "epilogue", (3, 21, 1), dict(act="sigmoid", cs=True), why="K = 1, 63 rows: fewer than 64"),
    _c("k512", "epilogue", (2, 30, 512), dict(act="lrelu", cs=True), why="K = 512, 60 rows"),
    _c("split_rows", "epilogue", (16, 256, 33), dict(act="tanh"),
       why="4096 rows over 64 blocks of 64 rows: yb atomics per column"),
    _c("split_k512", "epilogue", (8, 1000, 512), dict(act="relu", cs=True), why="8000 rows over 125 row blocks, K = 512"),
    # ---- index_ops.cu: Adam -----------------------------------------------------------------------------------------------
    _c("count0", "adam", (0,), why="no tensors: only the step advances"),
    _c("count1", "adam", (1,), dict(sizes=(ADAM_CHUNK + 1,)), why="one tensor of ADAM_CHUNK + 1: two blocks"),
    _c("count48", "adam", (48,), why="48 tensors: one full launch"),
    _c("count49", "adam", (49,), dict(step0=7), why="49 tensors: two launches, step starting at 7"),
    _c("cyclegan", "adam", (96,), dict(gscale=0.25),
       why="96 tensors, the CycleGAN optimizer over both generators: two launches; grad_scale 0.25"),
    _c("n1_step7", "adam", (3,), dict(sizes=(1,), step0=7), why="1-element tensors, step starting at 7"),
    _c("n0", "adam", (3,), dict(bad=(1, "n0")), error=True, why="a tensor with n = 0 is refused"),
    _c("null_p", "adam", (3,), dict(bad=(2, "null")), error=True, why="a tensor with a NULL pointer is refused"),
    _c("late_null", "adam", (96,), dict(bad=(60, "null")), error=True,
       why="a NULL pointer in the second launch's tensors is refused before the first launch runs"),
    _c("count_neg", "adam", (-1,), error=True, why="count < 0 is refused"),
]
