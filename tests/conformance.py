"""The conformance harness every kernel family's case table runs through.

A family supplies a case table (tests/*_cases.py, with its fp64 references) and a `Run` per case:
  prepare()       guards, NaN-filled outputs and workspaces, the inputs (Arena.prepare);
  call(stream)    the case's C ABI calls on that stream, returning the first non-zero code or 0;
  outputs()       copies of everything the call may write;
  check(what)     the outputs the last call left in the buffers against fp64, returning the worst |err| / bound;
and run_case() holds every case to one protocol:
  - a refused call returns one of the case's codes, leaves every guard intact and writes no byte of any output or
    workspace;
  - an accepted call returns 0, leaves every guard intact, its outputs pass check(), and its trace passes check_route();
  - the call captured in a CUDA graph on a side stream and replayed leaves every guard intact, repeats every output the
    case does not name as varying bit for bit, and passes check() again.

Buffers (Arena) are carved from one allocation, [guard | tensor | guard], every tensor 256-byte aligned behind a 4 KB
guard:
  - input guards hold NaN: a read past an input that feeds arithmetic shows up as NaN in the output;
  - outputs and workspaces start as NaN: an element the kernel never writes fails, and stale workspace contents
    cannot pass for zeros;
  - output / workspace / statistics / read-modify-write guards hold a sentinel bit pattern that must survive the call;
  - statistics start at known non-zero values: the header promises accumulation, not overwrite.

Also here: the TF32 models, the one element-wise checker, the profiler trace, and the source tooling the CPU tests
share (the csrc/ parser, the registry of case tables, ptxas).
"""
import glob
import json
import os
import re
import shutil
import subprocess
import tempfile

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "pytorch-gan_b200", "csrc")

GUARD_BYTES = 4096
ALIGN_BYTES = 256
SENTINEL = 0x7FC0DEAD          # a NaN bit pattern no kernel produces
STATS_FILL = (3.0, 5.0)        # prefill of stats[0..G) and stats[G..2G)


# ---- TF32 models -------------------------------------------------------------------------------------------------
def tf32_trunc(t):
    """what wgmma does to a raw fp32 operand: the low 13 mantissa bits are ignored"""
    return (t.contiguous().view(torch.int32) & ~0x1FFF).view(torch.float32)


def tf32_rna(t):
    """cvt.rna.tf32.f32: round to nearest, ties away from zero (the packed weights, round_tf32 outputs)"""
    return ((t.contiguous().view(torch.int32) + 0x1000) & ~0x1FFF).view(torch.float32)


def np_rna(a):
    a = np.ascontiguousarray(a, dtype=np.float32)
    return ((a.view(np.int32) + 0x1000) & ~0x1FFF).view(np.float32)


# ---- buffers -----------------------------------------------------------------------------------------------------
class Arena:
    """Tensors carved from one device allocation, each between two guards of GUARD_BYTES."""

    def __init__(self, specs):
        # specs: list of (name, numel, dtype, role) with role in {"in", "io", "out", "ws", "stats"}; "io" is a
        # read-modify-write operand: it holds its data, between sentinel guards
        self.specs = specs
        off = 0
        self.layout = {}
        for name, numel, dtype, role in specs:
            isz = torch.empty((), dtype=dtype).element_size()
            off += GUARD_BYTES
            nbytes = -(-max(numel, 1) * isz // ALIGN_BYTES) * ALIGN_BYTES
            self.layout[name] = (off, numel, dtype, role, nbytes)
            off += nbytes
        off += GUARD_BYTES
        self.buf = torch.empty(off // 4, dtype=torch.int32, device="cuda")
        self.t = {}
        for name, (o, numel, dtype, role, nbytes) in self.layout.items():
            raw = self.buf[o // 4:(o + nbytes) // 4]
            self.t[name] = raw.view(dtype)[:numel]

    def guards(self, name):
        o, numel, dtype, role, nbytes = self.layout[name]
        isz = torch.empty((), dtype=dtype).element_size()
        lo = self.buf[(o - GUARD_BYTES) // 4:o // 4]
        tail_start = o + numel * isz
        hi = self.buf[-(-tail_start // 4):(o + nbytes + GUARD_BYTES) // 4]
        return lo, hi

    def prepare(self, data):
        """guards, NaN / prefill of outputs and workspaces; data: name -> tensor for the inputs"""
        nan32 = torch.tensor(float("nan"), dtype=torch.float32).view(torch.int32).item()
        self.buf.fill_(nan32)
        for name, (o, numel, dtype, role, nbytes) in self.layout.items():
            lo, hi = self.guards(name)
            if role != "in":
                lo.fill_(SENTINEL)
                hi.fill_(SENTINEL)
            if role in ("in", "io"):
                self.t[name].copy_(data[name].reshape(-1))
            elif role == "stats":
                g = numel // 2
                self.t[name][:g] = STATS_FILL[0]
                self.t[name][g:] = STATS_FILL[1]
            else:
                self.t[name].fill_(float("nan"))

    def check_guards(self, what):
        for name, (o, numel, dtype, role, nbytes) in self.layout.items():
            if role == "in":
                continue
            for side, g in zip(("front", "back"), self.guards(name)):
                bad = (g != SENTINEL).nonzero()
                assert bad.numel() == 0, f"{what}: {name} guard ({side}) overwritten at word {bad[0].item()}"

    def ptr(self, name):
        return self.t[name].data_ptr() if name in self.t else None

    def outputs(self):
        """copies of every tensor the library may write"""
        return {k: v.clone() for k, v in self.t.items() if self.layout[k][3] != "in"}


# ---- checks ------------------------------------------------------------------------------------------------------
def check_elementwise(what, got, ref, bound, layout="", alt=None):
    """|got - ref| <= bound element by element, no NaN in got; where `alt` is not NaN, matching alt instead is
    accepted.  Returns the worst |err| / bound."""
    got = got.double().reshape(ref.shape)
    assert not torch.isnan(got).any(), f"{what}: NaN at {layout} {tuple(torch.isnan(got).nonzero()[0].tolist())} " \
                                       "(an element never written, or a guard read)"
    err = (got - ref).abs()
    if alt is not None:
        err = torch.where(torch.isnan(alt), err, torch.minimum(err, (got - alt).abs()))
    ratio = err / bound.clamp_min(1e-300)
    bad = ((err > bound) | torch.isnan(err)).nonzero()
    worst = ratio[~torch.isnan(ratio)].max().item() if ratio.numel() else 0.0
    if bad.numel():
        at = tuple(bad[0].tolist())
        raise AssertionError(f"{what}: |err| {err[at].item():.3e} > bound {bound[at].item():.3e} at {layout} {at}; "
                             f"got {got[at].item():.9g}, fp64 {ref[at].item():.9g}; worst |err|/bound {worst:.3g}")
    return worst


def not_vacuous(what, bound, terms):
    """median bound below the median magnitude of one term of the sum (a tap, an image, a product)"""
    t = terms[terms > 0]
    if t.numel() == 0:
        return
    med_b, med_t = bound.median().item(), t.median().item()
    assert med_b < med_t, f"{what}: vacuous bound: median bound {med_b:.3e} >= median one-term contribution {med_t:.3e}"


def bits_equal(what, got, want):
    got, want = got.reshape(-1).contiguous(), want.reshape(-1).contiguous().to(got.dtype)
    same = got.view(torch.int32) == want.view(torch.int32)
    if not same.all():
        i = same.logical_not().nonzero()[0].item()
        raise AssertionError(f"{what}: element {i}: {got[i].item()!r}, expected bit for bit {want[i].item()!r}")


def _same_bytes(a, b):
    return torch.equal(a.view(torch.uint8), b.view(torch.uint8))


# ---- profiler ----------------------------------------------------------------------------------------------------
def short_name(name):
    name = name.replace("(anonymous namespace)::", "")
    if name.startswith("void "):
        name = name[5:]
    head = name.split("(", 1)[0]
    return head.rsplit("::", 1)[-1] if "<" not in head else head[:head.index("<")].rsplit("::", 1)[-1] + \
        head[head.index("<"):]


def base_name(kernel):
    return kernel.split("<", 1)[0]


_PROFILER_WARM = []


def traced_kernels(fn):
    """(name, grid) of every kernel `fn` launches, in launch order, template arguments kept.

    The first CUDA activity session of a process can come back empty: a warm-up session runs once.  Once sessions have
    run, CUPTI hands a session its activity buffer while the session's first launch is in cudaLaunchKernel, and the
    kernel record of that launch can be lost while its runtime record stays.  So a marker goes first and its record,
    when there is one, is dropped here: every library kernel lives in namespace b200gan, the marker does not."""
    from torch.profiler import ProfilerActivity, profile
    if not _PROFILER_WARM:
        with profile(activities=[ProfilerActivity.CUDA]):
            torch.ones(1, device="cuda").add_(1)
            torch.cuda.synchronize()
        _PROFILER_WARM.append(True)
    marker = torch.zeros(1, device="cuda")
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        marker.zero_()
        fn()
        torch.cuda.synchronize()
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "trace.json")
        prof.export_chrome_trace(path)
        with open(path) as fh:
            trace = json.load(fh)
    events = [ev for ev in trace.get("traceEvents", []) if ev.get("cat") == "kernel"]
    if events and "b200gan::" not in events[0]["name"]:
        events = events[1:]
    return [(short_name(ev["name"]), tuple(ev.get("args", {}).get("grid", ()))) for ev in events]


def kernel_matches(expected, seen):
    """a table name with template arguments names one instance; without, any instance of the kernel"""
    return seen == expected if "<" in expected else base_name(seen) == expected


def first_grid(kernels, grid):
    """[(kernel, grid)] of a table that gives the grid of its first kernel only"""
    return [(k, grid if i == 0 else None) for i, k in enumerate(kernels)]


def check_route(what, call, launches, family=None, ordered=True, num_sms=None, prepare=None):
    """The kernels `call()` launches against the table's `launches`, [(kernel, grid or None)].

    family: name prefixes the comparison keeps (None: every kernel).  ordered: the kept trace is the table's launches in
    order; otherwise (the conv table) every traced kernel matches an entry and every entry is traced.  A grid of None,
    or a None in it, is not compared, and grids are compared only on a device with num_sms SMs (None: any device).

    A profiler session now and then comes back without some kernel records.  The call is the same every time, so an
    attempt whose records contradict the table fails at once, while one that only misses records is tried again, up to
    three times; the last must match exactly.  A trace without the table's kernels fails."""
    grids = num_sms is None or torch.cuda.get_device_properties(0).multi_processor_count == num_sms

    def fits(entry, rec):
        (name, grid), (n, g) = entry, rec
        return kernel_matches(name, n) and (not grids or grid is None or
                                            (len(grid) == len(g) and all(w is None or w == h for w, h in zip(grid, g))))

    seen = []
    for _ in range(3):
        if prepare is not None:
            prepare()
        seen = [r for r in traced_kernels(call) if family is None or r[0].startswith(family)]
        if ordered:   # an in-order subsequence of the table, matched greedily
            j = 0
            for rec in seen:
                while j < len(launches) and not fits(launches[j], rec):
                    j += 1
                assert j < len(launches), f"{what}: trace {seen} is not the table's {launches} in order " \
                                          f"({rec} out of place)"
                j += 1
            if len(seen) == len(launches):
                return
        else:
            for rec in seen:
                assert any(fits(e, rec) for e in launches), f"{what}: unexpected kernel {rec} (table: {launches})"
            if all(any(fits(e, rec) for rec in seen) for e in launches):
                return
    raise AssertionError(f"{what}: after three traces the trace {seen} still misses some of the table's {launches}")


# ---- the protocol ------------------------------------------------------------------------------------------------
def run_case(run, what, launches, refuse=(), varies=(), family=None, ordered=True, num_sms=None):
    """One case through the protocol of this module's docstring.  refuse: the codes a refusal case may return (empty for
    a case that must be accepted); varies: outputs that may differ between the eager call and the replay; launches,
    family, ordered, num_sms: the route, as check_route takes it."""
    stream = lambda: torch.cuda.current_stream().cuda_stream  # noqa: E731
    run.prepare()
    before = run.outputs()
    rc = run.call(stream())
    torch.cuda.synchronize()
    if refuse:
        assert rc in refuse, f"{what}: expected a refusal {refuse}, rc {rc}"
        run.arena.check_guards(what)
        for k, v in run.outputs().items():
            assert _same_bytes(v, before[k]), f"{what}: refused call wrote {k}"
        return
    assert rc == 0, f"{what}: rc {rc}: {run.lib.b200gan_last_error().decode()}"
    run.arena.check_guards(what)
    eager = run.outputs()
    worst = run.check(what + " eager")

    check_route(what, lambda: run.call(stream()), launches, family, ordered, num_sms, run.prepare)

    # a CUDA graph on a side stream, replayed once; a launch on the legacy stream fails the capture
    side = torch.cuda.Stream()
    run.prepare()
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=side):
        rc = run.call(side.cuda_stream)
    assert rc == 0, f"{what}: rc {rc} under capture: {run.lib.b200gan_last_error().decode()}"
    run.prepare()
    torch.cuda.synchronize()
    graph.replay()
    torch.cuda.synchronize()
    run.arena.check_guards(what + " graph")
    for k, v in run.outputs().items():
        if k not in varies:
            assert _same_bytes(v, eager[k]), f"{what}: graph replay differs from the eager call in {k}"
    worst = max(worst, run.check(what + " graph"))
    print(f"\n{what}: worst |err|/bound {worst:.3g}")


# ---- sources -----------------------------------------------------------------------------------------------------
def source(path):
    """the file without its // comments"""
    with open(path) as fh:
        return re.sub(r"//[^\n]*", "", fh.read())


def declared(path):
    """__global__ names, also behind a __launch_bounds__ whose arguments hold a call"""
    return set(re.findall(r"__global__\s+void\s+(?:__launch_bounds__\((?:[^()]|\([^()]*\))*\)\s*)?(\w+)\s*\(",
                          source(path)))


def declared_under_csrc():
    """kernel -> the file under csrc/ that declares it, over every .cu and .cuh at any depth"""
    return {k: os.path.relpath(p, CSRC) for ext in ("*.cu", "*.cuh")
            for p in glob.glob(os.path.join(CSRC, "**", ext), recursive=True) for k in declared(p)}


def functions(src):
    """name -> body of every function definition (static helpers and extern "C" entry points) in src"""
    src = re.sub(r"//[^\n]*", "", src)
    out = {}
    for m in re.finditer(r"\n(?:static|extern \"C\")[^;{]*?\b(\w+)\s*\([^;{]*\)\s*\{", src):
        depth, i = 1, m.end()
        while depth:
            depth += {"{": 1, "}": -1}.get(src[i], 0)
            i += 1
        out[m.group(1)] = src[m.end():i - 1]
    return out


NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
if not os.path.exists(NVCC):
    NVCC = shutil.which("nvcc")
needs_nvcc = pytest.mark.skipif(NVCC is None, reason="no nvcc")


def ptxas_report(path):
    """kernel -> dict(registers, stack, spills, smem) from ptxas -v, compiling `path` with the library's flags; a
    template instance of one integer argument is named `kernel<N>`"""
    import build as b200_build
    with tempfile.TemporaryDirectory() as d:
        r = subprocess.run([NVCC, *b200_build.FLAGS, "-Xptxas=-v", "-c", path, "-o", os.path.join(d, "k.o")],
                           capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-2000:]
    out = {}
    for chunk in r.stderr.split("Compiling entry function")[1:]:
        m = re.match(r" '_ZN7b200gan\d+(\w+?)(?:ILi(\d+)EE)?E", chunk)
        name = m.group(1) + (f"<{m.group(2)}>" if m.group(2) else "")
        stack, stores, loads = (int(v) for v in re.search(
            r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", chunk).groups())
        smem = re.search(r"(\d+) bytes smem", chunk)
        out[name] = dict(registers=int(re.search(r"Used (\d+) registers", chunk).group(1)), stack=stack,
                         spills=stores + loads, smem=int(smem.group(1)) if smem else 0)
    return out


# ---- the registry ------------------------------------------------------------------------------------------------
class Family:
    """a registered case table: its cases, a case's kernel names, the C ABI entry points its runs call, and the modules
    (the case table and its GPU conformance test) in which those calls are made"""

    def __init__(self, cases, names, entry_points, modules):
        self.cases, self.names, self.entry_points, self.modules = cases, names, tuple(entry_points), tuple(modules)


def case_tables():
    """family -> Family: every table whose kernels and entry points count as covered"""
    import chain_cases
    import class_head_cases
    import conv_cases
    import critic_cases
    import generator_cases
    import norm_cases
    import norm_conv_cases
    import pixel_loss_cases
    import stats_cases
    import stream_cases
    import tail_cases
    names = lambda c: c.kernels  # noqa: E731
    b = "b200gan_"
    return {
        "conv": Family(conv_cases.CASES, names,
                       [b + "conv2d_" + p for p in ("fprop", "dgrad", "wgrad", "wgrad_fused_bias")],
                       ["conv_cases.py", "test_gpu_conv_conformance.py"]),
        "chain": Family(chain_cases.CASES, names,
                        [b + "nb_" + p for p in ("fprop", "dz", "wgrad", "dgrad", "tail_fwd", "tail_bwd")],
                        ["chain_cases.py", "test_gpu_fused_conformance.py"]),
        "tail": Family(tail_cases.CASES, names, [b + "tail_fprop", b + "tail_bwd"],
                       ["tail_cases.py", "test_gpu_fused_conformance.py"]),
        "norm": Family(norm_cases.CASES, names, [b + "norm_" + p for p in ("stats", "finalize", "apply", "bwd")],
                       ["norm_cases.py", "test_gpu_norm_conformance.py"]),
        "norm conv": Family(norm_conv_cases.CASES, names, norm_conv_cases.ENTRY_POINTS,
                            ["norm_conv_cases.py", "test_gpu_norm_conv_conformance.py"]),
        "critic": Family(critic_cases.CASES, names,
                         [b + p for p in ("mlp_critic_fwd", "mlp_critic_bwd", "mlp_critic_dbwd", "critic_step_mlp")],
                         ["critic_cases.py", "test_gpu_critic_conformance.py"]),
        "stream": Family(stream_cases.CASES, names,
                         [b + p for p in ("epilogue_bwd", "bias_grad", "nchw_to_nhwc", "nhwc_to_nchw", "upsample2x_fwd",
                                          "upsample2x_bwd", "pad2d_fwd", "pad2d_bwd", "act_fwd", "linear1_fwd",
                                          "linear1_bwd", "bce_fwd", "bce_bwd", "adam_multi")],
                         ["stream_cases.py", "test_gpu_stream_conformance.py"]),
        "generator": Family(generator_cases.CASES, names, [b + "mlp_gen_fwd", b + "mlp_gen_bwd"],
                            ["generator_cases.py", "test_gpu_mlp_generator_conformance.py"]),
        "class head": Family(class_head_cases.CASES, names,
                             [b + p for p in ("class_head_fwd", "class_head_bwd", "cross_entropy_fwd",
                                              "cross_entropy_bwd")],
                             ["class_head_cases.py", "test_gpu_class_head_conformance.py"]),
        "pixel loss": Family(pixel_loss_cases.CASES, lambda c: [k for k, _ in c.kernels()],
                             [b + "pixel_loss_fwd", b + "pixel_loss_bwd"],
                             ["pixel_loss_cases.py", "test_gpu_pixel_loss_conformance.py"]),
        # the statistics every normalisation producer hands on: its entry points belong to norm, conv and chain
        "statistics": Family(stats_cases.CASES, names, [], ["stats_cases.py", "test_gpu_norm_statistics.py"]),
    }


def table_kernels(cases, names=lambda c: c.kernels):
    """the kernels a case table names, without template arguments"""
    return {base_name(k) for c in cases for k in names(c)}
