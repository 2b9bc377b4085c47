"""Every normalisation case of tests/norm_cases.py, element by element against torch float64.

Each case calls the C ABI directly on the guarded buffers of tests/conformance.py (Arena: NaN around the inputs,
outputs started as NaN, sentinels around everything the library writes) and runs its protocol: stats -> finalize ->
apply, then the backward, eagerly and replayed from a CUDA graph.  A LeakyReLU / ReLU backward gets scale_shift and no
saved output (the mask is recomputed from x); a Tanh / Sigmoid backward gets the saved output y.  Checked:
  - y, running_mean / running_var, num_batches_tracked, dx, dgamma / dbeta against fp64;
  - the statistics accumulator and the backward's sums workspace come back zeroed;
  - round_tf32 outputs are TF32-representable;
  - the trace shows the kernel instances, sample count and channel slices the table names.
The reference takes the activation's derivative from the kernel's own y (the mask of x * scale + shift in fp32, or
the saved output the library differentiates through), so an element next to a sign change cannot flip.  The checks
live in norm_cases.check_outputs, with bounds 2^-16 relative to the magnitudes that enter each value: an indexing
error, a wrong channel's parameters or a lost slice is O(1).  The statistics themselves, at the models' sizes and far
from zero, are held to their summation chains by tests/test_gpu_norm_statistics.py.
"""
import pytest

import norm_cases as nc
from conformance import run_case
from norm_cases import check_outputs

pytestmark = pytest.mark.gpu

class Run(nc.Run):
    def check(self, what):
        return check_outputs(self, what)


# the statistics and the backward's sums are fp64 atomics in no fixed order; everything formed from them may differ in
# its last bits between two calls
VARIES = ("y", "mean_rstd", "scale_shift", "dx", "dgb", "running_mean", "running_var")


def launches(c):
    """the table's kernel instances in launch order; a templated instance's grid has the samples (InstanceNorm: N) in y
    and the channel slices in z"""
    g = c.geom
    return [(k, (None, g.N if g.per_sample else 1, g.slices) if "<" in k else None) for k in c.kernels]


@pytest.mark.parametrize("case", nc.CASES, ids=lambda c: c.id)
def test_norm_case(case):
    run_case(Run(case), case.id, launches(case), varies=VARIES, family=("norm_",))
