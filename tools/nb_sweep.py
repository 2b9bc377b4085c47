"""Empirical check of the staged chain kernels' tile planner (csrc/narrow_block.cu: nb_plan): every (KT, PT, KG) candidate
of the four DCGAN discriminator layers, forward and data gradient, one pass (N = 128) and the grouped D-step pass
(N = 256, two statistics groups), CUDA-graph timed like tools/nb_bench.py.  Prints the planner's own choice next to the
best candidate.
    python tools/nb_sweep.py            # needs the GPU
"""
import os
import sys

import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "pytorch-gan_b200"))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from b200gan import ops  # noqa: E402
from b200gan.functional import ACT_LRELU, PACK_SIMT_DGRAD, PACK_SIMT_FPROP  # noqa: E402
from nb_bench import LAYERS, timed  # noqa: E402


def main():
    for groups, n in ((1, 128), (2, 256)):
        for name, _, c, h, k in LAYERS:
            a = torch.randn(n, c, h, h, device="cuda").contiguous(memory_format=torch.channels_last)
            w = torch.randn(k, c, 3, 3, device="cuda") * 0.1
            b = torch.zeros(k, device="cuda")
            g, _ = ops.make_geom((n, c, h, h), (k, c, 3, 3), 2, (1, 1, 1, 1))
            edge = None
            if c > 1:
                ad = a.double().view(groups, n // groups, c, h, h)
                stats = torch.cat([torch.cat([ad[q].sum((0, 2, 3)), (ad[q] * ad[q]).sum((0, 2, 3))]) for q in range(groups)])
                edge = ops.BnEdge(stats.contiguous(), torch.ones(c, device="cuda"), torch.zeros(c, device="cuda"), 0.8,
                                  n // groups * h * h, groups)
            pf, pd = ops.pack_weights(g, w, PACK_SIMT_FPROP), ops.pack_weights(g, w, PACK_SIMT_DGRAD)
            cs = torch.ones(n, k, device="cuda")
            dz = torch.randn(n, k, g.P, g.Q, device="cuda").contiguous(memory_format=torch.channels_last)
            runs = {"fprop": ("B200GAN_NB_FORCE_FPROP", lambda: ops.nb_fprop(g, a, pf, b, ACT_LRELU, 0.2, cs, edge, None, None,
                                                                            None, 0.1, True, groups)),
                    "dgrad": ("B200GAN_NB_FORCE_DGRAD", lambda: ops.nb_dgrad(g, dz, pd, edge, a))}
            for what, (var, fn) in runs.items():
                os.environ.pop(var, None)
                base = timed(fn, iters=10, reps=5)
                res = []
                for kt in (16, 8, 4, 1):
                    for pt in (4, 2, 1):
                        for kg in (8, 4, 2, 1):
                            os.environ[var] = f"{kt}:{pt}:{kg}"
                            try:
                                res.append((timed(fn, iters=10, reps=5), kt, pt, kg))
                            except RuntimeError:
                                pass
                os.environ.pop(var, None)
                res.sort()
                top = ", ".join(f"{t:.1f}us KT{kt} PT{pt} KG{kg}" for t, kt, pt, kg in res[:4])
                print(f"groups {groups} {name:<18} {what}: planner {base:.1f}us | best {top} | worst {res[-1][0]:.1f}us "
                      f"({len(res)} candidates)", flush=True)


if __name__ == "__main__":
    main()
