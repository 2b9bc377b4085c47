"""Per-kernel timing of the fused Discriminator chain (csrc/narrow_block.cu) on the four DCGAN blocks (dcgan.py:77-88) at
the BASELINE size (batch 128, 64x64): 20 launches captured in a CUDA graph, CUDA events around 10 replays (operands of one
layer fit in L2: these are the warm numbers the training step sees; the step's ncu launch list is the cold view).  Each
launch includes the wrapper's memset nodes (statistics / sums buffers).
    python tools/nb_bench.py            # needs the GPU
"""
import os
import sys

import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "pytorch-gan_b200"))
from b200gan import ops  # noqa: E402
from b200gan.functional import ACT_LRELU, PACK_SIMT_DGRAD, PACK_SIMT_FPROP  # noqa: E402

LAYERS = [("conv1 1->16 @64", 128, 1, 64, 16), ("conv2 16->32 @32", 128, 16, 32, 32), ("conv3 32->64 @16", 128, 32, 16, 64),
          ("conv4 64->128 @8", 128, 64, 8, 128)]


def timed(fn, iters=20, reps=10, warm=3):
    """GPU time per launch: `iters` launches captured in one CUDA graph (no host launch gaps), replayed `reps` times."""
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(side):
        fn()
        side.synchronize()
        with torch.cuda.graph(graph, stream=side):
            for _ in range(iters):
                fn()
    torch.cuda.synchronize()
    graph.replay()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    for _ in range(reps):
        graph.replay()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) * 1e3 / (iters * reps)


def main():
    print(f"{'layer':<20}{'fprop':>9}{'dz':>9}{'wgrad':>9}{'dgrad':>9}   us (MB moved: in+out activations)")
    tot = [0.0] * 4
    for name, n, c, h, k in LAYERS:
        a = torch.randn(n, c, h, h, device="cuda").contiguous(memory_format=torch.channels_last)
        w = torch.randn(k, c, 3, 3, device="cuda") * 0.1
        b = torch.zeros(k, device="cuda")
        g, _ = ops.make_geom((n, c, h, h), (k, c, 3, 3), 2, (1, 1, 1, 1))
        edge = None
        if c > 1:
            ad = a.double()
            stats = torch.cat([ad.sum((0, 2, 3)), (ad * ad).sum((0, 2, 3))]).contiguous()
            edge = ops.BnEdge(stats, torch.ones(c, device="cuda"), torch.zeros(c, device="cuda"), 0.8, n * h * h)
        pf, pd = ops.pack_weights(g, w, PACK_SIMT_FPROP), ops.pack_weights(g, w, PACK_SIMT_DGRAD)
        cs = torch.ones(n, k, device="cuda")
        y, st = ops.nb_fprop(g, a, pf, b, ACT_LRELU, 0.2, cs, edge, None, None, None, 0.1, True)
        out_edge = ops.BnEdge(st, torch.ones(k, device="cuda"), torch.zeros(k, device="cuda"), 0.8, n * g.P * g.Q)
        out_edge.sums = torch.zeros(2 * k, device="cuda", dtype=torch.float64)
        gy = torch.randn_like(y)
        dz, _ = ops.nb_dz(gy, y, cs, ACT_LRELU, 0.2, out_edge, True)
        t = [timed(lambda: ops.nb_fprop(g, a, pf, b, ACT_LRELU, 0.2, cs, edge, None, None, None, 0.1, True)),
             timed(lambda: ops.nb_dz(gy, y, cs, ACT_LRELU, 0.2, out_edge, True)),
             timed(lambda: ops.nb_wgrad(g, a, dz, edge, tuple(w.shape))),
             timed(lambda: ops.nb_dgrad(g, dz, pd, edge, a))]
        mb = (a.numel() + y.numel()) * 4 / 1e6
        print(f"{name:<20}" + "".join(f"{v:9.1f}" for v in t) + f"   ({mb:.1f} MB)")
        tot = [x + v for x, v in zip(tot, t)]
    print(f"{'sum':<20}" + "".join(f"{v:9.1f}" for v in tot))
    print("one D pass forward = sum(fprop); one D backward with parameter gradients = sum(dz + wgrad + dgrad)")


if __name__ == "__main__":
    main()
