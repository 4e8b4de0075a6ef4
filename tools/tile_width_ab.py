#!/usr/bin/env python
"""Gradient-kernel time with 256- vs 128-wide column tiles (SIGLIP_OPT_GRAD_TILE_N), and what auto mode (0) picks,
on one binary: the widths alternate inside each repetition so that they see the same clocks. CUDA-event time per
launch (SIGLIP_OPT_KERNEL_TIMING), median over the repetitions."""
import argparse, math, os, statistics, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from distributed_sigmoid_loss_b200 import SigmoidLossEngine, _capi

ap = argparse.ArgumentParser()
ap.add_argument("--shapes", default="16384x1024,16384x384,16384x768,16384x1152,4096x768")
ap.add_argument("--reps", type=int, default=5)
ap.add_argument("--iters", type=int, default=10)
a = ap.parse_args()
dev = torch.device("cuda", 0)
print(torch.cuda.get_device_name(0), flush=True)
for shape in a.shapes.split(","):
    B, D = (int(x) for x in shape.split("x"))
    g = torch.Generator().manual_seed(1234)
    img = torch.nn.functional.normalize(torch.randn(B, D, generator=g)).to(torch.bfloat16).to(dev)
    txt = torch.nn.functional.normalize(torch.randn(B, D, generator=g)).to(torch.bfloat16).to(dev)
    eng = SigmoidLossEngine(B, D, dev)
    tp, bs = torch.tensor([math.log(10.0)], device=dev), torch.tensor([-10.0], device=dev)
    res = {tn: ([], []) for tn in (256, 128, 0)}
    for _ in range(a.reps):
        for tn in (256, 128, 0):
            eng.set_option(_capi.SIGLIP_OPT_GRAD_TILE_N, tn)
            for _ in range(3):
                eng.fwd_bwd(img, txt, tp, bs, torch.bfloat16)
            torch.cuda.synchronize()
            eng.set_option(_capi.SIGLIP_OPT_KERNEL_TIMING, 1)
            for _ in range(a.iters):
                eng.fwd_bwd(img, txt, tp, bs, torch.bfloat16)
            lm, ln, gm, gn = eng.kernel_times()
            eng.set_option(_capi.SIGLIP_OPT_KERNEL_TIMING, 0)
            res[tn][0].append(1e3 * gm / gn)
            res[tn][1].append(1e3 * lm / ln)
    out = []
    for tn in (256, 128, 0):
        gr, lo = res[tn]
        out.append(f"tile_n={tn}: grad {statistics.median(gr):.1f} us [{min(gr):.1f}, {max(gr):.1f}], "
                   f"loss {statistics.median(lo):.1f} us")
    print(f"B={B} D={D}: " + " | ".join(out), flush=True)
    eng.close()
