#!/usr/bin/env python
"""Where does a launch of the wgmma kernels spend its time? globaltimer stamps of CTA 0 (SIGLIP_OPT_AUX_TRACE) for
back-to-back fused steps at one shape: gap since the previous launch ended, set-up, first operands, MMA issue span, tail
(last MMA issued -> last CTA done)."""
import argparse
import math
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from distributed_sigmoid_loss_b200 import SigmoidLossEngine, _capi

ap = argparse.ArgumentParser()
ap.add_argument("--B", type=int, default=4096)
ap.add_argument("--D", type=int, default=768)
ap.add_argument("--steps", type=int, default=40)
ap.add_argument("--pdl", type=int, default=1)
ap.add_argument("--split-k", type=int, default=0)
a = ap.parse_args()
dev = torch.device("cuda", 0)
g = torch.Generator().manual_seed(1234)
img = torch.nn.functional.normalize(torch.randn(a.B, a.D, generator=g)).to(torch.bfloat16).to(dev)
txt = torch.nn.functional.normalize(torch.randn(a.B, a.D, generator=g)).to(torch.bfloat16).to(dev)
tp = torch.tensor([math.log(10.0)], device=dev)
b = torch.tensor([-10.0], device=dev)
eng = SigmoidLossEngine(a.B, a.D, dev)
eng.set_option(_capi.SIGLIP_OPT_SPLIT_K, a.split_k)
eng.set_option(_capi.SIGLIP_OPT_PDL, a.pdl)
for _ in range(20):
    eng.fwd_bwd(img, txt, tp, b, torch.bfloat16)
torch.cuda.synchronize()
eng.set_option(_capi.SIGLIP_OPT_AUX_TRACE, 1)
for _ in range(a.steps):
    eng.fwd_bwd(img, txt, tp, b, torch.bfloat16)
tr = eng.aux_trace()
eng.set_option(_capi.SIGLIP_OPT_AUX_TRACE, 0)
names = ["loss", "grad"]
acc = {n: [] for n in names}
for i in range(2, len(tr)):
    t0, tflag, tdone, tend, tentry, tsetup, tfirst, tlast, tfirstcta, tmma_max, tmma_min, tepi, tent_max, tent_min, \
        tsetup_max, _ = tr[i]
    prev_end = tr[i - 1][3]
    acc[names[i % 2]].append((tentry - prev_end, tsetup - tentry, tfirst - tsetup, tlast - tfirst, tend - tlast,
                              tend - tentry, tdone - t0, tmma_max - tmma_min, tepi - tmma_max, tend - tepi,
                              tend - tfirstcta, tent_max - tent_min, tsetup_max - tent_min, tend - tent_min))
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
e0.record()
for _ in range(a.steps):
    eng.fwd_bwd(img, txt, tp, b, torch.bfloat16)
e1.record()
torch.cuda.synchronize()
print(f"pdl={a.pdl}: {e0.elapsed_time(e1) / a.steps * 1e3:.1f} us per fused step (CUDA events around {a.steps} back-to-back steps)")
print(f"B={a.B} D={a.D}: median over {len(acc['loss'])} launches (us): gap after previous launch | set-up | first operands | "
      "MMA issue span (CTA 0) | tail | kernel entry->end | aux jobs || spread of 'last MMA issued' over CTAs | latest MMA issue -> "
      "all tiles' epilogues done | -> kernel end | first CTA exit -> kernel end || first -> last CTA entry | first entry -> last "
      "set-up done | first entry -> kernel end")
for n in names:
    cols = list(zip(*acc[n]))
    med = [sorted(c)[len(c) // 2] / 1e3 for c in cols]
    print(f"  {n}: " + " | ".join(f"{m:7.2f}" for m in med))
eng.close()
