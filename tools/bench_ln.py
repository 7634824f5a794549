"""CUDA-event timings of the LayerNorm launches of one TTS step (rows = 32 x 313 decoder / 32 x 160 encoder tokens,
C = 768, bf16): forward with the fp32 residual stream, backward (dx + dgamma / dbeta, with and without the column sums
of dx that replace the out_proj / fc2 bias-gradient launches) and the separate column-sum kernel they replace. Each case
rotates over enough distinct buffers to exceed the 50 MB L2 (the step's LayerNorms read what a GEMM wrote a layer ago,
but timing one resident buffer would flatter an HBM-bound kernel). Output: algorithmic GB/s next to the data-sheet HBM bandwidth."""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from speecht5_b200 import kernels as K  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--out", default=None)
args = ap.parse_args()
dev = "cuda"


def timed(fns):
    """All calls of `fns` captured into ONE graph (no host gaps), replayed three times; returns us per call."""
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for f in fns[:2]:
            f()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        for f in fns:
            f()
    torch.cuda.synchronize()
    best = 1e30
    for _ in range(3):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        g.replay()
        e1.record()
        torch.cuda.synchronize()
        best = min(best, e0.elapsed_time(e1) / len(fns) * 1e3)
    return best


peak = 3350.0  # GB/s, HBM3 of the H100 SXM data sheet: a bound, not a rate reached
rows_out = []
for rows, C, drop in ((10016, 768, 0.1), (5120, 768, 0.1)):
    nbuf = max(4, int(400e6 / (rows * C * 2 * 4)))
    bufs = []
    for i in range(nbuf):
        x = torch.randn(rows, C, device=dev).bfloat16()
        bufs.append(dict(dy=torch.randn(rows, C, device=dev).bfloat16(), s=x, ds=torch.empty_like(x), dx=torch.empty_like(x),
                         y=torch.empty_like(x), res32=torch.randn(rows, C, device=dev), y32=torch.empty(rows, C, device=dev)))
    mean = torch.zeros(rows, device=dev)
    rstd = torch.ones(rows, device=dev)
    gamma, beta = torch.ones(C, device=dev), torch.zeros(C, device=dev)
    dg, db, dxs = torch.zeros(C, device=dev), torch.zeros(C, device=dev), torch.zeros(C, device=dev)
    e = 2 * rows * C  # bytes of one bf16 tensor
    cases = {
        "ln_bwd": (lambda b: K.ln_bwd(b["dy"], b["s"], mean, rstd, gamma, b["ds"], b["dx"], dg, db, drop, 1, 0), 4 * e),
        "ln_bwd_dxsum": (lambda b: K.ln_bwd(b["dy"], b["s"], mean, rstd, gamma, b["ds"], b["dx"], dg, db, drop, 1, 0, dxsum=dxs), 4 * e),
        "colsum": (lambda b: K.colsum(b["dx"], dxs, accumulate=True), e),
        "ln_fwd_stream": (lambda b: K.ln_fwd(b["dy"], None, gamma, beta, b["y"], b["ds"], mean, rstd, 1e-5, drop, 1, 0,
                                              residual_f32=b["res32"], y_f32=b["y32"]), 3 * e + 2 * 2 * e),
    }
    for name, (fn, nbytes) in cases.items():
        us = timed([(lambda b=b: fn(b)) for b in bufs for _ in range(2)])
        rec = dict(kernel=name, rows=rows, C=C, us=round(us, 2), algorithmic_mb=round(nbytes / 1e6, 1),
                   gbps=round(nbytes / us / 1e3, 1), frac_of_hbm_peak=(round(nbytes / us / 1e3 / peak, 3) if peak else None))
        rows_out.append(rec)
        print(json.dumps(rec))
if args.out:
    json.dump(rows_out, open(args.out, "w"), indent=1)
