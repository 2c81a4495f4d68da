#!/usr/bin/env python
"""Times the query-row dense layers of the decoder: di_rows_mlp_f32 vs the wgmma / FFMA dense kernels, each captured 20x
in a CUDA graph so that the figure is device time per launch, not the Python launch rate (needs an H100)."""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from deepinteraction_b200 import ops, fold  # noqa: E402

dev = torch.device('cuda:0')
g = torch.Generator().manual_seed(0)
REP = 20


def t(fn, n=20):
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        for _ in range(3):
            fn()
        s.synchronize()
        gr = torch.cuda.CUDAGraph()
        with torch.cuda.graph(gr, stream=s):
            for _ in range(REP):
                fn()
        gr.replay()
        s.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(s)
        for _ in range(n):
            gr.replay()
        b.record(s)
        s.synchronize()
    return a.elapsed_time(b) / (n * REP) * 1e3


for M, K, N1, N2 in [(200, 128, 384, 0), (200, 256, 384, 20), (200, 128, 512, 128), (200, 128, 128, 0), (200, 2, 128, 128),
                     (400, 128, 512, 128)]:
    x = torch.randn(M, K, generator=g).to(dev)
    W1, b1 = fold.Weight(torch.randn(N1, K, generator=g), dev), torch.randn(N1, generator=g).to(dev)
    W2 = fold.Weight(torch.randn(N2, N1, generator=g), dev) if N2 else None
    b2 = torch.randn(N2, generator=g).to(dev) if N2 else None

    def unfused():
        y = ops.linear([x], W1, b1, ops.ACT_RELU)
        return ops.linear([y], W2, b2) if N2 else y
    ops.TC_BF16[0] = False
    W1.wt
    if W2 is not None:
        W2.wt
    print('M%d K%d N1 %d N2 %d: rows_mlp %.1f us, dense kernels %.1f us (device time per launch, weights hot in L2)'
          % (M, K, N1, N2, t(lambda: ops.rows_mlp([x], W1, b1, ops.ACT_RELU, W2, b2)), t(unfused)), flush=True)
