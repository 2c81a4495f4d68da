"""Times the kernels of di_lcab_window_f32 (0 = bf16-split mma.sync, 1 = FFMA) at the bench shapes."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
from deepinteraction_b200 import ops, _lib

dev = torch.device('cuda:0')
L = _lib.lib()
junk = torch.empty(64 << 20, device=dev)
for (N, H, W, C) in ((6, 112, 200, 128), (1, 180, 180, 128)):
    q, k, v = (torch.randn(N * H * W, C, device=dev) for _ in range(3))
    for mode in (0, 1):
        L.di_set_window_ffma(mode)
        for _ in range(2):
            out = ops.lcab_window(q, k, v, N, H, W, C, 9)
        ts = []
        for _ in range(5):
            junk.zero_()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(); ops.lcab_window(q, k, v, N, H, W, C, 9, out=out); e1.record()
            torch.cuda.synchronize()
            ts.append(e0.elapsed_time(e1) * 1e3)
        us = float(np.median(ts))
        fl = 2 * 2 * 81 * N * H * W * C
        print('window %dx%dx%d C=%d kernel=%d: %.1f us  %.1f TFLOP/s useful  %.0f GB/s algorithmic' % (
            N, H, W, C, mode, us, fl / us / 1e6, 16.0 * N * H * W * C / us / 1e3))
    L.di_set_window_ffma(0)
