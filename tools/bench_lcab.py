#!/usr/bin/env python
"""Kernel- and module-level timing of LocalContextAttentionBlock (SURVEY.md 8(d) rows "LCAB self, image / BEV" and
the P2I cross block) at the base shapes, for the planar window path with the projection chain (default), without it, and the interleaved path
(DI_B200_WINDOW_TC=0).  Prints one JSON line per (shape, path): per-call kernel times from CUDA events, the module
time, and the module-boundary roofline fraction (2 F bytes for self attention, 3 F for cross: each distinct input map
read once, the output written once) against MEASURED_PEAKS.json.

    python tools/bench_lcab.py [--iters 20] [--only img|bev]      (needs an H100)
"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=20)
    ap.add_argument('--only', default='')
    args = ap.parse_args()
    from deepinteraction_b200 import mmri, ops, synth
    dev = torch.device('cuda:0')
    torch.set_grad_enabled(False)
    peak = 6650.0
    pth = os.path.join(ROOT, 'MEASURED_PEAKS.json')
    if os.path.exists(pth):
        peak = json.load(open(pth))['hbm_gbs']
    C = 128
    torch.manual_seed(5)
    holder = mmri.LocalContextAttentionBlock(C, C, 9)
    synth.randomize_norm_stats(holder, 5)
    pk = mmri._pack_lcab(holder.eval(), dev)
    flush = torch.empty(256 * 1024 * 1024 // 4, device=dev)          # > L2: evict between iterations
    shapes = [('img_self', 6, 112, 200, True), ('img_cross', 6, 112, 200, False), ('bev_self', 1, 180, 180, True)]
    for tag, N, H, W, self_attn in shapes:
        if args.only and not tag.startswith(args.only):
            continue
        M = N * H * W
        x = torch.randn(M, C, device=dev)
        y = x if self_attn else torch.randn(M, C, device=dev)
        for path in ('planar+proj', 'planar', 'interleaved'):
            ops.WINDOW_TC[0] = path != 'interleaved'
            ops.LCAB_PROJ[0] = path == 'planar+proj'
            for _ in range(3):
                out = mmri.lcab_forward(pk, x, y, N, H, W)
            torch.cuda.synchronize()
            tot = 0.0
            ops.PROFILE[0] = []
            for _ in range(args.iters):
                flush.zero_()
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                out = mmri.lcab_forward(pk, x, y, N, H, W)
                b.record()
                torch.cuda.synchronize()
                tot += a.elapsed_time(b)
            prof, ops.PROFILE[0] = ops.PROFILE[0], None
            per = {}
            for name, e0, e1, nb, fl, _mod in prof:
                d = per.setdefault(name, [0, 0.0])
                d[0] += 1
                d[1] += e0.elapsed_time(e1)
            F = M * C * 4
            mod_bytes = (2 if self_attn else 3) * F
            mod_us = tot / args.iters * 1e3
            win = [k for k in per if 'window' in k][0]
            win_us = per[win][1] / per[win][0] * 1e3
            print(json.dumps(dict(shape=tag, path=path, module_us=round(mod_us, 1), module_bytes_mb=round(mod_bytes / 1e6, 2),
                                  module_gbs=round(mod_bytes / (mod_us * 1e-6) / 1e9, 1),
                                  module_frac_of_hbm_peak=round(mod_bytes / (mod_us * 1e-6) / 1e9 / peak, 3),
                                  window_kernel=win, window_us=round(win_us, 1),
                                  window_kernel_gbs=round(4 * F / (win_us * 1e-6) / 1e9, 1),
                                  window_frac_of_hbm_peak=round(4 * F / (win_us * 1e-6) / 1e9 / peak, 3),
                                  kernels={k: round(v[1] / v[0] * 1e3, 1) for k, v in per.items()},
                                  out_checksum=float(out.double().abs().sum()))), flush=True)
    ops.WINDOW_TC[0] = True
    ops.LCAB_PROJ[0] = True


if __name__ == '__main__':
    main()
