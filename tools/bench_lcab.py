#!/usr/bin/env python
"""Per-stage timing of LocalContextAttentionBlock (C = 128) at the base shapes: the projection stage in both arms --
the fused kernel (ops.lcab_proj) and the five-launch chain of tests/lcab_chain.py -- and the planar window kernel
(ops.lcab_window_tc), each timed as separate calls with CUDA events, L2 flushed before every call.  Prints one JSON line
per shape.

Projection rates are quoted against the fused floor: each distinct input map read once and q, k, v written once,
4 F bytes for self attention and 5 F for cross attention (F = M * 128 * 4 bytes).  The peak is the H100 SXM data-sheet
HBM3 bandwidth (3.35 TB/s) unless MEASURED_PEAKS.json gives a measured one.  `proj_fused_ctas_qkv` is the number of
Q, K and V CTAs the fused kernel launched.

The window kernel's figures are computed from the shape and the kernel's tiling (8 x 16 queries per CTA, 8 warps of
2 x 8 queries): its HBM floor (q, k, v read once and out written once, 512 bytes per pixel each), its mma.sync
m16n8k16 count (per warp 4 chunks x 2 k16 steps x 20 key blocks x 3 split products for Q K^T plus 4 chunks x 10 halo
rows x 4 channel blocks x 3 for P V) and the time that count takes at the data-sheet dense bf16 rate (989 TFLOP/s),
its L2 -> shared-memory fill (per tile and 32-channel chunk: the 16 x 24 K halo and the 8 x 16 Q tile, then the V
halo, 128 bytes per pixel), and the fraction of the HBM floor the measured time reaches.

    python tools/bench_lcab.py [--iters 20] [--only img|bev]      (needs an H100)
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.append(os.path.join(ROOT, 'tests'))


def timed(fn, flush, iters):
    """Mean device time (us) of fn() over iters calls, each after an L2 flush."""
    for _ in range(3):
        fn()
    tot = 0.0
    for _ in range(iters):
        flush.zero_()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        tot += a.elapsed_time(b)
    return tot / iters * 1e3


BF16_TFLOPS = 989.0                                                # H100 SXM data sheet, dense


def window_counts(N, H, W, peak_gbs):
    """Shape-derived figures of the planar window kernel (C = 128)."""
    M = N * H * W
    tiles = N * -(-H // 8) * -(-W // 16)
    floor = 4 * M * 512
    mma = tiles * 8 * (4 * 2 * 20 * 3 + 4 * 10 * 4 * 3)
    fill = tiles * 4 * ((16 * 24 + 8 * 16) + 16 * 24) * 128
    return dict(tiles=tiles, hbm_floor_mb=round(floor / 1e6, 1), hbm_floor_us=round(floor / (peak_gbs * 1e9) * 1e6, 1),
                mma_sync=mma, mma_us_at_datasheet=round(mma * 4096 / (BF16_TFLOPS * 1e12) * 1e6, 1),
                l2_fill_mb=round(fill / 1e6, 1))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=20)
    ap.add_argument('--only', default='')
    args = ap.parse_args()
    from deepinteraction_b200 import _lib, mmri, ops, synth
    from lcab_chain import chain
    dev = torch.device('cuda:0')
    torch.set_grad_enabled(False)
    peak, peak_src = 3350.0, 'H100 SXM data sheet (3.35 TB/s)'
    pth = os.path.join(ROOT, 'MEASURED_PEAKS.json')
    if os.path.exists(pth):
        peak, peak_src = json.load(open(pth))['hbm_gbs'], 'MEASURED_PEAKS.json'
    gpu = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                         capture_output=True, text=True).stdout.strip().splitlines()
    C = 128
    torch.manual_seed(5)
    holder = mmri.LocalContextAttentionBlock(C, C, 9)
    synth.randomize_norm_stats(holder, 5)
    pk = mmri._pack_lcab(holder.eval(), dev)
    w = (pk['w_self'], pk['b_self'], pk['w_2'], pk['b_2'])
    flush = torch.empty(256 * 1024 * 1024 // 4, device=dev)          # > L2: evict between calls
    shapes = [('img_self', 6, 112, 200, True), ('img_cross', 6, 112, 200, False), ('bev_self', 1, 180, 180, True)]
    for tag, N, H, W, self_attn in shapes:
        if args.only and not tag.startswith(args.only):
            continue
        M = N * H * W
        x = torch.randn(M, C, device=dev)
        y = x if self_attn else torch.randn(M, C, device=dev)
        F = M * C * 4
        floor = (4 if self_attn else 5) * F
        res = dict(shape=tag, M=M, gpu=gpu[0] if gpu else None, peak_gbs=peak, peak_source=peak_src,
                   proj_floor_mb=round(floor / 1e6, 1), proj_floor_us=round(floor / (peak * 1e9) * 1e6, 1))
        roles = [ctypes.c_int() for _ in range(3)]
        _lib.check(_lib.lib().di_lcab_proj_grid(M, *[ctypes.byref(r) for r in roles]), 'di_lcab_proj_grid')
        res['proj_fused_ctas_qkv'] = [r.value for r in roles]
        outs = {}
        for arm, fn in (('fused', lambda: ops.lcab_proj(x, y, *w)), ('chain', lambda: chain(x, y, *w))):
            us = timed(fn, flush, args.iters)
            outs[arm] = [t.view(torch.int32) for t in fn()]
            gbs = floor / (us * 1e-6) / 1e9
            res['proj_' + arm] = dict(us=round(us, 1), gbs_vs_floor=round(gbs, 1), frac_of_peak=round(gbs / peak, 3))
        res['fused_equals_chain'] = all(torch.equal(a, b) for a, b in zip(outs['fused'], outs['chain']))
        q, k, v = (t.view(torch.float32) for t in outs['fused'])
        out = torch.empty(M, C, device=dev)
        res['window_us'] = round(timed(lambda: ops.lcab_window_tc(q, k, v, N, H, W, C, out=out), flush, args.iters), 1)
        win = window_counts(N, H, W, peak)
        win['frac_of_hbm_floor'] = round(win['hbm_floor_us'] / res['window_us'], 3)
        res['window'] = win
        print(json.dumps(res), flush=True)


if __name__ == '__main__':
    main()
