#!/usr/bin/env python
"""Per-stage timing of LocalContextAttentionBlock (C = 128) at the base shapes: the projection stage (ops.lcab_proj)
in both arms -- the fused kernel and the five-launch chain -- and the planar window kernel (ops.lcab_window_tc), each
timed as separate calls with CUDA events, L2 flushed before every call.  Prints one JSON line per shape.

Projection rates are quoted against the fused floor: each distinct input map read once and q, k, v written once,
4 F bytes for self attention and 5 F for cross attention (F = M * 128 * 4 bytes).  The peak is the H100 SXM data-sheet
HBM3 bandwidth (3.35 TB/s) unless MEASURED_PEAKS.json gives a measured one.

    python tools/bench_lcab.py [--iters 20] [--only img|bev]      (needs an H100)
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=20)
    ap.add_argument('--only', default='')
    args = ap.parse_args()
    from deepinteraction_b200 import mmri, ops, synth
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
        outs = {}
        for arm, fused in (('fused', True), ('chain', False)):
            ops.set_lcab_fused(fused)
            us = timed(lambda: ops.lcab_proj(x, y, *w), flush, args.iters)
            q, k, v = ops.lcab_proj(x, y, *w)
            outs[arm] = (q, k, v)
            gbs = floor / (us * 1e-6) / 1e9
            res['proj_' + arm] = dict(us=round(us, 1), gbs_vs_floor=round(gbs, 1), frac_of_peak=round(gbs / peak, 3))
        ops.set_lcab_fused(True)
        res['fused_equals_chain'] = all(torch.equal(a.view(torch.int32), b.view(torch.int32))
                                        for a, b in zip(outs['fused'], outs['chain']))
        q, k, v = outs['fused']
        out = torch.empty(M, C, device=dev)
        res['window_us'] = round(timed(lambda: ops.lcab_window_tc(q, k, v, N, H, W, C, out=out), flush, args.iters), 1)
        print(json.dumps(res), flush=True)


if __name__ == '__main__':
    main()
