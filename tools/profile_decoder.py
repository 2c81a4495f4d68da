#!/usr/bin/env python
"""Per-launch timing of ONE decoder forward at the base shapes (180x180 BEV, 6 x 112x200 image maps, 200 queries):
the launch sequence with CUDA-event times (eager), and the time of the whole decoder replayed from its CUDA graph.

    python tools/profile_decoder.py [--plusplus] [--batch 1]        (needs an H100)
"""
import argparse
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--plusplus', action='store_true')
    ap.add_argument('--batch', type=int, default=1)
    ap.add_argument('--iters', type=int, default=20)
    args = ap.parse_args()
    import projects.mmdet3d_plugin  # noqa: F401
    from projects.mmdet3d_plugin.registry import load_config, build_hot_path
    from deepinteraction_b200 import ops, synth, graph as di_graph
    torch.set_grad_enabled(False)
    dev = torch.device('cuda:0')
    cfg = load_config(os.path.join(ROOT, 'projects', 'configs', 'nuscenes',
                                   'di_b200_plusplus_hotpath.py' if args.plusplus else 'di_b200_base_hotpath.py'))
    torch.manual_seed(0)
    _, head = build_hot_path(cfg)
    synth.randomize_norm_stats(head, 0)
    head = head.to(dev).eval()
    B = args.batch
    g = torch.Generator().manual_seed(0)
    rig = synth.camera_rig(6, (448, 800))
    metas = [dict(lidar2img=[r.astype(np.float32) for r in rig], input_shape=(448, 800), img_shape=[(448, 800, 3)] * 6)] * B
    pts = [torch.randn(B, 180, 180, 128, generator=g).to(dev) for _ in range(2)]
    img = torch.randn(6 * B, 112, 200, 128, generator=g).to(dev)
    flush = torch.empty(256 * 1024 * 1024 // 4, device=dev)
    fwd = lambda: head.forward_nhwc(pts[0], pts[1], img, metas)
    for _ in range(3):
        fwd()
    torch.cuda.synchronize()
    tot = 0.0
    for _ in range(args.iters):
        flush.zero_()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fwd()
        b.record()
        torch.cuda.synchronize()
        tot += a.elapsed_time(b)
    print('decoder, CUDA-graph replay: %.1f us per forward (batch %d)' % (tot / args.iters * 1e3, B))
    di_graph.ENABLED[0] = False
    head._graphs.clear()
    fwd()
    seqs = []
    ops.PROFILE_FLUSH[0] = flush          # every launch from a cold L2 with the queue kept full (like an ncu launch list)
    for _ in range(args.iters):
        ops.PROFILE[0] = []
        fwd()
        torch.cuda.synchronize()
        seqs.append([(n, a.elapsed_time(b), mod) for n, a, b, nb, fl, mod in ops.PROFILE[0]])
    ops.PROFILE[0] = None
    n = len(seqs[0])
    assert all(len(s) == n for s in seqs)
    total = 0.0
    for i in range(n):
        us = float(np.median([s[i][1] for s in seqs])) * 1e3
        total += us
        mod = seqs[0][i][2]
        print('%3d %-34s %8.1f us   %s' % (i, seqs[0][i][0], us, mod[0] if isinstance(mod, tuple) else mod))
    print('sum of kernel times: %.1f us over %d launches' % (total, n))


if __name__ == '__main__':
    main()
