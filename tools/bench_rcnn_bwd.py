"""Time the backward of the decoder's V1 RCNN blocks on one GPU, next to the floors of their kernels.

    python tools/bench_rcnn_bwd.py [--block point|image] [--batches 1 2] [--iters 20] [--warmup 5] [--floors-only]

At the base shapes (P = 200 queries, C = 128) and per batch size, CUDA events time, for --block point (the default;
decode_head[1], a PointRCNNBlock on the 180 x 180 BEV map)
  * di_roi_align_bwd_f32 (the RoIAlign gradient into the BEV map),
  * di_dynconv_bwd_f32 (the DynamicConv gradient, forward recomputed per query),
  * the whole backward.point_rcnn_backward (eager re-run of the block + every gradient product),
  * the forward block (mmpi.DeepInteractionDecoder._rcnn_block as the schedule runs it), for comparison;
and for --block image (decode_head[0], an ImageRCNNBlock on 6 x 112 x 200 image maps of a 6-camera rig, 448 x 800 inputs)
  * di_mha_small_bwd_f32 with the block's view-group masks,
  * di_roi_align_bwd_f32 into the B * 6 image maps at scale 1/4,
  * the whole backward.image_rcnn_backward and the forward block.
The RoIAlign and DynamicConv gradients are printed with two floors computed from the shapes: their bytes at the data-sheet
HBM bandwidth of the H100 SXM (3.35 TB/s) and their fp32 FLOPs at the data-sheet dense FP32 rate (67 TFLOP/s); the larger
floor bounds the kernel.  The RoI rows come from prediction rows with boxes of 0.4 - 4.5 m (doubled in BEV mode, as the
block does) spread over the map.  The GPU name, power limit and maximum SM clock come from nvidia-smi in the same run.
There is no CPU path: without a GPU the script fails (after printing the floors with --floors-only).
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from tools.bench_decoder_layer_bwd import _decoder, _time, gpu_info   # noqa: E402

HBM_BPS = 3.35e12          # H100 SXM data sheet
FP32_FLOPS = 67e12         # H100 SXM data sheet, dense FP32 (FFMA)
P, Y, X, C = 200, 180, 180, 128
V, IMG_IN, IMG_HW = 6, (448, 800), (112, 200)
LI = {'point': 1, 'image': 0}      # decode_head[1]: the first PointRCNNBlock, decode_head[0]: the first ImageRCNNBlock


def floors(B, block='point'):
    """-> dict of (bytes, flops, floor_bytes_us, floor_flops_us) per kernel, from the shapes only."""
    n = B * P
    map_px = B * (V * IMG_HW[0] * IMG_HW[1] if block == 'image' else Y * X)
    roi_bytes = 4 * (n * 49 * C + map_px * C + n * 5)             # d_out read, d_maps written, RoI rows
    roi_flops = 2 * 4 * 4 * 49 * C * n                             # 4 samples x 4 taps per bin, one FMA per channel
    dyn_bytes = 4 * (3 * n * 49 * C + 2 * n * 2 * C * C + n * 4 * C)   # roi, d_out, d_roi; params, d_params; partials
    dyn_flops = 6 * 2 * n * 49 * C * C                             # 2 products recomputed, 4 gradient products
    out = {}
    kernels = [('roi_align_bwd', roi_bytes, roi_flops)] + ([('dynconv_bwd', dyn_bytes, dyn_flops)] if block == 'point' else [])
    for name, nbytes, flops in kernels:
        out[name] = dict(bytes=nbytes, flops=flops, floor_bytes_us=nbytes / HBM_BPS * 1e6, floor_flops_us=flops / FP32_FLOPS * 1e6)
    return out


def image_inputs(m, B, g, d):
    """-> (image maps [B*V, 112, 200, C], the camera metadata of synth.camera_rig(6, (448, 800)), prediction rows whose
    centres spread over the BEV map at heights of -1.5 - 0.5 m), drawn with the CPU generator g."""
    import numpy as np
    import torch
    from deepinteraction_b200 import synth
    n = B * P
    rig = synth.camera_rig(V, IMG_IN)
    metas = [dict(lidar2img=[r.astype(np.float32) for r in rig], input_shape=IMG_IN, img_shape=[(*IMG_IN, 3)] * V)
             for _ in range(B)]
    pred = torch.randn(n, m.NP, generator=g)
    pred[:, 0] = torch.rand(n, generator=g) * X
    pred[:, 1] = torch.rand(n, generator=g) * Y
    pred[:, 2] = torch.rand(n, generator=g) * 2 - 1.5
    pred[:, 3:6] = torch.rand(n, 3, generator=g) * 2.5 - 1.0
    img = torch.randn(B * V, *IMG_HW, C, generator=g)
    return img.to(d), metas, pred.to(d)


def run_image(B, iters, warmup):
    import torch
    from deepinteraction_b200 import backward, ops
    d = torch.device('cuda')
    g = torch.Generator().manual_seed(B)
    m = _decoder()
    bp = m.pack()['blocks'][LI['image']]
    n = B * P
    img, metas, pred = image_inputs(m, B, g, d)
    query, grad = (torch.randn(n, C, generator=g).to(d) for _ in range(2))
    sv = {}
    with backward._precise():
        backward._rcnn_forward(m, bp, query, pred, img, metas, B, P, saved=sv)
    qkv, da = sv['qkv'], torch.randn(n, C, generator=g).to(d)
    d_roi = torch.randn(n, 49, C, generator=g).to(d)
    res = {}
    res['mha_small_bwd_masked'] = _time(lambda: ops.mha_small_bwd(qkv[:, :C], qkv[:, C:2 * C], qkv[:, 2 * C:], da, B, P,
                                                                  m.num_heads, sv['onbits'], sv['win']), iters, warmup)
    res['roi_align_bwd'] = _time(lambda: ops.roi_align_bwd(d_roi, sv['rois'], B * V, *IMG_HW, 1.0 / m.out_size_factor_img),
                                 iters, warmup)
    res['image_rcnn_backward'] = _time(lambda: backward.image_rcnn_backward(m, LI['image'], query, pred, img, metas, grad),
                                       iters, warmup)

    def fwd():
        with backward._precise():                    # the schedule's precision: 3xTF32 products
            backward._rcnn_forward(m, bp, query, pred, img, metas, B, P)
    res['forward_block'] = _time(fwd, iters, warmup)
    live = sv['win'] >= 0
    print('B=%d view groups: %d of %d queries on a live view' % (B, int(live.sum()), n))
    return res


def run(B, iters, warmup):
    import torch
    from deepinteraction_b200 import backward, ops
    d = torch.device('cuda')
    g = torch.Generator(device=d).manual_seed(B)
    m = _decoder()
    li = LI['point']
    bp = m.pack()['blocks'][li]
    n = B * P
    pred = torch.randn(n, m.NP, device=d, generator=g)
    pred[:, 0] = torch.rand(n, device=d, generator=g) * X
    pred[:, 1] = torch.rand(n, device=d, generator=g) * Y
    pred[:, 3:6] = torch.rand(n, 3, device=d, generator=g) * 2.5 - 1.0
    query = torch.randn(n, C, device=d, generator=g)
    bev = torch.randn(B, Y, X, C, device=d, generator=g)
    grad = torch.randn(n, C, device=d, generator=g)
    prm = backward._bev_roi_params(m)
    rois = ops.rcnn_rois(pred, B, P, m.num_views, 1, prm)[0]
    d_roi = torch.randn(n, 49, C, device=d, generator=g)
    roi = ops.roi_align(bev, rois, 1.0)
    params = torch.randn(n, 2 * C * C, device=d, generator=g) / 11
    d_flat = torch.randn(n, 49 * C, device=d, generator=g)
    res = {}
    res['roi_align_bwd'] = _time(lambda: ops.roi_align_bwd(d_roi, rois, B, Y, X, 1.0), iters, warmup)
    res['dynconv_bwd'] = _time(lambda: ops.dynconv_bwd(roi, params, *bp['dn1'], *bp['dn2'], d_flat), iters, warmup)
    res['point_rcnn_backward'] = _time(lambda: backward.point_rcnn_backward(m, li, query, pred, bev, grad), iters, warmup)

    def fwd():
        with backward._precise():                    # the schedule's precision: 3xTF32 products
            m._rcnn_block(bp, query, pred, bev, None, B, P, prm, None, None)
    res['forward_block'] = _time(fwd, iters, warmup)
    return res


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split('\n')[0])
    ap.add_argument('--block', choices=['point', 'image'], default='point')
    ap.add_argument('--batches', type=int, nargs='+', default=[1, 2])
    ap.add_argument('--iters', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=5)
    ap.add_argument('--floors-only', action='store_true', help='print the floors and stop before touching the GPU')
    a = ap.parse_args(argv)
    fl = {B: floors(B, a.block) for B in a.batches}
    for B in a.batches:
        for name, f in fl[B].items():
            print('B=%d %-14s floors: bytes %.1f MB -> %.1f us, fp32 %.2f GFLOP -> %.1f us (bound: %s)' % (
                B, name, f['bytes'] / 1e6, f['floor_bytes_us'], f['flops'] / 1e9, f['floor_flops_us'],
                'bytes' if f['floor_bytes_us'] >= f['floor_flops_us'] else 'FLOPs'))
    if a.floors_only:
        return 0
    import torch
    if not torch.cuda.is_available():
        raise RuntimeError('bench_rcnn_bwd: no CUDA device (the kernels have no CPU path)')
    print('GPU (name, power limit, max SM clock):', gpu_info())
    for B in a.batches:
        res = (run_image if a.block == 'image' else run)(B, a.iters, a.warmup)
        for name, (med, best) in res.items():
            f = fl[B].get(name)
            extra = ''
            if f is not None:
                floor = max(f['floor_bytes_us'], f['floor_flops_us'])
                extra = ' | floor %.1f us (%s), %.0f%% of it' % (floor, 'bytes' if f['floor_bytes_us'] >= f['floor_flops_us'] else 'FLOPs',
                                                              100.0 * floor / med)
            print('B=%d %-22s median %8.1f us  best %8.1f us%s' % (B, name, med, best, extra))
        print(json.dumps(dict(B=B, **{k: v[0] for k, v in res.items()})))
    return 0


if __name__ == '__main__':
    sys.exit(main())
