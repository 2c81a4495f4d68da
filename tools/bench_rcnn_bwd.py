"""Time the backward of the decoder's PointRCNNBlock on one GPU, next to the floors of its two new kernels.

    python tools/bench_rcnn_bwd.py [--batches 1 2] [--iters 20] [--warmup 5] [--floors-only]

At the base shapes (P = 200 queries, 180 x 180 BEV, C = 128) and per batch size, CUDA events time
  * di_roi_align_bwd_f32 (the RoIAlign gradient into the BEV map),
  * di_dynconv_bwd_f32 (the DynamicConv gradient, forward recomputed per query),
  * the whole backward.point_rcnn_backward (eager re-run of the block + every gradient product),
  * the forward block (mmpi.DeepInteractionDecoder._rcnn_block as the schedule runs it), for comparison.
The two kernels are printed with two floors computed from the shapes: their bytes at the data-sheet HBM bandwidth of the
H100 SXM (3.35 TB/s) and their fp32 FLOPs at the data-sheet dense FP32 rate (67 TFLOP/s); the larger floor bounds the
kernel.  The RoI rows come from prediction rows with boxes of 0.4 - 4.5 m (doubled in BEV mode, as the block does) spread
over the map.  The GPU name, power limit and maximum SM clock come from nvidia-smi in the same run.  There is no CPU path:
without a GPU the script fails (after printing the floors with --floors-only).
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
LI = 1                     # decode_head[1]: the first PointRCNNBlock


def floors(B):
    """-> dict of (bytes, flops, floor_bytes_us, floor_flops_us) per kernel, from the shapes only."""
    n = B * P
    roi_bytes = 4 * (n * 49 * C + B * Y * X * C + n * 5)          # d_out read, d_maps written, RoI rows
    roi_flops = 2 * 4 * 4 * 49 * C * n                             # 4 samples x 4 taps per bin, one FMA per channel
    dyn_bytes = 4 * (3 * n * 49 * C + 2 * n * 2 * C * C + n * 4 * C)   # roi, d_out, d_roi; params, d_params; partials
    dyn_flops = 6 * 2 * n * 49 * C * C                             # 2 products recomputed, 4 gradient products
    out = {}
    for name, nbytes, flops in (('roi_align_bwd', roi_bytes, roi_flops), ('dynconv_bwd', dyn_bytes, dyn_flops)):
        out[name] = dict(bytes=nbytes, flops=flops, floor_bytes_us=nbytes / HBM_BPS * 1e6, floor_flops_us=flops / FP32_FLOPS * 1e6)
    return out


def run(B, iters, warmup):
    import torch
    from deepinteraction_b200 import backward, ops
    d = torch.device('cuda')
    g = torch.Generator(device=d).manual_seed(B)
    m = _decoder()
    bp = m.pack()['blocks'][LI]
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
    res['point_rcnn_backward'] = _time(lambda: backward.point_rcnn_backward(m, LI, query, pred, bev, grad), iters, warmup)

    def fwd():
        with backward._precise():                    # the schedule's precision: 3xTF32 products
            m._rcnn_block(bp, query, pred, bev, None, B, P, prm, None, None)
    res['forward_block'] = _time(fwd, iters, warmup)
    return res


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split('\n')[0])
    ap.add_argument('--batches', type=int, nargs='+', default=[1, 2])
    ap.add_argument('--iters', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=5)
    ap.add_argument('--floors-only', action='store_true', help='print the floors and stop before touching the GPU')
    a = ap.parse_args(argv)
    fl = {B: floors(B) for B in a.batches}
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
        res = run(B, a.iters, a.warmup)
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
