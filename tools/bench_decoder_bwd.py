"""Time the gradient of the base decoder's losses on one GPU, next to the byte floors of its two new kernels.

    python tools/bench_decoder_bwd.py [--batches 1 2] [--iters 20] [--warmup 5] [--floors-only] [--plusplus]

At the base shapes (P = 200 proposals, C = 128, 180 x 180 BEV maps, 6 x 112 x 200 image maps of a 6-camera rig, K = 10
classes, 4 MMPI layers) and per batch size, CUDA events time
  * di_mmpi_losses_bwd_f32 (the loss gradient: dense heat-map logits and prediction rows),
  * di_query_init_bwd_f32 (the top-k gather and class-encoding gradient),
  * backward.pred_head_backward of pred_head[0] (input [q | prev], 2C),
  * backward.heatmap_head_backward (two 3x3 convolutions on the 180 x 180 map),
  * the whole backward.decoder_backward (eager forward, loss, loss gradient and every block backward).
With --plusplus the ++ decoder (V2 RCNN blocks) at the same shapes is timed instead: di_pred_finish_pp_bwd_f32 (the
look-forward centre and fallback gradient), backward.pred_head_backward of pred_head[0] (input q, C) and the whole
backward.decoder_pp_backward.  The two kernels are printed with their byte floor at the data-sheet HBM bandwidth of the H100 SXM (3.35 TB/s).  The GPU
name, power limit and maximum SM clock come from nvidia-smi in the same run.  There is no CPU path: without a GPU the
script fails (after printing the floors with --floors-only).
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
P, Y, X, C, K, L, CODE = 200, 180, 180, 128, 10, 4, 10


def floors(B):
    """-> dict of (bytes, floor_us) per kernel, from the shapes only."""
    from deepinteraction_b200.loss import losses_bwd_bytes
    qi = 4 * (3 * B * P * C + K * C)          # d q0 read twice (gather, class sums), the selected rows read and written
    out = {}
    for name, nb in (('di_mmpi_losses_bwd_f32', losses_bwd_bytes(B, K, Y * X, L, P, CODE)), ('di_query_init_bwd_f32', qi)):
        out[name] = (nb, nb / HBM_BPS * 1e6)
    return out


def train_decoder(plusplus=False):
    """The base-shape decoder (plusplus: the ++ decoder) of tools/bench_decoder_layer_bwd.py with the reference's training
    configuration (Hungarian assignment, L1 loss weight 0.25)."""
    from deepinteraction_b200 import loss as Lm
    from tools import make_goldens as mg
    m = _decoder(plusplus)
    tc = dict(mg.DEC_TRAIN_CFG, grid_size=[1440, 1440, 40], voxel_size=[0.075, 0.075, 0.2])
    m.train_cfg = tc
    m.bbox_assigner = Lm._build(Lm.ASSIGNERS, tc['assigner'])
    m._loss_cfg['bbox'] = dict(mg.DEC_LOSSES['loss_bbox'])
    return m


def frame(m, B, g, d):
    """Encoder outputs, camera metadata and ground truth (30 boxes per sample, on the device) of one batch."""
    import torch
    from tools.bench_rcnn_bwd import image_inputs
    img, metas, _ = image_inputs(m, B, g, d)
    pts, new_pts = (torch.randn(B, Y, X, C, generator=g).to(d) for _ in range(2))
    gts, gls = [], []
    for _ in range(B):
        n = 30
        xy = torch.rand(n, 2, generator=g) * 80 - 40
        dims = torch.stack([torch.rand(n, generator=g) * 2 + 1, torch.rand(n, generator=g) * 4 + 2,
                            torch.rand(n, generator=g) + 1.2], 1)
        box = torch.cat([xy, torch.rand(n, 1, generator=g) * 2 - 2.5, dims, torch.rand(n, 1, generator=g) * 6.2 - 3.1,
                         torch.randn(n, 2, generator=g)], 1)
        gts.append(box.to(d))
        gls.append(torch.randint(0, K, (n,), generator=g).to(d))
    return pts, new_pts, img, metas, gts, gls


def plusplus_times(m, args, B, d):
    """{name: callable} of the ++ decoder's backward pieces at batch B."""
    import torch
    from deepinteraction_b200 import backward, ops
    backward.decoder_pp_backward(m, *args)                    # builds the per-pack tensors; leaves the loss targets
    _, d_pred = m.loss_backward()
    keep = torch.randint(0, 2, (L, B * P), device=d, dtype=torch.int32)
    q = torch.randn(B * P, C, device=d)
    return {
        'di_pred_finish_pp_bwd_f32': lambda: ops.pred_finish_pp_bwd(d_pred, keep),
        'pred_head_backward[0]': lambda: backward.pred_head_backward(m, 0, [q], d_pred[0]),
        'decoder_pp_backward': lambda: backward.decoder_pp_backward(m, *args),
    }


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split('\n')[0])
    ap.add_argument('--batches', type=int, nargs='+', default=[1, 2])
    ap.add_argument('--iters', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=5)
    ap.add_argument('--floors-only', action='store_true')
    ap.add_argument('--plusplus', action='store_true', help='time the ++ decoder\'s backward (decoder_pp_backward)')
    a = ap.parse_args(argv)
    for B in a.batches:
        for name, (nb, us) in floors(B).items():
            print(json.dumps(dict(B=B, kernel=name, bytes=nb, floor_bytes_us=round(us, 2))))
    if a.floors_only:
        return
    import torch
    from deepinteraction_b200 import backward, ops
    if not torch.cuda.is_available():
        raise SystemExit('no GPU: nothing is timed')
    d = torch.device('cuda:0')
    print(json.dumps(dict(gpu=gpu_info())))
    m = train_decoder(a.plusplus)
    for B in a.batches:
        g = torch.Generator().manual_seed(B)
        args = frame(m, B, g, d)
        pts, new_pts, img, metas, gts, gls = args
        if a.plusplus:
            times = plusplus_times(m, args, B, d)
            for name, fn in times.items():
                med, best = _time(fn, a.iters, a.warmup)
                print(json.dumps(dict(B=B, what=name, median_us=round(med, 1), min_us=round(best, 1))))
            continue
        r = backward.decoder_backward(m, *args)                 # builds the per-pack tensors; leaves the loss targets
        d_heat, d_pred = m.loss_backward()
        sv = {}
        with backward._precise():
            proj, aux = (t.to(d) for t in m._camera_consts(metas))
            out = m._schedule(pts, new_pts, img, (448, 800), proj, aux, sv)
        dq = torch.randn(B * P, C, generator=g).to(d)
        q = [sv['layer_query'][0], sv['query_feat1']]
        times = {
            'di_mmpi_losses_bwd_f32': lambda: m.loss_backward(),
            'di_query_init_bwd_f32': lambda: ops.query_init_bwd(dq, sv['top'], out['labels'], r['d_pts_conv'].view(B, -1, C), K),
            'pred_head_backward[0]': lambda: backward.pred_head_backward(m, 0, q, d_pred[0]),
            'heatmap_head_backward': lambda: backward.heatmap_head_backward(m, new_pts, d_heat),
            'decoder_backward': lambda: backward.decoder_backward(m, *args),
        }
        fl = floors(B)
        for name, fn in times.items():
            med, best = _time(fn, a.iters, a.warmup)
            row = dict(B=B, what=name, median_us=round(med, 1), min_us=round(best, 1))
            if name in fl:
                row['floor_bytes_us'] = round(fl[name][1], 2)
            print(json.dumps(row))


if __name__ == '__main__':
    main()
