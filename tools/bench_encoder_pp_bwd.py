"""Time the gradient of the ++ encoder (FusionTransformerv4) on one GPU, next to the byte floors of its new kernels.

    python tools/bench_encoder_pp_bwd.py [--batches 1 2] [--iters 20] [--warmup 3]

At config-4 shapes (image levels 6 x 112 x 200 and 6 x 56 x 100 of 256 channels, BEV maps of 180 x 180, hidden width
C = 128, two layers per modality with the polar block) and per batch size, CUDA events time (median of --iters calls)
  * di_msdeform_bwd_f32 of an image self attention (2 levels, every image pixel a query),
  * di_seq_attn_bwd_f32 of the polar block's cross attention (60 ray bins x 112 image rows per column),
  * di_polar_gather_bwd_f32 (the rays' gradient from the 180 x 180 BEV gradient),
  * the whole backward.encoder_pp_backward (eager forward with its intermediates, then the reverse walk),
  * one chained call: backward.decoder_pp_backward of the ++ decoder on the encoder's outputs, then
    encoder_pp_backward on its three gradients.
The kernels are printed with their byte floor at the data-sheet HBM bandwidth of the H100 SXM (3.35 TB/s; the
value-map and ray scatters count as a read and a write of their gradient maps).  The GPU name, power limit and maximum
SM clock come from nvidia-smi in the same run.  There is no CPU path.  The frame is built like bench.pp_host_frame
(copied here: bench.py stays as it is), with a 250k-point lidar cloud.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from tools.bench_decoder_layer_bwd import _time, gpu_info   # noqa: E402

HBM_BPS = 3.35e12          # H100 SXM data sheet
V, H0, W0, H1, W1, Y, X, C, R = 6, 112, 200, 56, 100, 180, 180, 128, 60


def host_frame(batch, seed, n_points=250000):
    """Config-4 inputs: image levels (B*6, 256, 112, 200), (B*6, 256, 56, 100); BEV maps [(B, 512, 180, 180),
    (B, 256, 180, 180), (B, 256, 180, 180)]; the base frame's cloud, pillars and camera rig (as bench.pp_host_frame)."""
    import torch
    from deepinteraction_b200 import synth
    fr = synth.make_frame_batch(seed, batch=batch, cloud='lidar', n_points=n_points, c_pts=256)
    g = torch.Generator().manual_seed(seed + 3)
    p1, p2 = fr['pts_feats'], torch.randn(batch, 256, 180, 180, generator=g)
    fr['img_levels'] = [fr['img_feats'], torch.randn(batch * 6, 256, 56, 100, generator=g)]
    fr['pts_levels'] = [torch.cat([p1, p2], 1), p1, p2]
    return fr


def encoder(d, seed=11):
    import torch
    from deepinteraction_b200 import mmri_pp
    from tools.make_goldens_pp import pp_layers, randomize_pp
    img_l, pts_l = pp_layers(True)
    torch.manual_seed(seed)
    enc = mmri_pp.FusionTransformerv4(2, 2, 256, 256, C, img_transformerlayers=img_l, pts_transformerlayers=pts_l)
    randomize_pp(enc, seed)
    return enc.to(d).eval()


def floors(B):
    """-> {kernel: bytes} from the shapes: inputs read once, outputs written once, scattered gradients read and written."""
    q, vals = B * V * H0 * W0, B * V * (H0 * W0 + H1 * W1) * C
    msda = 4 * (vals + 2 * vals + q * 192 + q * C + q * 192)              # values; d values (r+w); raw; dout; d raw
    mq, mk = B * V * R * W0, B * V * H0 * W0
    seq = 4 * (mq * C * 3 + mk * 2 * C + mq * C + mk * 2 * C)             # q, out, dout; k, v; dq; dk, dv
    rays = B * V * R * W0 * C
    gather = 4 * (B * Y * X * C + 2 * rays)
    return {'di_msdeform_bwd_f32': msda, 'di_seq_attn_bwd_f32': seq, 'di_polar_gather_bwd_f32': gather}


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split('\n')[0])
    ap.add_argument('--batches', type=int, nargs='+', default=[1, 2])
    ap.add_argument('--iters', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=3)
    a = ap.parse_args(argv)
    import torch
    from deepinteraction_b200 import backward, ops, synth
    from tools.bench_decoder_bwd import frame as dec_frame, train_decoder
    if not torch.cuda.is_available():
        raise SystemExit('no GPU: nothing is timed')
    d = torch.device('cuda:0')
    print(json.dumps(dict(gpu=gpu_info())))
    enc, dec = encoder(d), train_decoder(True)
    for B in a.batches:
        fr = host_frame(B, 100 + B)
        frd = synth.to_device(fr, d)
        il, pl = [t.to(d) for t in fr['img_levels']], [t.to(d) for t in fr['pts_levels']]
        metas, pm = frd['img_metas'], frd['pts_metas']
        g = torch.Generator().manual_seed(B)
        Gs = [torch.randn(s, generator=g).to(d) for s in ((B * V, H0, W0, C), (B, Y, X, C), (B, Y, X, C))]
        args = (enc, il, pl, metas, pm) + tuple(Gs)
        sv = {}
        with backward._precise():
            enc.pack()
            pillars, coors, npts, pts_list, consts = enc._frame(metas, pm, d)
            pmd = dict(pillars=pillars, pillar_coors=coors, pillars_num_points=npts, pts=pts_list)
            enc._schedule(il, pl, metas, pmd, [c.to(d) for c in consts] + [None], saved=sv)
        msda = sv['img'][0]['tape'][0][3]
        d_a = torch.randn(B * V * H0 * W0, C, generator=g).to(d)
        polar = next(s for op, i, _, s in sv['pts'][0]['tape'] if op == 'cross_attn' and 'rays' in s)
        kv, da2 = polar['kv'], torch.randn(polar['q2'].shape, generator=g).to(d)
        dq, dkv = torch.empty_like(polar['q2']), torch.empty_like(kv)
        BV = B * V
        gath = polar['gather']
        gts, gls = dec_frame(dec, B, g, d)[4:]

        def chained():
            img, pts_conv, pts = enc.forward_nhwc(il, pl, metas, pm)
            rd = backward.decoder_pp_backward(dec, pts_conv, pts, img, metas, gts, gls)
            backward.encoder_pp_backward(enc, il, pl, metas, pm, rd['d_img'], rd['d_pts_conv'], rd['d_new_pts'])
        times = {
            'di_msdeform_bwd_f32': lambda: ops.msdeform_bwd(msda['vals'], msda['raw'], d_a, BV, H0, W0),
            'di_seq_attn_bwd_f32': lambda: ops.seq_attn_bwd(polar['q2'], kv[:, :C], kv[:, C:], polar['a2'], da2, BV, W0, R,
                                                            H0, 8, dq, dkv[:, :C], dkv[:, C:]),
            'di_polar_gather_bwd_f32': lambda: ops.polar_gather_bwd(Gs[2], polar['rays_shape'], *gath),
            'encoder_pp_backward': lambda: backward.encoder_pp_backward(*args),
            'decoder_pp_backward+encoder_pp_backward': chained,
        }
        fl = floors(B)
        for name, fn in times.items():
            med, best = _time(fn, a.iters, a.warmup)
            row = dict(B=B, what=name, median_us=round(med, 1), min_us=round(best, 1))
            if name in fl:
                row.update(bytes=fl[name], floor_bytes_us=round(fl[name] / HBM_BPS * 1e6, 2))
            print(json.dumps(row), flush=True)


if __name__ == '__main__':
    main()
