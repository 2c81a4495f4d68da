"""Time the backward of the decoder's query x BEV transformer layer on one GPU, next to its floors.

    python tools/bench_decoder_layer_bwd.py [--batches 1 2] [--iters 20] [--warmup 5] [--floors-only]

At the base shapes (P = 200 queries, 180 x 180 BEV, C = 128, 8 heads of 16) and per batch size, CUDA events time
  * the attention-gradient kernel alone (di_xattn_bwd_f32: dO split, key-split kernel, dQ merge),
  * di_xattn_tc_lse_f32 next to di_xattn_tc_f32 (the forward with and without the row log-sum-exp),
  * the whole backward.decoder_layer_backward (eager re-run of the layer + every gradient product).
Each time is printed with two floors computed from the shapes: bytes of the gradient kernel at the data-sheet HBM bandwidth
of the H100 SXM (3.35 TB/s), and its MMA FLOPs (18 one-term bf16 products, xattn_bwd.cu) at the data-sheet dense bf16
rate (989 TFLOP/s); the larger floor is the one that bounds the kernel.  The floors of the forward entries use the same
rule (K and V planes read; 6 + 3 one-term products).  The GPU name, power limit and maximum SM clock come from nvidia-smi
in the same run.  There is no CPU path: without a GPU the script fails (after printing the floors with --floors-only).
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

HBM_BPS = 3.35e12          # H100 SXM data sheet
BF16_FLOPS = 989e12        # H100 SXM data sheet, dense
P, HW, C, HEADS = 200, 180 * 180, 128, 8
BWD_TERMS = 18             # S 6, dA 3, dV 3, dK 3, dQ 3 (xattn_bwd.cu)
FWD_TERMS = 9              # S 6, P V 3 (xattn_tc.cu)


def floors(B):
    """-> dict of (bytes, flops, floor_bytes_us, floor_flops_us) per timed item, from the shapes only."""
    one = 2.0 * P * HW * C                           # one contraction, one term, per sample (1.66 GFLOP)
    kplanes, vplanes = HW * 192 * 4, HW * 128 * 4     # bf16 hi | mid | lo and hi | mid planes
    bwd_bytes = B * (kplanes + vplanes + 2 * HW * C * 4)       # K, V planes read; dK, dV (fp32) written
    fwd_bytes = B * (kplanes + vplanes)
    out = {}
    for name, nbytes, flops in (('xattn_bwd', bwd_bytes, B * BWD_TERMS * one), ('xattn_tc_f32', fwd_bytes, B * FWD_TERMS * one),
                                ('xattn_tc_lse_f32', fwd_bytes, B * FWD_TERMS * one)):
        out[name] = dict(bytes=nbytes, flops=flops, floor_bytes_us=nbytes / HBM_BPS * 1e6, floor_flops_us=flops / BF16_FLOPS * 1e6)
    return out


def gpu_info():
    r = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True)
    return r.stdout.strip() if r.returncode == 0 else 'nvidia-smi failed: ' + r.stderr.strip()


def _time(fn, iters, warmup):
    import torch
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    times = []
    for _ in range(iters):
        e0.record()
        fn()
        e1.record()
        e1.synchronize()
        times.append(e0.elapsed_time(e1) * 1e3)
    times.sort()
    return times[len(times) // 2], times[0]


def _decoder(plusplus=False):
    import torch
    from deepinteraction_b200 import mmpi, synth
    test_cfg = dict(dataset='nuScenes', grid_size=[1440, 1440, 40], out_size_factor=8, pc_range=[-54.0, -54.0],
                    voxel_size=[0.075, 0.075], nms_type=None)
    coder = dict(type='TransFusionBBoxCoder', pc_range=[-54.0, -54.0], voxel_size=[0.075, 0.075], out_size_factor=8,
                 post_center_range=[-61.2, -61.2, -10.0, 61.2, 61.2, 10.0], score_threshold=0.0, code_size=10)
    torch.manual_seed(0)
    cls = mmpi.DeepInteractionPlusPlusDecoder if plusplus else mmpi.DeepInteractionDecoder
    m = cls(num_views=6, num_proposals=P, hidden_channel=C, num_classes=10, num_heads=HEADS,
                                    initialize_by_heatmap=True, nms_kernel_size=3, ffn_channel=256,
                                    common_heads=dict(center=(2, 2), height=(1, 2), dim=(3, 2), rot=(2, 2), vel=(2, 2)),
                                    loss_cls=dict(type='FocalLoss', use_sigmoid=True, gamma=2, alpha=0.25, reduction='mean'),
                                    bbox_coder=coder, test_cfg=test_cfg)
    synth.randomize_norm_stats(m, 0)
    return m.cuda().eval()


def run(B, iters, warmup):
    import torch
    from deepinteraction_b200 import backward, ops
    d = torch.device('cuda')
    g = torch.Generator(device=d).manual_seed(B)
    q = torch.randn(B * P, C, device=d, generator=g) * 0.05
    kv = torch.randn(B * HW, 2 * C, device=d, generator=g)
    dout = torch.randn(B * P, C, device=d, generator=g)
    out, lse, planes = ops.xattn_tc_lse(q, kv, B, P, HW, HEADS)
    res = {}
    res['xattn_bwd'] = _time(lambda: ops.xattn_bwd(planes, out, lse, dout, B, P, HW, HEADS), iters, warmup)
    res['xattn_tc_f32'] = _time(lambda: ops.xattn_tc(q, kv, B, P, HW, HEADS), iters, warmup)
    res['xattn_tc_lse_f32'] = _time(lambda: ops.xattn_tc_lse(q, kv, B, P, HW, HEADS), iters, warmup)
    m = _decoder()
    bev = torch.randn(B, 180, 180, C, device=d, generator=g)
    query = torch.randn(B * P, C, device=d, generator=g)
    pix = torch.randint(0, HW, (B * P,), device=d, generator=g)
    qpos = torch.stack([(pix % 180).float() + 0.5, (pix // 180).float() + 0.5], 1)
    res['decoder_layer_backward'] = _time(lambda: backward.decoder_layer_backward(m, query, qpos, bev, dout), iters, warmup)
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
            print('B=%d %-18s floors: bytes %.1f MB -> %.1f us, MMA %.1f GFLOP -> %.1f us (bound: %s)' % (
                B, name, f['bytes'] / 1e6, f['floor_bytes_us'], f['flops'] / 1e9, f['floor_flops_us'],
                'bytes' if f['floor_bytes_us'] >= f['floor_flops_us'] else 'MMA'))
    if a.floors_only:
        return 0
    import torch
    if not torch.cuda.is_available():
        raise RuntimeError('bench_decoder_layer_bwd: no CUDA device (the kernels have no CPU path)')
    print('GPU (name, power limit, max SM clock):', gpu_info())
    for B in a.batches:
        res = run(B, a.iters, a.warmup)
        for name, (med, best) in res.items():
            f = fl[B].get(name)
            extra = ''
            if f is not None:
                floor = max(f['floor_bytes_us'], f['floor_flops_us'])
                extra = ' | floor %.1f us (%s), %.0f%% of it' % (floor, 'bytes' if f['floor_bytes_us'] >= f['floor_flops_us'] else 'MMA',
                                                              100.0 * floor / med)
            print('B=%d %-24s median %8.1f us  best %8.1f us%s' % (B, name, med, best, extra))
        print(json.dumps(dict(B=B, **{k: v[0] for k, v in res.items()})))
    return 0


if __name__ == '__main__':
    sys.exit(main())
