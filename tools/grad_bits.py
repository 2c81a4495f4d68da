#!/usr/bin/env python
"""Fingerprint every gradient that backward.py and train.py compose, to compare two versions of them on one GPU.

    python tools/grad_bits.py --out DIR                          # writes DIR/hashes.json and DIR/encoder.pt
    python tools/grad_bits.py --compare DIR_A DIR_B [--spread DIR_A2]

From fixed seeds: lcab_backward (self and cross attention), LCABTrain forward + backward, decoder_layer_backward,
point_rcnn_backward, image_rcnn_backward and decoder_backward (base shapes, batch 2) run on deterministic kernels, so the SHA-256 of every
tensor they return is written and --compare asks the two runs to agree on every hash both have (a version without one of
the functions is compared on the others).  encoder_backward, encoder_train_step and encoder_pp_backward pass through
di_i2p_attend_bwd_f32 and di_bev_sample_bwd_f32 (the last also through the value and ray scatters of
di_msdeform_bwd_f32 and di_polar_gather_bwd_f32), which accumulate with atomicAdd and differ in the last bits from run to
run; their tensors are written as they are, and --compare reports per pair the largest max|a - b| / max|a| over the
tensors.  With --spread (a second run of version A) the A-B figure has to stay within twice the A-A2 figure.  The
train-mode gradients of the out_proj BatchNorm biases are left out of that figure: they are analytically zero (the next
layer's batch-mean subtraction cancels a per-channel constant), so what is computed is rounding noise without a scale.
"""
import argparse
import hashlib
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def flatten(x, prefix=''):
    """Nested dict / list / tuple of tensors -> {path: tensor} (None entries are kept as None)."""
    if torch.is_tensor(x) or x is None:
        return {prefix: x}
    items = x.items() if isinstance(x, dict) else enumerate(x)
    out = {}
    for k, v in items:
        out.update(flatten(v, f'{prefix}.{k}' if prefix else str(k)))
    return out


def sha(t):
    return None if t is None else hashlib.sha256(t.detach().contiguous().cpu().numpy().tobytes()).hexdigest()


def lcab_cases(d):
    from deepinteraction_b200 import backward, mmri, synth, train
    C, N, H, W = 128, 2, 12, 20
    for self_attn in (True, False):
        torch.manual_seed(31)
        blk = mmri.LocalContextAttentionBlock(C, C, 9)
        synth.randomize_norm_stats(blk, 31)
        blk = blk.to(d)
        g = torch.Generator().manual_seed(31)
        t, s, G = (torch.randn(N * H * W, C, generator=g).to(d) for _ in range(3))
        s = t if self_attn else s
        name = 'self' if self_attn else 'cross'
        yield 'lcab_backward.' + name, backward.lcab_backward(mmri._pack_lcab(blk.eval(), d), t, s, N, H, W, G)
        lt, grads = train.LCABTrain(blk.train()), {}
        with backward._precise(), torch.no_grad():
            out = lt.forward(t, s, N, H, W)
            d_t, d_s = lt.backward(G, grads)
        names = {id(p): n for n, p in blk.named_parameters()}
        yield 'lcab_train.' + name, dict(out=out, d_t=d_t, d_s=d_s, grads={names[k]: v for k, v in grads.items()})


def decoder_cases(d):
    from deepinteraction_b200 import backward
    from tools.bench_decoder_layer_bwd import _decoder, P, C
    m, B, Y, X = _decoder(), 2, 180, 180
    g = torch.Generator().manual_seed(7)
    query, grad = (torch.randn(B * P, C, generator=g).to(d) for _ in range(2))
    bev = torch.randn(B, Y, X, C, generator=g).to(d)
    pix = torch.randint(0, Y * X, (B * P,), generator=g)
    qpos = torch.stack([(pix % X).float() + 0.5, (pix // X).float() + 0.5], 1).to(d)
    yield 'decoder_layer_backward', backward.decoder_layer_backward(m, query, qpos, bev, grad)
    pred = torch.randn(B * P, m.NP, generator=g)
    pred[:, 0] = torch.rand(B * P, generator=g) * X
    pred[:, 1] = torch.rand(B * P, generator=g) * Y
    pred[:, 3:6] = torch.rand(B * P, 3, generator=g) * 2.5 - 1.0
    for li in (1, 3):
        yield f'point_rcnn_backward.{li}', backward.point_rcnn_backward(m, li, query, pred.to(d), bev, grad)
    if hasattr(backward, 'image_rcnn_backward'):
        from tools.bench_rcnn_bwd import image_inputs
        img, metas, pred_img = image_inputs(m, B, g, d)
        for li in (0, 2):
            yield f'image_rcnn_backward.{li}', backward.image_rcnn_backward(m, li, query, pred_img, img, metas, grad)
    if hasattr(backward, 'decoder_backward'):
        from tools.bench_decoder_bwd import frame, train_decoder
        mt = train_decoder()
        r = backward.decoder_backward(mt, *frame(mt, B, g, d))
        yield 'decoder_backward', {k: v for k, v in r.items() if k != 'losses'}


def encoder_cases(d):
    from deepinteraction_b200 import backward, mmri, synth, train
    from tools.make_goldens import small_frame
    fr = small_frame(1560, aug=True, views=2, c_img=64, c_pts=64, bev=36, batch=1)
    pm = {k: (v.to(d) if torch.is_tensor(v) else [p.to(d) for p in v]) for k, v in fr['pts_metas'].items()}
    g = torch.Generator().manual_seed(1560)
    Gs = [torch.randn(s, generator=g).to(d) for s in ((2, 28, 50, 128), (1, 36, 36, 128), (1, 36, 36, 128))]
    for mode in ('eval', 'train'):
        torch.manual_seed(1560)
        enc = mmri.DeepInteractionEncoder(2, 64, 64, 128)
        synth.randomize_norm_stats(enc, 1560)
        enc = enc.to(d).train(mode == 'train')
        args = (enc, fr['img_feats'].to(d), fr['pts_feats'].to(d), fr['img_metas'], pm)
        if mode == 'eval':
            yield 'encoder_backward', backward.encoder_backward(*args, *Gs)
        else:
            yield 'encoder_train_step', train.encoder_train_step(*args, lambda a, b, c: tuple(Gs))
            yield 'encoder_train_step.dropout', train.encoder_train_step(*args, lambda a, b, c: tuple(Gs), dropout_seed=7)
    if hasattr(backward, 'encoder_pp_backward'):
        from deepinteraction_b200 import mmri_pp
        from tools.make_goldens_pp import pp_frame, pp_layers, randomize_pp
        img_l, pts_l = pp_layers(True)
        torch.manual_seed(2100)
        enc = mmri_pp.FusionTransformerv4(2, 2, 16, 24, 128, img_transformerlayers=img_l, pts_transformerlayers=pts_l)
        randomize_pp(enc, 2100)
        enc = enc.to(d).eval()
        fr = pp_frame(2100, True)
        pm = {k: (v.to(d) if torch.is_tensor(v) else [p.to(d) for p in v]) for k, v in fr['pts_metas'].items()}
        yield 'encoder_pp_backward', backward.encoder_pp_backward(enc, [t.to(d) for t in fr['img_levels']],
                                                                  [t.to(d) for t in fr['pts_levels']], fr['img_metas'], pm, *Gs)


def run(out_dir):
    d = torch.device('cuda:0')
    os.makedirs(out_dir, exist_ok=True)
    hashes, tensors = {}, {}
    for cases, keep in ((lcab_cases, False), (decoder_cases, False), (encoder_cases, True)):
        for name, res in cases(d):
            for k, t in flatten(res, name).items():
                hashes[k] = sha(t)
                if keep and t is not None:
                    tensors[k] = t.detach().cpu()
    with open(os.path.join(out_dir, 'hashes.json'), 'w') as f:
        json.dump(hashes, f, indent=0, sort_keys=True)
    torch.save(tensors, os.path.join(out_dir, 'encoder.pt'))
    print('%d tensors hashed, %d encoder tensors kept -> %s' % (len(hashes), len(tensors), out_dir))


def worst_diff(dir_a, dir_b):
    """-> (largest max|a - b| / max|a| over the encoder tensors, its name, number of tensors that differ in any bit)."""
    a, b = (torch.load(os.path.join(p, 'encoder.pt')) for p in (dir_a, dir_b))
    assert set(a) == set(b), sorted(set(a) ^ set(b))
    worst, differ = (0.0, None), 0
    for k in a:
        assert a[k].shape == b[k].shape, k
        if not torch.equal(a[k], b[k]) and not k.endswith('out_proj.bn.bias'):
            differ += 1
            scale = float(a[k].abs().max())
            worst = max(worst, (float((a[k] - b[k]).abs().max()) / scale if scale > 0 else float('inf'), k))
    return worst[0], worst[1], differ


def compare(dir_a, dir_b, dir_a2):
    ha, hb = (json.load(open(os.path.join(p, 'hashes.json'))) for p in (dir_a, dir_b))
    only = sorted(set(ha) ^ set(hb))
    exact = [k for k in ha if k in hb and not k.startswith('encoder_')]
    bad = [k for k in exact if ha[k] != hb[k]]
    print('deterministic results: %d tensors in both runs, %d with a different SHA-256; %d in one run only' % (
        len(exact), len(bad), len(only)))
    for k in bad:
        print('  differs:', k)
    e_ab, k_ab, n_ab = worst_diff(dir_a, dir_b)
    print('encoder results A vs B : %d tensors differ in some bit, worst %.2e (%s)' % (n_ab, e_ab, k_ab))
    ok = not bad
    if dir_a2 is not None:
        e_aa, k_aa, n_aa = worst_diff(dir_a, dir_a2)
        print('encoder results A vs A2: %d tensors differ in some bit, worst %.2e (%s)' % (n_aa, e_aa, k_aa))
        ok = ok and e_ab <= 2 * e_aa
    print('OK' if ok else 'MISMATCH')
    return 0 if ok else 1


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split('\n')[0])
    ap.add_argument('--out', help='run on cuda:0 and write hashes.json and encoder.pt into this directory')
    ap.add_argument('--compare', nargs=2, metavar=('DIR_A', 'DIR_B'))
    ap.add_argument('--spread', metavar='DIR_A2', help='a second run of version A: the run-to-run spread of the encoder results')
    a = ap.parse_args(argv)
    if (a.out is None) == (a.compare is None):
        ap.error('give --out or --compare')
    if a.compare:
        return compare(*a.compare, a.spread)
    if not torch.cuda.is_available():
        raise RuntimeError('grad_bits: no CUDA device (the kernels have no CPU path)')
    run(a.out)
    return 0


if __name__ == '__main__':
    sys.exit(main())
