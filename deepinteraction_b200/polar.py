"""MMRI_I2P_Polar of the ++ encoder on libdi_b200 (reference models/necks/fusion_transformerv4.py:487-640).

Per camera every image COLUMN (h tokens) is decoded into a polar RAY (R = 60 radius bins) by one post-norm transformer
decoder layer whose queries are the BEV features sampled along that column's viewing ray; the rays are resampled onto
the BEV grid and averaged over the cameras that see a cell; + residual.  All six cameras run as one batch of
B*V*w column sequences; the maps are never transposed (the attention kernel walks the columns with a row stride).
The reference evaluates the two attentions with flash-attn 0.2.2 in fp16; here they are fp32 (di_seq_attn_f32).
"""
import math

import numpy as np
import torch

from . import fold, geom, ops


def sine_table(n_y, n_x, num_feats, temperature=10000.0):
    """TransSinePositionalEncoding (:420-485; normalize=False) for x = 0..n_x-1, y = 0..n_y-1 as a row table
    [(y * n_x + x), 2 * num_feats] = (pos_y | pos_x), float64 on the host (a constant of the module)."""
    dim_t = temperature ** (2 * (np.arange(num_feats) // 2) / num_feats)
    def enc(vals):
        p = vals[:, None] / dim_t
        out = np.empty_like(p)
        out[:, 0::2], out[:, 1::2] = np.sin(p[:, 0::2]), np.cos(p[:, 1::2])
        return out
    # the reference evaluates in fp32
    px, py = enc(np.arange(n_x, dtype=np.float32).astype(np.float32)), enc(np.arange(n_y, dtype=np.float32))
    tab = np.concatenate([np.repeat(py[:, None, :], n_x, 1), np.repeat(px[None, :, :], n_y, 0)], -1)
    return torch.from_numpy(tab.reshape(n_y * n_x, 2 * num_feats).astype(np.float32))


def _lin(m):
    return m.weight.detach().double().cpu(), m.bias.detach().double().cpu()


def _ln(m, device):
    return fold.dev(m.weight.detach().double().cpu(), device), fold.dev(m.bias.detach().double().cpu(), device), float(m.eps)


def pack_polar(a, device):
    tl = a.transformer_layers
    lay = tl.decoder.layers[0]
    W, d = (lambda t: fold.Weight(t, device)), (lambda t: fold.dev(t, device))
    C = a.embed_dims

    def mha(m):
        w, b = m.in_proj_weight.detach().double().cpu(), m.in_proj_bias.detach().double().cpu()
        wo, bo = _lin(m.out_proj)
        return dict(qkv=(W(w), d(b)), q=(W(w[:C]), d(b[:C])), kv=(W(w[C:]), d(b[C:])), out=(W(wo), d(bo)))
    w1, b1 = _lin(lay.linear1)
    w2, b2 = _lin(lay.linear2)
    return dict(kind='polar', C=C, R=a.radius, radius_range=list(a.radius_range), pc_range=list(a.pc_range), heads=8,
                enc_norm=_ln(tl.encoder.norm, device), self_attn=mha(lay.self_attn), cross=mha(lay.multihead_attn),
                ffn=(W(w1), d(b1), W(w2), d(b2)), norm1=_ln(lay.norm1, device), norm2=_ln(lay.norm2, device),
                norm3=_ln(lay.norm3, device), dec_norm=_ln(tl.decoder.norm, device), tables={}, device=device)


def polar_consts_host(img_metas):
    """Per-frame camera constants of the block (tiny 4x4 algebra on the host, like geom.camera_rows_host):
    cam [B*V, 26] = rows 0-1 of inverse(lidar2img) | camera centre xy (cam2lidar[:2, 3]) | rows 0-1 of the forward
    augmentation affine | pad;  undo [B, 12] = rows 0-2 of the reverse augmentation affine;  camc [B*V, 2]."""
    l2i = geom.lidar2img_array(img_metas)
    B, V = l2i.shape[:2]
    inv = torch.linalg.inv(torch.from_numpy(l2i)).numpy()          # fp32 inverse, as the reference (:561)
    cam = np.zeros((B, V, 26), np.float32)
    undo = np.zeros((B, 12), np.float32)
    for b, meta in enumerate(img_metas):
        Af, Ar = geom.aug_affine(meta, False), geom.aug_affine(meta, True)
        undo[b] = Ar[:3].reshape(12)
        c2l = np.asarray(meta['cam2lidar'], np.float32)
        for v in range(V):
            cam[b, v, 0:8] = inv[b, v, :2].reshape(8)
            cam[b, v, 8:10] = c2l[v][:2, 3]
            cam[b, v, 10:18] = Af[:2].reshape(8)
    cam_t = torch.from_numpy(cam.reshape(B * V, 26))
    return cam_t, torch.from_numpy(undo), cam_t[:, 8:10].contiguous()


def polar_forward(ap, lidar_map, img_map, ctx, saved=None):
    """lidar_map [B,Y,X,C] (queries / residual), img_map [B*V,h,w,C] (memory) -> [B,Y,X,C].  saved (a dict) receives
    what backward.encoder_pp_backward needs: the ray grid and constants, the rows between the steps and the pre-norm
    sums (recomputed by one more GEMM each; the returned map is the same either way)."""
    B, Y, X, C = lidar_map.shape
    BV, h, w, _ = img_map.shape
    V, R, H = BV // B, ap['R'], ap['heads']
    dev = lidar_map.device
    g = ctx['g']
    key = (h, w, R)
    if key not in ap['tables']:
        ap['tables'][key] = (sine_table(h, w, C // 2).to(dev), sine_table(R, w, C // 2).to(dev))
    img_pos, ray_pos = ap['tables'][key]
    if 'polar_consts' not in ctx:
        cam, undo, camc = polar_consts_host(ctx['img_metas'])
        ctx['polar_consts'] = (cam.to(dev, non_blocking=True), undo.to(dev, non_blocking=True), camc.to(dev, non_blocking=True))
    cam, undo, camc = ctx['polar_consts']
    rr = ap['radius_range']
    grid = ops.polar_grid(cam, BV, R, w, h, 4.0, rr[0], rr[2], ap['pc_range'], (Y, X))
    rays = ops.add_rows_mod(ops.bev_sample(lidar_map, grid, V).view(-1, C), ray_pos)          # tgt  [BV*R*w, C]
    cols = ops.add_rows_mod(img_map.view(-1, C), img_pos)                                      # src  [BV*h*w, C]
    ln = lambda pk, x, res=None: ops.rows_finish(x, res=res, gamma=pk[0], beta=pk[1], eps=pk[2])
    memory = ln(ap['enc_norm'], cols)
    sa = ap['self_attn']
    qkv = ops.linear([rays], *sa['qkv'])
    a1 = ops.seq_attn(qkv[:, :C], qkv[:, C:2 * C], qkv[:, 2 * C:], BV, w, R, R, H)
    x1 = ln(ap['norm1'], ops.linear([a1], *sa['out']), res=rays)
    ca = ap['cross']
    q2 = ops.linear([x1], *ca['q'])
    kv = ops.linear([memory], *ca['kv'])
    a2 = ops.seq_attn(q2, kv[:, :C], kv[:, C:], BV, w, R, h, H)
    x2 = ln(ap['norm2'], ops.linear([a2], *ca['out']), res=x1)
    w1, b1, w2, b2 = ap['ffn']
    f = ops.linear([x2], w1, b1, ops.ACT_RELU)
    x3 = ln(ap['norm3'], ops.linear([f], w2, b2), res=x2)
    if saved is not None:
        saved.update(grid=grid, bev_shape=(B, Y, X, C), rays_shape=(BV, R, w, C), cols=cols, rays=rays, qkv=qkv, a1=a1,
                     z1=ops.linear([a1], *sa['out'], res=rays), x1=x1, q2=q2, memory=memory, kv=kv, a2=a2,
                     z2=ops.linear([a2], *ca['out'], res=x1), x2=x2, f=f, z3=ops.linear([f], w2, b2, res=x2), x3=x3,
                     gather=(g.proj, undo, camc, V, g.in_hw, ap['pc_range'], rr[0], float(R)))
    x = ln(ap['dec_norm'], x3)
    return ops.polar_gather(x.view(BV, R, w, C), lidar_map, g.proj, undo, camc, V, g.in_hw, ap['pc_range'], rr[0], float(R))
