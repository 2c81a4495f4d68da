"""GPU parity: libdi_b200 decoder kernels (through the C ABI) vs the CPU oracle / reference goldens."""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from conftest import rel_err

pytestmark = pytest.mark.gpu
TOL = 1e-3
TIGHT = 5e-5
G = os.path.join(os.path.dirname(__file__), 'golden')


def dev():
    return torch.device('cuda:0')


def test_heatmap_nms_and_topk():
    from deepinteraction_b200 import ops
    g = torch.Generator().manual_seed(0)
    B, K, H, W, P = 2, 10, 36, 44, 50
    a, b = torch.randn(B, K, H, W, generator=g) * 2, torch.randn(B, K, H, W, generator=g) * 2
    heat = (a.sigmoid() + b.sigmoid()) / 2
    lm = torch.zeros_like(heat)
    lm[:, :, 1:-1, 1:-1] = F.max_pool2d(heat, 3, 1, 0)
    lm[:, 8], lm[:, 9] = heat[:, 8], heat[:, 9]
    ref = (heat * (heat == lm)).view(B, K, -1)
    pad = lambda t: F.pad(t.permute(0, 2, 3, 1), (0, 2)).contiguous().to(dev())       # pixel-major, ld = 12
    out, dense = ops.heatmap_nms(pad(a), pad(b), K, 3, (1 << 8) | (1 << 9))
    assert torch.equal(dense.cpu(), b)
    # same support; values equal to fp32 rounding of sigmoid
    assert torch.equal(out.cpu() > 0, ref > 0)
    assert float((out.cpu() - ref).abs().max()) < 1e-6
    top = ops.topk(out.view(B, -1), P).cpu().long()
    ref_top = out.cpu().view(B, -1).argsort(-1, descending=True)[:, :P]       # on the kernel's own scores
    assert torch.equal(top, ref_top)


def test_topk_edge_cases():
    from deepinteraction_b200 import ops
    g = torch.Generator().manual_seed(1)
    # many exact ties at the threshold and lots of zeros; ties resolve to the smaller index
    s = torch.zeros(1, 5000)
    s[0, torch.randperm(5000, generator=g)[:300]] = 0.5
    s[0, 7], s[0, 4000] = 0.9, 0.7
    top = ops.topk(s.to(dev()), 200).cpu().long()[0]
    assert top[0] == 7 and top[1] == 4000
    rest = top[2:]
    half = (s[0] == 0.5).nonzero().squeeze(1)
    assert torch.equal(rest, half[:198])
    # k == n, tiny positive values
    s2 = torch.rand(3, 64, generator=g) * 1e-6
    top2 = ops.topk(s2.to(dev()), 64).cpu().long()
    assert torch.equal(top2, s2.argsort(dim=-1, descending=True, stable=True))


def _mha_ref(q, k, v, heads, mask=None):
    M, C = q.shape
    d = C // heads
    qh, kh, vh = (t.view(M, heads, d).transpose(0, 1) for t in (q, k, v))
    s = qh @ kh.transpose(1, 2)
    if mask is not None:
        s = s.masked_fill(~mask[None], float('-inf'))
    return (s.softmax(-1) @ vh).transpose(0, 1).reshape(M, C)


def test_mha_small_with_and_without_group_mask():
    from deepinteraction_b200 import ops
    g = torch.Generator().manual_seed(2)
    B, P, C, H = 2, 200, 128, 8
    qkv = torch.randn(B * P, 3 * C, generator=g)
    onbits = torch.randint(0, 64, (B * P,), generator=g, dtype=torch.int32)
    win = torch.full((B * P,), -1, dtype=torch.int32)
    for i in range(B * P):
        bits = [v for v in range(6) if (int(onbits[i]) >> v) & 1]
        if bits:
            win[i] = bits[-1]
    qd = qkv.to(dev())
    out = ops.mha_small(qd[:, :C], qd[:, C:2 * C], qd[:, 2 * C:], B, P, H).cpu()
    out_m = ops.mha_small(qd[:, :C], qd[:, C:2 * C], qd[:, 2 * C:], B, P, H, onbits.to(dev()), win.to(dev())).cpu()
    for b in range(B):
        sl = slice(b * P, (b + 1) * P)
        q, k, v = qkv[sl, :C], qkv[sl, C:2 * C], qkv[sl, 2 * C:]
        assert rel_err(out[sl], _mha_ref(q, k, v, H)) < TIGHT
        w, ob = win[sl].long(), onbits[sl].long()
        mask = ((ob[None, :] >> w.clamp(min=0)[:, None]) & 1).bool()
        ref = _mha_ref(q, k, v, H, mask)
        live = w >= 0
        assert rel_err(out_m[sl][live], ref[live]) < TIGHT
        assert float(out_m[sl][~live].abs().max()) == 0.0


def test_cross_attention_matches_dense_softmax():
    from deepinteraction_b200 import ops
    g = torch.Generator().manual_seed(3)
    B, P, HW, C, H = 2, 200, 3000, 128, 8
    q = torch.randn(B * P, C, generator=g) * 0.5
    kv = torch.randn(B * HW, 2 * C, generator=g)
    out = ops.cross_attn(q.to(dev()), kv.to(dev()), B, P, HW, H, nsplit=7).cpu()
    for b in range(B):
        qb, kb, vb = q[b * P:(b + 1) * P], kv[b * HW:(b + 1) * HW, :C], kv[b * HW:(b + 1) * HW, C:]
        d = C // H
        s = torch.einsum('phd,khd->hpk', qb.view(P, H, d), kb.view(HW, H, d))
        ref = torch.einsum('hpk,khd->phd', s.softmax(-1), vb.view(HW, H, d)).reshape(P, C)
        assert rel_err(out[b * P:(b + 1) * P], ref) < TIGHT


@pytest.mark.parametrize('B,P,HW', [(1, 200, 32400), (2, 200, 3000), (1, 24, 1296), (3, 77, 64), (1, 256, 700)])
def test_cross_attention_tensor_core_matches_dense_softmax(B, P, HW):
    """di_xattn_tc_f32 (bf16 operand planes, six-term logits and three-term P V on mma.sync, online softmax, key splits) vs
    a float64 dense softmax; the K | V rows come from the 3xTF32 GEMM like in the decoder."""
    from deepinteraction_b200 import ops, fold
    g = torch.Generator().manual_seed(P + HW)
    C, H = 128, 8
    q = torch.randn(B * P, C, generator=g) * 0.7
    x = torch.randn(B * HW, C, generator=g)
    W = torch.randn(2 * C, C, generator=g) / C ** 0.5
    bias = torch.randn(2 * C, generator=g) * 0.1
    pos = torch.randn(HW, 2 * C, generator=g) * 0.3
    d = dev()
    kv32 = ops.linear([x.to(d)], fold.Weight(W, d), bias.to(d), res=pos.to(d), res_mod=HW)
    out = ops.xattn_tc(q.to(d), kv32, B, P, HW, H).cpu()
    kv = (x.double() @ W.double().t() + bias.double()).view(B, HW, 2 * C) + pos.double()[None]
    for b in range(B):
        qb, kb, vb = q[b * P:(b + 1) * P].double(), kv[b, :, :C], kv[b, :, C:]
        dh = C // H
        s = torch.einsum('phd,khd->hpk', qb.view(P, H, dh), kb.reshape(HW, H, dh))
        ref = torch.einsum('hpk,khd->phd', s.softmax(-1), vb.reshape(HW, H, dh)).reshape(P, C)
        assert rel_err(out[b * P:(b + 1) * P].double(), ref) < 2e-5, b


@pytest.mark.parametrize('M,Ks,N1,N2', [(200, (128,), 384, 0), (200, (128, 128), 384, 20), (37, (2,), 128, 128),
                                        (600, (128,), 512, 128), (5, (256,), 64, 0), (33, (128,), 128, 0), (200, (128,), 36, 12)])
def test_rows_mlp_matches_float64(M, Ks, N1, N2):
    """Query-row MLP kernel: two chained dense layers + residual + LayerNorm + activation + row masking in one launch."""
    from deepinteraction_b200 import ops, fold
    g = torch.Generator().manual_seed(M + N1)
    xs = [torch.randn(M, k, generator=g) for k in Ks]
    K = sum(Ks)
    W1, b1 = torch.randn(N1, K, generator=g) / K ** 0.5, torch.randn(N1, generator=g)
    N = N2 or N1
    res, gam, bet = torch.randn(M, N, generator=g), torch.rand(N, generator=g) + 0.5, torch.randn(N, generator=g)
    zin = torch.where(torch.rand(M, generator=g) < 0.2, -1, 3).to(torch.int32)
    x64 = torch.cat(xs, 1).double()
    h = F.gelu(x64 @ W1.double().t() + b1.double())
    if N2:
        W2, b2 = torch.randn(N2, N1, generator=g) / N1 ** 0.5, torch.randn(N2, generator=g)
        h = h @ W2.double().t() + b2.double()
    want = F.relu(F.layer_norm(h + res.double(), (N,), gam.double(), bet.double()))
    want[zin < 0] = 0
    d = dev()
    got = ops.rows_mlp([x.to(d) for x in xs], fold.Weight(W1, d), b1.to(d), ops.ACT_GELU,
                       fold.Weight(W2, d) if N2 else None, b2.to(d) if N2 else None, res.to(d), gam.to(d), bet.to(d),
                       ops.ACT_RELU, zin.to(d))
    assert rel_err(got.cpu().double(), want) < 2e-6
    plain = ops.rows_mlp([x.to(d) for x in xs], fold.Weight(W1, d), b1.to(d))          # single layer, nothing else
    assert rel_err(plain.cpu().double(), x64 @ W1.double().t() + b1.double()) < 2e-6


def test_rows_finish_layernorm():
    from deepinteraction_b200 import ops
    g = torch.Generator().manual_seed(4)
    x, r = torch.randn(333, 128, generator=g), torch.randn(333, 128, generator=g)
    gm, bt = torch.rand(128, generator=g) + 0.5, torch.randn(128, generator=g)
    ref = F.relu(F.layer_norm(x + r, (128,), gm, bt))
    out = ops.rows_finish(x.to(dev()), res=r.to(dev()), gamma=gm.to(dev()), beta=bt.to(dev()), act=ops.ACT_RELU)
    assert rel_err(out.cpu(), ref) < TIGHT


def test_roi_align_matches_oracle():
    from oracle.geometry import roi_align
    from deepinteraction_b200 import ops
    g = torch.Generator().manual_seed(5)
    maps = torch.randn(3, 128, 28, 50, generator=g)
    rois = torch.tensor([[0, 8.0, 12.0, 70.0, 49.0], [1, -30.0, -10.0, 20.0, 30.0], [2, 150.0, 60.0, 230.0, 140.0],
                         [1, 40.0, 40.0, 40.0, 40.0], [-1, 0.0, 0.0, 10.0, 10.0], [0, 190.0, 100.0, 260.0, 150.0]])
    out = ops.roi_align(maps.permute(0, 2, 3, 1).contiguous().to(dev()), rois.to(dev()), 0.25).cpu()   # [n,49,C]
    for i, r in enumerate(rois):
        if r[0] < 0:
            assert float(out[i].abs().max()) == 0.0
            continue
        ref = roi_align(maps[int(r[0])], r[None, 1:], 7, 0.25, 2)[0]            # (C,7,7)
        assert rel_err(out[i].t().reshape(128, 7, 7), ref) < TIGHT


def test_dynconv_matches_oracle():
    import oracle.mmpi as om
    from deepinteraction_b200 import ops
    torch.manual_seed(6)
    m = om.DynamicConv().eval()
    g = torch.Generator().manual_seed(6)
    n = 37
    pro = torch.randn(1, n, 128, generator=g)
    roi = torch.randn(49, n, 128, generator=g)
    with torch.no_grad():
        params = m.dynamic_layer(pro)[0]                                            # [n, 32768]
        feats = roi.permute(1, 0, 2)
        p1 = params[:, :16384].reshape(n, 128, 128)
        p2 = params[:, 16384:].reshape(n, 128, 128)
        f = F.relu(m.norm1(torch.bmm(feats, p1)))
        ref = F.relu(m.norm2(torch.bmm(f, p2))).flatten(1)
    d = lambda t: t.detach().contiguous().to(dev())
    out = ops.dynconv(d(feats), d(params), d(m.norm1.weight), d(m.norm1.bias), d(m.norm2.weight), d(m.norm2.bias))
    assert rel_err(out.cpu(), ref) < TIGHT


def _build(tag_seed, views, proposals, test_cfg=None, coder=None, plusplus=False):
    import oracle.mmpi as om
    import oracle.mmpi_pp as ompp
    from deepinteraction_b200 import mmpi, synth
    from tools import make_goldens as mg
    kw = dict(num_views=views, out_size_factor_img=4, num_proposals=proposals, auxiliary=True, hidden_channel=128,
              num_classes=10, num_mmpi=4, num_heads=8, initialize_by_heatmap=True, nms_kernel_size=3, ffn_channel=256,
              dropout=0.1, bn_momentum=0.1, activation='relu',
              common_heads=dict(center=(2, 2), height=(1, 2), dim=(3, 2), rot=(2, 2), vel=(2, 2)),
              loss_cls=dict(type='FocalLoss', use_sigmoid=True, gamma=2, alpha=0.25, reduction='mean', loss_weight=1.0),
              bbox_coder=dict(coder or mg.DEC_CODER), test_cfg=dict(test_cfg or mg.DEC_TEST_CFG))
    torch.manual_seed(tag_seed)
    o = (ompp.DeepInteractionPlusPlusDecoder if plusplus else om.DeepInteractionDecoder)(**kw).eval()
    synth.randomize_norm_stats(o, tag_seed)
    if plusplus:
        from test_oracle_golden import pp_scales
        pp_scales(o)
    m = (mmpi.DeepInteractionPlusPlusDecoder if plusplus else mmpi.DeepInteractionDecoder)(**kw)
    m.load_state_dict(o.state_dict(), strict=True)
    return o, m.to(dev()).eval()


def _compare(out, ref, tol):
    errs = {k: rel_err(out[k].cpu(), ref[k]) for k in ref}
    print({k: '%.1e' % v for k, v in errs.items()})
    for k, e in errs.items():
        assert e < tol, (k, e)


@pytest.mark.parametrize('tag', ['decoder_small', 'decoder_small_aug'])
def test_decoder_small_matches_reference_golden(tag):
    from tools.make_goldens import small_frame
    gold = torch.load(os.path.join(G, tag + '.pt'), weights_only=False)
    o, m = _build(gold['seed'], 2, 24)
    gen = torch.Generator().manual_seed(gold['seed'])
    fr = small_frame(gold['seed'], aug=gold['aug'], views=2, batch=2)
    pts_in = [torch.randn(2, 128, 36, 36, generator=gen), torch.randn(2, 128, 36, 36, generator=gen)]
    img_in = torch.randn(4, 128, 28, 50, generator=gen)
    out = m([p.to(dev()) for p in pts_in], img_in.to(dev()), fr['img_metas'])[0][0]
    assert torch.equal(m.query_labels.cpu(), gold['query_labels'])
    for a, b in zip(m.on_the_image_mask, gold['on_the_image_mask']):
        assert torch.equal(a.cpu(), b)
    _compare(out, gold['out'], TOL)


def test_decoder_stages_match_oracle():
    """Stage-by-stage (top-k, query init, transformer layer, every MMPI layer) on the small scene."""
    from tools.make_goldens import small_frame
    o, m = _build(1600, 2, 24)
    gen = torch.Generator().manual_seed(1600)
    fr = small_frame(1600, aug=True, views=2, batch=2)
    pts_in = [torch.randn(2, 128, 36, 36, generator=gen), torch.randn(2, 128, 36, 36, generator=gen)]
    img_in = torch.randn(4, 128, 28, 50, generator=gen)
    with torch.no_grad():
        ref, aux = o(pts_in, img_in, fr['img_metas'], return_aux=True)
    dbg = {}
    nhwc = lambda t: t.permute(0, 2, 3, 1).contiguous().to(dev())
    m.forward_nhwc(nhwc(pts_in[0]), nhwc(pts_in[1]), nhwc(img_in), fr['img_metas'], debug=dbg)
    B, P, C = 2, 24, 128
    assert torch.equal(dbg['top'].cpu().long(), aux['top'])
    assert rel_err(dbg['heat'].cpu(), aux['heatmap']) < 1e-5
    rows = lambda t: t.permute(0, 2, 1).reshape(B * P, -1)                       # (B,C,P) -> rows
    assert rel_err(dbg['query_feat0'].cpu(), rows(aux['query_feat0'])) < TIGHT
    assert torch.equal(dbg['query_pos0'].cpu(), aux['query_pos0'].reshape(B * P, 2))
    assert rel_err(dbg['query_feat1'].cpu(), rows(aux['query_feat1'])) < 2e-4
    first = torch.cat([aux['first_res'][k] for k in m.head_order], 1)
    assert rel_err(dbg['first_res'].cpu(), rows(first)) < 2e-4
    for l in range(4):
        e = rel_err(dbg['layer_query'][l].cpu(), rows(aux['layer_query'][l]))
        print('layer', l, 'query rel err %.2e' % e)
        assert e < TOL
    for a, b in zip(m.on_the_image_mask, aux['on_view']):
        assert torch.equal(a.cpu(), b != -1)


def test_decoder_base_shape_matches_oracle():
    """Base config shapes (180x180 BEV, 6 x 112x200 image maps, 200 queries), random feature maps."""
    from deepinteraction_b200 import synth
    test_cfg = dict(dataset='nuScenes', grid_size=[1440, 1440, 40], out_size_factor=8, pc_range=[-54.0, -54.0],
                    voxel_size=[0.075, 0.075], nms_type=None)
    coder = dict(type='TransFusionBBoxCoder', pc_range=[-54.0, -54.0], voxel_size=[0.075, 0.075], out_size_factor=8,
                 post_center_range=[-61.2, -61.2, -10.0, 61.2, 61.2, 10.0], score_threshold=0.0, code_size=10)
    o, m = _build(1601, 6, 200, test_cfg, coder)
    gen = torch.Generator().manual_seed(1601)
    rig = synth.camera_rig(6, (448, 800))
    metas = [dict(lidar2img=[r.astype(np.float32) for r in rig], input_shape=(448, 800),
                  img_shape=[(448, 800, 3)] * 6)]
    pts_in = [torch.randn(1, 128, 180, 180, generator=gen), torch.randn(1, 128, 180, 180, generator=gen)]
    img_in = torch.randn(6, 128, 112, 200, generator=gen)
    with torch.no_grad():
        ref = o(pts_in, img_in, metas)[0][0]
    out = m([p.to(dev()) for p in pts_in], img_in.to(dev()), metas)[0][0]
    assert torch.equal(m.query_labels.cpu(), o.query_labels)
    for a, b in zip(m.on_the_image_mask, o.on_the_image_mask):
        assert torch.equal(a.cpu(), b)
    _compare(out, ref, TOL)


def test_v2_leader_rows_and_branch_mix():
    """Kernels specific to the V2 RCNN blocks: first query of every (sample, view) group, the group self-attention for a
    list of (query row, group) pairs, row gather, and out = main * scale + leader_self * self_scale."""
    from deepinteraction_b200 import ops
    g = torch.Generator().manual_seed(8)
    B, P, C, H, V = 2, 100, 128, 8, 6
    qkv = torch.randn(B * P, 3 * C, generator=g)
    onbits = torch.randint(0, 64, (B * P,), generator=g, dtype=torch.int32)
    onbits[:7] &= ~1                       # view 0 of sample 0: leader is not query 0
    onbits[P:2 * P] &= ~(1 << 3)           # view 3 of sample 1: empty group
    win = torch.full((B * P,), -1, dtype=torch.int32)
    for i in range(B * P):
        bits = [v for v in range(V) if (int(onbits[i]) >> v) & 1]
        if bits:
            win[i] = bits[-1]
    d = dev()
    lrow, lwin = ops.rcnn_leaders(onbits.to(d), B, P, V)
    want_row = torch.full((B * V,), -1, dtype=torch.int32)
    for b in range(B):
        for v in range(V):
            hit = ((onbits[b * P:(b + 1) * P] >> v) & 1).nonzero()
            if len(hit):
                want_row[b * V + v] = b * P + int(hit[0])
    assert torch.equal(lrow.cpu(), want_row)
    assert torch.equal(lwin.cpu(), torch.where(want_row >= 0, torch.arange(B * V, dtype=torch.int32) % V, -1))
    assert int(want_row[0]) >= 7 and int(want_row[V + 3]) == -1
    qd = qkv.to(d)
    out = ops.mha_small_rows(qd[:, :C], qd[:, C:2 * C], qd[:, 2 * C:], B, P, H, onbits.to(d), lrow, lwin).cpu()
    for r in range(B * V):
        b, v, i = r // V, r % V, int(want_row[r])
        if i < 0:
            assert float(out[r].abs().max()) == 0.0
            continue
        sl = slice(b * P, (b + 1) * P)
        mask = ((onbits[sl].long() >> v) & 1).bool()[None].expand(P, P)
        ref = _mha_ref(qkv[sl, :C], qkv[sl, C:2 * C], qkv[sl, 2 * C:], H, mask)[i - b * P]
        assert rel_err(out[r], ref) < TIGHT
    src = torch.randn(B * P, 2 * C, generator=g)
    took = ops.take_rows(src.to(d)[:, :C], lrow).cpu()
    assert torch.equal(took, torch.where((want_row >= 0)[:, None], src[want_row.clamp(min=0).long(), :C], torch.zeros(1)))
    a, lead = torch.randn(B * P, C, generator=g), torch.randn(B * V, C, generator=g)
    sc, ssc = torch.tensor([0.61]), torch.tensor([0.37])
    mix = ops.branch_mix(a.to(d), lead.to(d), win.to(d), sc.to(d), ssc.to(d), P, V, True).cpu()
    grp = (torch.arange(B * P) // P) * V + win.clamp(min=0).long()
    want = a * sc + lead[grp] * ssc
    want[win < 0] = 0
    assert torch.equal(mix, want)                                   # two rounded products + one rounded sum, as torch


@pytest.mark.parametrize('tag', ['decoder_pp_small', 'decoder_pp_small_aug'])
def test_decoder_pp_small_matches_reference_golden(tag):
    """DeepInteractionPlusPlusDecoder vs outputs of the reference's own deepinteractionplusplus_decoder.py."""
    from tools.make_goldens import small_frame
    gold = torch.load(os.path.join(G, tag + '.pt'), weights_only=False)
    o, m = _build(gold['seed'], 2, 24, plusplus=True)
    gen = torch.Generator().manual_seed(gold['seed'])
    fr = small_frame(gold['seed'], aug=gold['aug'], views=2, batch=2)
    pts_in = [torch.randn(2, 128, 36, 36, generator=gen), torch.randn(2, 128, 36, 36, generator=gen)]
    img_in = torch.randn(4, 128, 28, 50, generator=gen)
    out = m([p.to(dev()) for p in pts_in], img_in.to(dev()), fr['img_metas'])[0][0]
    assert torch.equal(m.query_labels.cpu(), gold['query_labels'])
    assert len(m.on_the_image_mask) == 4
    for a, b in zip(m.on_the_image_mask, gold['on_the_image_mask']):
        assert torch.equal(a.cpu(), b)
    _compare(out, gold['out'], TOL)
    # replay from the captured graph gives the same bits
    out2 = m([p.to(dev()) for p in pts_in], img_in.to(dev()), fr['img_metas'])[0][0]
    out3 = m([p.to(dev()) for p in pts_in], img_in.to(dev()), fr['img_metas'])[0][0]
    for k in out:
        assert torch.equal(out2[k], out3[k]) and torch.equal(out[k], out3[k]), k


def test_decoder_pp_stages_match_oracle():
    from tools.make_goldens import small_frame
    o, m = _build(1700, 2, 24, plusplus=True)
    gen = torch.Generator().manual_seed(1700)
    fr = small_frame(1700, aug=True, views=2, batch=2)
    pts_in = [torch.randn(2, 128, 36, 36, generator=gen), torch.randn(2, 128, 36, 36, generator=gen)]
    img_in = torch.randn(4, 128, 28, 50, generator=gen)
    with torch.no_grad():
        ref, aux = o(pts_in, img_in, fr['img_metas'], return_aux=True)
    dbg = {}
    nhwc = lambda t: t.permute(0, 2, 3, 1).contiguous().to(dev())
    m.forward_nhwc(nhwc(pts_in[0]), nhwc(pts_in[1]), nhwc(img_in), fr['img_metas'], debug=dbg)
    B, P = 2, 24
    rows = lambda t: t.permute(0, 2, 1).reshape(B * P, -1)
    for l in range(4):
        e = rel_err(dbg['layer_query'][l].cpu(), rows(aux['layer_query'][l]))
        print('++ layer', l, 'query rel err %.2e' % e)
        assert e < TOL
    for a, b in zip(m.on_the_image_mask, o.on_the_image_mask):
        assert torch.equal(a.cpu(), b)


def test_decoder_pp_base_shape_matches_oracle():
    """++ decoder at the config-4 shapes (180x180 BEV, 6 x 112x200 image maps, 200 queries), batch 2."""
    from deepinteraction_b200 import synth
    test_cfg = dict(dataset='nuScenes', grid_size=[1440, 1440, 40], out_size_factor=8, pc_range=[-54.0, -54.0],
                    voxel_size=[0.075, 0.075], nms_type=None)
    coder = dict(type='TransFusionBBoxCoder', pc_range=[-54.0, -54.0], voxel_size=[0.075, 0.075], out_size_factor=8,
                 post_center_range=[-61.2, -61.2, -10.0, 61.2, 61.2, 10.0], score_threshold=0.0, code_size=10)
    rig = synth.camera_rig(6, (448, 800))
    metas = [dict(lidar2img=[r.astype(np.float32) for r in rig], input_shape=(448, 800),
                  img_shape=[(448, 800, 3)] * 6)] * 2
    nhwc = lambda t: t.permute(0, 2, 3, 1).contiguous().to(dev())
    for seed in (1701, 1702, 1703):
        o, m = _build(seed, 6, 200, test_cfg, coder, plusplus=True)
        with torch.no_grad():          # keep the heat-map logits out of sigmoid saturation (scores ~1 - 1e-7 all tie in fp32)
            o.heatmap_head[1].weight.mul_(0.2)
            o.heatmap_head_img[1].weight.mul_(0.2)
        m.load_state_dict(o.state_dict(), strict=True)
        gen = torch.Generator().manual_seed(seed)
        pts_in = [torch.randn(2, 128, 180, 180, generator=gen), torch.randn(2, 128, 180, 180, generator=gen)]
        img_in = torch.randn(12, 128, 112, 200, generator=gen)
        with torch.no_grad():
            ref, aux = o(pts_in, img_in, metas, return_aux=True)
        dbg = {}
        out = m.forward_nhwc(nhwc(pts_in[0]), nhwc(pts_in[1]), nhwc(img_in), metas, debug=dbg)[0][0]
        top, want = dbg['top'].cpu().long(), aux['top']
        # The proposal ORDER is only defined up to the fp32 rounding of the heat-map scores (they agree to ~1e-6; with
        # 2 x 200 ranks a swap of two neighbours is likely).  A differing rank must be a near tie in the oracle's own
        # scores.  The decoder is equivariant to the proposal order, so the outputs are compared after undoing the
        # swap; a near tie AT the cut (rank 200) changes the proposal set itself: next seed.
        hs = aux['heatmap'].reshape(2, -1)
        for b, r in (top != want).nonzero().tolist():
            assert abs(float(hs[b, top[b, r]] - hs[b, want[b, r]])) < 1e-5 * float(hs[b, want[b, r]]), (seed, b, r)
        if all(set(top[b].tolist()) == set(want[b].tolist()) for b in range(2)):
            break
        print('seed', seed, ': near tie at the top-k cut')
    else:
        raise AssertionError('no seed without a near tie at the cut')
    P = 200
    labels, masks = m.query_labels.cpu().clone(), [k.cpu().clone() for k in m.on_the_image_mask]
    out = {k: v.cpu().clone() for k, v in out.items()}
    for b in range(2):
        pos = {int(v): i for i, v in enumerate(top[b])}
        perm = torch.tensor([pos[int(v)] for v in want[b]])
        if not torch.equal(perm, torch.arange(P)):
            print('batch', b, 'ranks swapped:', (perm != torch.arange(P)).nonzero().flatten().tolist())
        labels[b] = labels[b][perm]
        for k in masks:
            k[b] = k[b][perm]
        for k, v in out.items():
            if k != 'dense_heatmap':
                v[b] = v[b][..., torch.cat([perm + c * P for c in range(v.shape[-1] // P)])]
    assert torch.equal(labels, o.query_labels)
    for a, b in zip(masks, o.on_the_image_mask):
        assert torch.equal(a, b)
    _compare(out, ref[0][0], TOL)


def test_get_bboxes_and_coder_match_reference_golden():
    """get_bboxes (decoder.py:549-638) and TransFusionBBoxCoder.decode/encode on the GPU vs the reference golden."""
    from tools.make_goldens import small_frame
    gold = torch.load(os.path.join(G, 'decoder_bboxes.pt'), weights_only=False)
    o, m = _build(gold['seed'], 2, 24)
    m.bbox_coder.score_threshold = gold['score_threshold']
    preds = {k: v.to(dev()) for k, v in gold['preds'].items()}
    m.query_labels = gold['query_labels'].to(dev())
    boxes, scores, labels = m.get_bboxes([[preds]], [dict()])[0]
    assert boxes.shape == gold['boxes'].shape and labels.dtype == torch.int32
    assert torch.equal(labels.cpu(), gold['labels'])
    assert rel_err(boxes.cpu(), gold['boxes']) < TIGHT and rel_err(scores.cpu(), gold['scores']) < TIGHT
    assert rel_err(m.bbox_coder.encode(gold['boxes'].to(dev())).cpu(), gold['encoded']) < TIGHT
    # end to end: forward on the GPU then get_bboxes == the reference's boxes for the same inputs
    gen = torch.Generator().manual_seed(gold['seed'])
    fr = small_frame(gold['seed'], aug=False, views=2, batch=1)
    pts_in = [torch.randn(1, 128, 36, 36, generator=gen), torch.randn(1, 128, 36, 36, generator=gen)]
    img_in = torch.randn(2, 128, 28, 50, generator=gen)
    out = m([p.to(dev()) for p in pts_in], img_in.to(dev()), fr['img_metas'])
    b2, s2, l2 = m.get_bboxes(out, fr['img_metas'])[0]
    assert torch.equal(l2.cpu(), gold['labels']) and rel_err(b2.cpu(), gold['boxes']) < TOL
    # box_type_3d wrapper and the unfiltered decode
    class Boxes:
        def __init__(self, t, box_dim=9):
            self.tensor, self.box_dim = t, box_dim
    b3 = m.get_bboxes(out, [dict(box_type_3d=Boxes)])[0][0]
    assert isinstance(b3, Boxes) and b3.box_dim == 9 and torch.equal(b3.tensor, b2)
    m.bbox_coder.score_threshold = 0.999                                  # nothing survives: empty, well-typed result
    b0, s0, l0 = m.get_bboxes(out, fr['img_metas'])[0]
    assert b0.shape == (0, 9) and s0.shape == (0,) and l0.shape == (0,) and l0.dtype == torch.int32
    assert m.bbox_coder.encode(b0).shape == (0, 10)
    m.bbox_coder.score_threshold = gold['score_threshold']
    full = m.bbox_coder.decode(*(preds[k][..., -24:] for k in ('heatmap', 'rot', 'dim', 'center', 'height', 'vel')))
    ref = o.bbox_coder.decode(*(gold['preds'][k][..., -24:] for k in ('heatmap', 'rot', 'dim', 'center', 'height', 'vel')))
    assert torch.equal(full[0]['labels'].cpu(), ref[0]['labels']) and rel_err(full[0]['bboxes'].cpu(), ref[0]['bboxes']) < TIGHT


def test_get_bboxes_circle_nms_matches_oracle():
    """nms_type='circle' (per-task greedy circle NMS) vs the oracle restatement, crowded random proposals."""
    import oracle.mmpi as om
    from tools import make_goldens as mg
    P = 300
    o, m = _build(5, 2, P, test_cfg=dict(mg.DEC_TEST_CFG, nms_type='circle'))
    g = torch.Generator().manual_seed(3)
    preds = dict(center=torch.rand(1, 2, P, generator=g) * 6 + 15, height=torch.randn(1, 1, P, generator=g),
                 dim=torch.randn(1, 3, P, generator=g) * 0.2, rot=torch.randn(1, 2, P, generator=g),
                 vel=torch.randn(1, 2, P, generator=g), heatmap=torch.randn(1, 10, P, generator=g),
                 query_heatmap_score=torch.rand(1, 10, P, generator=g))
    labels = torch.randint(6, 10, (1, P), generator=g)               # classes 8 and 9 have radius 0.175
    o.query_labels, m.query_labels = labels, labels.to(dev())
    rb, rs, rl = o.get_bboxes([[preds]], [dict()])[0]
    b, s_, l = m.get_bboxes([[{k: v.to(dev()) for k, v in preds.items()}]], [dict()])[0]
    assert 0 < rb.shape[0] < P and b.shape == rb.shape
    assert torch.equal(l.cpu(), rl) and rel_err(b.cpu(), rb) < TIGHT and rel_err(s_.cpu(), rs) < TIGHT
