"""Backward of the ++ decoder's V2 RCNN blocks (backward.point_rcnn_v2_backward, backward.image_rcnn_v2_backward and their
autograd Functions) and the four kernels only they use (di_branch_mix_bwd_f32, di_mha_small_rows_bwd_f32,
di_rows_scatter_add_f32, di_pred_finish_pp_bwd_f32), against float64 autograd.

The V2 block writes out = q3 * scale + s_l * self_scale, where s_l is the self branch of the FIRST query of the row's
(sample, view) group (the reference's (1,n,C) + (n,1,C) broadcast followed by [0], restated literally by oracle.mmpi_pp).
The blocks are compared with autograd through oracle.mmpi_pp's blocks run per group as the reference runs them, driven by
the product's decisions (RoI rectangles, win, onbits), at max(1e-4, 5x the error the same chain makes in fp32) like the
V1 block tests.  A ReLU pre-activation of ffn / self_ffn within 1e-5 of 0 (relative to the largest) takes the product's
side, as the heat-map head test does; every other element must agree.
"""
import math

import pytest
import torch

from conftest import rel_err
from kernel_check import record_calls, same_bits

pytestmark = pytest.mark.gpu

TOL = 1e-4
C, H = 128, 8


def dev():
    return torch.device('cuda:0')


def _ops():
    from deepinteraction_b200 import ops
    return ops


def _bar(got, want, f32, floor):
    return rel_err(got.double().cpu(), want.double().cpu()), max(floor, 5 * rel_err(f32.double().cpu(), want.double().cpu()))


# ---------------------------------------------------------------------------------------------------------------------
# 1. kernels
# ---------------------------------------------------------------------------------------------------------------------
def _group_draw(B, P, V, g):
    """onbits / win [B*P] with, per sample: query 0 on views 0 and 1 (it leads both; its win is 1), view V-1 empty (no
    leader), and queries on no view (win = -1)."""
    raw = (torch.randint(0, 1 << V, (B, P), generator=g) & torch.randint(0, 1 << V, (B, P), generator=g)) & ~(1 << (V - 1))
    raw[:, 0] = 0b11
    raw[:, 1:3] = 0
    win = torch.full((B, P), -1, dtype=torch.int64)
    for v in range(V):
        win = torch.where(((raw >> v) & 1) == 1, torch.full_like(win, v), win)
    return raw.reshape(-1).int(), win.reshape(-1).int()


def _branch_mix_oracle(a, lead, win, scale, self_scale, dout, P, V, zero_off, dtype):
    """autograd of the oracle's expression q_view * scale + self_view * self_scale ((1,n,C) + (n,1,C), then [0]) per
    (sample, view) group, row 0 of self_view being the group's leader row; rows with win < 0: 0 (image) or group 0."""
    d = dev()
    x = [t.to(d, dtype).requires_grad_(True) for t in (a, lead, scale, self_scale)]
    M = a.shape[0]
    g = torch.Generator().manual_seed(5)
    with torch.enable_grad():
        out = torch.zeros(M, C, device=d, dtype=dtype)
        for b in range(M // P):
            for v in range(V):
                w = win[b * P:(b + 1) * P].long()
                w = torch.where(w < 0, torch.full_like(w, -1 if zero_off else 0), w)
                rows = (w == v).nonzero().squeeze(1) + b * P
                n = rows.numel()
                if n == 0:
                    continue
                q_view = x[0][rows.to(d)].unsqueeze(0)
                self_view = torch.cat([x[1][b * V + v:b * V + v + 1], torch.randn(n - 1, C, generator=g).to(d, dtype)]).unsqueeze(1)
                out = out.index_put((rows.to(d),), (q_view * x[2] + self_view * x[3])[0])
        (out * dout.to(d, dtype)).sum().backward()
    return [t.grad for t in x]


@pytest.mark.parametrize('B,P,V,zero_off', [(2, 40, 2, True), (1, 200, 6, True), (2, 200, 1, False)])
def test_branch_mix_bwd_matches_float64_autograd(B, P, V, zero_off):
    ops = _ops()
    d = dev()
    g = torch.Generator().manual_seed(P + V)
    onbits, win = _group_draw(B, P, max(V, 2), g)
    if V == 1:
        win = torch.zeros_like(win)
    a, lead, dout = torch.randn(B * P, C, generator=g), torch.randn(B * V, C, generator=g), torch.randn(B * P, C, generator=g)
    scale, self_scale = torch.tensor([0.7]), torch.tensor([-1.3])
    got = ops.branch_mix_bwd(dout.to(d), a.to(d), lead.to(d), win.to(d), scale.to(d), self_scale.to(d), P, V, zero_off)
    want = _branch_mix_oracle(a, lead, win, scale, self_scale, dout, P, V, zero_off, torch.float64)
    f32 = _branch_mix_oracle(a, lead, win, scale, self_scale, dout, P, V, zero_off, torch.float32)
    for name, gt, w, f in zip(('da', 'dlead', 'dscale', 'dself_scale'), got, want, f32):
        e, bar = _bar(gt, w, f, 1e-5)
        print('%-12s %.1e (bar %.1e)' % (name, e, bar))
        assert e <= bar, (name, e, bar)
    if zero_off:
        assert bool((got[0][win.to(d) < 0] == 0).all())
    again = ops.branch_mix_bwd(dout.to(d), a.to(d), lead.to(d), win.to(d), scale.to(d), self_scale.to(d), P, V, zero_off)
    assert all(same_bits(x, y) for x, y in zip(got, again)), 'two calls differ'


def _rows_attn_oracle(qkv, dout, onbits, lrow, lwin, B, P, dtype):
    """autograd of row r's softmax attention (query qkv[lrow[r], :C], keys j of sample r // Vg with bit lwin[r]) ->
    (d q rows [R, C], d qkv [B*P, 3C] (k and v columns))."""
    d = dev()
    R = lrow.shape[0]
    Vg = R // B
    x = qkv.to(d, dtype).requires_grad_(True)
    lr = lrow.long()
    qr = x[lr.clamp(min=0).to(d), :C].detach().clone().requires_grad_(True)
    with torch.enable_grad():
        tot = 0
        for r in range(R):
            if lr[r] < 0:
                continue
            b = r // Vg
            keys = (((onbits[b * P:(b + 1) * P].long() >> int(lwin[r])) & 1) == 1).nonzero().squeeze(1) + b * P
            kh = x[keys.to(d), C:2 * C].view(-1, H, 16)
            vh = x[keys.to(d), 2 * C:].view(-1, H, 16)
            s = torch.einsum('hd,khd->hk', qr[r].view(H, 16), kh)
            o = torch.einsum('hk,khd->hd', s.softmax(-1), vh).reshape(C)
            tot = tot + (o * dout[r].to(d, dtype)).sum()
        tot.backward()
    return qr.grad, x.grad


@pytest.mark.parametrize('B,P,V', [(2, 24, 2), (2, 40, 3), (1, 200, 6), (1, 512, 6)])
def test_mha_small_rows_bwd_matches_float64_autograd(B, P, V):
    ops = _ops()
    d = dev()
    g = torch.Generator().manual_seed(70 + P + V)
    onbits, _ = _group_draw(B, P, V, g)
    lrow, lwin = ops.rcnn_leaders(onbits.to(d), B, P, V)
    lr = lrow.cpu()
    assert V < 3 or bool((lr == -1).any())                                  # view V-1 has no query
    assert all(int(lr[b * V]) == int(lr[b * V + 1]) == b * P for b in range(B))      # query 0 leads views 0 and 1
    qkv = torch.randn(B * P, 3 * C, generator=g)
    qkv[:, :C] *= 0.5
    dout = torch.randn(B * V, C, generator=g)
    base = torch.randn(B * P, 3 * C, generator=g)                            # the main attention's gradient, already there

    def run():
        qd, acc = qkv.to(d), base.to(d)
        dq = ops.mha_small_rows_bwd(qd[:, :C], qd[:, C:2 * C], qd[:, 2 * C:], dout.to(d), B, P, H, onbits.to(d), lrow, lwin,
                                    acc[:, C:2 * C], acc[:, 2 * C:])
        return dq, acc
    dq, acc = run()
    wq, wx = _rows_attn_oracle(qkv, dout, onbits, lr, lwin.cpu(), B, P, torch.float64)
    fq, fx = _rows_attn_oracle(qkv, dout, onbits, lr, lwin.cpu(), B, P, torch.float32)
    live = (lr >= 0).to(d)
    e, bar = _bar(dq[live], wq[live], fq[live], 1e-5)
    print('dq %.1e (bar %.1e)' % (e, bar))
    assert e <= bar and bool((dq[~live] == 0).all())
    for name, sl in (('dk', slice(C, 2 * C)), ('dv', slice(2 * C, 3 * C))):
        e, bar = _bar(acc[:, sl].double() - base[:, sl].double().to(d), wx[:, sl], fx[:, sl], 1e-5)
        print('%s %.1e (bar %.1e)' % (name, e, bar))
        assert e <= bar, (name, e, bar)
    assert same_bits(acc[:, :C], base[:, :C].to(d)), 'the q columns are not the kernel\'s to write'
    dq2, acc2 = run()
    assert same_bits(dq, dq2) and same_bits(acc, acc2), 'two calls differ'


def test_rows_scatter_add_adds_in_row_order_and_skips_minus_one():
    ops = _ops()
    d = dev()
    g = torch.Generator().manual_seed(9)
    idx = torch.tensor([3, -1, 0, 3, 7, 3, -1, 0], dtype=torch.int32)
    src = torch.randn(8, C, generator=g) * torch.logspace(-4, 4, 8)[:, None]
    dst = torch.randn(10, 3 * C, generator=g)
    want = dst.clone()
    for r in range(8):                                                      # fp32, ascending r: the kernel's order
        if idx[r] >= 0:
            want[idx[r], :C] = want[idx[r], :C] + src[r]
    got = dst.to(d)
    ops.rows_scatter_add(src.to(d), idx.to(d), got[:, :C])
    assert same_bits(got, want.to(d))
    got2 = dst.to(d)
    ops.rows_scatter_add(src.to(d), idx.to(d), got2[:, :C])
    assert same_bits(got, got2)


def _pp_chain_oracle(m, raw, first, wins, dpred, dtype):
    """autograd of oracle.mmpi_pp.DeepInteractionPlusPlusDecoder._mmpi's centre and fallback chain (:281-302), its blocks
    and heads replaced by the given rows: raw [L, M, NP] (each pred_head's output), first [M, NP] (prediction_heads[0]'s
    rows with the query position added), wins: per image layer the product's win [M] -> (d raw, d first)."""
    import oracle.mmpi_pp as ompp
    d = dev()
    L, M, NP = raw.shape
    B, P = M // m.num_proposals, m.num_proposals
    x, f = raw.to(d, dtype).requires_grad_(True), first.to(d, dtype).requires_grad_(True)

    def as_dict(rows):
        t, out, o = rows.view(B, P, NP).permute(0, 2, 1), {}, 0
        for h, n in zip(m.head_order, m.head_sizes):
            out[h] = t[:, o:o + n]
            o += n
        return out
    stub = type('Stub', (), {})()
    stub.num_mmpi = L
    win_it = iter(wins)
    feat = torch.zeros(1, device=d)
    stub.decode_head = [(lambda l: lambda *a: (feat, next(win_it).view(B, P).to(d) if l % 2 == 0 else None))(l) for l in range(L)]
    stub.pred_head = [(lambda l: lambda q: as_dict(x[l]))(l) for l in range(L)]
    aux = dict(layer_query=[])
    with torch.enable_grad():
        fr = as_dict(f)
        rets = ompp.DeepInteractionPlusPlusDecoder._mmpi(stub, feat, dict(fr), fr, None, None, None, None, None, aux)
        tot = 0
        for l, res in enumerate(rets):
            rows = torch.cat([res[h] for h in m.head_order], 1).permute(0, 2, 1).reshape(M, NP)
            tot = tot + (rows * dpred[l].to(d, dtype)).sum()
        tot.backward()
    keeps = [k.reshape(-1) for k in stub.on_the_image_mask]
    return x.grad, f.grad, torch.stack(keeps).int()


@pytest.mark.parametrize('B', [1, 2])
def test_pred_finish_pp_bwd_matches_the_oracle_chain(B):
    from test_gpu_rcnn_backward import _decoder
    ops = _ops()
    d = dev()
    m = _decoder(False, True)
    P, L, NP = m.num_proposals, 4, m.NP
    M = B * P
    g = torch.Generator().manual_seed(40 + B)
    raw, first, dpred = torch.randn(L, M, NP, generator=g), torch.randn(M, NP, generator=g), torch.randn(L, M, NP, generator=g)
    w0 = torch.randint(-1, 2, (M,), generator=g).int()
    w2 = torch.randint(-1, 2, (M,), generator=g).int()
    w2[(w0 >= 0).nonzero()[:3, 0]] = -1                       # rows kept at layer 1 and dropped at layer 2
    want_raw, want_first, keep = _pp_chain_oracle(m, raw, first, [w0, w2], dpred, torch.float64)
    k = keep.cpu()
    assert bool(((k[0] == 1) & (k[2] == 0)).any()) and bool((k[0] == 0).any()) and bool((k[3] == 1).any())
    d_delta, d_first = ops.pred_finish_pp_bwd(dpred.to(d), keep.to(d).contiguous())
    for name, gt, w in (('d_delta', d_delta, want_raw), ('d_first', d_first, want_first)):
        e = rel_err(gt.double().cpu(), w.cpu())
        print('%s %.1e' % (name, e))
        assert e <= 1e-6, (name, e)
    # the look-forward term: row m's centre gradient at layer l also takes keep_{l+1} dpred_{l+1}
    both = (k[0] == 1) & (k[1] == 1)
    assert bool(both.any()) and bool((want_raw[0, both.to(d), :2].cpu() != (dpred[0, both, :2]).double()).all())
    again = ops.pred_finish_pp_bwd(dpred.to(d), keep.to(d).contiguous())
    assert same_bits(again[0], d_delta) and same_bits(again[1], d_first)


# ---------------------------------------------------------------------------------------------------------------------
# 2. the blocks
# ---------------------------------------------------------------------------------------------------------------------
def _sided_ffn(ffn, side, log):
    """forward of a TransFFN (Linear-ReLU-Linear + identity) whose ReLU takes the product's side where side = (rows, h):
    on the selected rows of x (flattened to [n, C]), a pre-activation within 1e-5 max|z| of 0 takes the side of the product's
    hidden rows h; elsewhere the sides must agree."""
    l1, l2 = ffn.layers[0][0], ffn.layers[1]

    def fwd(x):
        z = l1(x)
        on = z > 0
        if side is not None:
            sel, h = side
            n = sel.shape[0]
            zf, onf = z.detach().reshape(n, -1), on.reshape(n, -1)
            theirs, s = h.to(zf.device).reshape(n, -1) > 0, sel.to(zf.device)[:, None]
            near = zf.abs() < 1e-5 * float(zf.abs().max())
            assert bool((~s | near | (onf == theirs)).all()), 'a ReLU side differs away from the kink'
            on = torch.where(s & near, theirs, onf).reshape(z.shape)
            log.append(int((s & near).sum()))
        return l2(z * on.to(z.dtype)) + x
    return fwd


def _saved(m, li, query, pred, maps, metas):
    from deepinteraction_b200 import backward
    d = dev()
    P = m.num_proposals
    bp, sv = m.pack()['blocks'][li], {}
    with backward._precise():
        backward._rcnn_forward(m, bp, query.to(d), pred.to(d), maps.to(d), metas, query.shape[0] // P, P, saved=sv)
    return sv


def _oracle_v2_grads(m, li, query, rois, win, onbits, maps, grad, sv, dtype):
    """autograd through oracle.mmpi_pp's V2 block (ImageRCNNBlockV2 per (sample, live view) group {j : bit v of onbits[j]}
    in ascending order, its output kept on the rows whose win == v; PointRCNNBlockV2 per sample) with
    oracle.geometry.roi_align on the product's rectangles.  sv: the product's saved values, for the ReLU sides.
    -> (dict of d_query, d_maps and 'grads.<name>', near-kink count)."""
    import oracle.mmpi_pp as ompp
    from oracle.geometry import roi_align
    d = dev()
    image = li % 2 == 0
    P = m.num_proposals
    B = query.shape[0] // P
    V = m.num_views if image else 1
    blk = (ompp.ImageRCNNBlockV2(m.num_views, P, m.out_size_factor_img, None, None, C, H, 0.1) if image
           else ompp.PointRCNNBlockV2(C, H, 0.1, None))
    blk.load_state_dict(m.decode_head[li].state_dict(), strict=True)
    blk = blk.to(device=d, dtype=dtype).eval()
    q = query.to(d, dtype).requires_grad_(True)
    fm = maps.to(d, dtype).permute(0, 3, 1, 2).contiguous().requires_grad_(True)
    f, fs, log = sv['f'], sv['fs'], []
    with torch.enable_grad():
        tot = 0
        for b in range(B):
            for v in range(V):
                if image:
                    grp = (((onbits >> v) & 1) == 1).nonzero().squeeze(1)
                    grp = grp[(grp >= b * P) & (grp < (b + 1) * P)]
                    if len(grp) == 0:
                        continue
                    won = win[grp] == v
                    rect = torch.where(won[:, None], rois[grp, 1:].double(), torch.tensor([1.0, 2.0, 30.0, 20.0], dtype=torch.float64))
                    roi = roi_align(fm[b * V + v], rect.to(d, dtype), 7, 1.0 / m.out_size_factor_img, 2)
                else:
                    grp = torch.arange(b * P, (b + 1) * P)
                    won = torch.ones(P, dtype=torch.bool)
                    roi = roi_align(fm[b], rois[grp, 1:].to(d, dtype), 7, 1.0, 2)
                lead = torch.zeros(len(grp), dtype=torch.bool)
                lead[0] = True
                blk.ffn.forward = _sided_ffn(blk.ffn, (won, f[grp.to(d)]), log)
                blk.self_ffn.forward = _sided_ffn(blk.self_ffn, (lead, fs[b * V + v].expand(len(grp), -1)), log)
                out = blk._tail(q[grp.to(d)].unsqueeze(1), roi)
                sel = won.to(d)
                tot = tot + (out[sel] * grad[grp].to(d, dtype)[sel]).sum()
        tot.backward()
    res = {'d_query': q.grad, 'd_maps': fm.grad.permute(0, 2, 3, 1)}
    res.update({'grads.' + n: p.grad for n, p in blk.named_parameters()})
    return res, sum(log)


def _image_draw(m, li, B, seed):
    """Image-block inputs (test_gpu_image_rcnn_backward's draw, every DynamicConv ReLU pre-activation 1e-6 from 0); with
    6 views query 1 sits in the overlap of views 0 and 1, so it leads both and its win is view 1."""
    from test_gpu_image_rcnn_backward import _block_inputs, _product_groups, _relu_margin
    tc = m.test_cfg
    cell, off = tc['out_size_factor'] * tc['voxel_size'][0], tc['pc_range'][0]
    for s in range(seed, seed + 64):
        query, pred, img, grad, metas = _block_inputs(m, B, s)
        if m.num_views == 6:
            az = 30.0 * math.pi / 180
            pred[1, 0], pred[1, 1], pred[1, 2] = (40 * math.cos(az) - off) / cell, (40 * math.sin(az) - off) / cell, -0.5
        rois, win, onbits = _product_groups(m, pred, metas, B)
        if _relu_margin(m, li, query, pred, img, metas, win) > 1e-6:
            return (query, pred, img, grad, metas), rois, win, onbits
    raise AssertionError('no draw with every DynamicConv ReLU pre-activation 1e-6 from 0 in 64 seeds')


def _point_draw(m, li, B, seed):
    from test_gpu_rcnn_backward import _block_inputs, _relu_margin
    for s in range(seed, seed + 64):
        query, pred, bev, grad = _block_inputs(m, B, s)
        if _relu_margin(m, li, query, pred, bev) > 1e-6:
            return query, pred, bev, grad
    raise AssertionError('no draw with every DynamicConv ReLU pre-activation 1e-6 from 0 in 64 seeds')


def _leader_coverage(sv, win, onbits, B, P, V):
    """-> dict: queries on 2+ live views, queries leading 2+ views, leaders whose win is another view, live groups in
    which no query wins, rows with win < 0."""
    from test_gpu_image_rcnn_backward import _coverage
    cov = _coverage(win, onbits, B, P, V)
    lrow = sv['lrow'].cpu().long()
    live = lrow[lrow >= 0]
    cov['double_leaders'] = int(live.numel() - live.unique().numel())
    cov['leader_wins_elsewhere'] = sum(int(lrow[g]) >= 0 and int(win[lrow[g]]) != g % V for g in range(B * V))
    return cov


@pytest.mark.parametrize('li', [0, 1, 2, 3])
@pytest.mark.parametrize('base_shape', [False, True], ids=['small', 'base_shape'])
def test_rcnn_v2_backward_matches_oracle_autograd(base_shape, li):
    from test_gpu_rcnn_backward import _decoder
    from deepinteraction_b200 import backward
    d = dev()
    m = _decoder(base_shape, True)
    B, P, V = (1 if base_shape else 2), m.num_proposals, m.num_views
    image = li % 2 == 0
    if image:
        (query, pred, maps, grad, metas), rois, win, onbits = _image_draw(m, li, B, 500 + 10 * li + base_shape)
        r = backward.image_rcnn_v2_backward(m, li, query.to(d), pred.to(d), maps.to(d), metas, grad.to(d))
        got = dict(d_query=r['d_query'], d_maps=r['d_img'])
    else:
        query, pred, maps, grad = _point_draw(m, li, B, 500 + 10 * li + base_shape)
        metas = None
        r = backward.point_rcnn_v2_backward(m, li, query.to(d), pred.to(d), maps.to(d), grad.to(d))
        got = dict(d_query=r['d_query'], d_maps=r['d_bev'])
    sv = _saved(m, li, query, pred, maps, metas)
    if not image:
        rois, win, onbits = sv['rois'].cpu(), sv['win'].cpu().long(), sv['onbits'].cpu().long()
    got.update({'grads.' + n: t for n, t in r['grads'].items()})
    if image:
        cov = _leader_coverage(sv, win, onbits, B, P, V)
        print(cov)
        assert cov['no_view'] > 0
        if base_shape:
            assert cov['multi_view'] > 0 and cov['double_leaders'] > 0 and cov['leader_wins_elsewhere'] > 0
            assert cov['idle_groups'] > 0
    want, near = _oracle_v2_grads(m, li, query, rois, win, onbits, maps, grad, sv, torch.float64)
    f32, _ = _oracle_v2_grads(m, li, query, rois.float(), win, onbits, maps, grad, sv, torch.float32)
    print('ffn / self_ffn ReLU elements within 1e-5 of the kink: %d' % near)
    sd = m.decode_head[li].state_dict()
    assert set(got) == set(want) and len(r['grads']) == 32 == len(sd)
    for k, w in want.items():
        if k.startswith('grads.'):
            assert got[k].shape == sd[k[6:]].shape, k
        e, bar = _bar(got[k], w, f32[k], TOL)
        print('%-45s %.1e (bar %.1e)' % (k, e, bar))
        assert e <= bar, (k, e, bar)
    if image:
        assert bool((r['d_query'][(win < 0).to(d)] == 0).all()), 'd_query of a query on no live view is not exactly 0'
    # repeat calls give the same bits
    if image:
        r2 = backward.image_rcnn_v2_backward(m, li, query.to(d), pred.to(d), maps.to(d), metas, grad.to(d))
    else:
        r2 = backward.point_rcnn_v2_backward(m, li, query.to(d), pred.to(d), maps.to(d), grad.to(d))
    assert same_bits(r2['d_query'], r['d_query']) and all(same_bits(r2['grads'][k], t) for k, t in r['grads'].items())


# ---------------------------------------------------------------------------------------------------------------------
# 3. autograd.Function, synchronisation, rejections
# ---------------------------------------------------------------------------------------------------------------------
def test_rcnn_v2_functions_forward_is_the_block_and_backward_matches():
    from test_gpu_rcnn_backward import _decoder
    from deepinteraction_b200 import backward
    from tools.make_goldens import small_frame
    m = _decoder(False, True)
    gen = torch.Generator().manual_seed(1811)
    fr = small_frame(1811, aug=True, views=2, batch=2)
    nhwc = lambda t: t.permute(0, 2, 3, 1).contiguous().to(dev())
    pts, new_pts = nhwc(torch.randn(2, 128, 36, 36, generator=gen)), nhwc(torch.randn(2, 128, 36, 36, generator=gen))
    img = nhwc(torch.randn(4, 128, 28, 50, generator=gen))
    dbg = {}
    out = m.forward_rows(pts, new_pts, img, fr['img_metas'], debug=dbg)
    qs = [dbg['query_feat1']] + dbg['layer_query']
    preds = [dbg['first_res']] + out['preds']
    for li in range(4):
        q0 = qs[li].clone().requires_grad_(True)
        image = li % 2 == 0
        maps = (img if image else new_pts).clone().requires_grad_(True)
        with torch.enable_grad():
            if image:
                y = backward.ImageRCNNV2Function.apply(m, li, q0, preds[li], maps, fr['img_metas'])
            else:
                y = backward.PointRCNNV2Function.apply(m, li, q0, preds[li], maps)
            assert same_bits(y.detach(), qs[li + 1]), li
            grad = torch.randn(y.shape, generator=gen).to(dev())
            (y * grad).sum().backward()
        if image:
            r = backward.image_rcnn_v2_backward(m, li, qs[li], preds[li], img, fr['img_metas'], grad)
            dm = r['d_img']
        else:
            r = backward.point_rcnn_v2_backward(m, li, qs[li], preds[li], new_pts, grad)
            dm = r['d_bev']
        assert same_bits(q0.grad, r['d_query']) and same_bits(maps.grad, dm), li


def test_rcnn_v2_backward_rejects_v1_blocks_other_kinds_and_shapes():
    from test_gpu_rcnn_backward import _decoder
    from test_gpu_image_rcnn_backward import _block_inputs
    from deepinteraction_b200 import backward
    d = dev()
    mpp, m = _decoder(False, True), _decoder(False)
    query, pred, img, grad, metas = _block_inputs(m, 2, 5)
    query, grad, img = query.to(d), grad.to(d), img.to(d)
    pred = pred[:, :mpp.NP].contiguous().to(d)
    bev = torch.randn(2, m.y_size, m.x_size, C, device=d)
    image_cases = [(mpp, li, query, grad) for li in (1, 3)] + [(m, li, query, grad) for li in (0, 2)]
    image_cases += [(mpp, 0, query.repeat(13, 1), grad.repeat(13, 1)), (mpp, 0, query[:, :64].contiguous(), grad[:, :64].contiguous())]
    point_cases = [(mpp, li, query, grad) for li in (0, 2)] + [(m, li, query, grad) for li in (1, 3)]
    m.pack()
    mpp.pack()
    with record_calls() as calls:
        for dec, li, q, gr in image_cases:
            p = pred.repeat(q.shape[0] // pred.shape[0], 1) if q.shape[0] != pred.shape[0] else pred
            with pytest.raises(NotImplementedError, match='ImageRCNNBlock'):
                backward.image_rcnn_v2_backward(dec, li, q, p, img, metas, gr)
            with pytest.raises(NotImplementedError, match='ImageRCNNBlock'):
                backward.ImageRCNNV2Function.apply(dec, li, q, p, img, metas)
        for dec, li, q, gr in point_cases:
            with pytest.raises(NotImplementedError, match='PointRCNNBlock'):
                backward.point_rcnn_v2_backward(dec, li, q, pred, bev, gr)
            with pytest.raises(NotImplementedError, match='PointRCNNBlock'):
                backward.PointRCNNV2Function.apply(dec, li, q, pred, bev)
    assert calls == [], calls


def test_rcnn_v2_backward_does_not_synchronise():
    from test_gpu_rcnn_backward import _decoder
    from test_gpu_image_rcnn_backward import _block_inputs
    from deepinteraction_b200 import backward
    m = _decoder(False, True)
    d = dev()
    query, pred, img, grad, metas = _block_inputs(m, 2, 6)
    args = (query.to(d), pred[:, :m.NP].contiguous().to(d), img.to(d), metas, grad.to(d))
    bev = torch.randn(2, m.y_size, m.x_size, C, device=d)
    backward.image_rcnn_v2_backward(m, 0, *args)               # warm-up: builds the per-pack tensors
    backward.point_rcnn_v2_backward(m, 1, args[0], args[1], bev, args[4])
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode('error')
    try:
        r = backward.image_rcnn_v2_backward(m, 0, *args)
        rp = backward.point_rcnn_v2_backward(m, 1, args[0], args[1], bev, args[4])
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
    assert bool(torch.isfinite(r['d_img']).all()) and bool(torch.isfinite(rp['d_bev']).all())
