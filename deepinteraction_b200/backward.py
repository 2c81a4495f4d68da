"""Backward of LocalContextAttentionBlock, of the encoder and of the decoder's query x BEV transformer layer on libdi_b200 (SURVEY.md 8(b) `di_lcab_backward`, the training side of the
hot module; forward: mmri.lcab_forward / di_lcab_forward_f32).

Reference: models/utils/encoder_utils.py:36-81 (autograd Functions around the window ops: similar_backward x 2,
weighting_backward_ori, weighting_backward_weight), :119-135 (the block), ops/locatt_ops kernels.cuh:44-119.

Scope: gradients of the block with BatchNorm in EVAL mode (running statistics, folded into the 1x1 convolutions -- the
form the forward kernels use): d/d target map, d/d source map, d/d folded weight and bias of the five Conv+BN layers.
The gradient of a folded weight maps to the convolution weight by the BN scale (dW_conv = dW_folded * gamma / sqrt(var +
eps)), and d beta = d bias_folded.  Train-mode BatchNorm (batch statistics with their own gradient) and dropout are not
covered.  The intermediates are recomputed in fp32 (q1, k1, q, k, v and the [P, 81] attention weights), the window
products run in the unfused kernels of csrc/lcab_bwd.cu, dense products on the wgmma / FFMA GEMMs.
"""
import contextlib

import torch

from . import fold, geom, ops


@contextlib.contextmanager
def _precise():
    """Gradient products run on the 3xTF32 split (error ~1e-7 per product) rather than the bf16 split of the inference
    path (~1e-5): the backward chains a dozen products per layer.  A context manager and a decorator; it nests (each use
    restores the mode it found) and restores the mode when the body raises."""
    saved, ops.TC_BF16[0] = ops.TC_BF16[0], False
    try:
        yield
    finally:
        ops.TC_BF16[0] = saved


def _transposed(w):
    """Weight [N, K] on the device (a fold.Weight or a tensor of any float type) -> fold.Weight [K, N] of the dX product
    dx = dy W, its splits built on first use."""
    w = getattr(w, 'w', w).detach()
    return fold.Weight(w.t().contiguous(), w.device, lazy=True)


_ONE = {}


def _add(a, b):
    """a + b on the device; None stands for zero."""
    if a is None or b is None:
        return b if a is None else a
    if a.device not in _ONE:
        _ONE[a.device] = torch.ones(1, device=a.device)
    return ops.axpy(a.contiguous(), b.contiguous(), _ONE[a.device])


_MINUS_ONE = {}


def _sub(a, b):
    """a - b on the device."""
    if a.device not in _MINUS_ONE:
        _MINUS_ONE[a.device] = torch.full((1,), -1.0, device=a.device)
    return ops.axpy(a.contiguous(), b.contiguous(), _MINUS_ONE[a.device])


def _bw_pack(pk):
    """Transposed weights for the dX products, built once per pack."""
    if '_bw' not in pk:
        pk['_bw'] = dict(q2=_transposed(pk['w_q2']), k2=_transposed(pk['w_k2']), q1=_transposed(pk['w_q1']),
                         kv1=_transposed(pk['w_kv1']), self1=_transposed(pk['w_self']))
    return pk['_bw']


def _wgrad(dy, x):
    """dy [M, N], x [M, K] (contiguous rows) -> dy^T x [N, K]: both operands transposed to channel-major, then a split-K
    product over the M pixels with a fixed-order sum of the partials."""
    M = dy.shape[0]
    dyt = ops.nhwc_to_nchw(dy.view(1, M, 1, dy.shape[1])).view(dy.shape[1], M)
    xt = ops.nhwc_to_nchw(x.view(1, M, 1, x.shape[1])).view(x.shape[1], M)
    splits = max(1, min(256, M // 512))
    if splits == 1:
        return ops.linear([dyt], xt)
    part = ops.linear([dyt], xt, splits=splits)
    return ops.rows_finish(part) if part.shape[0] > 1 else part[0]


def _layer_grads(dy, *xs):
    """Parameter gradients of the dense layer y = cat(xs, 1) W^T + b from its output gradient dy [M, N] and its inputs
    [M, K_i] -> (dW [N, sum K_i], db [N])."""
    dW = [_wgrad(dy, x.contiguous()) for x in xs]
    return (dW[0] if len(dW) == 1 else torch.cat(dW, 1)), ops.col_sum(dy)


def _window_backward(q, k, v, A, dO, dims, ks, scale):
    """Backward of out = gather(A, v), A = softmax(scale * dot(q, k)) over the ks x ks windows of a dims = (N, H, W) map:
    q / k / v / dO [N*H*W, C] rows, A [N*H*W, ks*ks] -> (dq, dk, dv)."""
    dA = ops.win_dot(dO, v, *dims, ks)
    dv = ops.win_scatter(A, dO, *dims, ks)
    dS = ops.win_softmax_bwd(A, dA, scale)
    return ops.win_gather(dS, k, *dims, ks), ops.win_scatter(dS, q, *dims, ks), dv


@_precise()
def lcab_backward(pk, target, source, N, H, W, grad_out):
    """target / source / grad_out: [N*H*W, C] fp32 pixel-major rows (same tensor object for target and source = self
    attention).  -> dict(d_target, d_source (None for self attention: summed into d_target), and per layer name in
    (q1, q2, k1, k2, v) a pair (dW_folded [C, C], db_folded [C]))."""
    C, ks = pk['C'], pk['ks']
    bw = _bw_pack(pk)
    self_attn = target is source
    x_t, x_s, dO = target.contiguous(), source.contiguous(), grad_out.contiguous()
    R = ops.ACT_RELU
    # forward intermediates in fp32 rows
    if self_attn:
        t = ops.linear([x_s], pk['w_self'], pk['b_self'], R)
        q1, k1, v = t[:, :C].contiguous(), t[:, C:2 * C].contiguous(), t[:, 2 * C:].contiguous()
    else:
        q1 = ops.linear([x_t], pk['w_q1'], pk['b_q1'], R)
        t = ops.linear([x_s], pk['w_kv1'], pk['b_kv1'], R)
        k1, v = t[:, :C].contiguous(), t[:, C:].contiguous()
    q = ops.linear([q1], pk['w_q2'], pk['b_q2'], R)
    k = ops.linear([k1], pk['w_k2'], pk['b_k2'], R)
    scale = 1.0 / float(C) ** 0.5
    A = ops.win_softmax(ops.win_dot(q, k, N, H, W, ks), scale)
    dq, dk, dv = _window_backward(q, k, v, A, dO, (N, H, W), ks, scale)
    # projections: ReLU masks from the saved outputs, dX on the GEMM kernels, dW as split-K products, db as column sums
    g = {}
    dq = ops.relu_bwd(dq, q)
    dk = ops.relu_bwd(dk, k)
    dv = ops.relu_bwd(dv, v)
    g['q2'] = _layer_grads(dq, q1)
    g['k2'] = _layer_grads(dk, k1)
    dq1 = ops.relu_bwd(ops.linear([dq], bw['q2']), q1)
    dk1 = ops.relu_bwd(ops.linear([dk], bw['k2']), k1)
    g['q1'] = _layer_grads(dq1, x_t)
    g['k1'] = _layer_grads(dk1, x_s)
    g['v'] = _layer_grads(dv, x_s)
    if self_attn:
        d_t, d_s = ops.linear([dq1, dk1, dv], bw['self1']), None
    else:
        d_t, d_s = ops.linear([dq1], bw['q1']), ops.linear([dk1, dv], bw['kv1'])
    return dict(d_target=d_t, d_source=d_s, **g)


@_precise()
def i2p_backward(i2p_pack, pts_nhwc, img_nhwc, pts_metas, proj, V, in_hw, grad_out, dropout=None):
    """Backward of the MMRI_I2P block as the product evaluates it (mmri.DeepInteractionEncoder.i2p; reference
    encoder_utils.py:216-320): rows = pts[coors]; qk = M1 rows + c1; s = attend(qk, image samples); o = M2 s + c2;
    out[coors] = o where a pillar saw >= 1 sample.  i2p_pack = (M1, c1, M2, c2) folded from nn.MultiheadAttention
    (fold.i2p_fold); proj: [B, V, 12] device camera rows (mmri.Geometry.proj).  grad_out [B, Y, X, C].
    -> dict(d_pts [B,Y,X,C], d_img [B*V,h,w,C], dM1, dc1, dM2, dc2); fold.i2p_unfold_grads maps the last four to the
    attention module's own parameters.  dropout = (p, seed): the training-mode attention dropout the forward used."""
    M1, c1, M2, c2 = i2p_pack
    coors = pts_metas['pillar_coors']
    pillars, npts = pts_metas['pillars'], pts_metas['pillars_num_points']
    d_pts = torch.zeros_like(pts_nhwc)
    d_img = torch.zeros_like(img_nhwc)
    if coors.shape[0] == 0:
        z = lambda t: torch.zeros_like(t.w if hasattr(t, 'w') else t)
        return dict(d_pts=d_pts, d_img=d_img, dM1=z(M1), dc1=z(c1), dM2=z(M2), dc2=z(c2))
    dev = pts_nhwc.device
    # a plain tensor (the [C, C + 4] output weight of the dropout form) stays on the FFMA path
    M2t = _transposed(M2) if hasattr(M2, 'w') else M2.detach().t().contiguous()
    # forward intermediates
    rows = ops.gather_rows(pts_nhwc, coors)
    qk = ops.linear([rows], M1, c1)
    s, cnt = ops.i2p_attend(qk, pillars, npts, coors, proj, img_nhwc, V, in_hw, dropout=dropout)
    # out = scatter(M2 s + c2) at pillars with cnt > 0
    do = ops.gather_rows_masked(grad_out.contiguous(), cnt, coors)
    dM2, dc2 = _layer_grads(do, s)
    ds = ops.linear([do], M2t)
    dqk = ops.i2p_attend_bwd(qk, ds, pillars, npts, coors, proj, img_nhwc, d_img, V, in_hw, dropout)
    dM1, dc1 = _layer_grads(dqk, rows)
    drows = ops.linear([dqk], _transposed(M1))
    ones = torch.ones(coors.shape[0], device=dev, dtype=torch.int32)
    ops.scatter_rows(drows, ones, coors, d_pts)             # one pillar per BEV cell: a plain store
    return dict(d_pts=d_pts, d_img=d_img, dM1=dM1, dc1=dc1, dM2=dM2, dc2=dc2)


def conv3x3_wgrad(x_nchw, g_rows, cout):
    """dW [Cout, Cin, 3, 3] and db of a 3x3 convolution: per tap a split-K product of the output gradient with the shifted
    input (dW[co, ci, ky, kx] = sum_p dY[p, co] X[p + (ky - 1, kx - 1), ci])."""
    return _conv3x3_wgrad_nhwc(ops.nchw_to_nhwc(x_nchw.contiguous()), g_rows, cout)


def _conv3x3_wgrad_nhwc(x_nhwc, g_rows, cout):
    """conv3x3_wgrad of a pixel-major input [N, H, W, Cin]."""
    cin = x_nhwc.shape[-1]
    dw = torch.empty(cout, cin, 3, 3, device=x_nhwc.device)
    for ky in range(3):
        for kx in range(3):
            xs = ops.shift_map(x_nhwc, ky - 1, kx - 1).view(-1, cin)
            dw[:, :, ky, kx] = _wgrad(g_rows, xs)
    return dw, ops.col_sum(g_rows)


def _encoder_geometry(enc, img_feats, pts_feats, img_metas, pts_metas):
    """Common start of the two encoder steps -> (V, pm, g): views per sample, pts_metas in the schedule's canonical form on
    the device (with the raw points, which the geometry reads) and the frame's mmri.Geometry, finished."""
    from . import mmri
    dev = img_feats.device
    (BV, _, h, w), (B, _, Y, X) = img_feats.shape, pts_feats.shape
    pm = enc._canon_pts_metas(pts_metas, dev)
    pm['pts'] = [p.to(dev) for p in pts_metas['pts']]
    g = mmri.Geometry(img_metas, pm, (h, w), (Y, X), dev)
    g.wait()
    return BV // B, pm, g


def _seed_rows(d_out, like):
    """Gradient of an output map as rows [M, C] (None = zero), the shape of the map `like` [..., C]."""
    C = like.shape[-1]
    return d_out.reshape(-1, C).contiguous() if d_out is not None else torch.zeros(like.numel() // C, C, device=like.device)


def _shared_conv_backward(g_rows, w_packed, x_nchw):
    """Backward of a shared 3x3 convolution y = conv3x3(x) from d y as rows [N*H*W, Cout] -> (d x [N, H, W, Cin],
    (dW [Cout, Cin, 3, 3], db)).  d x = conv3x3(d y, W^T flipped): the packed forward weight [Cout, (ky*3+kx)*Cin + ci]
    becomes the packed weight [Cin, (ky*3+kx)*Cout + co] with the taps flipped, on the device."""
    N, cin, H, W = x_nchw.shape
    cout = w_packed.shape[0]
    dx = ops.conv3x3(g_rows.view(N, H, W, cout), _flipped(w_packed), None, cout=cin, x_nhwc=True)
    return dx, conv3x3_wgrad(x_nchw, g_rows, cout)


def _flipped(w_packed, cout=None):
    """Packed 3x3 weight [Cout, (ky*3+kx)*Cin + ci] -> fold.Weight [Cin, (ky*3+kx)*cout + co] of the transposed convolution,
    taps flipped, on the device; cout > Cout pads the output channels of the forward with zero rows."""
    w = w_packed.w.detach()
    co, cin = w.shape[0], w.shape[1] // 9
    if cout is not None and cout > co:
        w = torch.cat([w, torch.zeros(cout - co, w.shape[1], device=w.device, dtype=w.dtype)], 0)
    cout = w.shape[0]
    wt = w.view(cout, 3, 3, cin).flip(1, 2).permute(3, 1, 2, 0).reshape(cin, 9 * cout)   # co, ky, kx, ci -> ci, ky', kx', co
    return fold.Weight(wt.contiguous(), w.device, lazy=True)


def _fuse_bw_pack(lp):
    """Transposed weights of the two fuse layers of an encoder layer pack, built once per pack."""
    if '_bw' not in lp:
        lp['_bw'] = dict(i_fuse=_transposed(lp['i_fuse'][0]), p_fuse=_transposed(lp['p_fuse'][0]))
    return lp['_bw']


@_precise()
def encoder_backward(enc, img_feats, pts_feats, img_metas, pts_metas, d_img, d_pts_conv, d_pts):
    """Backward of DeepInteractionEncoder.forward (base model, hidden width 128, BatchNorm in eval mode = the folded
    weights of the forward; reference deepinteraction_encoder.py:8-85).  img_feats (B*V, Ci, h, w), pts_feats
    (B, Cp, Y, X): the module's NCHW inputs on the GPU; pts_metas with pillars; d_img [B*V, h, w, C], d_pts_conv / d_pts
    [B, Y, X, C]: gradients of the three outputs (pixel-major; None = zero).
    -> dict(d_img_feats [B*V, h, w, Ci], d_pts_feats [B, Y, X, Cp] (pixel-major), layers = per encoder layer the folded
    parameter gradients: i2p (dM1, dc1, dM2, dc2), p_iml / p2i / i_iml (lcab_backward dicts), p_fuse / i_fuse (dW [C, 3C], db)).
    shared_conv = dict(img / pts -> (dW [C, Cin, 3, 3], db)).  The forward is re-run eagerly with its intermediates kept."""
    from . import mmri
    pk = enc.pack()
    C = enc.hidden_channel
    (BV, _, h, w), (B, _, Y, X) = img_feats.shape, pts_feats.shape
    V, pm, g = _encoder_geometry(enc, img_feats, pts_feats, img_metas, pts_metas)
    # ---- forward with saved intermediates
    img = ops.conv3x3(img_feats.contiguous(), *pk['shared_conv_img'], cout=C, x_nhwc=False)
    pts = ops.conv3x3(pts_feats.contiguous(), *pk['shared_conv_pts'], cout=C, x_nhwc=False)
    saved = []
    for lp in pk['layers']:
        img_r, pts_r = img.view(-1, C), pts.view(-1, C)
        i2p = enc.i2p(lp, pts, img, pm, g)
        p2p = mmri.lcab_forward(lp['p_iml'], pts_r, pts_r, B, Y, X)
        new_pts = ops.linear([i2p.view(-1, C), p2p, pts_r], *lp['p_fuse']).view(B, Y, X, C)
        warped = ops.bev_sample(pts, g.grid, V)
        p2i = mmri.lcab_forward(lp['p2i'], img_r, warped.view(-1, C), BV, h, w)
        i2i = mmri.lcab_forward(lp['i_iml'], img_r, img_r, BV, h, w)
        new_img = ops.linear([p2i, i2i, img_r], *lp['i_fuse']).view(BV, h, w, C)
        saved.append(dict(img=img, pts=pts, i2p=i2p, p2p=p2p, warped=warped, p2i=p2i, i2i=i2i))
        img, pts = new_img, new_pts
    # ---- backward
    gi, gp = _seed_rows(d_img, img), _seed_rows(d_pts, pts)
    layer_grads = []
    for lp, sv in zip(reversed(pk['layers']), reversed(saved)):
        img_r, pts_r = sv['img'].view(-1, C), sv['pts'].view(-1, C)
        lg = {}
        # fuse convolutions: new = Wf [a | b | c] + bf
        bw = _fuse_bw_pack(lp)
        di3 = ops.linear([gi], bw['i_fuse'])                           # [M_i, 3C] = d p2i | d i2i | d img (direct)
        dp3 = ops.linear([gp], bw['p_fuse'])                           # [M_p, 3C] = d i2p | d p2p | d pts (direct)
        lg['i_fuse'] = _layer_grads(gi, sv['p2i'], sv['i2i'], img_r)
        lg['p_fuse'] = _layer_grads(gp, sv['i2p'].view(-1, C), sv['p2p'], pts_r)
        d_p2i, d_i2i, d_img_dir = (di3[:, k * C:(k + 1) * C].contiguous() for k in range(3))
        d_i2p, d_p2p, d_pts_dir = (dp3[:, k * C:(k + 1) * C].contiguous() for k in range(3))
        # image side
        r_ii = lcab_backward(lp['i_iml'], img_r, img_r, BV, h, w, d_i2i)
        r_pi = lcab_backward(lp['p2i'], img_r, sv['warped'].view(-1, C), BV, h, w, d_p2i)
        r_ip = i2p_backward(lp['i2p'], sv['pts'], sv['img'], pm, g.proj, V, g.in_hw, d_i2p.view(B, Y, X, C))
        r_pp = lcab_backward(lp['p_iml'], pts_r, pts_r, B, Y, X, d_p2p)
        new_gi = _add(_add(_add(d_img_dir, r_ii['d_target']), r_pi['d_target']), r_ip['d_img'].view(-1, C))
        d_bev = ops.bev_sample_bwd(r_pi['d_source'].view(BV, h, w, C).contiguous(), g.grid, V, (B, Y, X, C))
        new_gp = _add(_add(_add(d_pts_dir, r_pp['d_target']), r_ip['d_pts'].view(-1, C)), d_bev.view(-1, C))
        lg.update(i_iml={k: v for k, v in r_ii.items() if not k.startswith('d_')},
                  p2i={k: v for k, v in r_pi.items() if not k.startswith('d_')},
                  p_iml={k: v for k, v in r_pp.items() if not k.startswith('d_')},
                  i2p=(r_ip['dM1'], r_ip['dc1'], r_ip['dM2'], r_ip['dc2']))
        layer_grads.append(lg)
        gi, gp = new_gi, new_gp
    layer_grads.reverse()
    if d_pts_conv is not None:
        gp = _add(gp, d_pts_conv.reshape(-1, C))
    d_img_feats, g_img = _shared_conv_backward(gi, pk['shared_conv_img'][0], img_feats)
    d_pts_feats, g_pts = _shared_conv_backward(gp, pk['shared_conv_pts'][0], pts_feats)
    return dict(d_img_feats=d_img_feats, d_pts_feats=d_pts_feats, layers=layer_grads, shared_conv=dict(img=g_img, pts=g_pts))


class LCABFunction(torch.autograd.Function):
    """autograd wrapper: out = LCAB(target, source) with the inference kernels, input gradients through lcab_backward.
    (Parameter gradients are returned by lcab_backward for the caller's optimiser on the folded weights.)"""

    @staticmethod
    def forward(ctx, pk, target, source, N, H, W):
        from .mmri import lcab_forward
        ctx.pk, ctx.dims, ctx.same = pk, (N, H, W), target is source
        ctx.save_for_backward(target, source)
        return lcab_forward(pk, target, source, N, H, W)

    @staticmethod
    def backward(ctx, grad_out):
        target, source = ctx.saved_tensors
        r = lcab_backward(ctx.pk, target, target if ctx.same else source, *ctx.dims, grad_out)
        return None, r['d_target'], r['d_source'], None, None, None


# ---- decoder: the steps the query x BEV layer and the RCNN blocks share ------------------------------------------------------
def _put(R, *named):
    """Store (module name, (d weight, d bias)) pairs under the modules' state_dict keys."""
    for module, (dW, db) in named:
        R[module + '.weight'], R[module + '.bias'] = dW, db


def _ffn_norm_backward(dy, z, gamma, f, act, x, w2t, w1t):
    """Backward of y = LayerNorm(z), z = x + linear2(f), f = act(linear1(x)) from the saved z, f and x, the norm's weight and
    the transposed weights; act = (ops.relu_bwd, saved output) or (ops.gelu_bwd, saved pre-activation).
    -> (dx, (d gamma, d beta), linear2's (dW, db), linear1's (dW, db)); the residual joins dx in the GEMM epilogue."""
    act_bwd, act_saved = act
    dz, dgamma, dbeta = ops.ln_bwd(dy, z, gamma)
    g2 = _layer_grads(dz, f)
    dh = act_bwd(ops.linear([dz], w2t), act_saved)
    g1 = _layer_grads(dh, x)
    return ops.linear([dh], w1t, res=dz), (dgamma, dbeta), g2, g1


def _self_attn_backward(dz, a, qkv, out_t, B, P, H, onbits=None, win=None):
    """Backward of out_proj(a), a = attention over the P queries of each sample (within the view groups of onbits / win
    when given) with the saved projections qkv [B*P, 3C] -> (d qkv, out_proj's (dW, db)).  The in-projection stays with
    the caller: its sources differ."""
    g_out = _layer_grads(dz, a)
    C = qkv.shape[1] // 3
    da = ops.linear([dz], out_t)
    return ops.mha_small_bwd(qkv[:, :C], qkv[:, C:2 * C], qkv[:, 2 * C:], da, B, P, H, onbits, win), g_out


# ---- decoder: TransformerDecoderLayer (query x BEV) ---------------------------------------------------------------------
def _dec_bw_pack(dec, pk):
    """Transposed weights of the layer's dX products and the constants of fold.decoder_layer_unfold, built once per pack."""
    if '_bw' in pk:
        return pk['_bw']
    layer = dec.decoder[0]
    C = dec.hidden_channel
    T = _transposed
    # the forward's weights as packed: q rows with head_dim^-0.5 folded in, and [W | W] over two sources where the same
    # projection reads a row and its positional embedding
    pk['_bw'] = dict(ffn1=T(pk['ffn'][0]), ffn2=T(pk['ffn'][2]), cross_out=T(pk['cross_out'][0]), self_out=T(pk['self_attn'][2]),
                     cross_q=T(pk['cross_q'][0].w[:, :C]), kv=T(pk['cross_kv'][0]), self_in=T(pk['self_attn'][0].w[:, :C]),
                     spe2=T(pk['self_pe'][2]), cpe2=T(layer.cross_posembed.position_embedding_head[3].weight.flatten(1)),
                     unfold=fold.decoder_layer_unfold_consts(layer, dec.num_heads, pk['bce'].device))
    return pk['_bw']


@_precise()
def decoder_layer_backward(dec, query, query_pos, bev, grad_out):
    """Backward of the decoder's TransformerDecoderLayer (reference models/utils/decoder_utils.py:35-113, 116-495; the call
    self.decoder[0](query_feat, lidar_feat_flatten, query_pos, bev_pos) of deepinteraction_decoder.py), shared by the base
    and the ++ decoder, with BatchNorm in eval mode (the folded weights of the forward) and dropout off.
    dec: DeepInteractionDecoder / DeepInteractionPlusPlusDecoder on the GPU; query [B*P, C] and query_pos [B*P, 2]: the rows
    the forward feeds the layer; bev [B, Y, X, C]: pts_conv (pixel-major); grad_out [B*P, C].
    -> dict(d_query [B*P, C], d_bev [B, Y, X, C] (through K and V), grads = {name: tensor} for the 30 parameters of
    dec.decoder[0], keyed and shaped as in its state_dict).  query_pos gets no gradient (a gather of the constant bev_pos).
    The layer is re-run eagerly with its intermediates kept; everything stays on the device, without host synchronisation
    after the first call of a pack."""
    pk = dec.pack()
    C, H = dec.hidden_channel, dec.num_heads
    B, Y, X, _ = bev.shape
    HW, M = Y * X, query.shape[0]
    P = M // B
    if H != 8 or C != 128 or P > 256 or P * B != M:
        raise NotImplementedError('decoder_layer_backward: the cross-attention gradient kernel takes 8 heads x 16 channels and '
                                  f'P <= 256 queries per sample (got heads={H}, C={C}, rows={M}, B={B})')
    bw = _dec_bw_pack(dec, pk)
    query, query_pos, bev = query.contiguous(), query_pos.contiguous(), bev.contiguous()
    sv = {}
    dec._layer(pk, query, query_pos, bev, B, P, saved=sv)
    R, F = {}, {}
    # norm3, FFN (ReLU)
    dq2, n3, l2, l1 = _ffn_norm_backward(grad_out.contiguous(), sv['z3'], pk['norm3'][0], sv['f'], (ops.relu_bwd, sv['f']),
                                         sv['q2'], bw['ffn2'], bw['ffn1'])
    _put(R, ('norm3', n3), ('linear2', l2), ('linear1', l1))
    # norm2, query x BEV cross attention
    dz2, R['norm2.weight'], R['norm2.bias'] = ops.ln_bwd(dq2, sv['z2'], pk['norm2'][0])
    _put(R, ('multihead_attn.out_proj', _layer_grads(dz2, sv['a2'])))
    da2 = ops.linear([dz2], bw['cross_out'])
    dqc, dkv = ops.xattn_bwd(sv['planes'], sv['a2'], sv['lse'], da2, B, P, HW, H)
    F['cross_q'] = _layer_grads(dqc, torch.cat([sv['q1'], sv['qpe']], 1))
    F['cross_kv'] = _layer_grads(dkv, sv['kk'])
    tq = ops.linear([dqc], bw['cross_q'])               # the [Wq | Wq] pack: the same gradient for q1 and qpe
    d_bev = ops.linear([dkv], bw['kv'])                 # d kk [B*HW, C] = d bev
    # constant key positional embedding: d kpe = sum over the batch of d kk, back through its MLP over the grid positions
    dkpe = d_bev[:HW]
    for b in range(1, B):
        dkpe = _add(dkpe, d_bev[b * HW:(b + 1) * HW])
    cpe = pk['cross_pe']
    dh = ops.relu_bwd(ops.linear([dkpe.contiguous()], bw['cpe2']), cpe['hidden'])
    F['cross_posembed'] = _layer_grads(dh, cpe['pos']) + _layer_grads(dkpe, cpe['hidden'])
    # norm1, self attention over the queries
    dz1, R['norm1.weight'], R['norm1.bias'] = ops.ln_bwd(_add(dz2, tq), sv['z1'], pk['norm1'][0])
    dqkv, g_out = _self_attn_backward(dz1, sv['a1'], sv['qkv'], bw['self_out'], B, P, H)
    _put(R, ('self_attn.out_proj', g_out))
    F['self_in'] = _layer_grads(dqkv, torch.cat([query, sv['qpe']], 1))
    ts = ops.linear([dqkv], bw['self_in'])              # the [W | W] pack: the same gradient for query and qpe
    d_query = _add(dz1, ts)
    dqpe = _add(tq, ts)
    # self positional MLP
    dhs = ops.relu_bwd(ops.linear([dqpe], bw['spe2']), sv['hs'])
    F['self_posembed'] = _layer_grads(dhs, query_pos) + _layer_grads(dqpe, sv['hs'])
    R.update(fold.decoder_layer_unfold(bw['unfold'], F))
    return dict(d_query=d_query, d_bev=d_bev.view(B, Y, X, C), grads=R)


class DecoderLayerFunction(torch.autograd.Function):
    """autograd wrapper: out [B*P, C] = the decoder's TransformerDecoderLayer (the forward schedule's kernels, bit for bit);
    backward -> (d_query, d_bev) through decoder_layer_backward.  Parameter gradients are returned by decoder_layer_backward."""

    @staticmethod
    def forward(ctx, dec, query, query_pos, bev):
        ctx.dec = dec
        ctx.save_for_backward(query, query_pos, bev)
        with _precise():
            pk = dec.pack()
            B = bev.shape[0]
            return dec._layer(pk, query.contiguous(), query_pos.contiguous(), bev.contiguous(), B, query.shape[0] // B)

    @staticmethod
    def backward(ctx, grad_out):
        query, query_pos, bev = ctx.saved_tensors
        r = decoder_layer_backward(ctx.dec, query, query_pos, bev, grad_out)
        return None, r['d_query'], None, r['d_bev']


# ---- decoder: the V1 RCNN blocks, PointRCNNBlock (BEV) and ImageRCNNBlock (camera views) --------------------------------
def _rcnn_bw_pack(dec, bp):
    """Transposed weights of the block's dX products, built once per pack.  The DynamicConv generator's transpose
    [C, 2*128*128] stays a plain tensor: its dX product (K = 32768 over B*P rows) runs as a split-K FFMA product."""
    if '_bw' in bp:
        return bp['_bw']
    C = dec.hidden_channel
    T = _transposed
    s = float(C // dec.num_heads) ** -0.5           # folded into the q rows of the packed in-projection (_pack_mha)
    qscale = torch.cat([torch.full((C,), s, dtype=torch.float64), torch.ones(2 * C, dtype=torch.float64)])
    bw = dict(ffn1=T(bp['ffn'][0]), ffn2=T(bp['ffn'][2]), dout=T(bp['dout'][0]), dyn=bp['dyn'][0].w.t().contiguous(),
              attn_in=T(bp['attn'][0]), attn_out=T(bp['attn'][2]), qscale=fold.dev(qscale, bp['norm1'][0].device))
    if bp['v2']:
        bw.update(sffn1=T(bp['self_ffn'][0]), sffn2=T(bp['self_ffn'][2]))
    bp['_bw'] = bw
    return bw


# the dX product of the DynamicConv generator: d q1 [B*P, C] = d params [B*P, 32768] W_dyn.  The tensor-core GEMM has no
# split-K, and at M ~ 200 - 400 rows and N = 128 it would run on 2 - 4 CTAs over the whole K; 64 splits of 512 give
# 128 - 256 CTAs of the FFMA kernel, reduced in a fixed order by di_rows_finish_f32 together with the residual gradient.
_DYN_SPLITS = 64


def _rcnn_block_of(dec, li, query, maps, image, v2=False):
    """-> (block pack, B, P) of decode_head[li], an ImageRCNNBlock[V2] (image) or PointRCNNBlock[V2] (not image) read from
    maps ([B*V, h, w, C] image maps or the [B, Y, X, C] BEV map); NotImplementedError before any launch for what the
    backward of that block does not cover."""
    fn, kind = ('image_rcnn', 'ImageRCNNBlock') if image else ('point_rcnn', 'PointRCNNBlock')
    fn, kind = (fn + '_v2_backward', kind + 'V2') if v2 else (fn + '_backward', 'V1 ' + kind)
    bp = dec.pack()['blocks'][li]
    if bp['image'] != image or bp['v2'] != v2:
        raise NotImplementedError('%s covers the %s only (decode_head[%d] is %s)'
                                  % (fn, kind, li, type(dec.decode_head[li]).__name__))
    C, M = dec.hidden_channel, query.shape[0]
    B = maps.shape[0] // dec.num_views if image else maps.shape[0]
    P = M // max(B, 1)
    if (C != 128 or maps.shape[3] != C or query.shape[1] != C or P > 512 or P * B != M
            or (image and B * dec.num_views != maps.shape[0])):
        raise NotImplementedError(f'{fn}: the {kind} gradient takes C = 128 and P <= 512 queries per sample '
                                  f'(got C={query.shape[1]}, rows={M}, maps={maps.shape[0]})')
    return bp, B, P


def _bev_roi_params(dec):
    return dec._roi_params((0, 0))          # the image size enters the image-mode RoIs only


def _rcnn_forward(dec, bp, query, pred, maps, img_metas, B, P, saved=None):
    """dec._rcnn_block on the block's maps: the BEV map, or the image maps, whose RoIs also need the camera constants of
    img_metas.  Those go to the device from pinned memory, without a host synchronisation (a pageable source would make
    the copy synchronous)."""
    if not bp['image']:
        return dec._rcnn_block(bp, query, pred, maps, None, B, P, _bev_roi_params(dec), None, None, saved=saved)
    proj, aux = (t.pin_memory().to(maps.device, non_blocking=True) for t in dec._camera_consts(img_metas))
    prm = dec._roi_params(geom.input_hw(img_metas))
    return dec._rcnn_block(bp, query, pred, None, maps, B, P, prm, proj, aux, saved=saved)


def _rcnn_middle_backward(dec, bp, bw, sv, maps, B, P, dq2, masks, R):
    """The section of an RCNN block's backward that V1 and V2 blocks share, from d q2 down: norm2, DynamicConv (norm3 +
    ReLU, out_layer, the dynamic convolution, the parameter generator), RoIAlign, norm1 and the self attention over the
    queries of a sample (within the view groups of masks = (onbits, win) when given).  -> (dz1 [B*P, C]: the gradient
    of norm1's input sum, whose residual part reaches the block's input; dqkv [B*P, 3C]: the gradient of the packed
    in-projection's output; d_maps); the gradients of norm2, dyconv, norm1 and out_proj are stored in R."""
    image = bp['image']
    C, H = dec.hidden_channel, dec.num_heads
    x = '' if image else '_pts'
    dz2, R[f'norm2{x}.weight'], R[f'norm2{x}.bias'] = ops.ln_bwd(dq2, sv['z2'], bp['norm2'][0])
    D = f'dyconv{x}.'
    dzd3, R[D + 'norm3.weight'], R[D + 'norm3.bias'] = ops.ln_bwd(ops.relu_bwd(dz2, sv['t']), sv['zd3'], bp['dn3'][0])
    _put(R, (D + 'out_layer', _layer_grads(dzd3, sv['flat'])))
    d_roi, d_params, d_norm = ops.dynconv_bwd(sv['roi'], sv['params'], *bp['dn1'], *bp['dn2'], ops.linear([dzd3], bw['dout']))
    dn = ops.col_sum(d_norm).view(4, C)
    R[D + 'norm1.weight'], R[D + 'norm1.bias'], R[D + 'norm2.weight'], R[D + 'norm2.bias'] = dn.unbind(0)
    _put(R, (D + 'dynamic_layer', _layer_grads(d_params, sv['q1'])))
    dq1 = ops.rows_finish(ops.linear([d_params], bw['dyn'], splits=_DYN_SPLITS), res=dz2)
    d_maps = ops.roi_align_bwd(d_roi, sv['rois'], *maps.shape[:3], 1.0 / dec.out_size_factor_img if image else 1.0)
    dz1, R[f'norm1{x}.weight'], R[f'norm1{x}.bias'] = ops.ln_bwd(dq1, sv['z1'], bp['norm1'][0])
    dqkv, g_out = _self_attn_backward(dz1, sv['a'], sv['qkv'], bw['attn_out'], B, P, H, *masks)
    _put(R, (f'dyconv_pre_self_attn{x}.out_proj', g_out))
    return dz1, dqkv, d_maps


def _in_proj_backward(bp, bw, query, dqkv, dz1, R):
    """The block's input gradient d query = dqkv W_in + dz1 and the in-projection's gradients (into R)."""
    A = 'dyconv_pre_self_attn%s.' % ('' if bp['image'] else '_pts')
    d_query = ops.linear([dqkv], bw['attn_in'], res=dz1)
    # dqkv is the gradient of the packed projection, whose q rows carry head_dim^-0.5
    dW_in, db_in = _layer_grads(dqkv, query)
    R[A + 'in_proj_weight'], R[A + 'in_proj_bias'] = dW_in * bw['qscale'][:, None], db_in * bw['qscale']
    return d_query


def _v1_rcnn_backward(dec, bp, B, P, query, pred, maps, img_metas, grad_out):
    """Backward of a V1 RCNN block (reference models/utils/decoder_utils.py:632-761 image, :765-841 BEV), LayerNorms as
    they are, dropout off -> (d_query, d_maps, grads).  The block is re-run eagerly with its intermediates kept.  The two
    kinds differ where _rcnn_block does: the maps the RoIs read and their scale, the view-group masks (image blocks:
    attention within a view group, rows on no live view written as 0) and the parameter names."""
    image = bp['image']
    query, pred, maps, grad_out = (t.contiguous() for t in (query, pred, maps, grad_out))
    sv = {}
    _rcnn_forward(dec, bp, query, pred, maps, img_metas, B, P, saved=sv)
    bw = _rcnn_bw_pack(dec, bp)
    x = '' if image else '_pts'
    masks = (sv['onbits'], sv['win']) if image else ()
    if image:
        grad_out = ops.rows_finish(grad_out, zero_if_neg=sv['win'])     # the forward writes those rows as 0 by selection
    R = {}
    # norm3, FFN (GELU)
    dq2, n3, l2, l1 = _ffn_norm_backward(grad_out, sv['z3'], bp['norm3'][0], sv['f'], (ops.gelu_bwd, sv['h']), sv['q2'],
                                         bw['ffn2'], bw['ffn1'])
    _put(R, ('norm3' + x, n3), ('linear2' + x, l2), ('linear1' + x, l1))
    dz1, dqkv, d_maps = _rcnn_middle_backward(dec, bp, bw, sv, maps, B, P, dq2, masks, R)
    return _in_proj_backward(bp, bw, query, dqkv, dz1, R), d_maps, R


def _v2_rcnn_backward(dec, bp, B, P, query, pred, maps, img_metas, grad_out):
    """Backward of a V2 RCNN block (reference models/utils/decoder_utils.py:844-991 image, :995-1089 BEV; oracle/mmpi_pp.py),
    LayerNorms as they are, dropout off -> (d_query, d_maps, grads).  out = q3 * scale + s_l * self_scale, where q3 is
    the V1 path up to q2 followed by norm3(q2 + ffn(q2)) (ReLU) and s_l = self_norm(q1_l + self_ffn(q1_l)) is the self
    branch of the FIRST query of the row's (sample, view) group, q1_l = norm1(prev[lead] + out_proj(attention of the
    leader over its group)).  The leader branch shares norm1, out_proj, the in-projection and the group's keys and values
    with the main path, so its gradients are added to the main path's; a query that leads two views gets both."""
    image = bp['image']
    query, pred, maps, grad_out = (t.contiguous() for t in (query, pred, maps, grad_out))
    C, H = dec.hidden_channel, dec.num_heads
    sv = {}
    _rcnn_forward(dec, bp, query, pred, maps, img_metas, B, P, saved=sv)
    bw = _rcnn_bw_pack(dec, bp)
    x = '' if image else '_pts'
    Vg = dec.num_views if image else 1
    R = {}
    # the branch mix: image rows on no live view are written as 0 and take no gradient
    dq3, d_s, R['scale'], R['self_scale'] = ops.branch_mix_bwd(grad_out, sv['q3'], sv['s_l'], sv['win'], bp['scale'],
                                                               bp['self_scale'], P, Vg, image)
    # main path: norm3, FFN (ReLU), then the section V1 blocks share
    dq2, n3, l2, l1 = _ffn_norm_backward(dq3, sv['z3'], bp['norm3'][0], sv['f'], (ops.relu_bwd, sv['f']), sv['q2'],
                                         bw['ffn2'], bw['ffn1'])
    _put(R, ('norm3' + x, n3), ('ffn.layers.1', l2), ('ffn.layers.0.0', l1))
    dz1, dqkv, d_maps = _rcnn_middle_backward(dec, bp, bw, sv, maps, B, P, dq2, (sv['onbits'], sv['win']) if image else (), R)
    # leader branch on the B*Vg leader rows: self_norm, self FFN (ReLU), norm1, out_proj, the group attention
    dq1_l, sn, s2, s1 = _ffn_norm_backward(d_s, sv['zs'], bp['self_norm'][0], sv['fs'], (ops.relu_bwd, sv['fs']), sv['q1_l'],
                                           bw['sffn2'], bw['sffn1'])
    _put(R, ('self_norm' + x, sn), ('self_ffn.layers.1', s2), ('self_ffn.layers.0.0', s1))
    dz1_l, dg, db = ops.ln_bwd(dq1_l, sv['z1_l'], bp['norm1'][0])
    R[f'norm1{x}.weight'], R[f'norm1{x}.bias'] = _add(R[f'norm1{x}.weight'], dg), _add(R[f'norm1{x}.bias'], db)
    A = f'dyconv_pre_self_attn{x}.out_proj.'
    dW, db = _layer_grads(dz1_l, sv['a_l'])
    R[A + 'weight'], R[A + 'bias'] = _add(R[A + 'weight'], dW), _add(R[A + 'bias'], db)
    da_l = ops.linear([dz1_l], bw['attn_out'])
    qkv = sv['qkv']
    dq_l = ops.mha_small_rows_bwd(qkv[:, :C], qkv[:, C:2 * C], qkv[:, 2 * C:], da_l, B, P, H, sv['onbits'], sv['lrow'],
                                  sv['lwin'], dqkv[:, C:2 * C], dqkv[:, 2 * C:])
    ops.rows_scatter_add(dq_l, sv['lrow'], dqkv[:, :C])           # the leader's own query row
    ops.rows_scatter_add(dz1_l, sv['lrow'], dz1)                  # norm1's residual: prev[lead]
    return _in_proj_backward(bp, bw, query, dqkv, dz1, R), d_maps, R


@_precise()
def point_rcnn_backward(dec, li, query, pred, bev, grad_out):
    """Backward of the base decoder's PointRCNNBlock (reference models/utils/decoder_utils.py:765-841; dec.decode_head[li],
    li = 1 or 3 in the base configuration), LayerNorms as they are, dropout off.
    dec: DeepInteractionDecoder on the GPU; query [B*P, C]: the rows the block reads; pred [B*P, NP]: the prediction rows its
    RoIs come from (di_rcnn_rois_f32, BEV mode); bev [B, Y, X, C]: new_pts (pixel-major); grad_out [B*P, C].
    -> dict(d_query [B*P, C], d_bev [B, Y, X, C] (through RoIAlign), grads = {name: tensor} for the 24 parameters of
    dec.decode_head[li], keyed and shaped as in its state_dict).  The RoIs are constants (the reference computes them
    from detached predictions), so pred gets no gradient.  The block is re-run eagerly with its intermediates kept;
    everything stays on the device, without host synchronisation after the first call of a pack."""
    bp, B, P = _rcnn_block_of(dec, li, query, bev, False)
    d_query, d_bev, R = _v1_rcnn_backward(dec, bp, B, P, query, pred, bev, None, grad_out)
    return dict(d_query=d_query, d_bev=d_bev, grads=R)


@_precise()
def image_rcnn_backward(dec, li, query, pred, img, img_metas, grad_out):
    """Backward of the base decoder's ImageRCNNBlock (reference models/utils/decoder_utils.py:632-761; dec.decode_head[li],
    li = 0 or 2 in the base configuration), LayerNorms as they are, dropout off.
    dec: DeepInteractionDecoder on the GPU; query [B*P, C]: the rows the block reads; pred [B*P, NP]: the prediction rows its
    RoIs come from (di_rcnn_rois_f32, image mode); img [B*V, h, w, C]: the image maps (pixel-major, as forward_rows takes
    them); img_metas: the frame's camera metadata; grad_out [B*P, C].
    -> dict(d_query [B*P, C], d_img [B*V, h, w, C] (through RoIAlign at 1 / out_size_factor_img), grads = {name: tensor}
    for the 24 parameters of dec.decode_head[li], keyed and shaped as in its state_dict).  A query with win = w >= 0 (the
    last live view it is on) attends over the queries of its sample on view w and reads its RoI from map b*V + w; a query
    on no live view outputs the constant 0, so its grad_out row is ignored and its d_query row is 0.  The RoIs and view
    groups are constants (the reference computes them from detached predictions), so pred gets no gradient.  Everything
    stays on the device, without host synchronisation after the first call of a pack."""
    bp, B, P = _rcnn_block_of(dec, li, query, img, True)
    d_query, d_img, R = _v1_rcnn_backward(dec, bp, B, P, query, pred, img, img_metas, grad_out)
    return dict(d_query=d_query, d_img=d_img, grads=R)


class PointRCNNFunction(torch.autograd.Function):
    """autograd wrapper: out [B*P, C] = dec.decode_head[li] (a V1 PointRCNNBlock) with the forward schedule's kernels, bit
    for bit; backward -> (d_query, d_bev) through point_rcnn_backward, no gradient for pred (the RoIs are constants).
    Parameter gradients are returned by point_rcnn_backward."""

    @staticmethod
    def forward(ctx, dec, li, query, pred, bev):
        bp, B, P = _rcnn_block_of(dec, li, query, bev, False)
        ctx.dec, ctx.li = dec, li
        ctx.save_for_backward(query, pred, bev)
        with _precise():
            return _rcnn_forward(dec, bp, query.contiguous(), pred.contiguous(), bev.contiguous(), None, B, P)[0]

    @staticmethod
    def backward(ctx, grad_out):
        query, pred, bev = ctx.saved_tensors
        r = point_rcnn_backward(ctx.dec, ctx.li, query, pred, bev, grad_out)
        return None, None, r['d_query'], None, r['d_bev']


class ImageRCNNFunction(torch.autograd.Function):
    """autograd wrapper: out [B*P, C] = dec.decode_head[li] (a V1 ImageRCNNBlock) with the forward schedule's kernels, bit
    for bit; backward -> (d_query, d_img) through image_rcnn_backward, no gradient for pred or img_metas (the RoIs and view
    groups are constants).  Parameter gradients are returned by image_rcnn_backward."""

    @staticmethod
    def forward(ctx, dec, li, query, pred, img, img_metas):
        bp, B, P = _rcnn_block_of(dec, li, query, img, True)
        ctx.dec, ctx.li, ctx.img_metas = dec, li, img_metas
        ctx.save_for_backward(query, pred, img)
        with _precise():
            return _rcnn_forward(dec, bp, query.contiguous(), pred.contiguous(), img.contiguous(), img_metas, B, P)[0]

    @staticmethod
    def backward(ctx, grad_out):
        query, pred, img = ctx.saved_tensors
        r = image_rcnn_backward(ctx.dec, ctx.li, query, pred, img, ctx.img_metas, grad_out)
        return None, None, r['d_query'], None, r['d_img'], None


# ---- decoder: the V2 RCNN blocks of the ++ decoder, PointRCNNBlockV2 and ImageRCNNBlockV2 --------------------------------
@_precise()
def point_rcnn_v2_backward(dec, li, query, pred, bev, grad_out):
    """Backward of the ++ decoder's PointRCNNBlockV2 (reference models/utils/decoder_utils.py:995-1089; dec.decode_head[li],
    li = 1 or 3), LayerNorms as they are, dropout off.  Arguments as point_rcnn_backward's.  -> dict(d_query [B*P, C],
    d_bev [B, Y, X, C], grads = {name: tensor} for the 32 parameters of dec.decode_head[li], keyed and shaped as in its
    state_dict, scale and self_scale included).  One view group per sample: every row receives the self branch of the
    sample's first query.  The RoIs are constants, so pred gets no gradient; no host synchronisation after the first call
    of a pack."""
    bp, B, P = _rcnn_block_of(dec, li, query, bev, False, v2=True)
    d_query, d_bev, R = _v2_rcnn_backward(dec, bp, B, P, query, pred, bev, None, grad_out)
    return dict(d_query=d_query, d_bev=d_bev, grads=R)


@_precise()
def image_rcnn_v2_backward(dec, li, query, pred, img, img_metas, grad_out):
    """Backward of the ++ decoder's ImageRCNNBlockV2 (reference models/utils/decoder_utils.py:844-991; dec.decode_head[li],
    li = 0 or 2), LayerNorms as they are, dropout off.  Arguments as image_rcnn_backward's.  -> dict(d_query [B*P, C],
    d_img [B*V, h, w, C], grads = {name: tensor} for the 32 parameters of dec.decode_head[li]).  A query with win = w >= 0
    receives the self branch of the first query on live view w of its sample; a query on no live view outputs 0, so its
    grad_out row is ignored.  The RoIs and view groups are constants; no host synchronisation after the first call of a
    pack."""
    bp, B, P = _rcnn_block_of(dec, li, query, img, True, v2=True)
    d_query, d_img, R = _v2_rcnn_backward(dec, bp, B, P, query, pred, img, img_metas, grad_out)
    return dict(d_query=d_query, d_img=d_img, grads=R)


class PointRCNNV2Function(torch.autograd.Function):
    """autograd wrapper: out [B*P, C] = dec.decode_head[li] (a PointRCNNBlockV2) with the forward schedule's kernels, bit
    for bit; backward -> (d_query, d_bev) through point_rcnn_v2_backward.  Parameter gradients are returned by
    point_rcnn_v2_backward."""

    @staticmethod
    def forward(ctx, dec, li, query, pred, bev):
        bp, B, P = _rcnn_block_of(dec, li, query, bev, False, v2=True)
        ctx.dec, ctx.li = dec, li
        ctx.save_for_backward(query, pred, bev)
        with _precise():
            return _rcnn_forward(dec, bp, query.contiguous(), pred.contiguous(), bev.contiguous(), None, B, P)[0]

    @staticmethod
    def backward(ctx, grad_out):
        query, pred, bev = ctx.saved_tensors
        r = point_rcnn_v2_backward(ctx.dec, ctx.li, query, pred, bev, grad_out)
        return None, None, r['d_query'], None, r['d_bev']


class ImageRCNNV2Function(torch.autograd.Function):
    """autograd wrapper: out [B*P, C] = dec.decode_head[li] (an ImageRCNNBlockV2) with the forward schedule's kernels, bit
    for bit; backward -> (d_query, d_img) through image_rcnn_v2_backward.  Parameter gradients are returned by
    image_rcnn_v2_backward."""

    @staticmethod
    def forward(ctx, dec, li, query, pred, img, img_metas):
        bp, B, P = _rcnn_block_of(dec, li, query, img, True, v2=True)
        ctx.dec, ctx.li, ctx.img_metas = dec, li, img_metas
        ctx.save_for_backward(query, pred, img)
        with _precise():
            return _rcnn_forward(dec, bp, query.contiguous(), pred.contiguous(), img.contiguous(), img_metas, B, P)[0]

    @staticmethod
    def backward(ctx, grad_out):
        query, pred, img = ctx.saved_tensors
        r = image_rcnn_v2_backward(ctx.dec, ctx.li, query, pred, img, ctx.img_metas, grad_out)
        return None, None, r['d_query'], None, r['d_img'], None


# ---- decoder: prediction heads, heat-map head, query init and the whole decoder from its loss ---------------------
def _pred_bw_pack(dec, li, pack):
    """Transposed weights of a prediction FFN's two dX products and, per head, its row / column ranges in the packed
    weights (mmpi._pack_pred) with the constants of fold.conv_bn_unfold, built once per pack.  li: index into
    dec.pred_head, or None for dec.prediction_heads[0]."""
    pk = dec.pack()
    holder = pk if li is None else pk['blocks'][li]
    if '_bw_pred' not in holder:
        ffn = dec.prediction_heads[0] if li is None else dec.pred_head[li]
        dev_ = pk['bce'].device
        heads, r, c = [], 0, 0
        for h in dec.head_order:
            seq = getattr(ffn, h)
            n1, n2 = seq[0].conv.weight.shape[0], seq[1].weight.shape[0]
            consts = tuple(t.to(device=dev_, dtype=torch.float32) for t in fold.conv_bn_unfold_consts(seq[0].conv, seq[0].bn))
            heads.append((h, slice(r, r + n1), slice(c, c + n2), consts))
            r, c = r + n1, c + n2
        holder['_bw_pred'] = dict(w1=_transposed(pack[0]), w2=_transposed(pack[2]), heads=heads)
    return holder['_bw_pred']


@_precise()
def pred_head_backward(dec, li, srcs, grad_out):
    """Backward of a prediction FFN (reference models/utils/decoder_utils.py:498-581; per head ConvBN1d(cin -> 64) + ReLU,
    Conv1d(64 -> k), BatchNorm in eval mode) as the forward packs it: one [sum 64, cin] layer over every head, then a
    block-diagonal [NP, sum 64] one.  li: index into dec.pred_head (input cat([query, previous query]), :289), or None for
    dec.prediction_heads[0] (input the query).  srcs: the input rows [B*P, C] as the forward feeds them; grad_out
    [B*P, NP]: gradient of the head's output rows (head order, before the forward adds query_pos to the centre, which
    passes it unchanged).  -> dict(d_srcs = [d src], grads = {name: tensor} for '{h}.0.conv.weight', '{h}.0.bn.weight',
    '{h}.0.bn.bias', '{h}.1.weight', '{h}.1.bias' of every head h, shaped as in the FFN's state_dict).  The hidden rows are
    re-run for the ReLU mask; only the diagonal blocks of the second layer's weight gradient are parameters."""
    pk = dec.pack()
    pack = pk['pred0'] if li is None else pk['blocks'][li]['pred']
    bw = _pred_bw_pack(dec, li, pack)
    srcs = [s.contiguous() for s in srcs]
    dy = grad_out.contiguous()
    W1, b1 = pack[0], pack[1]
    h = dec._mlp(srcs, W1, b1, ops.ACT_RELU)
    dW2, db2 = _layer_grads(dy, h)
    dh = ops.relu_bwd(ops.linear([dy], bw['w2']), h)
    dW1, db1 = _layer_grads(dh, *srcs)
    dx = ops.linear([dh], bw['w1'])
    R = {}
    for name, rows, cols, consts in bw['heads']:
        dW0, _, dgamma, dbeta = fold.conv_bn_unfold(consts, dW1[rows], db1[rows])
        R[name + '.0.conv.weight'] = dW0.unsqueeze(-1)
        R[name + '.0.bn.weight'], R[name + '.0.bn.bias'] = dgamma, dbeta
        R[name + '.1.weight'] = dW2[cols, rows].unsqueeze(-1)
        R[name + '.1.bias'] = db2[cols]
    k, d_srcs = 0, []
    for s in srcs:
        d_srcs.append(dx[:, k:k + s.shape[1]].contiguous())
        k += s.shape[1]
    return dict(d_srcs=d_srcs, grads=R)


def _heat_bw_pack(dec, pk):
    """Flipped, transposed weights of the two heat-map convolutions (the second padded to 32 output channels, the
    layout of the loss gradient) and the constants of fold.conv_bn_unfold, built once per pack."""
    if '_bw_heat' not in pk:
        seq = dec.heatmap_head_img
        w0, _, w1, _ = pk['heatmap_head_img']
        consts = tuple(t.to(device=w0.w.device, dtype=torch.float32) for t in fold.conv_bn_unfold_consts(seq[0].conv, seq[0].bn))
        pk['_bw_heat'] = dict(w0=_flipped(w0), w1=_flipped(w1, 32), unfold=consts)
    return pk['_bw_heat']


@_precise()
def heatmap_head_backward(dec, new_pts, grad_out):
    """Backward of dec.heatmap_head_img (reference deepinteraction_decoder.py:224: ConvBN2d(C -> C, 3x3) + ReLU, Conv2d(C
    -> K, 3x3), BatchNorm in eval mode).  new_pts [B, Y, X, C] (pixel-major); grad_out [B, Y, X, 32]: gradient of the
    dense logits, channels K..31 zero (LossMixin.loss_backward); the weight gradient reads its first K channels.  -> dict(d_new_pts [B, Y, X, C], grads = {name: tensor}
    for '0.conv.weight', '0.bn.weight', '0.bn.bias', '1.weight', '1.bias', shaped as in its state_dict).  The first
    convolution is re-run for the ReLU mask; input gradients go through the transposed, tap-flipped convolutions."""
    pk = dec.pack()
    bw = _heat_bw_pack(dec, pk)
    B, Y, X, C = new_pts.shape
    K = dec.heatmap_head_img[1].weight.shape[0]
    x = new_pts.contiguous()
    g = grad_out.contiguous()
    w0, b0, _, _ = pk['heatmap_head_img']
    h = ops.conv3x3(x, w0, b0, C, True, False, ops.ACT_RELU)
    dh = ops.relu_bwd(ops.conv3x3(g, bw['w1'], None, cout=C, x_nhwc=True), h)
    dW1, db1 = _conv3x3_wgrad_nhwc(h, g.view(-1, 32)[:, :K].contiguous(), K)     # the pad channels are no parameters
    dx = ops.conv3x3(dh, bw['w0'], None, cout=C, x_nhwc=True)
    dW0, db0 = _conv3x3_wgrad_nhwc(x, dh.view(-1, C), C)
    dWc, _, dgamma, dbeta = fold.conv_bn_unfold(bw['unfold'], dW0.reshape(C, -1), db0)
    R = {'0.conv.weight': dWc.view(C, C, 3, 3), '0.bn.weight': dgamma, '0.bn.bias': dbeta, '1.weight': dW1, '1.bias': db1}
    return dict(d_new_pts=dx, grads=R)


def _decoder_checks(dec, pts_conv, new_pts, img, plusplus=False):
    """NotImplementedError before any launch for what decoder_backward (plusplus: decoder_pp_backward) does not cover,
    including what the block backwards reject (_rcnn_block_of): the maps' shapes and channels."""
    fn = 'decoder_pp_backward' if plusplus else 'decoder_backward'
    B, P, C = pts_conv.shape[0], dec.num_proposals, dec.hidden_channel
    bev = (B, dec.y_size, dec.x_size, C)
    if (pts_conv.dim() != 4 or tuple(pts_conv.shape) != bev or tuple(new_pts.shape) != bev or img.dim() != 4
            or img.shape[0] != B * dec.num_views or img.shape[3] != C or P > 512):
        raise NotImplementedError(f'{fn}: pts_conv and new_pts must be [B, {dec.y_size}, {dec.x_size}, {C}] and '
                                  f'img [B*{dec.num_views}, h, w, {C}], pixel-major (got {tuple(pts_conv.shape)}, '
                                  f'{tuple(new_pts.shape)}, {tuple(img.shape)})')
    from .mmpi import DeepInteractionPlusPlusDecoder
    v2 = [getattr(b, 'v2', False) for b in dec.decode_head]
    if not plusplus and (isinstance(dec, DeepInteractionPlusPlusDecoder) or any(v2)):
        raise NotImplementedError('decoder_backward covers the base DeepInteractionDecoder only (the V2 RCNN blocks of the '
                                  '++ decoder have no backward)')
    if plusplus and not (isinstance(dec, DeepInteractionPlusPlusDecoder) and all(v2)):
        raise NotImplementedError('decoder_pp_backward covers the DeepInteractionPlusPlusDecoder only (the base decoder: '
                                  'decoder_backward)')
    if not dec.auxiliary:
        raise NotImplementedError(f'{fn} needs auxiliary=True (a loss on every layer), as both reference configs')
    if dec.num_heads != 8 or dec.hidden_channel != 128 or P > 256 or dec.num_classes_heat > 32 or B < 1:
        raise NotImplementedError(f'{fn}: the gradient kernels take 8 heads x 16 channels, P <= 256 proposals '
                                  f'and K <= 32 classes (got heads={dec.num_heads}, C={dec.hidden_channel}, P={P}, '
                                  f'K={dec.num_classes_heat})')


def _prefixed(R, prefix, grads):
    for k, v in grads.items():
        R[prefix + k] = v


def _decoder_loss_forward(dec, pts_conv, new_pts, img, img_metas, gt_bboxes_3d, gt_labels_3d, grad_losses):
    """The forward with the values the chain needs (the forward schedule's own kernels, run eagerly), the loss and its
    gradient -> (saved values, forward result, losses, d dense heat-map logits, d prediction rows [L, B*P, NP])."""
    proj, aux = (t.pin_memory().to(pts_conv.device, non_blocking=True) for t in dec._camera_consts(img_metas))
    sv = {}
    r = dec._schedule(pts_conv, new_pts, img, geom.input_hw(img_metas), proj, aux, sv)
    losses = dec.loss(gt_bboxes_3d, gt_labels_3d, dec._outputs(r, pts_conv.shape[0]))
    d_heat, d_pred = dec.loss_backward(grad_losses)
    return sv, r, losses, d_heat, d_pred


@_precise()
def decoder_backward(dec, pts_conv, new_pts, img, img_metas, gt_bboxes_3d, gt_labels_3d, grad_losses=None):
    """Gradient of the base decoder's losses (reference deepinteraction_decoder.py:201-313 forward, :484-547 loss) with
    BatchNorm in eval mode (the folded weights of the forward) and dropout off.
    dec: DeepInteractionDecoder on the GPU with train_cfg; pts_conv, new_pts [B, Y, X, C], img [B*V, h, w, C]: the encoder's
    outputs (pixel-major, as forward_rows takes them); img_metas; gt_bboxes_3d / gt_labels_3d as dec.loss takes them;
    grad_losses [2 + 2L] (device): the upstream gradient of the loss dict's values in their order (None = ones: mmdet's
    sum of every key containing 'loss'; matched_ious takes none).
    -> dict(losses = dec.loss(...) of this forward, d_pts_conv [B, Y, X, C], d_new_pts [B, Y, X, C], d_img [B*V, h, w, C],
    grads = {name: tensor} keyed and shaped as dec.state_dict() for every parameter but heatmap_head.* (the heat map the
    loss reads comes from heatmap_head_img; heatmap_head only ranks proposals, through .detach(), so autograd gives it
    None)).  Proposals, RoIs, view groups and the assignment are constants, as in the reference.  The prediction rows of
    queries on no live view take prediction_heads[0]'s rows by selection, so their gradient goes to that head; they
    carry weight 0 under the on-image mask, so its gradient is exactly zero in the base decoder.  Everything stays on the device, without host synchronisation after
    the first call of a pack (ground truth and img_metas as the forward and loss take them; boxes given on the device)."""
    B, P = pts_conv.shape[0], dec.num_proposals
    _decoder_checks(dec, pts_conv, new_pts, img)
    pk = dec.pack()
    pts_conv, new_pts, img = pts_conv.contiguous(), new_pts.contiguous(), img.contiguous()
    sv, r, losses, d_heat, d_pred = _decoder_loss_forward(dec, pts_conv, new_pts, img, img_metas, gt_bboxes_3d,
                                                          gt_labels_3d, grad_losses)
    # ---- MMPI layers in reverse: pred_head[l] reads [q_{l+1} | q_l]; block l maps q_l to q_{l+1} with the RoIs of the
    # previous layer's (detached) predictions
    qs = [sv['query_feat1']] + sv['layer_query']
    R = {}
    dq, d_img, d_new_pts, d_first = None, None, None, None
    wins = iter(reversed(r['wins']))
    for li in reversed(range(len(pk['blocks']))):
        bp = pk['blocks'][li]
        d_rows = d_pred[li]
        if bp['image']:
            # rows on no live view are prediction_heads[0]'s rows, selected (pred_finish): their gradient goes there
            d_head = ops.rows_finish(d_rows, zero_if_neg=next(wins))
            d_first = _add(d_first, _sub(d_rows, d_head))
            d_rows = d_head
        ph = pred_head_backward(dec, li, [qs[li + 1], qs[li]], d_rows)
        _prefixed(R, 'pred_head.%d.' % li, ph['grads'])
        pred_in = r['preds'][li - 1] if li > 0 else sv['first_res']
        d_out = _add(dq, ph['d_srcs'][0])
        if bp['image']:
            d_q, d_maps, g = _v1_rcnn_backward(dec, bp, B, P, qs[li], pred_in, img, img_metas, d_out)
            d_img = _add(d_img, d_maps)
        else:
            d_q, d_maps, g = _v1_rcnn_backward(dec, bp, B, P, qs[li], pred_in, new_pts, None, d_out)
            d_new_pts = _add(d_new_pts, d_maps)
        _prefixed(R, 'decode_head.%d.' % li, g)
        dq = _add(d_q, ph['d_srcs'][1])
    # prediction_heads[0] reads the layer's output q1 and feeds the fallback rows (its RoIs are constants).  Under the
    # on-image mask those rows carry weight 0, so this is exactly zero in the base decoder; it is computed all the same.
    d_first = d_first if d_first is not None else torch.zeros_like(d_pred[0])
    d_pts_conv, d_new_pts, d_img = _decoder_tail(dec, sv, r, R, dq, d_first, d_heat, pts_conv, new_pts, img, d_new_pts, d_img)
    return dict(losses=losses, d_pts_conv=d_pts_conv, d_new_pts=d_new_pts, d_img=d_img, grads=R)


def _decoder_tail(dec, sv, r, R, dq, d_first, d_heat, pts_conv, new_pts, img, d_new_pts, d_img):
    """The part of the decoder's gradient the base and the ++ decoder share, from d q1 (the transformer layer's output,
    without prediction_heads[0]'s part) and d first (that head's output rows): prediction_heads[0], the transformer layer,
    query init and the heat-map head.  -> (d_pts_conv, d_new_pts, d_img) with the MMPI layers' d_new_pts / d_img (None =
    zero) added; parameter gradients are stored in R."""
    B = pts_conv.shape[0]
    pf = pred_head_backward(dec, None, [sv['query_feat1']], d_first)
    _prefixed(R, 'prediction_heads.0.', pf['grads'])
    dq = _add(dq, pf['d_srcs'][0])
    rl = decoder_layer_backward(dec, sv['query_feat0'], sv['query_pos0'], pts_conv, dq)
    _prefixed(R, 'decoder.0.', rl['grads'])
    d_pts_conv = rl['d_bev'].contiguous()
    d_wce, d_bce = ops.query_init_bwd(rl['d_query'], sv['top'], r['labels'], d_pts_conv.view(B, -1, dec.hidden_channel),
                                      dec.num_classes_heat)
    R['class_encoding.weight'], R['class_encoding.bias'] = d_wce.unsqueeze(-1), d_bce
    hh = heatmap_head_backward(dec, new_pts, d_heat)
    _prefixed(R, 'heatmap_head_img.', hh['grads'])
    d_new_pts = _add(d_new_pts, hh['d_new_pts'])
    if d_img is None:
        d_img = torch.zeros_like(img)
    return d_pts_conv, d_new_pts, d_img


class DecoderLossFunction(torch.autograd.Function):
    """autograd wrapper: the base decoder's summed loss (mmdet's sum of every loss key) from the encoder outputs
    pts_conv, new_pts [B, Y, X, C] and img [B*V, h, w, C]; backward -> (d_pts_conv, d_new_pts, d_img) through
    decoder_backward.  Parameter gradients are returned by decoder_backward."""

    @staticmethod
    def forward(ctx, dec, pts_conv, new_pts, img, img_metas, gt_bboxes_3d, gt_labels_3d):
        _decoder_checks(dec, pts_conv, new_pts, img)
        ctx.dec, ctx.args = dec, (img_metas, gt_bboxes_3d, gt_labels_3d)
        ctx.save_for_backward(pts_conv, new_pts, img)
        losses = dec.loss(gt_bboxes_3d, gt_labels_3d, dec.forward_nhwc(pts_conv, new_pts, img, img_metas))
        return torch.stack([v for k, v in losses.items() if 'loss' in k]).sum()

    @staticmethod
    def backward(ctx, grad):
        pts_conv, new_pts, img = ctx.saved_tensors
        L = len(ctx.dec.decode_head)
        g = grad.reshape(1).float().expand(2 + 2 * L).contiguous()
        r = decoder_backward(ctx.dec, pts_conv, new_pts, img, *ctx.args, grad_losses=g)
        return None, r['d_pts_conv'], r['d_new_pts'], r['d_img'], None, None, None


@_precise()
def decoder_pp_backward(dec, pts_conv, new_pts, img, img_metas, gt_bboxes_3d, gt_labels_3d, grad_losses=None):
    """Gradient of the ++ decoder's losses (reference deepinteractionplusplus_decoder.py:200-319 forward, the base loss with
    every layer's weights multiplied by that layer's on-image mask), BatchNorm in eval mode and dropout off.  Arguments
    and result as decoder_backward's: dict(losses, d_pts_conv, d_new_pts, d_img, grads for every parameter but
    heatmap_head.*).  Layer l's prediction rows are pred_head[l](q_{l+1}) with the look-forward centre (centre_l =
    delta_l + look_l, look_{l+1} = delta_l + qpos_l, qpos and the first look detached), rows outside the cumulative mask
    keep_l taking prediction_heads[0]'s rows at every layer (di_pred_finish_pp_bwd_f32 routes the gradient).  Those rows
    carry weight 0 under the masks, so prediction_heads[0]'s gradient is exactly zero; it is computed all the same.
    Proposals, RoIs, view groups, masks and the assignment are constants.  Everything stays on the device, without host
    synchronisation after the first call of a pack."""
    B, P = pts_conv.shape[0], dec.num_proposals
    _decoder_checks(dec, pts_conv, new_pts, img, plusplus=True)
    pk = dec.pack()
    pts_conv, new_pts, img = pts_conv.contiguous(), new_pts.contiguous(), img.contiguous()
    sv, r, losses, d_heat, d_pred = _decoder_loss_forward(dec, pts_conv, new_pts, img, img_metas, gt_bboxes_3d,
                                                          gt_labels_3d, grad_losses)
    d_delta, d_first = ops.pred_finish_pp_bwd(d_pred, torch.stack(r['keeps']))
    # ---- MMPI layers in reverse: pred_head[l] reads q_{l+1}; block l maps q_l to q_{l+1} with the RoIs of the previous
    # layer's (detached) predictions
    qs = [sv['query_feat1']] + sv['layer_query']
    R = {}
    dq, d_img, d_new_pts = None, None, None
    for li in reversed(range(len(pk['blocks']))):
        bp = pk['blocks'][li]
        ph = pred_head_backward(dec, li, [qs[li + 1]], d_delta[li])
        _prefixed(R, 'pred_head.%d.' % li, ph['grads'])
        pred_in = r['preds'][li - 1] if li > 0 else sv['first_res']
        maps, metas = (img, img_metas) if bp['image'] else (new_pts, None)
        dq, d_maps, g = _v2_rcnn_backward(dec, bp, B, P, qs[li], pred_in, maps, metas, _add(dq, ph['d_srcs'][0]))
        if bp['image']:
            d_img = _add(d_img, d_maps)
        else:
            d_new_pts = _add(d_new_pts, d_maps)
        _prefixed(R, 'decode_head.%d.' % li, g)
    d_pts_conv, d_new_pts, d_img = _decoder_tail(dec, sv, r, R, dq, d_first, d_heat, pts_conv, new_pts, img, d_new_pts, d_img)
    return dict(losses=losses, d_pts_conv=d_pts_conv, d_new_pts=d_new_pts, d_img=d_img, grads=R)


class DecoderPPLossFunction(torch.autograd.Function):
    """autograd wrapper: the ++ decoder's summed loss from the encoder outputs pts_conv, new_pts [B, Y, X, C] and img
    [B*V, h, w, C]; backward -> (d_pts_conv, d_new_pts, d_img) through decoder_pp_backward.  Parameter gradients are
    returned by decoder_pp_backward."""

    @staticmethod
    def forward(ctx, dec, pts_conv, new_pts, img, img_metas, gt_bboxes_3d, gt_labels_3d):
        _decoder_checks(dec, pts_conv, new_pts, img, plusplus=True)
        ctx.dec, ctx.args = dec, (img_metas, gt_bboxes_3d, gt_labels_3d)
        ctx.save_for_backward(pts_conv, new_pts, img)
        losses = dec.loss(gt_bboxes_3d, gt_labels_3d, dec.forward_nhwc(pts_conv, new_pts, img, img_metas))
        return torch.stack([v for k, v in losses.items() if 'loss' in k]).sum()

    @staticmethod
    def backward(ctx, grad):
        pts_conv, new_pts, img = ctx.saved_tensors
        L = len(ctx.dec.decode_head)
        g = grad.reshape(1).float().expand(2 + 2 * L).contiguous()
        r = decoder_pp_backward(ctx.dec, pts_conv, new_pts, img, *ctx.args, grad_losses=g)
        return None, r['d_pts_conv'], r['d_new_pts'], r['d_img'], None, None, None


# ---- the ++ encoder: FusionTransformerv4 -----------------------------------------------------------------------------
def _tr(cache, key, w):
    """_transposed(w), built once per pack under `key` of the pack's cache dict."""
    if key not in cache:
        cache[key] = _transposed(w)
    return cache[key]


def _msda_backward(ap, sv, dy, B, hq, wq, R, prefix):
    """Backward of msda_forward (out = output_proj(msdeform(value_proj(maps), raw(q))) + q) from its saved values ->
    (d q rows, [d map rows per level]).  The fused raw weight's gradient is split back into sampling_offsets.* and
    attention_weights.*; value_proj's gradient sums over the levels."""
    cache = ap.setdefault('_bw', {})
    _put(R, (prefix + 'output_proj', _layer_grads(dy, sv['a'])))
    da = ops.linear([dy], _tr(cache, 'out', ap['out'][0]))
    d_raw, d_vals = ops.msdeform_bwd(sv['vals'], sv['raw'], da, B, hq, wq, ap['heads'], ap['points'])
    dW, db = _layer_grads(d_raw, sv['q'])
    n_off = ap['heads'] * ap['L'] * ap['points'] * 2
    R[prefix + 'sampling_offsets.weight'], R[prefix + 'sampling_offsets.bias'] = dW[:n_off], db[:n_off]
    R[prefix + 'attention_weights.weight'], R[prefix + 'attention_weights.bias'] = dW[n_off:], db[n_off:]
    d_q = ops.linear([d_raw], _tr(cache, 'raw', ap['raw'][0]), res=dy)
    dWv = dbv = None
    d_maps = []
    for m, dv in zip(sv['maps'], d_vals):
        C = m.shape[-1]
        dWl, dbl = _layer_grads(dv.view(-1, C), m.reshape(-1, C))
        dWv, dbv = _add(dWv, dWl), _add(dbv, dbl)
        d_maps.append(ops.linear([dv.view(-1, C)], _tr(cache, 'value', ap['value'][0])))
    _put(R, (prefix + 'value_proj', (dWv, dbv)))
    return d_q, d_maps


def _ffn_backward(pk, sv, dy, cache, key, R, prefix):
    """Backward of ffn_forward (out = linear2(relu(linear1(x))) + x) -> d x; parameter gradients into R."""
    w1, _, w2, _ = pk
    _put(R, (prefix + 'layers.1', _layer_grads(dy, sv['h'])))
    dh = ops.relu_bwd(ops.linear([dy], _tr(cache, key + '2', w2)), sv['h'])
    _put(R, (prefix + 'layers.0.0', _layer_grads(dh, sv['x'])))
    return ops.linear([dh], _tr(cache, key + '1', w1), res=dy)


def _polar_backward(ap, sv, dy, R, prefix):
    """Backward of polar.polar_forward from d out [B*Y*X, C] rows -> (d lidar rows (the residual, plus the ray queries'
    sampling), d image-map rows (through the memory)).  The block is evaluated in fp32 as its forward, dropout off."""
    cache = ap.setdefault('_bw', {})
    C = dy.shape[1]
    BV, Rr, w, _ = sv['rays_shape']
    h = sv['cols'].shape[0] // (BV * w)
    T = 'transformer_layers.'
    D = prefix + T + 'decoder.layers.0.'
    sa, ca = ap['self_attn'], ap['cross']
    d_lidar = dy.contiguous()
    proj, undo, camc, V, in_hw, pc, r0, r_cnt = sv['gather']
    bev = sv['bev_shape']
    d_x4 = ops.polar_gather_bwd(d_lidar.view(bev), sv['rays_shape'], proj, undo, camc, V, in_hw, pc, r0, r_cnt)
    d_x3, R[prefix + T + 'decoder.norm.weight'], R[prefix + T + 'decoder.norm.bias'] = ops.ln_bwd(
        d_x4.view(-1, C), sv['x3'], ap['dec_norm'][0])
    w1, _, w2, _ = ap['ffn']
    d_x2, n3, l2, l1 = _ffn_norm_backward(d_x3, sv['z3'], ap['norm3'][0], sv['f'], (ops.relu_bwd, sv['f']), sv['x2'],
                                          _tr(cache, 'ffn2', w2), _tr(cache, 'ffn1', w1))
    _put(R, (D + 'norm3', n3), (D + 'linear2', l2), (D + 'linear1', l1))
    # norm2, cross attention over the image column (memory)
    dz2, R[D + 'norm2.weight'], R[D + 'norm2.bias'] = ops.ln_bwd(d_x2, sv['z2'], ap['norm2'][0])
    _put(R, (D + 'multihead_attn.out_proj', _layer_grads(dz2, sv['a2'])))
    da2 = ops.linear([dz2], _tr(cache, 'cross_out', ca['out'][0]))
    kv = sv['kv']
    dq2 = torch.empty_like(sv['q2'])
    dkv = torch.empty_like(kv)
    ops.seq_attn_bwd(sv['q2'], kv[:, :C], kv[:, C:], sv['a2'], da2, BV, w, Rr, h, ap['heads'], dq2, dkv[:, :C], dkv[:, C:])
    dWq, dbq = _layer_grads(dq2, sv['x1'])
    dWkv, dbkv = _layer_grads(dkv, sv['memory'])
    R[D + 'multihead_attn.in_proj_weight'] = torch.cat([dWq, dWkv], 0)
    R[D + 'multihead_attn.in_proj_bias'] = torch.cat([dbq, dbkv], 0)
    d_x1 = ops.linear([dq2], _tr(cache, 'cross_q', ca['q'][0]), res=dz2)
    d_mem = ops.linear([dkv], _tr(cache, 'cross_kv', ca['kv'][0]))
    d_cols, R[prefix + T + 'encoder.norm.weight'], R[prefix + T + 'encoder.norm.bias'] = ops.ln_bwd(
        d_mem, sv['cols'], ap['enc_norm'][0])
    # norm1, self attention along the ray
    dz1, R[D + 'norm1.weight'], R[D + 'norm1.bias'] = ops.ln_bwd(d_x1, sv['z1'], ap['norm1'][0])
    _put(R, (D + 'self_attn.out_proj', _layer_grads(dz1, sv['a1'])))
    da1 = ops.linear([dz1], _tr(cache, 'self_out', sa['out'][0]))
    qkv = sv['qkv']
    dqkv = torch.empty_like(qkv)
    ops.seq_attn_bwd(qkv[:, :C], qkv[:, C:2 * C], qkv[:, 2 * C:], sv['a1'], da1, BV, w, Rr, Rr, ap['heads'],
                     dqkv[:, :C], dqkv[:, C:2 * C], dqkv[:, 2 * C:])
    R[D + 'self_attn.in_proj_weight'], R[D + 'self_attn.in_proj_bias'] = _layer_grads(dqkv, sv['rays'])
    d_rays = ops.linear([dqkv], _tr(cache, 'self_in', sa['qkv'][0]), res=dz1)
    d_bev = ops.bev_sample_bwd(d_rays.view(BV, Rr, w, C), sv['grid'], V, bev)
    return _add(d_lidar, d_bev.view(-1, C)), d_cols


def _pp_cross_backward(layer, ap, idx, sv, dy, ctx, R, prefix):
    """Backward of FusionTransformerv4._cross -> (d query rows, d value-map rows or None)."""
    C = dy.shape[1]
    g = ctx['g']
    if ap['kind'] == 'p2i':             # 1-level MSDA over the BEV map sampled at the warp grid
        Bq, hq, wq, _ = sv['maps'][0].shape
        d_q, (d_warped,) = _msda_backward(ap, sv, dy, Bq, hq, wq, R, prefix + 'Local.')
        d_bev = ops.bev_sample_bwd(d_warped.view(Bq, hq, wq, C), g.grid, g.V, sv['value_shape'])
        return d_q, d_bev.view(-1, C)
    if ap['kind'] == 'i2p':             # + residual (:364)
        qm = sv['query_map']
        r = i2p_backward(ap['w'], qm, sv['value_map'], ctx['pm'], g.proj, g.V, g.in_hw, dy.view(qm.shape))
        mha = layer.attentions[idx].learnedAlign
        with fold.on_device():
            u = fold.i2p_unfold_grads(mha, r['dM1'], r['dc1'], r['dM2'], r['dc2'])
        f32 = lambda *ts: torch.cat(ts, 0).float()
        A = prefix + 'learnedAlign.'
        R[A + 'in_proj_weight'], R[A + 'in_proj_bias'] = f32(u['Wq'], u['Wk'], u['Wv']), f32(u['bq'], u['bk'], u['bv'])
        R[A + 'out_proj.weight'], R[A + 'out_proj.bias'] = u['Wo'].float(), u['bo'].float()
        return _add(dy, r['d_pts'].view(-1, C)), r['d_img'].view(-1, C)
    return _polar_backward(ap, sv, dy, R, prefix)


def _pp_layer_backward(layer, lp, sv, d_out, ctx, R, prefix):
    """Backward of FusionTransformerv4._layer from its saved tape: d out rows -> (d query rows, d value-map rows or
    None, [d multi-scale map rows per level or None]).  out = self_feat + scale * query; self_feat is the self
    attention's output, so the gradient of its branch joins the query's there."""
    cache = lp.setdefault('_bw', {})
    d_q, R[prefix + 'scale'] = ops.axpy_bwd(d_out, sv['query'], lp['scale'])
    grads = dict(query=d_q, self=d_out)
    Bq, hq, wq, _ = sv['shape']
    d_value, d_ms = None, None
    for op, idx, stream, s in reversed(sv['tape']):
        gr = grads[stream]
        if op == 'self_attn':
            gr = _add(gr, grads['self'])
            grads['self'] = None
            gr, d_maps = _msda_backward(lp['attn'][idx], s, gr, Bq, hq, wq, R, prefix + 'attentions.%d.' % idx)
            d_ms = d_maps if d_ms is None else [_add(a, b) for a, b in zip(d_ms, d_maps)]
        elif op == 'norm':
            gr, R[prefix + 'norms.%d.weight' % idx], R[prefix + 'norms.%d.bias' % idx] = ops.ln_bwd(gr, s['x'], lp['norms'][idx][0])
        elif op == 'ffn':
            gr = _ffn_backward(lp['ffns'][idx], s, gr, cache, 'ffn%d.' % idx, R, prefix + 'ffns.%d.' % idx)
        else:
            gr, dv = _pp_cross_backward(layer, lp['attn'][idx], idx, s, gr, ctx, R, prefix + 'attentions.%d.' % idx)
            d_value = _add(d_value, dv)
        grads[stream] = gr
    return grads['query'], d_value, d_ms


def _encoder_pp_checks(enc, img_levels, pts_levels, d_img, d_pts_conv, d_pts):
    """NotImplementedError before any launch for what encoder_pp_backward does not cover."""
    from . import mmri_pp
    if not isinstance(enc, mmri_pp.FusionTransformerv4):
        raise NotImplementedError('encoder_pp_backward covers the ++ encoder mmri_pp.FusionTransformerv4 only (the base '
                                  f'DeepInteractionEncoder: encoder_backward; got {type(enc).__name__})')
    C = enc.hidden_channel
    if C != 128:
        raise NotImplementedError(f'encoder_pp_backward: the gradient kernels take hidden_channel = 128 (got {C})')
    for blocks in (enc.img_fusion_blocks, enc.pts_fusion_blocks):
        for layer in blocks:
            for a in layer.attentions:
                m = a.Local if isinstance(a, mmri_pp.MMRI_P2I) else a
                if isinstance(m, mmri_pp.MultiScaleDeformableAttention) and not (
                        m.num_heads == 8 and m.num_points == 4 and m.num_levels in (1, 2) and m.embed_dims == 128):
                    raise NotImplementedError('encoder_pp_backward: the deformable-attention gradient takes 8 heads, 4 points '
                                              f'and 1 or 2 levels (got {m.num_heads}, {m.num_points}, {m.num_levels})')
    img_levels, pts_levels = list(img_levels), list(pts_levels)
    lv = lambda blocks: {a.num_levels for l in blocks for a in l.attentions if isinstance(a, mmri_pp.MultiScaleDeformableAttention)}
    if lv(enc.img_fusion_blocks) != {len(img_levels)} or lv(enc.pts_fusion_blocks) != {len(pts_levels) - 1}:
        raise NotImplementedError(f'encoder_pp_backward: {len(img_levels)} image and {len(pts_levels)} point-cloud levels do '
                                  'not match the layers (self attention over every image level and every point-cloud level '
                                  'after the first)')
    ci, cp, cs = (enc.multi_scale_conv_img.in_channels, enc.multi_scale_conv_pts.in_channels,
                  enc.shared_conv_pts.in_channels)
    shapes = [tuple(t.shape) for t in img_levels + pts_levels]
    B = pts_levels[0].shape[0] if pts_levels[0].dim() == 4 else 0
    ok = (all(t.dim() == 4 for t in img_levels + pts_levels) and B > 0 and img_levels[0].shape[0] % B == 0
          and all(t.shape[1] == ci and t.shape[0] == img_levels[0].shape[0] for t in img_levels)
          and pts_levels[0].shape[1] == cs
          and all(t.shape[1] == cp and t.shape[0] == B and t.shape[2:] == pts_levels[0].shape[2:] for t in pts_levels[1:]))
    if ok:
        BV, _, h, w = img_levels[0].shape
        _, _, Y, X = pts_levels[0].shape
        want = ((d_img, (BV, h, w, C)), (d_pts_conv, (B, Y, X, C)), (d_pts, (B, Y, X, C)))
        ok = all(d is None or tuple(d.shape) == s for d, s in want)
    if not ok:
        raise NotImplementedError(f'encoder_pp_backward: image levels [B*V, {ci}, h, w], point-cloud levels [B, {cs}, Y, X] '
                                  f'then [B, {cp}, Y, X], output gradients [B*V, h, w, {C}] / [B, Y, X, {C}] pixel-major '
                                  f'(got {shapes})')


@_precise()
def encoder_pp_backward(enc, img_levels, pts_levels, img_metas, pts_metas, d_img, d_pts_conv, d_pts):
    """Backward of the ++ encoder FusionTransformerv4.forward (reference fusion_transformerv4.py:25-640) with dropout off;
    it has no BatchNorm, so this is the training gradient of the neck.  img_levels [B*V, Ci, h_l, w_l] and pts_levels
    ([B, 2 Cp, Y, X] concat, then [B, Cp, Y, X] maps): the module's NCHW inputs on the GPU; pts_metas with pillars;
    d_img [B*V, h, w, C], d_pts_conv / d_pts [B, Y, X, C]: gradients of the three outputs, pixel-major (None = zero;
    decoder_pp_backward's d_img, d_pts_conv, d_new_pts).
    -> dict(d_img_levels, d_pts_levels: pixel-major [N, H, W, C_in] per input level, grads = {name: tensor} keyed and
    shaped as enc.state_dict(), every parameter present).  The forward is re-run eagerly (FusionTransformerv4._schedule
    with saved=) and its operation tape walked in reverse; both layers' self attentions read the same multi-scale maps, so
    their value gradients add up per level.  Everything stays on the device, without host synchronisation after the
    first call of a pack (pts_metas given on the device)."""
    _encoder_pp_checks(enc, img_levels, pts_levels, d_img, d_pts_conv, d_pts)
    pk = enc.pack()
    C = enc.hidden_channel
    img_levels, pts_levels = [t.contiguous() for t in img_levels], [t.contiguous() for t in pts_levels]
    dev = img_levels[0].device
    pillars, coors, npts, pts_list, consts = enc._frame(img_metas, pts_metas, dev)
    pm = dict(pillars=pillars, pillar_coors=coors, pillars_num_points=npts, pts=pts_list)
    # pinned sources keep the uploads asynchronous; no live counts: the point arrays have their exact sizes
    consts = [c.pin_memory().to(dev, non_blocking=True) for c in consts] + [None]
    sv = {}
    img, pts_conv, pts = enc._schedule(img_levels, pts_levels, img_metas, pm, consts, saved=sv)
    ctx = sv['ctx']
    R = {}
    gi, gp = _seed_rows(d_img, img), _seed_rows(d_pts, pts)
    d_ms_img = d_ms_pts = None
    add_all = lambda acc, new: new if acc is None else [_add(a, b) for a, b in zip(acc, new)]
    for i in reversed(range(enc.num_layers)):
        # t_pts reads (new_pts, new_img) and t_img reads (new_img, new_pts) of the previous layer
        dq_p, dv_p, dms_p = _pp_layer_backward(enc.pts_fusion_blocks[i], pk['pts'][i], sv['pts'][i], gp, ctx, R,
                                               'pts_fusion_blocks.%d.' % i)
        dq_i, dv_i, dms_i = _pp_layer_backward(enc.img_fusion_blocks[i], pk['img'][i], sv['img'][i], gi, ctx, R,
                                               'img_fusion_blocks.%d.' % i)
        d_ms_img, d_ms_pts = add_all(d_ms_img, dms_i), add_all(d_ms_pts, dms_p)
        gi, gp = _add(dq_i, dv_p), _add(dq_p, dv_i)
    d_ms_img[0], d_ms_pts[0] = _add(d_ms_img[0], gi), _add(d_ms_pts[0], gp)     # level 0 is the first layer's query

    def convs(name, xs, gs):
        dxs, dW, db = [], None, None
        for x, g in zip(xs, gs):
            dx, (w, b) = _shared_conv_backward(g.contiguous(), pk[name][0], x)
            dxs.append(dx)
            dW, db = _add(dW, w), _add(db, b)
        R[name + '.weight'], R[name + '.bias'] = dW, db
        return dxs
    d_img_levels = convs('multi_scale_conv_img', img_levels, d_ms_img)
    d_pts_levels = (convs('shared_conv_pts', pts_levels[:1], [_seed_rows(d_pts_conv, pts_conv)])
                    + convs('multi_scale_conv_pts', pts_levels[1:], d_ms_pts))
    return dict(d_img_levels=d_img_levels, d_pts_levels=d_pts_levels, grads=R)


class EncoderPPFunction(torch.autograd.Function):
    """autograd wrapper: EncoderPPFunction.apply(enc, img_metas, pts_metas, n_img, *img_levels, *pts_levels) ->
    (img [B*V, h, w, C], pts_conv, pts [B, Y, X, C]) = enc.forward_nhwc(...) with the forward schedule's kernels;
    backward -> the input levels' gradients in their NCHW layout through encoder_pp_backward.  Parameter gradients are
    returned by encoder_pp_backward."""

    @staticmethod
    def forward(ctx, enc, img_metas, pts_metas, n_img, *levels):
        _encoder_pp_checks(enc, levels[:n_img], levels[n_img:], None, None, None)
        ctx.enc, ctx.metas, ctx.n_img = enc, (img_metas, pts_metas), n_img
        ctx.save_for_backward(*levels)
        return enc.forward_nhwc(list(levels[:n_img]), list(levels[n_img:]), img_metas, pts_metas)

    @staticmethod
    def backward(ctx, d_img, d_pts_conv, d_pts):
        levels, n = ctx.saved_tensors, ctx.n_img
        r = encoder_pp_backward(ctx.enc, levels[:n], levels[n:], *ctx.metas, d_img, d_pts_conv, d_pts)
        grads = [ops.nhwc_to_nchw(d.contiguous()) for d in r['d_img_levels'] + r['d_pts_levels']]
        return (None, None, None, None) + tuple(grads)
