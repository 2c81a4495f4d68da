"""Training-mode step of the base encoder on libdi_b200: forward with BatchNorm batch statistics (running statistics
updated), backward to the module's OWN parameters (SURVEY.md 8 row 'training path', config 3).

Reference: models/necks/deepinteraction_encoder.py:8-85 run under `model.train()` -- every ConvBNReLU
(models/utils/encoder_utils.py:11-34) normalises with the statistics of the current batch, and autograd differentiates
through them; the gradient of the whole model is then all-reduced (tools/train.py:157 -> shard.GradBuckets here).

Eval-mode BatchNorm folds into the 1x1 convolutions (the inference kernels; backward.py differentiates that form).
Batch statistics depend on the data, so this path keeps the layers apart: raw 1x1 product on the wgmma / FFMA GEMMs
(3xTF32 split), column moments (di_bn_stats_f32), normalise + ReLU (di_bn_apply_f32), and on the way back
di_bn_bwd_f32 + the weight / input products.  The window attention runs in the unfused kernels of csrc/lcab_bwd.cu with
the [P, 81] weights kept for the backward; I2P, BEVWarp sampling and the 3x3 shared convolutions have no norm and
reuse backward.py.

The attention dropout of MMRI_I2P (encoder_utils.py:223, p = 0.1 in the reference config) is applied when a
`dropout_seed` is given: the mask is a counter-based hash regenerated in the backward (di_i2p_attend_dropout_f32); it is
not torch's Philox stream, so a step equals the reference's in distribution, and exactly when the same mask is used
(tests/test_gpu_backward.py injects it into the oracle).  Not covered: the decoder's backward.  First-version kernels:
every intermediate is materialised.
"""
import torch

from . import backward as bw
from . import fold, ops


DEBUG = [False]      # tools/debug_train_step.py: keep the projections and their gradients of every attention block


class ConvBNTrain:
    """One ConvBN holder (1x1 convolution without bias + BatchNorm2d in training mode [+ ReLU]) on pixel-major rows."""

    def __init__(self, cb, relu):
        self.cb, self.relu = cb, relu
        self.saved = None

    def forward(self, srcs):
        conv, bn = self.cb.conv, self.cb.bn
        dev = conv.weight.device
        w = conv.weight.detach().reshape(conv.weight.shape[0], -1)
        W = fold.Weight(w, dev, lazy=True)
        y = ops.linear(srcs, W)
        mean, var = ops.bn_stats(y, bn.running_mean, bn.running_var, bn.momentum)
        if bn.num_batches_tracked is not None:
            bn.num_batches_tracked += 1
        z = ops.bn_apply(y, mean, var, bn.weight, bn.bias, bn.eps, self.relu)
        self.saved = (list(srcs), y, mean, var, z, w)
        return z

    def backward(self, dz, grads):
        """-> d cat(srcs, 1) [M, K]; parameter gradients are written into `grads` keyed by the parameter tensor's id."""
        conv, bn = self.cb.conv, self.cb.bn
        srcs, y, mean, var, z, w = self.saved
        self.saved = None
        dy, dg, db = ops.bn_bwd(dz.contiguous(), z if self.relu else None, y, mean, var, bn.weight, bn.eps)
        dw = torch.cat([bw._wgrad(dy, s.contiguous()) for s in srcs], 1)
        grads[id(conv.weight)] = dw.view_as(conv.weight)
        if bn.weight is not None:
            grads[id(bn.weight)], grads[id(bn.bias)] = dg, db
        return ops.linear([dy], bw._transposed(w))


class LCABTrain:
    """LocalContextAttentionBlock (encoder_utils.py:84-135) in training mode."""

    def __init__(self, blk):
        self.ks = blk.kernel_size
        self.q1, self.q2 = ConvBNTrain(blk.query_project[0], True), ConvBNTrain(blk.query_project[1], True)
        self.k1, self.k2 = ConvBNTrain(blk.key_project[0], True), ConvBNTrain(blk.key_project[1], True)
        self.v = ConvBNTrain(blk.value_project, True)

    def forward(self, target, source, N, H, W):
        q = self.q2.forward([self.q1.forward([target])])
        k = self.k2.forward([self.k1.forward([source])])
        v = self.v.forward([source])
        self.scale = 1.0 / float(q.shape[1]) ** 0.5
        A = ops.win_softmax(ops.win_dot(q, k, N, H, W, self.ks), self.scale)
        self.saved = (q, k, v, A, (N, H, W))
        if DEBUG[0]:
            self.dbg = dict(q=q, k=k, v=v)
        return ops.win_gather(A, v, N, H, W, self.ks)

    def backward(self, dO, grads):
        """-> (d target, d source)"""
        q, k, v, A, dims = self.saved
        self.saved = None
        dO = dO.contiguous()
        dq, dk, dv = bw._window_backward(q, k, v, A, dO, dims, self.ks, self.scale)
        if DEBUG[0]:
            self.dbg.update(dq=dq, dk=dk, dv=dv, dO=dO)
        d_t = self.q1.backward(self.q2.backward(dq, grads), grads)
        d_s = self.k1.backward(self.k2.backward(dk, grads), grads)
        return d_t, bw._add(d_s, self.v.backward(dv, grads))


class FuseTrain:
    """new = integration(cat(out_proj(cat(a, b)), c)) -- two ConvBN layers without activation
    (deepinteraction_encoder.py:14-15,18-19,26-27,30-31)."""

    def __init__(self, out_proj, integration):
        self.o, self.i = ConvBNTrain(out_proj, False), ConvBNTrain(integration, False)

    def forward(self, a, b, c):
        return self.i.forward([self.o.forward([a, b]), c])

    def backward(self, dy, grads):
        """-> (da, db, dc)"""
        d2 = self.i.backward(dy, grads)
        C = d2.shape[1] // 2
        d1 = self.o.backward(d2[:, :C].contiguous(), grads)
        return d1[:, :C].contiguous(), d1[:, C:].contiguous(), d2[:, C:].contiguous()


class GradSink(dict):
    """Gradient store that reports every parameter gradient the moment the backward produces it (last layer first), e.g. to
    shard.GradBuckets.add -- so the all-reduce of full buckets overlaps the rest of the backward (SURVEY.md 8(e); the reference
    gets this from MMDistributedDataParallel).  on_grad(name, tensor): tensor is the contiguous gradient kept in this dict; an
    in-place update of it (the averaged result) is what encoder_train_step returns."""

    def __init__(self, names, on_grad):
        super().__init__()
        self.names, self.on_grad = names, on_grad

    def __setitem__(self, key, grad):
        grad = grad.contiguous()
        super().__setitem__(key, grad)
        self.on_grad(self.names[key], grad)


def encoder_train_step(enc, img_feats, pts_feats, img_metas, pts_metas, grad_fn, debug=None, dropout_seed=None, on_grad=None):
    """One training-mode forward + backward of DeepInteractionEncoder (base model).

    enc: mmri.DeepInteractionEncoder on the GPU (the parameter holder; its BatchNorm running statistics are updated as
    torch's training mode does).  img_feats (B*V, Ci, h, w), pts_feats (B, Cp, Y, X): NCHW inputs on the GPU.
    grad_fn(img [B*V,h,w,C], pts_conv [B,Y,X,C], pts [B,Y,X,C]) -> (d_img, d_pts_conv, d_pts), same shapes (None = zero):
    the gradient of the loss w.r.t. the three outputs (pixel-major), e.g. from the decoder.  debug: dict that receives the
    per-layer branch outputs ('fwd') and their gradients ('bwd') as pixel-major rows.  dropout_seed: None = no attention
    dropout in MMRI_I2P (deterministic step); an integer (e.g. the iteration number) = dropout with the module's rate
    (`learnedAlign.dropout`, 0.1 in the reference config) and a mask derived from (seed, layer, pillar, key).
    on_grad(name, tensor): called for every parameter gradient as soon as the backward has it (GradSink), e.g.
    `lambda n, t: buckets.add(t)` to overlap the bucketed all-reduce with the backward.
    -> dict(outputs=(img, pts_conv, pts), d_img_feats [B*V,h,w,Ci], d_pts_feats [B,Y,X,Cp],
            grads={parameter name: gradient} for every parameter of `enc` the output depends on)."""
    with bw._precise(), torch.no_grad(), fold.on_device():
        return _encoder_train_step(enc, img_feats, pts_feats, img_metas, pts_metas, grad_fn, debug, dropout_seed, on_grad)


def _encoder_train_step(enc, img_feats, pts_feats, img_metas, pts_metas, grad_fn, debug=None, dropout_seed=None, on_grad=None):
    dev = img_feats.device
    C = enc.hidden_channel
    (BV, _, h, w), (B, _, Y, X) = img_feats.shape, pts_feats.shape
    V, pm, g = bw._encoder_geometry(enc, img_feats, pts_feats, img_metas, pts_metas)
    Wt = lambda t: fold.Weight(t, dev, lazy=True)
    d = lambda t: fold.dev(t, dev)
    conv_pack = lambda conv: (Wt(fold.pack_conv3x3(conv.weight.detach())), d(conv.bias.detach()))
    pk_img, pk_pts = conv_pack(enc.shared_conv_img), conv_pack(enc.shared_conv_pts)
    # ---- forward
    img = ops.conv3x3(img_feats.contiguous(), *pk_img, cout=C, x_nhwc=False)
    pts = ops.conv3x3(pts_feats.contiguous(), *pk_pts, cout=C, x_nhwc=False)
    pts_conv = pts
    layers = []
    for blk in enc.fusion_blocks:
        L = dict(p_iml=LCABTrain(blk.P_IML), p2i=LCABTrain(blk.P2I_block.Local), i_iml=LCABTrain(blk.I_IML),
                 p_fuse=FuseTrain(blk.P_out_proj, blk.P_integration), i_fuse=FuseTrain(blk.I_out_proj, blk.I_integration))
        mha = blk.I2P_block.learnedAlign
        use_drop = dropout_seed is not None and float(mha.dropout) > 0
        if not use_drop:
            M1, c1, M2, c2 = fold.i2p_fold(mha)
            L['i2p'] = (Wt(M1), d(c1), Wt(M2), d(c2))
        else:                                   # dropout form: [C, C + 4] output weight (FFMA path), bias = b_o alone
            M1, c1, M2x, bo = fold.i2p_fold(mha, split_bias=True)
            L['i2p'] = (Wt(M1), d(c1), d(M2x), d(bo))
        img_r, pts_r = img.view(-1, C), pts.view(-1, C)
        L['drop'] = (float(mha.dropout), int(dropout_seed) * 131 + len(layers)) if use_drop else None
        i2p = enc.i2p(L, pts, img, pm, g, dropout=L['drop'])
        p2p = L['p_iml'].forward(pts_r, pts_r, B, Y, X)
        new_pts = L['p_fuse'].forward(i2p.view(-1, C), p2p, pts_r).view(B, Y, X, C)
        warped = ops.bev_sample(pts, g.grid, V)
        p2i = L['p2i'].forward(img_r, warped.view(-1, C), BV, h, w)
        i2i = L['i_iml'].forward(img_r, img_r, BV, h, w)
        new_img = L['i_fuse'].forward(p2i, i2i, img_r).view(BV, h, w, C)
        L.update(img=img, pts=pts, mha=mha)
        if debug is not None:
            debug.setdefault('fwd', []).append(dict(i2p=i2p, p2p=p2p, warped=warped, p2i=p2i, i2i=i2i, blocks=L))
        layers.append(L)
        img, pts = new_img, new_pts
    outputs = (img, pts_conv, pts)
    d_img, d_pts_conv, d_pts = grad_fn(*outputs)
    # ---- backward
    names = {id(p): n for n, p in enc.named_parameters()}
    grads = {} if on_grad is None else GradSink(names, on_grad)
    gi, gp = bw._seed_rows(d_img, img), bw._seed_rows(d_pts, pts)
    for L in reversed(layers):
        d_p2i, d_i2i, d_img_dir = L['i_fuse'].backward(gi, grads)
        d_i2p, d_p2p, d_pts_dir = L['p_fuse'].backward(gp, grads)
        t_ii, s_ii = L['i_iml'].backward(d_i2i, grads)
        t_pi, s_pi = L['p2i'].backward(d_p2i, grads)
        r_ip = bw.i2p_backward(L['i2p'], L['pts'], L['img'], pm, g.proj, V, g.in_hw, d_i2p.view(B, Y, X, C), L['drop'])
        t_pp, s_pp = L['p_iml'].backward(d_p2p, grads)
        gi = bw._add(bw._add(bw._add(bw._add(d_img_dir, t_ii), s_ii), t_pi), r_ip['d_img'].view(-1, C))
        d_bev = ops.bev_sample_bwd(s_pi.view(BV, h, w, C).contiguous(), g.grid, V, (B, Y, X, C))
        gp = bw._add(bw._add(bw._add(bw._add(d_pts_dir, t_pp), s_pp), r_ip['d_pts'].view(-1, C)), d_bev.view(-1, C))
        if debug is not None:
            debug.setdefault('bwd', []).insert(0, dict(p2i=d_p2i, i2i=d_i2i, i2p=d_i2p, p2p=d_p2p, warped=s_pi))
        mha = L['mha']
        u = fold.i2p_unfold_grads(mha, r_ip['dM1'], r_ip['dc1'], r_ip['dM2'], r_ip['dc2'])
        f32 = lambda t: t.to(torch.float32).to(dev)
        if mha._qkv_same_embed_dim:
            grads[id(mha.in_proj_weight)] = f32(torch.cat([u['Wq'], u['Wk'], u['Wv']], 0))
        else:
            grads[id(mha.q_proj_weight)], grads[id(mha.k_proj_weight)], grads[id(mha.v_proj_weight)] = f32(u['Wq']), f32(u['Wk']), f32(u['Wv'])
        grads[id(mha.in_proj_bias)] = f32(torch.cat([u['bq'], u['bk'], u['bv']], 0))
        grads[id(mha.out_proj.weight)], grads[id(mha.out_proj.bias)] = f32(u['Wo']), f32(u['bo'])
    if d_pts_conv is not None:
        gp = bw._add(gp, d_pts_conv.reshape(-1, C))
    d_img_feats, g_img = bw._shared_conv_backward(gi, pk_img[0], img_feats)
    d_pts_feats, g_pts = bw._shared_conv_backward(gp, pk_pts[0], pts_feats)
    for conv, g_conv in ((enc.shared_conv_img, g_img), (enc.shared_conv_pts, g_pts)):
        grads[id(conv.weight)], grads[id(conv.bias)] = g_conv
    return dict(outputs=outputs, d_img_feats=d_img_feats, d_pts_feats=d_pts_feats,
                grads={names[k]: v for k, v in grads.items()})
