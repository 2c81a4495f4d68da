"""The ++ ("deformable") MMRI encoder of DeepInteraction++ on libdi_b200 (BASELINE.json config 4).

Reference: projects/mmdet3d_plugin/models/necks/fusion_transformerv4.py -- FusionTransformerv4 :25-138,
DeepInteractionLayer :142-218, MMRI_P2I (BEVWarp + 1-level deformable attention) :220-240, MMRI_I2P (+ residual)
:242-364, MMRI_I2P_Polar :487-640 -- and the mmcv 1.3.18 bricks they are assembled from (MultiScaleDeformableAttention,
FFN, BaseTransformerLayer; SURVEY.md Appendix C.4 / C.5).  Parameter names equal the reference's, so a ++ checkpoint
loads unchanged (`img_fusion_blocks.N.attentions.M...`, `...ffns.K.layers.0.0`, `...norms.J`, `...scale`).

Schedule (pixel-major rows, fp32; no torch math on device tensors):
  * the three 3x3 convs on the wgmma implicit-GEMM kernel; per layer and modality
    value_proj / (sampling_offsets | attention_weights) / output_proj / FFN as tensor-core GEMMs (the two query-side
    Linear layers are ONE GEMM), di_msdeform_f32 for the sampling core, LayerNorm + residual in di_rows_finish_f32;
  * MMRI_P2I: the BEVWarp geometry of the base encoder (depth scatter, GPU depth completion, lifting: once per frame)
    + di_bev_sample_f32 + a 1-level deformable attention; MMRI_I2P: the folded single-head pillar attention of the
    base encoder + residual scatter-add; MMRI_I2P_Polar: see PolarBlock below.
"""
import math

import torch
import torch.nn as nn

from . import fold, geom, ops
from .graph import GraphCache
from .mmri import Geometry, MMRI_I2P as _I2PHolder, _pow2_cap, POINT_CAP_MIN

PC_RANGE = (-54.0, -54.0, -5.0, 54.0, 54.0, 3.0)


# ------------------------------------------------------------------------------------------------
# parameter holders (names == reference state_dict keys; they never run torch math)
# ------------------------------------------------------------------------------------------------
class MultiScaleDeformableAttention(nn.Module):
    def __init__(self, embed_dims=256, num_heads=8, num_levels=4, num_points=4, im2col_step=64, dropout=0.1,
                 batch_first=False, norm_cfg=None, init_cfg=None):
        super().__init__()
        self.embed_dims, self.num_heads, self.num_levels, self.num_points = embed_dims, num_heads, num_levels, num_points
        self.sampling_offsets = nn.Linear(embed_dims, num_heads * num_levels * num_points * 2)
        self.attention_weights = nn.Linear(embed_dims, num_heads * num_levels * num_points)
        self.value_proj = nn.Linear(embed_dims, embed_dims)
        self.output_proj = nn.Linear(embed_dims, embed_dims)


class FFN(nn.Module):
    def __init__(self, embed_dims=256, feedforward_channels=1024, num_fcs=2, act_cfg=None, ffn_drop=0., **kw):
        super().__init__()
        assert num_fcs == 2
        self.embed_dims = embed_dims
        self.layers = nn.Sequential(
            nn.Sequential(nn.Linear(embed_dims, feedforward_channels), nn.ReLU(inplace=True), nn.Dropout(ffn_drop)),
            nn.Linear(feedforward_channels, embed_dims), nn.Dropout(ffn_drop))


class BEVWarp(nn.Module):
    pass


class MMRI_P2I(nn.Module):
    def __init__(self, embed_dims, batch_first=True):
        super().__init__()
        self.embed_dims = embed_dims
        self.Warp = BEVWarp()
        self.Local = MultiScaleDeformableAttention(embed_dims, num_levels=1, batch_first=batch_first)


class MMRI_I2P(_I2PHolder):
    def __init__(self, embed_dims, dropout, batch_first=True, fp16_enabled=False, flash_attn=False,
                 group_attn_enabled=False):
        if flash_attn:
            raise NotImplementedError('MMRI_I2P(flash_attn=True) is not used by the ++ config and not built')
        super().__init__(embed_dims, embed_dims, dropout)
        self.embed_dims = embed_dims


class _MHAHolder(nn.Module):
    def __init__(self, d):
        super().__init__()
        self.in_proj_weight = nn.Parameter(torch.empty(3 * d, d))
        self.in_proj_bias = nn.Parameter(torch.zeros(3 * d))
        self.out_proj = nn.Linear(d, d)
        nn.init.xavier_uniform_(self.in_proj_weight)


class _DecoderLayerHolder(nn.Module):
    def __init__(self, d, ff):
        super().__init__()
        self.self_attn, self.multihead_attn = _MHAHolder(d), _MHAHolder(d)
        self.linear1, self.linear2 = nn.Linear(d, ff), nn.Linear(ff, d)
        self.norm1, self.norm2, self.norm3 = nn.LayerNorm(d), nn.LayerNorm(d), nn.LayerNorm(d)


class _NormHolder(nn.Module):
    def __init__(self, d):
        super().__init__()
        self.norm = nn.LayerNorm(d)


class _DecoderHolder(nn.Module):
    def __init__(self, d, ff):
        super().__init__()
        self.layers = nn.ModuleList([_DecoderLayerHolder(d, ff)])
        self.norm = nn.LayerNorm(d)


class _TransformerHolder(nn.Module):
    def __init__(self, d, ff):
        super().__init__()
        self.encoder, self.decoder = _NormHolder(d), _DecoderHolder(d, ff)


class MMRI_I2P_Polar(nn.Module):
    def __init__(self, embed_dims, dropout, batch_first=True, radius_range=(1., 61., 1.0), num_decoder_layers=1,
                 pc_range=PC_RANGE):
        super().__init__()
        assert num_decoder_layers == 1
        self.embed_dims, self.radius_range, self.pc_range = embed_dims, list(radius_range), list(pc_range)
        self.radius = int((radius_range[1] - radius_range[0]) / radius_range[-1])
        self.transformer_layers = _TransformerHolder(embed_dims, embed_dims * 4)


ATTENTIONS = dict(MultiScaleDeformableAttention=MultiScaleDeformableAttention, MMRI_P2I=MMRI_P2I, MMRI_I2P=MMRI_I2P,
                  MMRI_I2P_Polar=MMRI_I2P_Polar)


class DeepInteractionLayer(nn.Module):
    """Holder with mmcv BaseTransformerLayer's attribute layout (attentions / ffns / norms) + `scale`."""

    def __init__(self, attn_cfgs, ffn_cfgs, operation_order=None, norm_cfg=None, batch_first=True, **kw):
        super().__init__()
        self.operation_order = tuple(operation_order)
        if self.operation_order[0] == 'norm' or not batch_first:
            raise NotImplementedError('DeepInteractionLayer: only the post-norm, batch_first layout of the ++ config is built')
        self.attentions = nn.ModuleList()
        for cfg in attn_cfgs:
            cfg = dict(cfg)
            self.attentions.append(ATTENTIONS[cfg.pop('type')](**cfg))
        self.embed_dims = self.attentions[0].embed_dims
        ffn_cfg = {k: v for k, v in dict(ffn_cfgs).items() if k != 'type'}
        self.ffns = nn.ModuleList(FFN(**dict(ffn_cfg)) for _ in range(self.operation_order.count('ffn')))
        self.norms = nn.ModuleList(nn.LayerNorm(self.embed_dims) for _ in range(self.operation_order.count('norm')))
        self.scale = nn.Parameter(torch.ones(1))


# ------------------------------------------------------------------------------------------------
# weight packs + building blocks of the schedule
# ------------------------------------------------------------------------------------------------
def _lin(m):
    return m.weight.detach().double().cpu(), m.bias.detach().double().cpu()


def _pack_msda(m, device):
    wv, bv = _lin(m.value_proj)
    wo, bo = _lin(m.output_proj)
    ws, bs = _lin(m.sampling_offsets)
    wa, ba = _lin(m.attention_weights)
    W, d = (lambda t: fold.Weight(t, device)), (lambda t: fold.dev(t, device))
    return dict(kind='msda', L=m.num_levels, heads=m.num_heads, points=m.num_points, value=(W(wv), d(bv)), out=(W(wo), d(bo)),
                raw=(W(torch.cat([ws, wa], 0)), d(torch.cat([bs, ba], 0))))     # offsets | logits in ONE GEMM


def _pack_ffn(m, device):
    w1, b1 = _lin(m.layers[0][0])
    w2, b2 = _lin(m.layers[1])
    return (fold.Weight(w1, device), fold.dev(b1, device), fold.Weight(w2, device), fold.dev(b2, device))


def _pack_ln(m, device):
    return fold.dev(m.weight.detach().double().cpu(), device), fold.dev(m.bias.detach().double().cpu(), device), float(m.eps)


def msda_forward(pk, query_rows, value_maps, B, hq, wq, saved=None):
    """mmcv MultiScaleDeformableAttention.forward (identity = query, batch_first): value_maps = list of [B,H_l,W_l,C].
    saved (a dict) receives the query rows, the value maps, their projections, raw and the sampled rows."""
    C = query_rows.shape[1]
    vals = [ops.linear([v.view(-1, C)], *pk['value']).view(v.shape) for v in value_maps]
    raw = ops.linear([query_rows], *pk['raw'])
    a = ops.msdeform(vals, raw, B, hq, wq, pk['heads'], pk['points'])
    if saved is not None:
        saved.update(q=query_rows, maps=list(value_maps), vals=vals, raw=raw, a=a)
    return ops.linear([a], *pk['out'], res=query_rows)


def ffn_forward(pk, x, saved=None):
    """FFN (identity = x); saved (a dict) receives the input and the hidden rows."""
    w1, b1, w2, b2 = pk
    h = ops.linear([x], w1, b1, ops.ACT_RELU)
    if saved is not None:
        saved.update(x=x, h=h)
    return ops.linear([h], w2, b2, res=x)


def ln_forward(pk, x):
    return ops.rows_finish(x, gamma=pk[0], beta=pk[1], eps=pk[2])


class FusionTransformerv4(nn.Module):
    """Drop-in for the reference ``FusionTransformerv4`` (NECKS): same constructor, state_dict, forward signature
    (img_feats: list of levels, pts_feats: [concat, map_1, map_2, ...]) and return structure; inference only."""

    def __init__(self, num_layers=2, num_lidar_maps=2, in_channels_img=64, in_channels_pts=128 * 3, hidden_channel=128,
                 bn_momentum=0.1, bias='auto', img_transformerlayers=None, pts_transformerlayers=None):
        super().__init__()
        use_bias = True if bias == 'auto' else bool(bias)
        self.shared_conv_pts = nn.Conv2d(in_channels_pts * num_lidar_maps, hidden_channel, 3, padding=1, bias=use_bias)
        self.multi_scale_conv_img = nn.Conv2d(in_channels_img, hidden_channel, 3, padding=1, bias=use_bias)
        self.multi_scale_conv_pts = nn.Conv2d(in_channels_pts, hidden_channel, 3, padding=1, bias=use_bias)
        self.num_layers, self.hidden_channel, self.bn_momentum = num_layers, hidden_channel, bn_momentum
        mk = lambda cfg: DeepInteractionLayer(**{k: v for k, v in dict(cfg).items() if k != 'type'})
        self.img_fusion_blocks = nn.ModuleList(mk(img_transformerlayers) for _ in range(num_layers))
        self.pts_fusion_blocks = nn.ModuleList(mk(pts_transformerlayers) for _ in range(num_layers))
        self._pack = None
        self._pack_key = None
        self._side_streams = {}
        self.last_geometry = None
        self._graphs = GraphCache()

    # -- packing -----------------------------------------------------------------------------------
    def _state_key(self):
        return tuple((p.data_ptr(), p._version) for p in list(self.parameters()) + list(self.buffers()))

    def _pack_layer(self, layer, device):
        attn = []
        for a in layer.attentions:
            if isinstance(a, MultiScaleDeformableAttention):
                attn.append(_pack_msda(a, device))
            elif isinstance(a, MMRI_P2I):
                attn.append(dict(_pack_msda(a.Local, device), kind='p2i'))
            elif isinstance(a, MMRI_I2P_Polar):
                from .polar import pack_polar
                attn.append(pack_polar(a, device))
            elif isinstance(a, MMRI_I2P):
                M1, c1, M2, c2 = fold.i2p_fold(a.learnedAlign)
                attn.append(dict(kind='i2p', w=(fold.Weight(M1, device), fold.dev(c1, device), fold.Weight(M2, device),
                                                fold.dev(c2, device))))
            else:
                raise NotImplementedError(type(a).__name__)
        return dict(order=layer.operation_order, attn=attn, ffns=[_pack_ffn(f, device) for f in layer.ffns],
                    norms=[_pack_ln(n, device) for n in layer.norms], scale=fold.dev(layer.scale.detach().double().cpu(), device))

    def pack(self, force=False):
        key = self._state_key()
        if self._pack is not None and key == self._pack_key and not force:
            return self._pack
        device = self.shared_conv_pts.weight.device
        if device.type != 'cuda':
            raise RuntimeError('FusionTransformerv4 (libdi_b200) runs on CUDA only; move the module to a GPU')
        pk = {}
        for name in ('shared_conv_pts', 'multi_scale_conv_img', 'multi_scale_conv_pts'):
            W, b = fold.conv_bn(getattr(self, name))
            pk[name] = (fold.Weight(fold.pack_conv3x3(W), device), fold.dev(b, device))
        pk['img'] = [self._pack_layer(l, device) for l in self.img_fusion_blocks]
        pk['pts'] = [self._pack_layer(l, device) for l in self.pts_fusion_blocks]
        self._pack, self._pack_key = pk, key
        self._graphs.clear()
        return pk

    # -- forward -----------------------------------------------------------------------------------
    def _layer(self, lp, query_map, value_map, ms_maps, ctx, saved=None):
        """DeepInteractionLayer.forward (:161-218) on pixel-major maps.  query_map [Bq,hq,wq,C] (Bq = B*V or B).
        saved (a dict) selects the eager re-run of backward.encoder_pp_backward: saved['tape'] then lists every applied
        operation as (op, module index, 'query' or 'self' (the self_feat branch), its saved values), in order; the
        returned map is the same either way."""
        Bq, hq, wq, C = query_map.shape
        query = query_map.view(-1, C)
        order = lp['order']
        ni = ai = fi = 0
        self_feat = None
        tape = None if saved is None else saved.setdefault('tape', [])
        for op in order[:-2]:
            sv = None if saved is None else {}
            idx = None
            if op == 'self_attn':
                query, idx = msda_forward(lp['attn'][ai], query, ms_maps, Bq, hq, wq, saved=sv), ai
                ai += 1
                self_feat = query
            elif op == 'norm':
                if sv is not None:
                    sv['x'] = query
                query, idx = ln_forward(lp['norms'][ni], query), ni
                ni += 1
            elif op == 'cross_attn':
                query = self._cross(lp['attn'][ai], query.view(Bq, hq, wq, C), value_map, ctx, saved=sv).view(-1, C)
                idx = ai
                ai += 1
            elif op == 'ffn':
                query, idx = ffn_forward(lp['ffns'][fi], query, saved=sv), fi
                fi += 1
            if tape is not None and idx is not None:
                tape.append((op, idx, 'query', sv))
        for op in order[-2:]:
            sv = None if saved is None else {}
            idx = None
            if op == 'norm':
                if sv is not None:
                    sv['x'] = self_feat
                self_feat, idx = ln_forward(lp['norms'][ni], self_feat), ni
                ni += 1
            elif op == 'ffn':
                self_feat, idx = ffn_forward(lp['ffns'][fi], self_feat, saved=sv), fi
                fi += 1
            if tape is not None and idx is not None:
                tape.append((op, idx, 'self', sv))
        if saved is not None:
            saved.update(self_feat=self_feat, query=query, shape=(Bq, hq, wq, C))
        return ops.axpy(self_feat, query, lp['scale']).view(Bq, hq, wq, C)

    def _cross(self, ap, query_map, value_map, ctx, saved=None):
        g, pm, counts = ctx['g'], ctx['pm'], ctx['counts']
        Bq, hq, wq, C = query_map.shape
        if ap['kind'] == 'p2i':            # query = image maps [B*V,h,w,C], value = BEV map [B,Y,X,C]
            g.wait()
            warped = ops.bev_sample(value_map, g.grid, g.V)
            if saved is not None:
                saved['value_shape'] = tuple(value_map.shape)
            return msda_forward(ap, query_map.view(-1, C), [warped], Bq, hq, wq, saved=saved).view(Bq, hq, wq, C)
        if ap['kind'] == 'i2p':            # query = BEV map, value = image maps; + residual (:364)
            n_dev = None if counts is None else counts[0:1]
            coors = pm['pillar_coors']
            if saved is not None:
                saved.update(query_map=query_map, value_map=value_map)
            out = query_map.clone()
            if coors.shape[0] == 0:
                return out
            M1, c1, M2, c2 = ap['w']
            rows = ops.gather_rows(query_map, coors, n_dev)
            qk = ops.linear([rows], M1, c1)
            s, cnt = ops.i2p_attend(qk, pm['pillars'], pm['pillars_num_points'], coors, g.proj, value_map, g.V, g.in_hw, n_dev)
            o = ops.linear([s], M2, c2)
            return ops.scatter_rows_add(o, cnt, coors, out, n_dev)
        if ap['kind'] == 'polar':
            from .polar import polar_forward
            return polar_forward(ap, query_map, value_map, ctx, saved=saved)
        raise NotImplementedError(ap['kind'])

    def forward_nhwc(self, img_feats, pts_feats, img_metas, pts_metas):
        """-> img [B*V,h,w,C], pts_conv [B,Y,X,C], pts [B,Y,X,C] (pixel-major, fp32).  The kernel schedule is replayed
        from a CUDA graph once an input signature repeats (graph.py: feature maps bound by address, per-frame pillar /
        point arrays staged at fixed capacities, camera constants uploaded per replay)."""
        if self.training:
            raise NotImplementedError('libdi_b200 FusionTransformerv4 is forward/eval only (call .eval())')
        self.pack()
        img_feats, pts_feats = [t.contiguous() for t in img_feats], [t.contiguous() for t in pts_feats]
        dev_ = img_feats[0].device
        pillars, coors, npts, pts_list, consts = self._frame(img_metas, pts_metas, dev_)
        B_, _, Y_, X_ = pts_feats[0].shape
        staged = [pillars, coors, npts] + pts_list
        caps = [_pow2_cap(pillars.shape[0], B_ * Y_ * X_)] * 3 + [_pow2_cap(p.shape[0], POINT_CAP_MIN) for p in pts_list]
        consts.append(torch.tensor([pillars.shape[0]] + [p.shape[0] for p in pts_list], dtype=torch.int32))
        n_img = len(img_feats)
        inputs = img_feats + pts_feats
        sig = (tuple(tuple(t.shape) for t in inputs), tuple(tuple(t.shape[1:]) for t in staged), geom.input_hw(img_metas),
               id(self._pack))

        def fn(ins, cs, st):
            pm = dict(pillars=st[0], pillar_coors=st[1], pillars_num_points=st[2], pts=list(st[3:]))
            return self._schedule(list(ins[:n_img]), list(ins[n_img:]), img_metas, pm, cs)
        return self._graphs.run(sig, inputs, consts, fn, staged=staged, caps=caps)

    def _frame(self, img_metas, pts_metas, dev_):
        """-> (pillars, coors, npts, pts list) on the device in the schedule's dtypes, and the frame's host constants:
        the camera rows and, when a layer has a polar block, its constants (polar.polar_consts_host)."""
        pillars = pts_metas['pillars'].to(device=dev_, dtype=torch.float32).contiguous()
        coors = pts_metas['pillar_coors'].to(device=dev_, dtype=torch.int32).contiguous()
        npts = pts_metas['pillars_num_points'].to(device=dev_, dtype=torch.int32).contiguous()
        pts_list = [p.to(device=dev_, dtype=torch.float32) for p in pts_metas['pts']]
        proj_h, i2l_h = geom.camera_rows_host(img_metas)
        consts = [proj_h, i2l_h]
        if any(a['kind'] == 'polar' for l in self._pack['pts'] for a in l['attn']):
            from .polar import polar_consts_host
            consts += list(polar_consts_host(img_metas))
        return pillars, coors, npts, pts_list, consts

    def _schedule(self, img_feats, pts_feats, img_metas, pm, consts, saved=None):
        """The kernel schedule.  consts: device tensors (camera rows, polar constants when present, then the live counts
        or None for exact-size point arrays).  saved (a dict) selects the eager re-run of backward.encoder_pp_backward:
        it receives the geometry, the context, the multi-scale maps and per layer the saved dict of _layer."""
        pk = self._pack
        dev_ = img_feats[0].device
        C = self.hidden_channel
        counts = consts[-1]
        BV, _, h, w = img_feats[0].shape
        B, _, Y, X = pts_feats[0].shape
        cur_id = torch.cuda.current_stream().cuda_stream
        if cur_id not in self._side_streams:
            self._side_streams[cur_id] = torch.cuda.Stream(device=dev_)
        g = Geometry(img_metas, pm, (h, w), (Y, X), dev_, side_stream=self._side_streams[cur_id], cams=(consts[0], consts[1]),
                     counts=counts)
        self.last_geometry = g
        conv = lambda x, name: ops.conv3x3(x, *pk[name], cout=C, x_nhwc=False)
        pts_conv = conv(pts_feats[0], 'shared_conv_pts')
        ms_img = [conv(f, 'multi_scale_conv_img') for f in img_feats]
        ms_pts = [conv(f, 'multi_scale_conv_pts') for f in pts_feats[1:]]
        new_img, new_pts = ms_img[0], ms_pts[0]
        ctx = dict(g=g, pm=pm, counts=counts, img_metas=img_metas, B=B, V=BV // B)
        if len(consts) > 3:
            ctx['polar_consts'] = tuple(consts[2:5])
        if saved is not None:
            saved.update(g=g, ctx=ctx, ms_img=ms_img, ms_pts=ms_pts, pts_conv=pts_conv, img=[], pts=[])
        for i in range(self.num_layers):
            s_img, s_pts = (None, None) if saved is None else ({}, {})
            if saved is not None:
                saved['img'].append(s_img)
                saved['pts'].append(s_pts)
            t_img = self._layer(pk['img'][i], new_img, new_pts, ms_img, ctx, saved=s_img)
            t_pts = self._layer(pk['pts'][i], new_pts, new_img, ms_pts, ctx, saved=s_pts)
            new_img, new_pts = t_img, t_pts
        return new_img, pts_conv, new_pts

    def forward(self, img_feats, pts_feats, img_metas, pts_metas):
        img, pts_conv, pts = self.forward_nhwc(img_feats, pts_feats, img_metas, pts_metas)
        return img.permute(0, 3, 1, 2), [pts_conv.permute(0, 3, 1, 2), pts.permute(0, 3, 1, 2)]
