"""MMPI decoder on libdi_b200: parameter holders with the reference's state_dict schema and the kernel
schedule of one forward pass.

Reference: projects/mmdet3d_plugin/models/dense_heads/deepinteraction_decoder.py:19-313 (forward
:201-313) and models/utils/decoder_utils.py (PositionEmbeddingLearned :16-32, TransformerDecoderLayer
:35-113, MultiheadAttention :116-495, FFN :498-581, DynamicConv :584-629, ImageRCNNBlock :632-761,
PointRCNNBlock :765-841), core/bbox/coders/transfusion_bbox_coder.py.

Differences from the reference schedule (results unchanged, fp32):
  * queries are rows [B*P, C]; maps are pixel-major, so the top-k gather, RoIAlign and the cross
    attention read contiguous 512-byte rows;
  * the key positional embedding of the query x BEV cross attention depends only on the BEV grid, so
    its K/V contribution is precomputed once (pack time) and added in the K/V GEMM epilogue;
  * the per-sample / per-view Python loops of the RCNN blocks become ONE batched pass: every query is
    pooled from the view that wins it ("later views overwrite", decoder_utils.py:759) and attends to
    the queries of that view through a group mask -- no data-dependent host control flow, no syncs;
  * the 324k-element argsort is a radix select + 1024-slot bitonic sort in one CTA.
"""
import copy

import numpy as np
import os

import torch
import torch.nn as nn

from . import fold, geom, ops
from .loss import LossMixin
from .graph import GraphCache
from .mmri import ConvBN


# ------------------------------------------------------------------------------------------------
# parameter holders
# ------------------------------------------------------------------------------------------------
class PositionEmbeddingLearned(nn.Module):
    def __init__(self, cin, c):
        super().__init__()
        self.position_embedding_head = nn.Sequential(nn.Conv1d(cin, c, 1), nn.BatchNorm1d(c), nn.ReLU(inplace=True),
                                                     nn.Conv1d(c, c, 1))


class MultiheadAttention(nn.Module):
    def __init__(self, embed_dim, num_heads):
        super().__init__()
        self.embed_dim, self.num_heads = embed_dim, num_heads
        self.in_proj_weight = nn.Parameter(torch.empty(3 * embed_dim, embed_dim))
        self.in_proj_bias = nn.Parameter(torch.zeros(3 * embed_dim))
        self.out_proj = nn.Linear(embed_dim, embed_dim)
        nn.init.xavier_uniform_(self.in_proj_weight)
        nn.init.constant_(self.out_proj.bias, 0.0)


class TransformerDecoderLayer(nn.Module):
    def __init__(self, d_model, nhead, dim_ff):
        super().__init__()
        self.self_attn = MultiheadAttention(d_model, nhead)
        self.multihead_attn = MultiheadAttention(d_model, nhead)
        self.linear1 = nn.Linear(d_model, dim_ff)
        self.linear2 = nn.Linear(dim_ff, d_model)
        self.norm1, self.norm2, self.norm3 = nn.LayerNorm(d_model), nn.LayerNorm(d_model), nn.LayerNorm(d_model)
        self.self_posembed = PositionEmbeddingLearned(2, d_model)
        self.cross_posembed = PositionEmbeddingLearned(2, d_model)


class FFN(nn.Module):
    """Prediction heads: per head Sequential(ConvBN1d(in->64), Conv1d(64->k))."""

    def __init__(self, cin, heads, head_conv=64):
        super().__init__()
        self.heads = heads
        for name, (classes, num_conv) in heads.items():
            layers, c = [], cin
            for _ in range(num_conv - 1):
                layers.append(ConvBN(c, head_conv, 1, dims=1))
                c = head_conv
            layers.append(nn.Conv1d(c, classes, 1))
            setattr(self, name, nn.Sequential(*layers))


class DynamicConv(nn.Module):
    def __init__(self):
        super().__init__()
        self.dynamic_layer = nn.Linear(128, 2 * 128 * 128)
        self.norm1, self.norm2 = nn.LayerNorm(128), nn.LayerNorm(128)
        self.out_layer = nn.Linear(128 * 49, 128)
        self.norm3 = nn.LayerNorm(128)


def _rcnn_holder(blk, sfx, c, heads, dropout):
    setattr(blk, 'dyconv' + sfx, DynamicConv())
    setattr(blk, 'dyconv_pre_self_attn' + sfx, nn.MultiheadAttention(c, heads, dropout=dropout))
    for i in (1, 2, 3):
        setattr(blk, f'norm{i}' + sfx, nn.LayerNorm(c))
    setattr(blk, 'linear1' + sfx, nn.Linear(c, 4 * c))
    setattr(blk, 'linear2' + sfx, nn.Linear(4 * c, c))


class ImageRCNNBlock(nn.Module):
    sfx = ''

    def __init__(self, c, heads, dropout):
        super().__init__()
        _rcnn_holder(self, '', c, heads, dropout)


class PointRCNNBlock(nn.Module):
    sfx = '_pts'

    def __init__(self, c, heads, dropout):
        super().__init__()
        _rcnn_holder(self, '_pts', c, heads, dropout)


class TransFFN(nn.Module):
    """Holder with mmcv 1.3.18 FFN's parameter names (`layers.0.0`, `layers.1`): Linear-ReLU-Linear + identity."""

    def __init__(self, c, hidden, drop=0.):
        super().__init__()
        self.layers = nn.Sequential(nn.Sequential(nn.Linear(c, hidden), nn.ReLU(inplace=True), nn.Dropout(drop)),
                                    nn.Linear(hidden, c), nn.Dropout(drop))


def _rcnn_holder_v2(blk, sfx, c, heads, dropout):
    """decoder_utils.py:859-882 / :1004-1026 (`ffn`, `self_ffn`, `scale`, `self_scale` carry no `_pts` suffix)."""
    setattr(blk, 'dyconv' + sfx, DynamicConv())
    setattr(blk, 'dyconv_pre_self_attn' + sfx, nn.MultiheadAttention(c, heads, dropout=dropout))
    for i in (1, 2, 3):
        setattr(blk, f'norm{i}' + sfx, nn.LayerNorm(c))
    setattr(blk, 'self_norm' + sfx, nn.LayerNorm(c))
    blk.ffn = TransFFN(c, 4 * c, dropout)
    blk.self_ffn = TransFFN(c, 4 * c, dropout)
    blk.scale = nn.Parameter(torch.ones(1) * 0.5)
    blk.self_scale = nn.Parameter(torch.ones(1) * 0.5)


class ImageRCNNBlockV2(nn.Module):
    sfx, v2 = '', True

    def __init__(self, c, heads, dropout):
        super().__init__()
        _rcnn_holder_v2(self, '', c, heads, dropout)


class PointRCNNBlockV2(nn.Module):
    sfx, v2 = '_pts', True

    def __init__(self, c, heads, dropout):
        super().__init__()
        _rcnn_holder_v2(self, '_pts', c, heads, dropout)


class TransFusionBBoxCoder:
    """Drop-in for core/bbox/coders/transfusion_bbox_coder.py:8-126: same constructor, ``decode`` and ``encode``
    (CUDA tensors; kernels di_bbox_decode_f32 / di_bbox_encode_f32).  Unlike the reference, ``decode`` does not
    write into its ``center`` / ``dim`` arguments.  Inside the forward the RCNN blocks decode in di_rcnn_rois_f32."""

    def __init__(self, pc_range, out_size_factor, voxel_size, post_center_range=None, score_threshold=None,
                 code_size=8, **unused):
        self.pc_range, self.out_size_factor, self.voxel_size = pc_range, out_size_factor, voxel_size
        self.post_center_range, self.score_threshold, self.code_size = post_center_range, score_threshold, code_size

    def _scale(self):
        return (self.out_size_factor * self.voxel_size[0], self.out_size_factor * self.voxel_size[1],
                self.pc_range[0], self.pc_range[1])

    def encode(self, dst_boxes):
        return ops.bbox_encode(dst_boxes, self.code_size, *self._scale())

    def _decode_all(self, heatmap, rot, dim, center, height, vel, filter, qscore=None, qlabel=None):
        if filter and self.post_center_range is None:
            raise NotImplementedError('Need to reorganize output as a batch, only support post_center_range is not None for now!')
        rng = None if not filter else [float(v) for v in (self.post_center_range.tolist() if torch.is_tensor(
            self.post_center_range) else self.post_center_range)]
        return ops.bbox_decode(heatmap, rot, dim, center, height, vel, *self._scale(), post_range=rng,
                               score_thr=self.score_threshold if filter else None, qscore=qscore, qlabel=qlabel)

    def decode(self, heatmap, rot, dim, center, height, vel, filter=False):
        boxes, scores, labels, keep = self._decode_all(heatmap, rot, dim, center, height, vel, filter)
        labels = labels.long()
        if not filter:
            return [dict(bboxes=boxes[i], scores=scores[i], labels=labels[i]) for i in range(boxes.shape[0])]
        return [dict(bboxes=boxes[i, keep[i]], scores=scores[i, keep[i]], labels=labels[i, keep[i]])
                for i in range(boxes.shape[0])]


NMS_TASKS = {   # deepinteraction_decoder.py:575-586: (class indices, radius)
    'nuScenes': [((0, 1, 2, 3, 4, 5, 6, 7), -1.0), ((8,), 0.175), ((9,), 0.175)],
    'Waymo': [((0,), 0.7), ((1,), 0.7), ((2,), 0.7)],
}


HEAD_ORDER = ('center', 'height', 'dim', 'rot', 'vel', 'heatmap')


# The DynamicConv parameter generator streams a 32768 x 128 weight per MMPI layer; its output only feeds the
# (LayerNorm-ed) dynamic convolution, no index or softmax decision, so it may run the cheaper bf16 split.
_DYN_BF16 = os.environ.get('DI_B200_DYN_BF16', '0') != '0'


class DeepInteractionDecoder(nn.Module, LossMixin):
    """Drop-in for the reference ``DeepInteractionDecoder`` (HEADS): same constructor kwargs, state_dict
    and forward contract (``forward(pts_inputs, img_inputs, img_metas) -> [[dict]]``; side attributes
    ``query_labels`` and ``on_the_image_mask``); ``get_bboxes``, ``get_targets`` and ``loss`` (forward values,
    deepinteraction_b200/loss.py).  The forward is inference (eval) only."""
    _BLOCKS = (ImageRCNNBlock, PointRCNNBlock)
    _PRED_SRCS = 2          # prediction heads of the MMPI layers read cat([query, previous query]) (:289)

    def __init__(self, num_views=0, out_size_factor_img=4, num_proposals=128, auxiliary=True, hidden_channel=128,
                 num_classes=4, num_mmpi=4, num_decoder_layers=1, num_heads=8, learnable_query_pos=False,
                 initialize_by_heatmap=False, nms_kernel_size=1, ffn_channel=256, dropout=0.1, bn_momentum=0.1,
                 activation='relu', common_heads=dict(), num_heatmap_convs=2, conv_cfg=dict(type='Conv1d'),
                 norm_cfg=dict(type='BN1d'), bias='auto', loss_cls=dict(type='GaussianFocalLoss', reduction='mean'),
                 loss_bbox=dict(type='L1Loss', reduction='mean'),
                 loss_heatmap=dict(type='GaussianFocalLoss', reduction='mean'), train_cfg=None, test_cfg=None,
                 bbox_coder=None, ret_idx=None):
        super().__init__()
        if not initialize_by_heatmap:
            raise NotImplementedError('only initialize_by_heatmap=True (both reference configs) is supported')
        if hidden_channel != 128:
            raise NotImplementedError('DynamicConv is hard-coded to 128 channels in the reference (decoder_utils.py:589)')
        if activation != 'relu' or num_decoder_layers != 1 or num_mmpi % 2 != 0 or num_heatmap_convs != 2:
            raise NotImplementedError('unsupported decoder configuration for the libdi_b200 path')
        self.num_classes_heat = num_classes
        self.num_classes = num_classes + (0 if loss_cls.get('use_sigmoid', False) else 1)
        self.num_proposals, self.auxiliary, self.num_heads = num_proposals, auxiliary, num_heads
        self.num_decoder_layers, self.num_mmpi, self.num_views = num_decoder_layers, num_mmpi, num_views
        self.out_size_factor_img, self.nms_kernel_size = out_size_factor_img, nms_kernel_size
        self.train_cfg, self.test_cfg = train_cfg, test_cfg
        self.bbox_coder = TransFusionBBoxCoder(**{k: v for k, v in bbox_coder.items() if k != 'type'})
        c = hidden_channel
        self.hidden_channel = c
        use_bias = True if bias == 'auto' else bool(bias)
        self.heatmap_head = nn.Sequential(ConvBN(c, c, 3), nn.Conv2d(c, num_classes, 3, padding=1, bias=use_bias))
        self.heatmap_head_img = copy.deepcopy(self.heatmap_head)
        self.class_encoding = nn.Conv1d(num_classes, c, 1)
        self.decoder = nn.ModuleList(TransformerDecoderLayer(c, num_heads, ffn_channel)
                                     for _ in range(num_decoder_layers))
        heads = copy.deepcopy(common_heads)
        heads.update(dict(heatmap=(self.num_classes, num_heatmap_convs)))
        self.heads = heads
        self.prediction_heads = nn.ModuleList(FFN(c, heads) for _ in range(num_decoder_layers))
        self.decode_head, self.pred_head = nn.ModuleList(), nn.ModuleList()
        for _ in range(num_mmpi // 2):
            self.decode_head.append(self._BLOCKS[0](c, num_heads, dropout))
            self.pred_head.append(FFN(self._PRED_SRCS * c, heads))
            self.decode_head.append(self._BLOCKS[1](c, num_heads, dropout))
            self.pred_head.append(FFN(self._PRED_SRCS * c, heads))
        self.x_size = test_cfg['grid_size'][0] // test_cfg['out_size_factor']
        self.y_size = test_cfg['grid_size'][1] // test_cfg['out_size_factor']
        for p in self.decoder.parameters():          # reference :171-175
            if p.dim() > 1:
                nn.init.xavier_uniform_(p)
        for m in self.modules():
            if isinstance(m, (nn.BatchNorm2d, nn.BatchNorm1d)):
                m.momentum = bn_momentum
        order = [h for h in HEAD_ORDER if h in heads]
        assert order[:4] == ['center', 'height', 'dim', 'rot'] and set(order) == set(heads), \
            'prediction heads must be center, height, dim, rot[, vel], heatmap'
        self.head_order = order
        self.head_sizes = [heads[h][0] for h in order]
        self.NP = sum(self.head_sizes)
        self.query_labels = None
        self.on_the_image_mask = []
        self._pack, self._pack_key = None, None
        self._graphs = GraphCache()
        self._init_loss(train_cfg, loss_cls, loss_bbox, loss_heatmap)

    # -- packing -----------------------------------------------------------------------------------
    def _state_key(self):
        return tuple((p.data_ptr(), p._version) for p in list(self.parameters()) + list(self.buffers()))

    def _pack_pred(self, ffn, d):
        W1, b1, blocks, b2 = [], [], [], []
        for h in self.head_order:
            seq = getattr(ffn, h)
            w, b = fold.conv_bn(seq[0].conv, seq[0].bn)
            W1.append(w.reshape(w.shape[0], -1))
            b1.append(b)
            blocks.append(fold._d(seq[1].weight).reshape(seq[1].weight.shape[0], -1))
            b2.append(fold._d(seq[1].bias))
        dev_ = d(b1[0]).device
        return (fold.Weight(torch.cat(W1, 0), dev_), d(torch.cat(b1, 0)), fold.Weight(torch.block_diag(*blocks), dev_),
                d(torch.cat(b2, 0)))

    def _pack_mha(self, in_w, in_b, out_proj, d, two_source_q=False):
        C, h = self.hidden_channel, self.num_heads
        W, b = fold._d(in_w).clone(), fold._d(in_b).clone()
        s = float(C // h) ** -0.5
        W[:C] *= s          # q = (Wq x + bq) * head_dim^-0.5  (decoder_utils.py:407; same in nn.MultiheadAttention)
        b[:C] *= s
        dev_ = d(b).device
        return W, b, fold.Weight(fold._d(out_proj.weight), dev_), d(fold._d(out_proj.bias))

    def pack(self, force=False):
        key = self._state_key()
        if self._pack is not None and key == self._pack_key and not force:
            return self._pack
        device = self.class_encoding.weight.device
        if device.type != 'cuda':
            raise RuntimeError('DeepInteractionDecoder (libdi_b200) runs on CUDA only; move the module to a GPU')
        d = lambda t: fold.dev(t, device)
        C = self.hidden_channel
        pk = dict()
        for name in ('heatmap_head', 'heatmap_head_img'):
            seq = getattr(self, name)
            w0, b0 = fold.conv_bn(seq[0].conv, seq[0].bn)
            w1, b1 = fold.conv_bn(seq[1])
            # second conv: pad Cout to a multiple of 4 (zero rows) so that it can take the tensor-core path
            w1p, kpad = fold.pack_conv3x3(w1), (-w1.shape[0]) % 4
            w1p = torch.cat([w1p, torch.zeros(kpad, w1p.shape[1], dtype=w1p.dtype)], 0)
            b1p = torch.cat([b1, torch.zeros(kpad, dtype=b1.dtype)], 0)
            pk[name] = (fold.Weight(fold.pack_conv3x3(w0), device), d(b0), fold.Weight(w1p, device), d(b1p))
        pk['wce_t'] = d(fold._d(self.class_encoding.weight)[:, :, 0].t())
        pk['bce'] = d(fold._d(self.class_encoding.bias))
        layer = self.decoder[0]
        lin = lambda m: (d(fold._d(m.weight)), d(fold._d(m.bias)))
        linw = lambda m: (fold.Weight(fold._d(m.weight), device), d(fold._d(m.bias)))

        def pe_pack(pe):
            seq = pe.position_embedding_head
            w1, b1 = fold.conv_bn(seq[0], seq[1])
            return (fold.Weight(w1.reshape(w1.shape[0], -1), device), d(b1),
                    fold.Weight(fold._d(seq[3].weight)[:, :, 0], device), d(fold._d(seq[3].bias)))
        pk['self_pe'] = pe_pack(layer.self_posembed)
        W, b, wo, bo = self._pack_mha(layer.self_attn.in_proj_weight, layer.self_attn.in_proj_bias,
                                      layer.self_attn.out_proj, d)
        pk['self_attn'] = (fold.Weight(torch.cat([W, W], 1), device), d(b), wo, bo)   # sources [query | query_pos_embed]
        W, b, wo, bo = self._pack_mha(layer.multihead_attn.in_proj_weight, layer.multihead_attn.in_proj_bias,
                                      layer.multihead_attn.out_proj, d)
        pk['cross_q'] = (fold.Weight(torch.cat([W[:C], W[:C]], 1), device), d(b[:C]))
        w_kv, b_kv = fold.Weight(W[C:], device), d(b[C:])
        # constant key positional embedding -> its K/V contribution (the bev grid is fixed).  Folded ONCE on the host
        # in float64: this constant sits inside every cross-attention logit, so it must not carry kernel rounding.
        ys, xs = torch.meshgrid(torch.arange(self.y_size, dtype=torch.float64),
                                torch.arange(self.x_size, dtype=torch.float64), indexing='ij')
        bev_pos = torch.stack([xs + 0.5, ys + 0.5], -1).view(-1, 2)                  # flatten index = y*X + x (:162-169)
        seq = layer.cross_posembed.position_embedding_head
        w1, b1 = fold.conv_bn(seq[0], seq[1])
        h = torch.relu(bev_pos @ w1.reshape(w1.shape[0], -1).t() + b1)
        kpe = h @ fold._d(seq[3].weight)[:, :, 0].t() + fold._d(seq[3].bias)
        pk['cross_kv'] = (w_kv, b_kv, d(kpe @ fold._d(W[C:]).t()))
        pk['cross_pe'] = dict(pos=d(bev_pos), hidden=d(h), kpe=d(kpe))     # the backward's kk = bev + kpe and kpe's MLP
        pk['cross_out'] = (wo, bo)
        for i in (1, 2, 3):
            pk[f'norm{i}'] = lin(getattr(layer, f'norm{i}'))
        pk['ffn'] = linw(layer.linear1) + linw(layer.linear2)
        pk['pred0'] = self._pack_pred(self.prediction_heads[0], d)
        blocks = []
        for blk, ph in zip(self.decode_head, self.pred_head):
            g = lambda n: getattr(blk, n + blk.sfx)
            mha = g('dyconv_pre_self_attn')
            W, b, wo, bo = self._pack_mha(mha.in_proj_weight, mha.in_proj_bias, mha.out_proj, d)
            dy = g('dyconv')
            bp = dict(image=blk.sfx == '', attn=(fold.Weight(W, device), d(b), wo, bo), norm1=lin(g('norm1')),
                      norm2=lin(g('norm2')), norm3=lin(g('norm3')), dyn=linw(dy.dynamic_layer),
                      dn1=lin(dy.norm1), dn2=lin(dy.norm2), dout=lin(dy.out_layer), dn3=lin(dy.norm3),
                      pred=self._pack_pred(ph, d), v2=getattr(blk, 'v2', False))
            if bp['v2']:
                bp.update(ffn=linw(blk.ffn.layers[0][0]) + linw(blk.ffn.layers[1]),
                          self_ffn=linw(blk.self_ffn.layers[0][0]) + linw(blk.self_ffn.layers[1]),
                          self_norm=lin(g('self_norm')), scale=d(fold._d(blk.scale)), self_scale=d(fold._d(blk.self_scale)))
            else:
                bp.update(ffn=linw(g('linear1')) + linw(g('linear2')))
            blocks.append(bp)
        pk['blocks'] = blocks
        self._pack, self._pack_key = pk, key
        self._graphs.clear()                 # captured graphs hold pointers into the previous pack
        return pk

    # -- forward -----------------------------------------------------------------------------------
    def _pred(self, pack, srcs):
        w1, b1, w2, b2 = pack
        return self._mlp(srcs, w1, b1, ops.ACT_RELU, w2, b2)

    @staticmethod
    def _mlp(srcs, W1, b1, act1=ops.ACT_NONE, W2=None, b2=None, res=None, ln=None, act_out=ops.ACT_NONE, zero_if_neg=None):
        """act_out(LN(act1(cat(srcs) W1^T + b1) [W2^T + b2] + res)): ONE launch of the query-row MLP kernel when the
        shapes fit it (a few hundred query rows), otherwise the general dense-layer + rows_finish kernels."""
        M, K = srcs[0].shape[0], sum(t.shape[1] for t in srcs)
        if ops.can_rows_mlp(M, K, W1.shape[0], 0 if W2 is None else W2.shape[0]) and len(srcs) <= 2:
            return ops.rows_mlp(srcs, W1, b1, act1, W2, b2, res, None if ln is None else ln[0], None if ln is None else ln[1],
                                act_out, zero_if_neg)
        y = ops.linear(srcs, W1, b1, act1)
        if W2 is not None:
            y = ops.linear([y], W2, b2)
        if res is None and ln is None and act_out == ops.ACT_NONE and zero_if_neg is None:
            return y
        return ops.rows_finish(y, res=res, gamma=None if ln is None else ln[0], beta=None if ln is None else ln[1],
                               act=act_out, zero_if_neg=zero_if_neg)

    def _roi_params(self, in_hw):
        bc, tc = self.bbox_coder, self.test_cfg
        return [bc.out_size_factor * bc.voxel_size[0], bc.out_size_factor * bc.voxel_size[1], bc.pc_range[0],
                bc.pc_range[1], tc['out_size_factor'] * tc['voxel_size'][0], tc['pc_range'][0], in_hw[0], in_hw[1],
                bc.voxel_size[0] * bc.out_size_factor, bc.pc_range[0]]

    def _camera_consts(self, img_metas):
        """Host-side constants of one call: camera rows (B,V,12) and per-sample (crop_x, crop_y, flip, orig_w)."""
        proj, _ = geom.camera_rows_host(img_metas)
        aux = torch.tensor([[*(np.asarray(m.get('img_crop_offset', (0.0, 0.0)), np.float32).reshape(-1)[:2]),
                             1.0 if m.get('flip', False) else 0.0,
                             float(m['img_shape'][0][1]) if m.get('flip', False) else 0.0] for m in img_metas],
                           dtype=torch.float32)
        return proj, aux

    def forward_rows(self, pts_conv, new_pts, img, img_metas, debug=None):
        """pts_conv, new_pts [B,Y,X,C]; img [B*V,h,w,C] (pixel-major) -> dict(preds [B*P, NP] per layer, ...).
        Replayed from a CUDA graph once the input signature repeats (graph.py)."""
        if self.training:
            raise NotImplementedError('libdi_b200 DeepInteractionDecoder is forward/eval only (call .eval())')
        self.pack()
        proj_h, aux_h = self._camera_consts(img_metas)
        in_hw = geom.input_hw(img_metas)
        if debug is not None:
            dev_ = pts_conv.device
            return self._schedule(pts_conv, new_pts, img, in_hw, proj_h.to(dev_), aux_h.to(dev_), debug)
        inputs = [pts_conv, new_pts, img]
        sig = (tuple(tuple(t.shape) for t in inputs), in_hw, id(self._pack))

        def fn(ins, consts, staged):
            return self._schedule(ins[0], ins[1], ins[2], in_hw, consts[0], consts[1], None)
        return self._graphs.run(sig, inputs, [proj_h, aux_h], fn)

    def _schedule(self, pts_conv, new_pts, img, in_hw, proj, aux, debug):
        """Precision policy: every tensor-core product of the decoder uses the 3xTF32 split (error ~1e-7), not the
        bf16 split the encoder's image-sized layers use (~1e-5): the heatmap logits feed an index-exact top-k, the
        cross-attention logits go through exp over 32400 keys, and the query-level GEMMs are latency-bound anyway
        (measured: base-shape decoder outputs 1.1e-3 off with bf16 split, ~1e-4 with 3xTF32)."""
        bf_saved = ops.TC_BF16[0]
        ops.TC_BF16[0] = False
        try:
            return self._schedule_impl(pts_conv, new_pts, img, in_hw, proj, aux, debug)
        finally:
            ops.TC_BF16[0] = bf_saved

    def _schedule_impl(self, pts_conv, new_pts, img, in_hw, proj, aux, debug):
        pk = self._pack
        B, Y, X, C = pts_conv.shape
        assert (Y, X) == (self.y_size, self.x_size), 'BEV size must equal test_cfg grid_size // out_size_factor'
        HW, P, V, K, H = Y * X, self.num_proposals, self.num_views, self.num_classes_heat, self.num_heads
        dev_ = pts_conv.device
        # module tags + module-boundary bytes (SURVEY.md 8(d)) for bench.py's roofline table; no effect otherwise
        F_b, F_i = 4 * B * HW * C, 4 * img.numel()
        ops._MODULE[0] = ('heatmap_heads+nms+topk+query_init', 2 * F_b + 2 * 4 * K * B * HW, 2 * 2 * B * HW * 9 * C * (C + K))
        # heatmaps, NMS, top-k, query init
        w0, b0, w1, b1 = pk['heatmap_head']
        Kp = w1.shape[0]
        logit_a = ops.conv3x3(ops.conv3x3(pts_conv, w0, b0, C, True, False, ops.ACT_RELU), w1, b1, Kp, True, False)
        w0, b0, w1, b1 = pk['heatmap_head_img']
        logit_b = ops.conv3x3(ops.conv3x3(new_pts, w0, b0, C, True, False, ops.ACT_RELU), w1, b1, Kp, True, False)
        ds = self.test_cfg['dataset']
        no_nms = {'nuScenes': (1 << 8) | (1 << 9), 'Waymo': (1 << 1) | (1 << 2)}.get(ds, 0)
        heat, dense_b = ops.heatmap_nms(logit_a, logit_b, K, self.nms_kernel_size, no_nms)
        top = ops.topk(heat.view(B, K * HW), P)
        q, qpos, labels, qscore = ops.query_init(pts_conv.view(B, HW, C), top, heat, pk['wce_t'], pk['bce'], X)
        if debug is not None:
            debug.update(top=top, heat=heat, query_feat0=q.clone(), query_pos0=qpos.clone())
        # transformer decoder layer
        ops._MODULE[0] = ('TransformerDecoderLayer (query x BEV cross-attn)', F_b + 4 * (2 * C * C + 2 * HW * C),
                          2 * B * HW * C * 2 * C + 4 * B * P * HW * C)
        q = self._layer(pk, q, qpos, pts_conv, B, P)
        ops._MODULE[0] = ('prediction_heads', 0, 0)
        pred = self._pred(pk['pred0'], [q])
        ops.pred_finish(pred, qpos)
        first = pred
        if debug is not None:
            debug.update(query_feat1=q.clone(), first_res=first.clone())
        # MMPI layers
        prm = self._roi_params(in_hw)
        preds, wins, keeps = [], [], []
        if pk['blocks'] and pk['blocks'][0]['v2']:
            look = qpos.clone()                                   # deepinteractionplusplus_decoder.py:281
            keep = torch.empty(B * P, device=dev_, dtype=torch.int32)
        for li, bp in enumerate(pk['blocks']):
            prev = q
            # RoI reads <= one map; DynamicConv parameter generator weights 128 x 32768 (+ out_layer 6272 x 128) read once
            ops._MODULE[0] = ('ImageRCNNBlock' if bp['image'] else 'PointRCNNBlock',
                              4 * (B * P * 49 * C) + 4 * (C * 2 * C * C + 49 * C * C), 2 * B * P * (C * 2 * C * C + 2 * 49 * C * C + 49 * C * C))
            q, rois, win = self._rcnn_block(bp, prev, pred, new_pts, img, B, P, prm, proj, aux)
            if bp['v2']:
                ops._MODULE[0] = ('prediction_heads', 0, 0)
                pred = self._pred(bp['pred'], [q])
                ops.pred_finish_pp(pred, qpos, look, first, win if bp['image'] else None, keep, li == 0)
                keeps.append(keep.clone())
            else:
                ops._MODULE[0] = ('prediction_heads', 0, 0)
                pred = self._pred(bp['pred'], [q, prev])
                ops.pred_finish(pred, qpos, first if bp['image'] else None, win if bp['image'] else None)
            preds.append(pred)
            if bp['image']:
                wins.append(win)
            if debug is not None:
                debug.setdefault('layer_query', []).append(q.clone())
                debug.setdefault('rois', []).append(rois)
        ops._MODULE[0] = None
        return dict(preds=preds, wins=wins, keeps=keeps, qscore=qscore, dense_heatmap=dense_b, labels=labels)

    def _layer(self, pk, q, qpos, bev, B, P, saved=None):
        """TransformerDecoderLayer (decoder_utils.py:35-113) on query rows: q [B*P, C], qpos [B*P, 2], bev [B, Y, X, C]
        (pts_conv) -> [B*P, C].  The one implementation of the layer, for the forward schedule and for the eager re-run of
        backward.decoder_layer_backward.  saved (a dict) selects the re-run: the cross attention then always runs through
        xattn_tc_lse, so that its output O and row log-sum-exp come from one kernel, and the values the backward needs are
        stored in `saved`; the returned rows are the same either way."""
        C, H = self.hidden_channel, self.num_heads
        HW = bev.shape[1] * bev.shape[2]
        pw1, pb1, pw2, pb2 = pk['self_pe']
        qpe = self._mlp([qpos], pw1, pb1, ops.ACT_RELU, pw2, pb2)
        w, b, wo, bo = pk['self_attn']
        qkv = self._mlp([q, qpe], w, b)
        a = ops.mha_small(qkv[:, :C], qkv[:, C:2 * C], qkv[:, 2 * C:], B, P, H)
        q1 = self._mlp([a], wo, bo, res=q, ln=pk['norm1'])
        qc = self._mlp([q1, qpe], *pk['cross_q'])
        w_kv, b_kv, ckv = pk['cross_kv']
        kv = ops.linear([bev.view(B * HW, C)], w_kv, b_kv, res=ckv, res_mod=HW)
        if saved is not None:
            a2, lse, planes = ops.xattn_tc_lse(qc, kv, B, P, HW, H)
        elif ops.can_xattn_tc(P, C, H, B * HW):
            a2 = ops.xattn_tc(qc, kv, B, P, HW, H)                  # tensor-core attention kernel (xattn_tc.cu)
        else:
            a2 = ops.cross_attn(qc, kv, B, P, HW, H)
        q2 = self._mlp([a2], *pk['cross_out'], res=q1, ln=pk['norm2'])
        f1w, f1b, f2w, f2b = pk['ffn']
        q3 = self._mlp([q2], f1w, f1b, ops.ACT_RELU, f2w, f2b, res=q2, ln=pk['norm3'])
        if saved is not None:
            # pre-norm sums and the hidden rows of the two-layer MLPs, which the fused row kernels do not return
            f = self._mlp([q2], f1w, f1b, ops.ACT_RELU)
            saved.update(qpe=qpe, hs=self._mlp([qpos], pw1, pb1, ops.ACT_RELU), qkv=qkv, a1=a,
                         z1=self._mlp([a], wo, bo, res=q), q1=q1, a2=a2, lse=lse, planes=planes,
                         z2=self._mlp([a2], *pk['cross_out'], res=q1), q2=q2, f=f, z3=self._mlp([f], f2w, f2b, res=q2),
                         kk=ops.add_rows_mod(bev.reshape(B * HW, C), pk['cross_pe']['kpe']))
        return q3

    def _rcnn_block(self, bp, prev, pred, new_pts, img, B, P, prm, proj, aux, saved=None):
        """One RCNN block of the MMPI layers (decoder_utils.py:632-1089) on query rows: prev [B*P, C], pred [B*P, NP] (the
        previous layer's predictions, which give the RoIs), new_pts [B, Y, X, C] (BEV blocks) or img [B*V, h, w, C] (image
        blocks) -> (rows [B*P, C], rois [B*P, 5], win [B*P]).  The one implementation of the block, for the forward
        schedule and for the eager re-run of the block backwards in backward.py; saved (a dict) additionally stores the
        values the backward needs, with the returned rows unchanged."""
        C, H, V = self.hidden_channel, self.num_heads, self.num_views
        if bp['image']:
            rois, win, onbits = ops.rcnn_rois(pred, B, P, V, 0, prm, proj, aux)
            roi = ops.roi_align(img, rois, 1.0 / self.out_size_factor_img)
        else:
            rois, win, onbits = ops.rcnn_rois(pred, B, P, V, 1, prm)
            roi = ops.roi_align(new_pts, rois, 1.0)
        w, b, wo, bo = bp['attn']
        qkv = self._mlp([prev], w, b)
        a = ops.mha_small(qkv[:, :C], qkv[:, C:2 * C], qkv[:, 2 * C:], B, P, H, onbits, win)
        q1 = self._mlp([a], wo, bo, res=prev, ln=bp['norm1'])
        ops.TC_BF16[0] = _DYN_BF16                       # parameter generator (M=P, N=32768): see _DYN_BF16
        params = ops.linear([q1], *bp['dyn'])
        ops.TC_BF16[0] = False
        flat = ops.dynconv(roi, params, *bp['dn1'], *bp['dn2'])
        part = ops.linear([flat], bp['dout'][0], splits=49)
        t = ops.rows_finish(part, bias=bp['dout'][1], gamma=bp['dn3'][0], beta=bp['dn3'][1], act=ops.ACT_RELU)
        q2 = ops.rows_finish(t, res=q1, gamma=bp['norm2'][0], beta=bp['norm2'][1])
        f1w, f1b, f2w, f2b = bp['ffn']
        if saved is not None:
            # pre-norm sums and the hidden rows of the two-layer MLPs, which the fused row kernels do not return
            saved.update(rois=rois, win=win, onbits=onbits, qkv=qkv, a=a, z1=self._mlp([a], wo, bo, res=prev), q1=q1, params=params, roi=roi,
                         flat=flat, part=part, zd3=ops.rows_finish(part, bias=bp['dout'][1]), t=t,
                         z2=ops.rows_finish(t, res=q1), q2=q2)
        if bp['v2']:
            # decoder_utils.py:971-988 / :1071-1085.  The self branch every query of a (sample, view) group receives
            # is the one of the group's FIRST query (the reference's (1,n,C) + (n,1,C) broadcast followed by [0];
            # oracle/mmpi_pp.py), so it is evaluated on the B*V "leader" rows only.
            q3 = self._mlp([q2], f1w, f1b, ops.ACT_RELU, f2w, f2b, res=q2, ln=bp['norm3'])
            Vg = V if bp['image'] else 1
            lrow, lwin = ops.rcnn_leaders(onbits, B, P, Vg)
            a_l = ops.mha_small_rows(qkv[:, :C], qkv[:, C:2 * C], qkv[:, 2 * C:], B, P, H, onbits, lrow, lwin)
            q1_l = self._mlp([a_l], wo, bo, res=ops.take_rows(prev, lrow), ln=bp['norm1'])
            s1w, s1b, s2w, s2b = bp['self_ffn']
            s_l = self._mlp([q1_l], s1w, s1b, ops.ACT_RELU, s2w, s2b, res=q1_l, ln=bp['self_norm'])
            if saved is not None:
                f = self._mlp([q2], f1w, f1b, ops.ACT_RELU)
                fs = self._mlp([q1_l], s1w, s1b, ops.ACT_RELU)
                saved.update(f=f, z3=self._mlp([f], f2w, f2b, res=q2), q3=q3, lrow=lrow, lwin=lwin, a_l=a_l,
                             z1_l=self._mlp([a_l], wo, bo, res=ops.take_rows(prev, lrow)), q1_l=q1_l, fs=fs,
                             zs=self._mlp([fs], s2w, s2b, res=q1_l), s_l=s_l)
            return ops.branch_mix(q3, s_l, win, bp['scale'], bp['self_scale'], P, Vg, bp['image']), rois, win
        q = self._mlp([q2], f1w, f1b, ops.ACT_GELU, f2w, f2b, res=q2, ln=bp['norm3'],
                      zero_if_neg=win if bp['image'] else None)
        if saved is not None:
            h = self._mlp([q2], f1w, f1b)
            f = self._mlp([q2], f1w, f1b, ops.ACT_GELU)
            saved.update(h=h, f=f, z3=self._mlp([f], f2w, f2b, res=q2))
        return q, rois, win

    def _to_dict(self, pred, B, P):
        t = pred.view(B, P, self.NP).permute(0, 2, 1)
        out, o = {}, 0
        for h, n in zip(self.head_order, self.head_sizes):
            out[h] = t[:, o:o + n]
            o += n
        return out

    def forward_nhwc(self, pts_conv, new_pts, img, img_metas, debug=None):
        r = self.forward_rows(pts_conv, new_pts, img, img_metas, debug)
        return self._outputs(r, pts_conv.shape[0])

    def _outputs(self, r, B):
        """forward_rows' result -> the reference's [[dict]] output; sets query_labels and on_the_image_mask."""
        P = self.num_proposals
        self.query_labels = r['labels'].long()
        if r['keeps']:                                            # ++: one cumulative mask per layer (:295-299)
            self.on_the_image_mask = [(k.view(B, P) != 0) for k in r['keeps']]
        else:
            self.on_the_image_mask = [(w.view(B, P) != -1) for w in r['wins']]
        rets = [self._to_dict(p, B, P) for p in r['preds']]
        rets[0]['query_heatmap_score'] = r['qscore']
        rets[0]['dense_heatmap'] = r['dense_heatmap']
        if not self.auxiliary:
            return [rets[-1]]
        merged = {}
        for key in rets[0]:
            if key in ('dense_heatmap', 'dense_heatmap_old', 'query_heatmap_score'):
                merged[key] = rets[0][key]
            else:
                merged[key] = torch.cat([r_[key] for r_ in rets], -1)
        return [[merged]]

    def get_bboxes(self, preds_dicts, img_metas, img=None, rescale=False, for_roi=False):
        """deepinteraction_decoder.py:549-638 on the forward's output: last-layer score composition + box decode +
        range/score filter in one kernel, optional per-task circle NMS (nms_type 'circle'), one boolean compaction at
        the end (the only host synchronisation: the result length is data dependent).  Batch size 1 and a single
        layer, as the reference asserts (:631-632).  -> [[boxes, scores, labels.int()]]."""
        assert len(preds_dicts) == 1, 'get_bboxes expects the single merged layer the forward returns'
        p0, P = preds_dicts[0][0], self.num_proposals
        assert p0['heatmap'].shape[0] == 1, 'the reference get_bboxes supports batch size 1 (:632)'
        last = lambda k: p0[k][..., -P:]
        coder = self.bbox_coder
        boxes, scores, labels, keep = coder._decode_all(last('heatmap'), last('rot'), last('dim'), last('center'),
                                                        last('height'), last('vel') if 'vel' in p0 else None, True,
                                                        qscore=p0['query_heatmap_score'], qlabel=self.query_labels)
        nms = self.test_cfg['nms_type']
        if nms is not None:
            if nms != 'circle':
                raise NotImplementedError("nms_type %r: only None and 'circle' are provided (rotated NMS is mmdet3d's nms_gpu)" % nms)
            for classes, radius in NMS_TASKS[self.test_cfg['dataset']]:
                if radius > 0:
                    keep = ops.circle_nms(boxes, scores, labels, keep, sum(1 << c for c in classes), radius)
        k = keep[0]
        boxes, scores, labels = boxes[0, k], scores[0, k], labels[0, k]
        wrap = img_metas[0].get('box_type_3d') if isinstance(img_metas[0], dict) else None
        if wrap is not None:
            boxes = wrap(boxes, box_dim=boxes.shape[-1])
        return [[boxes, scores, labels.int()]]

    def forward(self, pts_inputs, img_inputs, img_metas):
        """pts_inputs: [pts_feat_conv, new_pts_feat] (B,C,Y,X); img_inputs (B*V,C,h,w).  NCHW tensors that are
        channels-last views (what DeepInteractionEncoder returns) are used in place; true NCHW is transposed."""
        def nhwc(t):
            p = t.permute(0, 2, 3, 1)
            return p if p.is_contiguous() else ops.nchw_to_nhwc(t.contiguous())
        return self.forward_nhwc(nhwc(pts_inputs[0]), nhwc(pts_inputs[1]), nhwc(img_inputs), img_metas)


class DeepInteractionPlusPlusDecoder(DeepInteractionDecoder):
    """Drop-in for the reference ``DeepInteractionPlusPlusDecoder`` (HEADS; models/dense_heads/
    deepinteractionplusplus_decoder.py:19-319): V2 RCNN blocks (decoder_utils.py:844-1089), prediction heads on C
    channels (:140, :147), look-forward centre update (:281-294), cumulative on-image mask and first-layer fallback at
    every layer (:295-302; ``on_the_image_mask`` holds num_mmpi masks).  Same constructor kwargs and state_dict."""
    _BLOCKS = (ImageRCNNBlockV2, PointRCNNBlockV2)
    _PRED_SRCS = 1
    _PP_MASKS = True          # loss: every layer's weights are multiplied by that layer's mask (:513-514)
