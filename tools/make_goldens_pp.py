#!/usr/bin/env python
"""Goldens of the ++ ("deformable") encoder from the REFERENCE's own models/necks/fusion_transformerv4.py, loaded by path
and unmodified (build container only; same mechanism as tools/make_goldens.py).

Additional stubs, i.e. third-party semantics this golden does NOT pin (SURVEY.md Appendix C.4-C.6):
  * mmcv 1.3.18 MultiScaleDeformableAttention, FFN, BaseTransformerLayer, build_transformer_layer, the ATTENTION /
    TRANSFORMER_LAYER registries -> the restatements in oracle/mmri_pp.py (so the golden pins the reference's OWN
    classes -- FusionTransformerv4, DeepInteractionLayer, MMRI_P2I, MMRI_I2P, MMRI_I2P_Polar, positional encoding,
    FlashMultiheadAttention wiring -- on top of those bricks);
  * flash-attn 0.2.2 `flash_attn_unpadded_kvpacked_func` (an fp16 GPU kernel) -> softmax attention on fp16-rounded
    q / kv with fp16-rounded probabilities and output (what the kernel's interface guarantees), evaluated in fp32;
  * mmcv `auto_fp16`: casts the named tensor arguments to half when the module has `fp16_enabled = True`, and the
    result back to float (out_fp32=True) -- true for FlashAttention only (fusion_transformerv4.py:665-667).

  * torch 1.9.1 `nn.Transformer` / `TransformerEncoder` / `TransformerDecoder` / `TransformerDecoderLayer`: the
    reference builds `nn.Transformer(num_encoder_layers=0, custom_decoder=...)` and a decoder layer whose attention
    modules it replaces (fusion_transformerv4.py:500-505,762-768).  torch 2.x's classes index `layers[0]` of the empty
    encoder and pass `is_causal` to the replaced attention, so they cannot run this file; the generator substitutes
    minimal classes with torch 1.9.1's documented forward (post-norm decoder layer; the layer-less encoder still
    applies its final LayerNorm -- Appendix C.6) before the reference file is loaded.

    python tools/make_goldens_pp.py        -> tests/golden/encoder_pp_small.pt, encoder_pp_nopolar.pt
"""
import copy
import functools
import inspect
import math
import os
import sys

import torch
import torch.nn as nn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))
sys.path.insert(0, os.path.join(ROOT, 'tests'))

import make_goldens as mg                 # noqa: E402
import oracle.mmri_pp as opp               # noqa: E402
from deepinteraction_b200 import synth     # noqa: E402


class _OnGpu(torch.Tensor):
    """CPU tensor that answers is_cuda = True: the reference asserts it (fusion_transformerv4.py:679) right before
    the flash-attn call, which is stubbed here."""
    is_cuda = property(lambda self: True)


def auto_fp16(apply_to=None, out_fp32=False):
    def wrap(fn):
        names = inspect.getfullargspec(fn).args

        @functools.wraps(fn)
        def inner(self, *args, **kw):
            if not getattr(self, 'fp16_enabled', False):
                return fn(self, *args, **kw)
            args = list(args)
            for i, a in enumerate(args):
                if names[i + 1] in apply_to and torch.is_tensor(a):
                    args[i] = a.half().as_subclass(_OnGpu)
            kw = {k: (v.half().as_subclass(_OnGpu) if k in apply_to and torch.is_tensor(v) else v) for k, v in kw.items()}
            out = fn(self, *args, **kw)
            if out_fp32:
                f = lambda o: o.as_subclass(torch.Tensor).float() if torch.is_tensor(o) else o
                out = tuple(f(o) for o in out) if isinstance(out, tuple) else f(out)
            return out
        return inner
    return wrap


def flash_attn_unpadded_kvpacked_func(q, kv, cu_q, cu_k, max_sq, max_sk, dropout_p, softmax_scale=None, causal=False):
    """q (B*Sq, H, D) fp16, kv (B*Sk, 2, H, D) fp16 with equal-length sequences -> (B*Sq, H, D) fp16."""
    q, kv = q.as_subclass(torch.Tensor), kv.as_subclass(torch.Tensor)
    nb = cu_q.numel() - 1
    H, D = q.shape[1], q.shape[2]
    qf = q.float().view(nb, max_sq, H, D).transpose(1, 2)
    k = kv[:, 0].float().view(nb, max_sk, H, D).transpose(1, 2)
    v = kv[:, 1].float().view(nb, max_sk, H, D).transpose(1, 2)
    scale = softmax_scale if softmax_scale is not None else 1.0 / math.sqrt(D)
    p = torch.softmax(qf @ k.transpose(-1, -2) * scale, -1).half().float()
    return (p @ v).transpose(1, 2).reshape(nb * max_sq, H, D).half()


class T19DecoderLayer(nn.Module):
    """torch 1.9.1 nn.TransformerDecoderLayer (norm_first did not exist: post-norm)."""

    def __init__(self, d_model, nhead, dim_feedforward=2048, dropout=0.1, activation='relu', layer_norm_eps=1e-5,
                 batch_first=False, device=None, dtype=None):
        super().__init__()
        self.self_attn = nn.MultiheadAttention(d_model, nhead, dropout=dropout, batch_first=batch_first)
        self.multihead_attn = nn.MultiheadAttention(d_model, nhead, dropout=dropout, batch_first=batch_first)
        self.linear1, self.dropout, self.linear2 = nn.Linear(d_model, dim_feedforward), nn.Dropout(dropout), nn.Linear(dim_feedforward, d_model)
        self.norm1, self.norm2, self.norm3 = (nn.LayerNorm(d_model, eps=layer_norm_eps) for _ in range(3))
        self.dropout1, self.dropout2, self.dropout3 = nn.Dropout(dropout), nn.Dropout(dropout), nn.Dropout(dropout)
        assert activation == 'relu'

    def forward(self, tgt, memory, tgt_mask=None, memory_mask=None, tgt_key_padding_mask=None, memory_key_padding_mask=None):
        t2 = self.self_attn(tgt, tgt, tgt, attn_mask=tgt_mask, key_padding_mask=tgt_key_padding_mask)[0]
        tgt = self.norm1(tgt + self.dropout1(t2))
        t2 = self.multihead_attn(tgt, memory, memory, attn_mask=memory_mask, key_padding_mask=memory_key_padding_mask)[0]
        tgt = self.norm2(tgt + self.dropout2(t2))
        t2 = self.linear2(self.dropout(torch.relu(self.linear1(tgt))))
        return self.norm3(tgt + self.dropout3(t2))


class T19Stack(nn.Module):
    """torch 1.9.1 nn.TransformerEncoder / nn.TransformerDecoder: N cloned layers, then the optional final norm."""

    def __init__(self, layer, num_layers, norm=None):
        super().__init__()
        self.layers = nn.ModuleList(copy.deepcopy(layer) for _ in range(num_layers))
        self.num_layers, self.norm = num_layers, norm

    def forward(self, x, *a, **k):
        for m in self.layers:
            x = m(x, *a, **k)
        return self.norm(x) if self.norm is not None else x


class T19Transformer(nn.Module):
    def __init__(self, d_model=512, nhead=8, num_encoder_layers=6, num_decoder_layers=6, dim_feedforward=2048, dropout=0.1,
                 activation='relu', custom_encoder=None, custom_decoder=None, layer_norm_eps=1e-5, batch_first=False):
        super().__init__()
        assert custom_encoder is None and custom_decoder is not None and num_encoder_layers == 0
        self.encoder = T19Stack(nn.Identity(), 0, nn.LayerNorm(d_model, eps=layer_norm_eps))
        self.decoder = custom_decoder

    def forward(self, src, tgt):
        return self.decoder(tgt, self.encoder(src))


def install_pp_stubs(ref):
    mg.install_stubs(ref)
    nn.TransformerDecoderLayer, nn.TransformerDecoder, nn.TransformerEncoder, nn.Transformer = \
        T19DecoderLayer, T19Stack, T19Stack, T19Transformer
    sm = sys.modules
    for n in ['flash_attn', 'flash_attn.flash_attn_interface', 'flash_attn.bert_padding', 'mmcv.cnn.bricks.registry']:
        mg._mod(n)
    sm['flash_attn.flash_attn_interface'].flash_attn_unpadded_kvpacked_func = flash_attn_unpadded_kvpacked_func
    for n in ('unpad_input', 'pad_input', 'index_first_axis'):
        setattr(sm['flash_attn.bert_padding'], n, None)
    sm['mmcv.runner'].auto_fp16 = auto_fp16

    class BaseModule(nn.Module):
        def __init__(self, init_cfg=None):
            super().__init__()
    sm['mmcv.runner'].BaseModule = BaseModule
    attention, layers = mg._Registry(), mg._Registry()
    attention.d['MultiScaleDeformableAttention'] = opp.MultiScaleDeformableAttention
    sm['mmcv.cnn.bricks.registry'].ATTENTION = attention
    sm['mmcv.cnn.bricks.registry'].TRANSFORMER_LAYER = layers

    class BaseTransformerLayer(nn.Module):                      # mmcv 1.3.18 constructor semantics (Appendix C.5)
        def __init__(self, attn_cfgs=None, ffn_cfgs=None, operation_order=None, norm_cfg=None, init_cfg=None,
                     batch_first=False, **kw):
            super().__init__()
            self.batch_first, self.operation_order = batch_first, operation_order
            self.pre_norm = operation_order[0] == 'norm'
            self.attentions = nn.ModuleList()
            for cfg in attn_cfgs:
                cfg = copy.deepcopy(cfg)
                cfg.setdefault('batch_first', batch_first)
                self.attentions.append(attention.build(cfg))
            self.embed_dims = self.attentions[0].embed_dims
            self.ffns = nn.ModuleList()
            for _ in range(operation_order.count('ffn')):
                cfg = {k: v for k, v in copy.deepcopy(dict(ffn_cfgs)).items() if k != 'type'}
                cfg.setdefault('embed_dims', self.embed_dims)
                self.ffns.append(opp.FFN(**cfg))
            self.norms = nn.ModuleList(nn.LayerNorm(self.embed_dims) for _ in range(operation_order.count('norm')))
    tr = sm['mmcv.cnn.bricks.transformer']
    tr.FFN, tr.BaseTransformerLayer = opp.FFN, BaseTransformerLayer
    tr.MultiScaleDeformableAttention = opp.MultiScaleDeformableAttention
    tr.build_transformer_layer = layers.build
    ft = mg._load('projects.mmdet3d_plugin.models.necks.fusion_transformerv4',
                  os.path.join(ref, mg.PLUGIN, 'models/necks/fusion_transformerv4.py'))
    return ft


def pp_layers(polar=True, hidden=128):
    msda = dict(type='MultiScaleDeformableAttention', embed_dims=hidden, num_levels=2, batch_first=True)
    ffn = dict(type='FFN', embed_dims=hidden, feedforward_channels=4 * hidden, num_fcs=2, ffn_drop=0.1,
               act_cfg=dict(type='ReLU', inplace=True))
    img = dict(type='DeepInteractionLayer', attn_cfgs=[msda, dict(type='MMRI_P2I', embed_dims=hidden, batch_first=True)],
               ffn_cfgs=ffn, operation_order=('self_attn', 'norm', 'cross_attn', 'norm', 'ffn', 'norm', 'ffn', 'norm'))
    attn = [msda]
    order = ['self_attn', 'norm']
    if polar:
        attn.append(dict(type='MMRI_I2P_Polar', embed_dims=hidden, dropout=0.1, batch_first=True))
        order += ['cross_attn', 'norm']
    attn.append(dict(type='MMRI_I2P', embed_dims=hidden, dropout=0.1, batch_first=True, fp16_enabled=True,
                     group_attn_enabled=True))
    order += ['cross_attn', 'norm', 'ffn', 'norm']
    pts = dict(type='DeepInteractionLayer', attn_cfgs=attn, ffn_cfgs=ffn, operation_order=tuple(order))
    return img, pts


def randomize_pp(model, seed):
    """Non-degenerate deformable attention: mmcv initialises sampling_offsets.weight / attention_weights to zero."""
    synth.randomize_norm_stats(model, seed)
    g = torch.Generator().manual_seed(seed + 17)
    for m in model.modules():
        if hasattr(m, 'sampling_offsets') and hasattr(m, 'attention_weights'):
            m.sampling_offsets.weight.data = torch.randn(m.sampling_offsets.weight.shape, generator=g) * 0.05
            m.attention_weights.weight.data = torch.randn(m.attention_weights.weight.shape, generator=g) * 0.1
            m.attention_weights.bias.data = torch.randn(m.attention_weights.bias.shape, generator=g) * 0.1
        if isinstance(m, nn.LayerNorm):
            m.weight.data = 1 + 0.2 * torch.randn(m.weight.shape, generator=g)
            m.bias.data = 0.1 * torch.randn(m.bias.shape, generator=g)
    for n, p in model.named_parameters():
        if n.endswith('scale'):
            p.data.fill_(0.7)


def pp_frame(seed, aug, views=2, c_img=16, c_pts=24, bev=36, batch=1):
    """Small ++ scene: image levels 28x50 and 14x25, three BEV maps (concat of the two SECONDFPN maps first)."""
    fr = mg.small_frame(seed, aug=aug, views=views, c_img=c_img, c_pts=c_pts, bev=bev, batch=batch)
    g = torch.Generator().manual_seed(seed + 3)
    lvl1 = torch.randn(batch * views, c_img, 14, 25, generator=g)
    p1, p2 = fr['pts_feats'], torch.randn(batch, c_pts, bev, bev, generator=g)
    fr['img_levels'] = [fr['img_feats'], lvl1]
    fr['pts_levels'] = [torch.cat([p1, p2], 1), p1, p2]
    return fr


def main():
    ft = install_pp_stubs('/root/reference')
    torch.set_grad_enabled(False)
    out_dir = os.path.join(ROOT, 'tests', 'golden')
    cmp = lambda a, b: float((a - b).abs().max() / b.abs().max().clamp_min(1e-12))
    for tag, polar, aug in (('encoder_pp_small', True, True), ('encoder_pp_nopolar', False, False)):
        seed = 2100 + int(polar)
        img_l, pts_l = pp_layers(polar)
        torch.manual_seed(seed)
        om = opp.FusionTransformerv4(2, 2, 16, 24, 128, img_transformerlayers=img_l, pts_transformerlayers=pts_l).eval()
        randomize_pp(om, seed)
        rm = ft.FusionTransformerv4(num_layers=2, num_lidar_maps=2, in_channels_img=16, in_channels_pts=24,
                                    hidden_channel=128, img_transformerlayers=img_l, pts_transformerlayers=pts_l).eval()
        rm.load_state_dict(om.state_dict(), strict=True)
        fr = pp_frame(seed, aug)
        r_img, (r_p0, r_p1) = rm(list(fr['img_levels']), list(fr['pts_levels']), fr['img_metas'], fr['pts_metas'])
        o_img, (o_p0, o_p1) = om(list(fr['img_levels']), list(fr['pts_levels']), fr['img_metas'], fr['pts_metas'])
        print(tag, 'oracle vs reference: img %.2e pts_conv %.2e pts %.2e' % (cmp(o_img, r_img), cmp(o_p0, r_p0), cmp(o_p1, r_p1)))
        sub = 1 if polar else 4            # the second golden keeps every 4th channel (fixture size)
        from golden_sample import shrink           # sampled storage of the larger maps (tests/golden_sample.py)
        torch.save(shrink(dict(seed=seed, aug=aug, polar=polar, checksum=mg.state_checksum(om.state_dict()), channel_step=sub,
                               img=r_img[:, ::sub].clone(), pts_conv=r_p0[:, ::sub].clone(), pts=r_p1[:, ::sub].clone())),
                   os.path.join(out_dir, tag + '.pt'))
        print(tag, '%.0f KiB' % (os.path.getsize(os.path.join(out_dir, tag + '.pt')) / 1024))


if __name__ == '__main__':
    main()
