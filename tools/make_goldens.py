#!/usr/bin/env python
"""Generate tests/golden/*.pt from the REFERENCE's own Python files.

Runs only in the build container (needs /root/reference, read-only).  The
reference package cannot be imported (mmcv/mmdet/mmdet3d/detectron2/spconv are
absent), so its hot-path files are loaded BY PATH, unmodified, under their real
dotted names with small ``sys.modules`` stubs for the absent third-party imports
(SURVEY.md Appendix B).  What each stub assumes is documented next to it.

Every golden stores: the config, the seed, a checksum of the weights, the inputs
that are not re-creatable from the seed, and the reference outputs.  Weights are
created by the ORACLE modules under the seed and loaded into the reference
modules with ``load_state_dict(strict=True)`` -- which also pins state-dict key
compatibility.  tests/test_oracle_golden.py re-creates them from the seed.

Usage:  python tools/make_goldens.py [--ref /root/reference] [--out tests/golden]
"""
import argparse
import hashlib
import importlib.util
import copy
import os
import sys
import types

import numpy as np
import torch
import torch.nn as nn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))

import oracle.geometry as og          # noqa: E402
import oracle.mmri as ommri            # noqa: E402
import oracle.mmpi as ommpi            # noqa: E402
from oracle.mmri_pp import FFN as ompp_ffn   # noqa: E402
import oracle.loss as oloss            # noqa: E402
from deepinteraction_b200 import synth  # noqa: E402

PLUGIN = 'projects/mmdet3d_plugin'


def _mod(name):
    m = types.ModuleType(name)
    sys.modules[name] = m
    return m


def _load(name, path):
    spec = importlib.util.spec_from_file_location(name, path)
    m = importlib.util.module_from_spec(spec)
    sys.modules[name] = m
    spec.loader.exec_module(m)
    return m


class _Registry:
    def __init__(self):
        self.d = {}

    def register_module(self, *a, **k):
        def deco(cls):
            self.d[cls.__name__] = cls
            return cls
        return deco

    def build(self, cfg):
        cfg = dict(cfg)
        return self.d[cfg.pop('type')](**cfg)


def install_stubs(ref):
    np.bool = bool                                    # depth_map_utils.py:209,226 (numpy<1.24 alias)
    for n in ['projects', 'projects.mmdet3d_plugin', 'projects.mmdet3d_plugin.models',
              'projects.mmdet3d_plugin.models.utils', 'projects.mmdet3d_plugin.models.utils.ops',
              'projects.mmdet3d_plugin.models.utils.ip_basic', 'projects.mmdet3d_plugin.models.necks',
              'projects.mmdet3d_plugin.models.dense_heads', 'projects.mmdet3d_plugin.core',
              'projects.mmdet3d_plugin.core.bbox', 'projects.mmdet3d_plugin.core.bbox.coders',
              'mmcv', 'mmcv.cnn', 'mmcv.cnn.bricks', 'mmcv.cnn.bricks.transformer', 'mmcv.runner',
              'mmdet3d', 'mmdet3d.models', 'mmdet3d.models.fusion_layers', 'mmdet3d.models.builder',
              'mmdet3d.models.utils', 'mmdet3d.core', 'mmdet3d.ops', 'mmdet3d.ops.iou3d',
              'mmdet3d.ops.iou3d.iou3d_utils', 'mmdet', 'mmdet.core', 'mmdet.core.bbox', 'mmdet.core.bbox.builder',
              'mmdet.core.bbox.assigners', 'mmdet.core.bbox.match_costs', 'mmdet.core.bbox.match_costs.builder',
              'mmdet.core.bbox.iou_calculators', 'projects.mmdet3d_plugin.core.bbox.assigners',
              'detectron2', 'detectron2.modeling', 'detectron2.modeling.poolers', 'detectron2.structures']:
        _mod(n)
    sm = sys.modules
    # mmdet3d 0.17.1 coord transform: restated in oracle.geometry (third party, unpinned)
    sm['mmdet3d.models.fusion_layers'].apply_3d_transformation = \
        lambda pcd, coords_type, img_meta, reverse=False: og.apply_3d_transformation(pcd, img_meta, reverse)

    # locatt_ops has no CPU path: semantics of kernels.cuh:4-80 via the oracle's shifted-MAC ops
    # The three backward entry points (kernels.cuh:44-119, bound in similar.cu:43-92 / weighting.cu:44-121) are the vector-Jacobian
    # products of the two forward ops, which are bilinear -- evaluated through autograd of the oracle's ops.  (The oracle's ops
    # and the product's backward kernels are pinned to the reference's own CUDA extension in tests/test_gpu_backward.py.)
    def _vjp(fn, wrt_like, cot):
        with torch.enable_grad():
            x = torch.zeros_like(wrt_like).requires_grad_(True)
            return torch.autograd.grad(fn(x), x, cot)[0]

    class _LA:
        similar_forward = staticmethod(lambda q, k, kh, kw: ommri.window_similarity(q, k, kh))
        weighting_forward = staticmethod(lambda v, w, kh, kw: ommri.window_weighting(v, w, kh))
        # similar_backward(x, grad, kH, kW, is_ori): is_ori -> x is x_loc, returns d x_ori; else x is x_ori, returns d x_loc
        similar_backward = staticmethod(lambda x, g, kh, kw, is_ori: (
            _vjp(lambda q: ommri.window_similarity(q, x, kh), x, g) if is_ori
            else _vjp(lambda k: ommri.window_similarity(x, k, kh), x, g)))
        # weighting_backward_ori(x_weight, grad): d v;  weighting_backward_weight(x_ori = v, grad): d weight
        weighting_backward_ori = staticmethod(lambda w, g, kh, kw: _vjp(lambda v: ommri.window_weighting(v, w, kh), g, g))
        weighting_backward_weight = staticmethod(lambda v, g, kh, kw: _vjp(
            lambda w: ommri.window_weighting(v, w, kh), torch.zeros(v.shape[0], v.shape[2], v.shape[3], kh * kw, dtype=v.dtype), g))
    ops = sm['projects.mmdet3d_plugin.models.utils.ops']
    ops.locatt_ops = types.SimpleNamespace(localattention=_LA)

    # mmcv 1.3.18
    def build_conv_layer(cfg, *a, **k):
        k = dict(k)
        if k.get('bias', True) == 'auto':
            k['bias'] = True
        return getattr(nn, cfg['type'])(*a, **k)

    class ConvModule(nn.Module):
        def __init__(self, cin, cout, kernel_size, stride=1, padding=0, bias='auto', conv_cfg=None, norm_cfg=None,
                     **kw):
            super().__init__()
            with_norm = norm_cfg is not None
            if bias == 'auto':
                bias = not with_norm
            dim = conv_cfg['type'][-2:]
            self.conv = getattr(nn, 'Conv' + dim)(cin, cout, kernel_size, stride, padding, bias=bias)
            if with_norm:
                self.bn = getattr(nn, 'BatchNorm' + dim)(cout)
            self.activate = nn.ReLU(inplace=True)

        def forward(self, x):
            x = self.conv(x)
            if hasattr(self, 'bn'):
                x = self.bn(x)
            return self.activate(x)
    sm['mmcv.cnn'].build_conv_layer = build_conv_layer
    sm['mmcv.cnn'].ConvModule = ConvModule
    sm['mmcv.cnn'].kaiming_init = lambda *a, **k: None
    sm['mmcv.cnn.bricks.transformer'].FFN = ompp_ffn      # mmcv 1.3.18 FFN (third party): oracle.mmri_pp.FFN restates it
    sm['mmcv.runner'].force_fp32 = lambda *a, **k: (lambda f: f)
    necks, heads, coders = _Registry(), _Registry(), _Registry()
    sm['mmdet3d.models.builder'].NECKS = necks
    sm['mmdet3d.models.builder'].HEADS = heads
    # losses / target utilities of mmdet 2.14 and mmdet3d 0.17.1 (third party): restated in oracle.loss, part 2
    sm['mmdet3d.models.builder'].build_loss = oloss.build_loss
    sm['mmdet3d.models.utils'].clip_sigmoid = oloss.clip_sigmoid
    sm['mmdet3d.ops.iou3d.iou3d_utils'].nms_gpu = None
    for n in ['circle_nms', 'xywhr2xyxyr']:
        setattr(sm['mmdet3d.core'], n, None)
    sm['mmdet3d.core'].draw_heatmap_gaussian = oloss.draw_heatmap_gaussian
    sm['mmdet3d.core'].gaussian_radius = oloss.gaussian_radius
    sm['mmdet3d.core'].PseudoSampler = oloss.PseudoSampler

    class LiDARInstance3DBoxes:                       # mmdet3d 0.17.1 (third party, unpinned)
        def __init__(self, tensor, box_dim=7):
            self.tensor = tensor

        @property
        def corners(self):
            return og.lidar_box_corners(self.tensor)
    sm['mmdet3d.core'].LiDARInstance3DBoxes = LiDARInstance3DBoxes
    sm['mmdet.core.bbox'].BaseBBoxCoder = object
    sm['mmdet.core.bbox.builder'].BBOX_CODERS = coders
    sm['mmdet.core'].build_bbox_coder = coders.build
    assigners, costs = _Registry(), _Registry()
    costs.register_module()(oloss.FocalLossCost)
    sm['mmdet.core.bbox.builder'].BBOX_ASSIGNERS = assigners
    sm['mmdet.core.bbox.assigners'].AssignResult = oloss.AssignResult
    sm['mmdet.core.bbox.assigners'].BaseAssigner = object
    sm['mmdet.core.bbox.match_costs'].build_match_cost = costs.build
    sm['mmdet.core.bbox.match_costs.builder'].MATCH_COST = costs
    sm['mmdet.core.bbox.iou_calculators'].build_iou_calculator = \
        lambda cfg: oloss.BboxOverlaps3D(**{k: v for k, v in cfg.items() if k != 'type'})
    sm['mmdet.core'].multi_apply = oloss.multi_apply
    sm['mmdet.core'].build_assigner = assigners.build
    sm['mmdet.core'].build_sampler = None
    sm['mmdet.core'].AssignResult = oloss.AssignResult

    # detectron2 ROIPooler(ROIAlignV2, one level) == torchvision roi_align(aligned=True)
    import torchvision.ops as tvo

    class Boxes:
        def __init__(self, t):
            self.tensor = t

    class ROIPooler:
        def __init__(self, output_size, scales, sampling_ratio, pooler_type):
            self.o, self.s, self.r = output_size, scales[0], sampling_ratio

        def __call__(self, feats, boxes):
            return tvo.roi_align(feats[0], [b.tensor for b in boxes], self.o, self.s, self.r, aligned=True)
    sm['detectron2.modeling.poolers'].ROIPooler = ROIPooler
    sm['detectron2.structures'].Boxes = Boxes

    P = os.path.join(ref, PLUGIN)
    _load('projects.mmdet3d_plugin.models.utils.ip_basic.depth_map_utils',
          os.path.join(P, 'models/utils/ip_basic/depth_map_utils.py'))
    sm['projects.mmdet3d_plugin.models.utils.ip_basic'].depth_map_utils = \
        sm['projects.mmdet3d_plugin.models.utils.ip_basic.depth_map_utils']
    eu = _load('projects.mmdet3d_plugin.models.utils.encoder_utils', os.path.join(P, 'models/utils/encoder_utils.py'))
    enc = _load('projects.mmdet3d_plugin.models.necks.deepinteraction_encoder',
                os.path.join(P, 'models/necks/deepinteraction_encoder.py'))
    _load('projects.mmdet3d_plugin.core.bbox.coders.transfusion_bbox_coder',
          os.path.join(P, 'core/bbox/coders/transfusion_bbox_coder.py'))
    _load('projects.mmdet3d_plugin.core.bbox.assigners.hungarian_assigner',
          os.path.join(P, 'core/bbox/assigners/hungarian_assigner.py'))
    du = _load('projects.mmdet3d_plugin.models.utils.decoder_utils', os.path.join(P, 'models/utils/decoder_utils.py'))
    dec = _load('projects.mmdet3d_plugin.models.dense_heads.deepinteraction_decoder',
                os.path.join(P, 'models/dense_heads/deepinteraction_decoder.py'))
    decpp = _load('projects.mmdet3d_plugin.models.dense_heads.deepinteractionplusplus_decoder',
                  os.path.join(P, 'models/dense_heads/deepinteractionplusplus_decoder.py'))
    dec.PlusPlus = decpp.DeepInteractionPlusPlusDecoder
    return eu, enc, du, dec


def state_checksum(sd):
    h = hashlib.sha256()
    for k in sorted(sd):
        h.update(k.encode())
        h.update(sd[k].detach().cpu().contiguous().numpy().tobytes())
    return h.hexdigest()[:16]


# ---- golden cases (shared with tests/test_oracle_golden.py through golden_cases()) ----------------

DEC_TEST_CFG = dict(dataset='nuScenes', grid_size=[288, 288, 40], out_size_factor=8, pc_range=[-54.0, -54.0],
                    voxel_size=[0.375, 0.375], nms_type=None)
DEC_CODER = dict(type='TransFusionBBoxCoder', pc_range=[-54.0, -54.0], voxel_size=[0.375, 0.375], out_size_factor=8,
                 post_center_range=[-61.2, -61.2, -10.0, 61.2, 61.2, 10.0], score_threshold=0.0, code_size=10)


def small_frame(seed, aug=False, views=2, c_img=16, c_pts=24, bev=36, batch=1, n_points=6000):
    """Small scene: input images 112x200 (features 28x50), BEV bev x bev over +-54 m."""
    fr = synth.make_frame_batch(seed, batch=batch, num_views=views, in_hw=(112, 200), stride=4, c_img=c_img,
                                c_pts=c_pts, bev_hw=(bev, bev), n_points=n_points, cloud='lidar', aug=aug)
    # re-pillarise at the small BEV resolution
    pil, coors, npts = synth.pillarize([p.numpy() for p in fr['pts_metas']['pts']], pillar=108.0 / bev)
    fr['pts_metas'].update(pillars=torch.from_numpy(pil), pillar_coors=torch.from_numpy(coors),
                           pillars_num_points=torch.from_numpy(npts))
    return fr


DEC_TRAIN_CFG = dict(dataset='nuScenes',
                     assigner=dict(type='HungarianAssigner3D', iou_calculator=dict(type='BboxOverlaps3D', coordinate='lidar'),
                                   cls_cost=dict(type='FocalLossCost', gamma=2, alpha=0.25, weight=0.15),
                                   reg_cost=dict(type='BBoxBEVL1Cost', weight=0.25), iou_cost=dict(type='IoU3DCost', weight=0.25)),
                     pos_weight=-1, gaussian_overlap=0.1, min_radius=2, grid_size=[288, 288, 40], voxel_size=[0.375, 0.375, 0.2],
                     out_size_factor=8, code_weights=[1.0, 1.0, 1.0, 1.0, 1.0, 1.0, 1.0, 1.0, 0.2, 0.2],
                     point_cloud_range=[-54.0, -54.0, -5.0, 54.0, 54.0, 3.0])
DEC_LOSSES = dict(loss_cls=dict(type='FocalLoss', use_sigmoid=True, gamma=2, alpha=0.25, reduction='mean', loss_weight=1.0),
                  loss_bbox=dict(type='L1Loss', reduction='mean', loss_weight=0.25),
                  loss_heatmap=dict(type='GaussianFocalLoss', reduction='mean', loss_weight=1.0))


def loss_case_gt(preds, coder, seed, counts=(7, 5)):
    """Synthetic ground truth of the loss goldens: per sample, boxes drawn at random inside the range plus three
    jittered copies of decoded last-layer predictions (non-zero IoU entries)."""
    g = torch.Generator().manual_seed(seed)
    P = preds['query_heatmap_score'].shape[-1]
    last = {k: preds[k][..., -P:] for k in ('heatmap', 'rot', 'dim', 'center', 'height', 'vel')}
    dec = coder.decode(*(last[k].clone() for k in ('heatmap', 'rot', 'dim', 'center', 'height', 'vel')))
    boxes, labels = [], []
    for b, n in enumerate(counts):
        xy = torch.rand(n, 2, generator=g) * 90 - 45
        z = torch.rand(n, 1, generator=g) * 2 - 2.5
        dims = torch.stack([torch.rand(n, generator=g) * 1.5 + 1.5, torch.rand(n, generator=g) * 3 + 3,
                            torch.rand(n, generator=g) * 0.8 + 1.4], 1)
        yaw = torch.rand(n, 1, generator=g) * 6.2 - 3.1
        vel = torch.randn(n, 2, generator=g)
        bx = torch.cat([xy, z, dims, yaw, vel], 1)
        pick = torch.randperm(P, generator=g)[:3]
        near = dec[b]['bboxes'][pick].clone()
        near[:, :2] += torch.randn(3, 2, generator=g) * 0.3
        near[:, 3:6] *= 1 + 0.1 * torch.randn(3, 3, generator=g)
        near[:, 6] += 0.1 * torch.randn(3, generator=g)
        boxes.append(torch.cat([bx, near], 0))
        labels.append(torch.randint(0, 10, (n + 3,), generator=g))
    return boxes, labels


def make_decoder(cls, views=2, proposals=24, **extra):
    return cls(**extra, num_views=views, out_size_factor_img=4, num_proposals=proposals, auxiliary=True, hidden_channel=128,
               num_classes=10, num_mmpi=4, num_heads=8, initialize_by_heatmap=True, nms_kernel_size=3,
               ffn_channel=256, dropout=0.1, bn_momentum=0.1, activation='relu',
               common_heads=dict(center=(2, 2), height=(1, 2), dim=(3, 2), rot=(2, 2), vel=(2, 2)),
               loss_cls=dict(type='FocalLoss', use_sigmoid=True, gamma=2, alpha=0.25, reduction='mean',
                             loss_weight=1.0),
               bbox_coder=dict(DEC_CODER), test_cfg=dict(DEC_TEST_CFG))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--ref', default='/root/reference')
    ap.add_argument('--out', default=os.path.join(ROOT, 'tests', 'golden'))
    ap.add_argument('--only', default='', help='comma-separated golden names to (re)generate; default: all')
    args = ap.parse_args()
    only = set(x for x in args.only.split(',') if x)
    os.makedirs(args.out, exist_ok=True)
    eu, enc, du, dec = install_stubs(args.ref)
    torch.set_grad_enabled(False)
    report = []

    def save(name, obj):
        if only and name not in only:
            return
        if name.startswith('encoder_'):                # full-map outputs: sampled storage (tests/golden_sample.py)
            from golden_sample import shrink
            obj = shrink(obj)
        torch.save(obj, os.path.join(args.out, name + '.pt'))
        sz = os.path.getsize(os.path.join(args.out, name + '.pt'))
        report.append(f'{name}: {sz / 1024:.0f} KiB')

    def cmp(a, b):
        return float((a - b).abs().max() / b.abs().max().clamp_min(1e-12))

    # --- G1: config 1 of BASELINE.json: single MMRI_I2P, 32x32 BEV C=64, 1 cam 64x64 ---------------
    for tag, aug in (('i2p_cfg1', False), ('i2p_cfg1_aug', True)):
        seed = 1235
        torch.manual_seed(seed)
        om = ommri.MMRI_I2P(64, 64, 0.1).eval()
        synth.randomize_norm_stats(om, seed)
        rm = eu.MMRI_I2P(64, 64, 0.1).eval()
        rm.load_state_dict(om.state_dict(), strict=True)
        fr = synth.make_frame_batch(seed, batch=2, num_views=1, in_hw=(256, 256), stride=4, c_img=64, c_pts=64,
                                    bev_hw=(32, 32), n_points=20000, aug=aug)
        pil, coors, npts = synth.pillarize([p.numpy() for p in fr['pts_metas']['pts']], pillar=108.0 / 32)
        fr['pts_metas'].update(pillars=torch.from_numpy(pil), pillar_coors=torch.from_numpy(coors),
                               pillars_num_points=torch.from_numpy(npts))
        lidar = fr['pts_feats']
        img = fr['img_feats'].view(2, 1, 64, 64, 64)
        ref_out = rm(lidar, img, fr['img_metas'], fr['pts_metas'])
        ora_out = om(lidar, img, fr['img_metas'], fr['pts_metas'])
        print(tag, 'oracle vs reference rel err', cmp(ora_out, ref_out), 'pillars', len(npts))
        save(tag, dict(seed=seed, aug=aug, checksum=state_checksum(om.state_dict()), out=ref_out))

    # --- G2: LocalContextAttentionBlock, cross (target != source) ----------------------------------
    seed = 1300
    torch.manual_seed(seed)
    om = ommri.LocalContextAttentionBlock(32, 32, 9).eval()
    synth.randomize_norm_stats(om, seed)
    rm = eu.LocalContextAttentionBlock(32, 32, 9).eval()
    rm.load_state_dict(om.state_dict(), strict=True)
    g = torch.Generator().manual_seed(seed)
    tgt, src = torch.randn(2, 32, 13, 21, generator=g), torch.randn(2, 32, 13, 21, generator=g)
    ref_out = rm(tgt, src)
    print('lcab oracle vs reference', cmp(om(tgt, src), ref_out))
    save('lcab', dict(seed=seed, checksum=state_checksum(om.state_dict()), out=ref_out))

    # --- G3: BEVWarp (incl. cv2 depth completion) ---------------------------------------------------
    for tag, aug in (('bevwarp', False), ('bevwarp_aug', True)):
        seed = 1400
        fr = small_frame(seed, aug=aug, views=2, c_img=8, c_pts=8, bev=36)
        lidar = fr['pts_feats']
        img = fr['img_feats'].view(1, 2, 8, 28, 50)
        ref_out = eu.BEVWarp()(lidar, img, fr['img_metas'], fr['pts_metas'])
        ora_out = ommri.BEVWarp()(lidar, img, fr['img_metas'], fr['pts_metas'])
        print(tag, 'oracle vs reference', cmp(ora_out, ref_out), 'nonzero frac', float((ref_out != 0).float().mean()))
        save(tag, dict(seed=seed, aug=aug, out=ref_out))

    # --- G4: full small encoder ----------------------------------------------------------------------
    for tag, aug in (('encoder_small', False), ('encoder_small_aug', True)):
        seed = 1500
        torch.manual_seed(seed)
        om = ommri.DeepInteractionEncoder(2, 16, 24, 32).eval()
        synth.randomize_norm_stats(om, seed)
        rm = enc.DeepInteractionEncoder(num_layers=2, in_channels_img=16, in_channels_pts=24, hidden_channel=32).eval()
        rm.load_state_dict(om.state_dict(), strict=True)
        fr = small_frame(seed, aug=aug, views=2, c_img=16, c_pts=24, bev=36, batch=2)
        r_img, (r_p0, r_p1) = rm(fr['img_feats'], fr['pts_feats'], fr['img_metas'], fr['pts_metas'])
        o_img, (o_p0, o_p1) = om(fr['img_feats'], fr['pts_feats'], fr['img_metas'], fr['pts_metas'])
        print(tag, 'oracle vs reference', cmp(o_img, r_img), cmp(o_p0, r_p0), cmp(o_p1, r_p1))
        save(tag, dict(seed=seed, aug=aug, checksum=state_checksum(om.state_dict()), img=r_img, pts_conv=r_p0,
                       pts=r_p1))

    # --- G4b: encoder at the base model's hidden width (C = 128: the planar window kernel's only width) -------------
    if not only or 'encoder_c128' in only:
        seed = 1550
        torch.manual_seed(seed)
        om = ommri.DeepInteractionEncoder(2, 16, 24, 128).eval()
        synth.randomize_norm_stats(om, seed)
        rm = enc.DeepInteractionEncoder(num_layers=2, in_channels_img=16, in_channels_pts=24, hidden_channel=128).eval()
        rm.load_state_dict(om.state_dict(), strict=True)
        fr = small_frame(seed, aug=True, views=2, c_img=16, c_pts=24, bev=36, batch=1)
        r_img, (r_p0, r_p1) = rm(fr['img_feats'], fr['pts_feats'], fr['img_metas'], fr['pts_metas'])
        o_img, (o_p0, o_p1) = om(fr['img_feats'], fr['pts_feats'], fr['img_metas'], fr['pts_metas'])
        print('encoder_c128 oracle vs reference', cmp(o_img, r_img), cmp(o_p0, r_p0), cmp(o_p1, r_p1))
        save('encoder_c128', dict(seed=seed, aug=True, checksum=state_checksum(om.state_dict()), img=r_img, pts_conv=r_p0,
                                  pts=r_p1))

    # --- G9: TRAINING mode of the reference modules (BatchNorm batch statistics, the autograd wiring of the window Functions;
    # I2P attention dropout set to 0 so the step is deterministic): outputs, running statistics after the step, input and
    # parameter gradients of a fixed linear functional.  Pins the oracle's .train() behaviour (tests/test_oracle_golden.py),
    # which is what the product's training step is compared with on the GPU.
    def train_step(m, inputs, cots, call):
        """-> outputs, grads of sum(out * cot) w.r.t. inputs and parameters, state after the step"""
        with torch.enable_grad():
            xs = [x.clone().requires_grad_(True) for x in inputs]
            outs = call(m, xs)
            sum((o * c).sum() for o, c in zip(outs, cots)).backward()
        return dict(outs=[o.detach() for o in outs], d_in=[x.grad for x in xs],
                    grads={n: p.grad.clone() for n, p in m.named_parameters()},
                    buffers={n: b.clone() for n, b in m.named_buffers()})

    if not only or 'lcab_train' in only:
        seed = 1810
        torch.manual_seed(seed)
        om = ommri.LocalContextAttentionBlock(32, 32, 9)
        synth.randomize_norm_stats(om, seed)
        rm = eu.LocalContextAttentionBlock(32, 32, 9)
        rm.load_state_dict(om.state_dict(), strict=True)
        ck = state_checksum(om.state_dict())
        om.train(), rm.train()
        g = torch.Generator().manual_seed(seed)
        tgt, src, cot = (torch.randn(2, 32, 9, 12, generator=g) for _ in range(3))
        src[:, :, :2] = 0.0
        call = lambda m, xs: [m(xs[0], xs[1])]
        r, o = train_step(rm, [tgt, src], [cot], call), train_step(om, [tgt, src], [cot], call)
        print('lcab_train oracle vs reference: out', cmp(o['outs'][0], r['outs'][0]), 'd_in',
              [cmp(a, b) for a, b in zip(o['d_in'], r['d_in'])], 'worst param grad',
              max(cmp(o['grads'][n], r['grads'][n]) for n in r['grads']))
        save('lcab_train', dict(seed=seed, checksum=ck, **r))          # inputs / cotangent: regenerated from the seed

    if not only or 'encoder_train' in only:
        seed = 1820
        torch.manual_seed(seed)
        om = ommri.DeepInteractionEncoder(2, 16, 24, 32)
        synth.randomize_norm_stats(om, seed)
        rm = enc.DeepInteractionEncoder(num_layers=2, in_channels_img=16, in_channels_pts=24, hidden_channel=32)
        rm.load_state_dict(om.state_dict(), strict=True)
        ck = state_checksum(om.state_dict())
        for m in (om, rm):
            m.train()
            for blk in m.fusion_blocks:
                blk.I2P_block.learnedAlign.dropout = 0.0
        fr = small_frame(seed, aug=True, views=2, batch=2)
        g = torch.Generator().manual_seed(seed)
        call = lambda m, xs: (lambda r_: [r_[0], r_[1][0], r_[1][1]])(m(xs[0], xs[1], fr['img_metas'], fr['pts_metas']))
        with torch.no_grad():
            shapes = [t.shape for t in call(ommri.DeepInteractionEncoder(2, 16, 24, 32).eval(), [fr['img_feats'], fr['pts_feats']])]
        cots = [torch.randn(sh, generator=g) for sh in shapes]
        r = train_step(rm, [fr['img_feats'], fr['pts_feats']], cots, call)
        o = train_step(om, [fr['img_feats'], fr['pts_feats']], cots, call)
        print('encoder_train oracle vs reference: outs', [cmp(a, b) for a, b in zip(o['outs'], r['outs'])], 'd_in',
              [cmp(a, b) for a, b in zip(o['d_in'], r['d_in'])], 'worst param grad',
              max((cmp(o['grads'][n], r['grads'][n]), n) for n in r['grads'] if not n.endswith('out_proj.bn.bias')),
              'worst running stat', max(cmp(o['buffers'][n].float(), r['buffers'][n].float()) for n in r['buffers']))
        save('encoder_train', dict(seed=seed, checksum=ck, **r))       # frame / cotangents: regenerated from the seed

    # --- G10: HeuristicAssigner3D (hungarian_assigner.py:50-91) run unmodified (its IoU calculator is the restated BboxOverlaps3D) ---
    if not only or 'heuristic_assign' in only:
        ha = sys.modules['projects.mmdet3d_plugin.core.bbox.assigners.hungarian_assigner']
        g = torch.Generator().manual_seed(1900)

        def boxes(n, spread):
            xy = torch.rand(n, 2, generator=g) * 2 * spread - spread
            z = torch.rand(n, 1, generator=g) * 2 - 2.5
            dims = torch.stack([torch.rand(n, generator=g) * 2 + 1, torch.rand(n, generator=g) * 4 + 2, torch.rand(n, generator=g) + 1.2], 1)
            return torch.cat([xy, z, dims, torch.rand(n, 1, generator=g) * 6.2 - 3.1, torch.randn(n, 2, generator=g)], 1)
        pred = boxes(150, 30.0)
        gt = torch.cat([boxes(22, 30.0), pred[:8] + 0.3 * torch.randn(8, 9, generator=g)], 0)
        gt[:, 3:6] = gt[:, 3:6].abs() + 0.5
        gt[5, :2] = gt[4, :2] + 0.01                        # two boxes compete for one prediction
        gl, ql = torch.randint(0, 4, (30,), generator=g), torch.randint(0, 4, (150,), generator=g)
        cases = {}
        for name, q in (('plain', None), ('same_class', ql)):
            r = ha.HeuristicAssigner3D(dist_thre=20).assign(pred, gt, None, gl, q)
            o = oloss.HeuristicAssigner3D(dist_thre=20).assign(pred, gt, None, gl, q)
            print('heuristic_assign', name, 'matched', int((r.gt_inds > 0).sum()), 'oracle == reference',
                  bool(torch.equal(o.gt_inds, r.gt_inds) and torch.equal(o.labels, r.labels)), cmp(o.max_overlaps, r.max_overlaps))
            cases[name] = dict(gt_inds=r.gt_inds, max_overlaps=r.max_overlaps, labels=r.labels)
        save('heuristic_assign', dict(pred=pred, gt=gt, gt_labels=gl, query_labels=ql, dist_thre=20, cases=cases))

    # --- G5: decoder (hidden 128 is hard-coded in DynamicConv) ----------------------------------------
    for tag, aug in (('decoder_small', False), ('decoder_small_aug', True)):
        seed = 1600
        torch.manual_seed(seed)
        om = make_decoder(ommpi.DeepInteractionDecoder).eval()
        synth.randomize_norm_stats(om, seed)
        rm = make_decoder(dec.DeepInteractionDecoder).eval()
        missing = rm.load_state_dict(om.state_dict(), strict=True)
        g = torch.Generator().manual_seed(seed)
        fr = small_frame(seed, aug=aug, views=2, batch=2)
        pts_in = [torch.randn(2, 128, 36, 36, generator=g), torch.randn(2, 128, 36, 36, generator=g)]
        img_in = torch.randn(4, 128, 28, 50, generator=g)
        r = rm(pts_in, img_in, fr['img_metas'])[0][0]
        o = om(pts_in, img_in, fr['img_metas'])[0][0]
        for k in r:
            print(tag, k, tuple(r[k].shape), 'oracle vs reference', cmp(o[k], r[k]))
        print(tag, 'labels equal', bool((rm.query_labels == om.query_labels).all()),
              'on-image', [int(m.sum()) for m in rm.on_the_image_mask])
        save(tag, dict(seed=seed, aug=aug, checksum=state_checksum(om.state_dict()), out=r,
                       query_labels=rm.query_labels, on_the_image_mask=rm.on_the_image_mask))
    # --- G7: the ++ decoder (V2 RCNN blocks, look-forward centres, cumulative on-image mask) -----------------
    from oracle import mmpi_pp as ommpi_pp
    for tag, aug in (('decoder_pp_small', False), ('decoder_pp_small_aug', True)):
        if only and tag not in only:
            continue
        seed = 1700
        torch.manual_seed(seed)
        om = make_decoder(ommpi_pp.DeepInteractionPlusPlusDecoder).eval()
        synth.randomize_norm_stats(om, seed)
        with torch.no_grad():                      # the two branch scales start equal (0.5); make them distinguishable
            for i, blk in enumerate(om.decode_head):
                blk.scale.fill_(0.6 + 0.05 * i)
                blk.self_scale.fill_(0.35 - 0.03 * i)
        rm = make_decoder(dec.PlusPlus).eval()
        rm.load_state_dict(om.state_dict(), strict=True)
        g = torch.Generator().manual_seed(seed)
        fr = small_frame(seed, aug=aug, views=2, batch=2)
        pts_in = [torch.randn(2, 128, 36, 36, generator=g), torch.randn(2, 128, 36, 36, generator=g)]
        img_in = torch.randn(4, 128, 28, 50, generator=g)
        r = rm(pts_in, img_in, fr['img_metas'])[0][0]
        o = om(pts_in, img_in, fr['img_metas'])[0][0]
        for k in r:
            print(tag, k, tuple(r[k].shape), 'oracle vs reference', cmp(o[k], r[k]))
        print(tag, 'labels equal', bool((rm.query_labels == om.query_labels).all()),
              'masks equal', all(bool((a == b).all()) for a, b in zip(rm.on_the_image_mask, om.on_the_image_mask)),
              'on-image', [int(m.sum()) for m in rm.on_the_image_mask])
        save(tag, dict(seed=seed, aug=aug, checksum=state_checksum(om.state_dict()), out=r,
                       query_labels=rm.query_labels, on_the_image_mask=rm.on_the_image_mask))
    # --- G8: loss path (targets, Hungarian assignment, gaussian heat-map targets, focal / L1 / gaussian-focal losses):
    #     the reference's get_targets / loss / HungarianAssigner3D run UNMODIFIED on oracle.loss part 2 (third party)
    from oracle import mmpi_pp as ommpi_pp2
    for tag, rcls, ocls, pp in (('decoder_loss', dec.DeepInteractionDecoder, ommpi.DeepInteractionDecoder, False),
                                ('decoder_pp_loss', dec.PlusPlus, ommpi_pp2.DeepInteractionPlusPlusDecoder, True)):
        if only and tag not in only:
            continue
        seed = 1600
        torch.manual_seed(seed)
        om = make_decoder(ocls).eval()
        synth.randomize_norm_stats(om, seed)
        rm = make_decoder(rcls, train_cfg=oloss.ConfigDict(DEC_TRAIN_CFG), loss_bbox=DEC_LOSSES['loss_bbox'],
                          loss_heatmap=DEC_LOSSES['loss_heatmap']).eval()
        rm.load_state_dict(om.state_dict(), strict=True)
        g = torch.Generator().manual_seed(seed)
        fr = small_frame(seed, aug=False, views=2, batch=2)
        pts_in = [torch.randn(2, 128, 36, 36, generator=g), torch.randn(2, 128, 36, 36, generator=g)]
        img_in = torch.randn(4, 128, 28, 50, generator=g)
        preds = rm(pts_in, img_in, fr['img_metas'])
        boxes, labels = loss_case_gt(preds[0][0], om.bbox_coder, seed)
        gt = [oloss.LiDARBoxes(b) for b in boxes]
        saved = {k: v.clone() for k, v in preds[0][0].items()}
        tg = rm.get_targets(gt, labels, preds[0])
        ld = rm.loss(gt, labels, preds)
        lh = oloss.LossHead(10, 24, 4, om.bbox_coder, DEC_TRAIN_CFG, auxiliary=True, plusplus=pp, **DEC_LOSSES)
        lh.query_labels, lh.on_the_image_mask = rm.query_labels, rm.on_the_image_mask
        lo = lh.loss(gt, labels, [[{k: v.clone() for k, v in saved.items()}]])
        for k in ld:
            print(tag, k, float(ld[k]), 'oracle vs reference', cmp(lo[k], ld[k]))
        print(tag, 'num_pos', int(tg[5]), 'assignment equal', bool((lo['_targets']['labels'] == tg[0]).all()),
              'heatmap targets equal', bool((lo['_targets']['heatmap'] == tg[7]).all()))
        save(tag, dict(seed=seed, preds=saved, query_labels=rm.query_labels, on_the_image_mask=rm.on_the_image_mask,
                       gt_boxes=boxes, gt_labels=labels, losses={k: v.clone() for k, v in ld.items()},
                       targets=dict(labels=tg[0], label_weights=tg[1], bbox_targets=tg[2], bbox_weights=tg[3], ious=tg[4],
                                    num_pos=int(tg[5]), matched_ious=float(tg[6]), heatmap=tg[7])))
    # --- G6: get_bboxes + bbox coder (A16, SURVEY 8f): batch 1 (the reference asserts it, :631-632), nms_type None ---
    class Boxes:                                    # stands in for img_metas['box_type_3d'] (mmdet3d LiDARInstance3DBoxes)
        def __init__(self, tensor, box_dim=9):
            self.tensor, self.box_dim = tensor, box_dim
    seed = 1610
    torch.manual_seed(seed)
    om = make_decoder(ommpi.DeepInteractionDecoder).eval()
    synth.randomize_norm_stats(om, seed)
    rm = make_decoder(dec.DeepInteractionDecoder).eval()
    rm.load_state_dict(om.state_dict(), strict=True)
    rm.bbox_coder.score_threshold = om.bbox_coder.score_threshold = 0.27       # filters about half of the proposals
    g = torch.Generator().manual_seed(seed)
    fr = small_frame(seed, aug=False, views=2, batch=1)
    pts_in = [torch.randn(1, 128, 36, 36, generator=g), torch.randn(1, 128, 36, 36, generator=g)]
    img_in = torch.randn(2, 128, 28, 50, generator=g)
    metas = [dict(m, box_type_3d=Boxes) for m in fr['img_metas']]
    r_out = rm(pts_in, img_in, metas)
    o_out = om(pts_in, img_in, metas)
    preds = copy.deepcopy(r_out)                                      # the reference decode() writes into its inputs
    rb = rm.get_bboxes(copy.deepcopy(r_out), metas)
    ob = om.get_bboxes(o_out, metas)
    print('get_bboxes kept', tuple(rb[0][0].tensor.shape), 'oracle vs reference', cmp(ob[0][0].tensor, rb[0][0].tensor),
          cmp(ob[0][1], rb[0][1]), 'labels equal', bool((ob[0][2] == rb[0][2]).all()))
    enc_r = rm.bbox_coder.encode(rb[0][0].tensor)
    enc_o = om.bbox_coder.encode(ob[0][0].tensor)
    print('encode oracle vs reference', cmp(enc_o, enc_r))
    save('decoder_bboxes', dict(seed=seed, checksum=state_checksum(om.state_dict()), preds=preds[0][0],
                                query_labels=rm.query_labels, boxes=rb[0][0].tensor, scores=rb[0][1], labels=rb[0][2],
                                encoded=enc_r, score_threshold=0.27))
    print('\n'.join(report))


if __name__ == '__main__':
    main()
