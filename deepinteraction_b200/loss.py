"""MMPI loss path on libdi_b200 (SURVEY.md 8(f) rank 3): matching costs, Hungarian assignment, targets, gaussian
heat-map targets and the focal / L1 / gaussian-focal losses of the decoder head, computed on the GPU without a host
round trip.

Reference: projects/mmdet3d_plugin/core/bbox/assigners/hungarian_assigner.py (BBox3DL1Cost :14-21, BBoxBEVL1Cost
:24-37, IoU3DCost :40-47, HeuristicAssigner3D :50-91, HungarianAssigner3D :94-153) and
models/dense_heads/deepinteraction_decoder.py get_targets :315-353, get_targets_single :355-482, loss :484-547
(deepinteractionplusplus_decoder.py:513-514 for the ++ mask rule).  The reference copies every cost matrix to the CPU
and calls scipy.optimize.linear_sum_assignment once per layer and sample; here all (sample, layer) problems are solved by
one kernel launch (di_hungarian_f32).  LossMixin.loss_backward gives the gradient of the three losses with respect to
the dense heat-map logits and the prediction rows (di_mmpi_losses_bwd_f32); backward.decoder_backward chains it through
the whole base decoder.

The classes below carry the names the reference registers (MATCH_COST / BBOX_ASSIGNERS), so `train_cfg.assigner` of
Fusion_0075_*.py builds unchanged; the cost objects are parameter holders (the arithmetic is fused in
di_match_cost_f32).
"""
import ctypes

import torch

from . import ops


class FocalLossCost:
    """mmdet 2.14 FocalLossCost (constructor kwargs)."""

    def __init__(self, weight=1., alpha=0.25, gamma=2, eps=1e-12):
        self.weight, self.alpha, self.gamma, self.eps = weight, alpha, gamma, eps


class BBox3DL1Cost:
    kind = 1

    def __init__(self, weight):
        self.weight = weight


class BBoxBEVL1Cost:
    kind = 0

    def __init__(self, weight):
        self.weight = weight


class IoU3DCost:
    def __init__(self, weight):
        self.weight = weight


MATCH_COSTS = dict(FocalLossCost=FocalLossCost, BBox3DL1Cost=BBox3DL1Cost, BBoxBEVL1Cost=BBoxBEVL1Cost, IoU3DCost=IoU3DCost)


def _build(table, cfg):
    if not isinstance(cfg, dict):
        return cfg
    cfg = dict(cfg)
    return table[cfg.pop('type')](**cfg)


def _f(vals):
    return (ctypes.c_float * len(vals))(*[float(v) for v in vals])


def _to_device(t, device):
    """Host tensor -> device through pinned memory, without a host synchronisation (a pageable source makes the copy
    synchronous)."""
    return t.pin_memory().to(device, non_blocking=True) if torch.device(device).type == 'cuda' else t.to(device)


def pad_gt(gt_boxes, gt_labels, device):
    """list of (G_b, nb) boxes / (G_b,) labels -> padded [B, Gmax, nb] fp32, [B, Gmax] int32, counts [B] int32.  Boxes
    already on the device are padded there; no host synchronisation either way."""
    B = len(gt_boxes)
    nb = gt_boxes[0].shape[-1]
    G = max(1, max(int(b.shape[0]) for b in gt_boxes))
    on_dev = all(b.is_cuda for b in gt_boxes)
    boxes = torch.zeros(B, G, nb, dtype=torch.float32, device=device if on_dev else 'cpu')
    labels = torch.zeros(B, G, dtype=torch.int32, device=device if on_dev else 'cpu')
    counts = torch.tensor([int(b.shape[0]) for b in gt_boxes], dtype=torch.int32)
    for i, (b, l) in enumerate(zip(gt_boxes, gt_labels)):
        n = int(b.shape[0])
        if n:
            boxes[i, :n] = b.to(boxes.device, torch.float32)
            labels[i, :n] = l.to(labels.device, torch.int32)
    if not on_dev:
        boxes, labels = _to_device(boxes, device), _to_device(labels, device)
    return boxes, labels, _to_device(counts, device)


def losses_bwd_bytes(B, K, HW, L, P, code):
    """Algorithmic traffic of di_mmpi_losses_bwd_f32: the dense logits and targets read twice (count, gradient), the
    [B, HW, 32] heat-map gradient written; per prediction row its K + code predictions, label and weight (int64), box
    targets and weights read, its gradient row written."""
    rows = B * L * P
    return 4 * (2 * 2 * B * K * HW + B * HW * 32) + rows * (4 * (K + code) + 16 + 8 * code + 4 * (K + code))


class HungarianAssigner3D:
    """Drop-in for hungarian_assigner.py:94-153.  ``assign`` keeps the reference signature (one layer of one sample) and
    returns (gt_inds, max_overlaps, labels) tensors -- the fields of mmdet's AssignResult; ``assign_batch`` solves all
    (sample, layer) problems of a head output in one launch."""

    def __init__(self, cls_cost=dict(type='ClassificationCost', weight=1.), reg_cost=dict(type='BBoxBEVL1Cost', weight=1.0),
                 iou_cost=dict(type='IoU3DCost', weight=1.0), iou_calculator=dict(type='BboxOverlaps3D')):
        if isinstance(cls_cost, dict) and cls_cost.get('type') != 'FocalLossCost':
            raise NotImplementedError("cls_cost %r: only FocalLossCost (both reference configs) is provided" % cls_cost.get('type'))
        self.cls_cost, self.reg_cost, self.iou_cost = (_build(MATCH_COSTS, c) for c in (cls_cost, reg_cost, iou_cost))
        ic = dict(iou_calculator)
        if ic.get('type') != 'BboxOverlaps3D' or ic.get('coordinate', 'lidar') != 'lidar':
            raise NotImplementedError('iou_calculator: only BboxOverlaps3D(coordinate="lidar") is provided')

    def _params(self, train_cfg):
        r = train_cfg['point_cloud_range']
        return _f([self.cls_cost.weight, self.cls_cost.alpha, self.cls_cost.gamma, self.cls_cost.eps, self.reg_cost.weight,
                   self.reg_cost.kind, self.iou_cost.weight, r[0], r[1], r[3] - r[0], r[4] - r[1]])

    def assign_batch(self, boxes, score, gt, gt_labels, n_gt, L, train_cfg):
        """boxes [B, L*P, nb] decoded predictions, score [B, K, L*P] logits, gt [B, Gmax, nb], gt_labels [B, Gmax] int32,
        n_gt [B] int32 -> gt_inds [B, L*P] int64 (0 = background, j + 1 = box j), max_overlaps [B, L*P], cost, iou."""
        B, LP, nb = boxes.shape
        K, G = score.shape[1], gt.shape[1]
        dev = boxes.device
        cost = torch.zeros(B, LP, G, device=dev, dtype=torch.float32)
        iou = torch.zeros(B, LP, G, device=dev, dtype=torch.float32)
        ops._call('di_match_cost_f32', ops._ptr(boxes), nb, ops._ptr(score), K, ops._ptr(gt), ops._ptr(gt_labels), ops._ptr(n_gt),
                  B, LP, G, self._params(train_cfg), ops._ptr(cost), ops._ptr(iou), ops._stream())
        gt_inds = torch.empty(B, LP, device=dev, dtype=torch.int64)
        overlaps = torch.empty(B, LP, device=dev, dtype=torch.float32)
        ops._call('di_hungarian_f32', ops._ptr(cost), ops._ptr(iou), ops._ptr(n_gt), B, L, LP // L, G, ops._ptr(gt_inds),
                  ops._ptr(overlaps), ops._stream())
        return gt_inds, overlaps, cost, iou

    def assign(self, bboxes, gt_bboxes, gt_labels, cls_pred, train_cfg):
        """bboxes (P, nb), gt_bboxes (G, nb), gt_labels (G,), cls_pred (1, K, P) -> gt_inds (P,) int64, max_overlaps (P,),
        labels (P,) int64 (-1 where unassigned)."""
        dev = bboxes.device
        gt, gl, n = pad_gt([gt_bboxes], [gt_labels], dev)
        gt_inds, ov, _, _ = self.assign_batch(bboxes[None].contiguous().float(), cls_pred.contiguous().float(), gt, gl, n, 1, train_cfg)
        gt_inds, ov = gt_inds[0], ov[0]
        labels = torch.where(gt_inds > 0, gl[0].long()[(gt_inds - 1).clamp(min=0)], torch.full_like(gt_inds, -1))
        return gt_inds, ov, labels


class HeuristicAssigner3D:
    """Drop-in for hungarian_assigner.py:50-91 (di_heuristic_assign_f32): every ground-truth box claims its nearest prediction
    (BEV distance, same-class constraint when query_labels is given); returns (gt_inds int64, max_overlaps, labels float) --
    the fields of mmdet's AssignResult."""

    def __init__(self, dist_thre=100, iou_calculator=dict(type='BboxOverlaps3D')):
        self.dist_thre = dist_thre

    def assign(self, bboxes, gt_bboxes, gt_bboxes_ignore=None, gt_labels=None, query_labels=None):
        P, G, dev = bboxes.shape[0], gt_bboxes.shape[0], bboxes.device
        gt_inds = torch.zeros(P, device=dev, dtype=torch.int64)
        overlaps = torch.zeros(P, device=dev, dtype=torch.float32)
        labels = torch.full((P,), -1.0, device=dev, dtype=torch.float32)
        if P == 0 or G == 0:
            return gt_inds, overlaps, labels
        b, g = bboxes.contiguous().float(), gt_bboxes.to(dev).contiguous().float()
        gl = gt_labels.to(dev, torch.int32).contiguous()
        ql = None if query_labels is None else query_labels.to(dev, torch.int32).contiguous()
        work = torch.empty(2 * G, device=dev, dtype=torch.int32)
        ops._call('di_heuristic_assign_f32', ops._ptr(b), b.shape[1], P, ops._ptr(g), ops._ptr(gl), G, ops._ptr(ql),
                  float(self.dist_thre), ops._ptr(gt_inds), ops._ptr(overlaps), ops._ptr(labels), ops._ptr(work), ops._stream())
        return gt_inds, overlaps, labels


ASSIGNERS = dict(HungarianAssigner3D=HungarianAssigner3D, HeuristicAssigner3D=HeuristicAssigner3D)


class LossMixin:
    """get_targets / loss of DeepInteractionDecoder and DeepInteractionPlusPlusDecoder (forward values)."""
    _PP_MASKS = False

    def _init_loss(self, train_cfg, loss_cls, loss_bbox, loss_heatmap):
        for name, cfg, kind in (('loss_cls', loss_cls, 'FocalLoss'), ('loss_bbox', loss_bbox, 'L1Loss'),
                                ('loss_heatmap', loss_heatmap, 'GaussianFocalLoss')):
            if cfg.get('type') != kind:
                raise NotImplementedError('%s: only %s (both reference configs) is provided, got %r' % (name, kind, cfg.get('type')))
            if cfg.get('reduction', 'mean') != 'mean':
                raise NotImplementedError('%s: reduction must be "mean"' % name)
        if not loss_cls.get('use_sigmoid', False):
            raise NotImplementedError('loss_cls: use_sigmoid=True (both reference configs) is required')
        self._loss_cfg = dict(cls=dict(loss_cls), bbox=dict(loss_bbox), heat=dict(loss_heatmap))
        self.bbox_assigner = None
        if train_cfg is not None and train_cfg.get('assigner') is not None:
            self.bbox_assigner = _build(ASSIGNERS, train_cfg['assigner'])

    def _gt_tensors(self, gt_bboxes_3d, gt_labels_3d, device):
        boxes = [g.tensor if hasattr(g, 'tensor') else g for g in gt_bboxes_3d]
        return pad_gt(boxes, gt_labels_3d, device)

    def _targets(self, gt_bboxes_3d, gt_labels_3d, pd, use_masks):
        if self.bbox_assigner is None or not isinstance(self.bbox_assigner, HungarianAssigner3D):
            raise RuntimeError('loss / get_targets need train_cfg.assigner = HungarianAssigner3D')
        tc, coder = self.train_cfg, self.bbox_coder
        dev = pd['center'].device
        cont = lambda k: pd[k].contiguous().float()
        heat, rot, dim, center, height = cont('heatmap'), cont('rot'), cont('dim'), cont('center'), cont('height')
        vel = cont('vel') if 'vel' in pd else None
        B, K, LP = heat.shape
        P = self.num_proposals
        L = LP // P if self.auxiliary else 1
        boxes, _, _, _ = coder._decode_all(heat, rot, dim, center, height, vel, False)
        gt, gl, n_gt = self._gt_tensors(gt_bboxes_3d, gt_labels_3d, dev)
        gt_inds, overlaps, cost, iou = self.bbox_assigner.assign_batch(boxes.contiguous(), heat, gt, gl, n_gt, L, tc)
        code, nb = coder.code_size, gt.shape[-1]
        labels = torch.empty(B, LP, device=dev, dtype=torch.int64)
        label_w = torch.empty(B, LP, device=dev, dtype=torch.int64)
        bbox_t = torch.empty(B, LP, code, device=dev, dtype=torch.float32)
        bbox_w = torch.empty(B, LP, code, device=dev, dtype=torch.float32)
        ious = torch.empty(B, LP, device=dev, dtype=torch.float32)
        num_pos = torch.zeros(L, device=dev, dtype=torch.float32)
        iou_sum = torch.zeros(B, device=dev, dtype=torch.float32)
        pos_cnt = torch.zeros(B, device=dev, dtype=torch.int32)
        mask, mode = None, 0
        if use_masks and self.on_the_image_mask is not None and len(self.on_the_image_mask):
            mask = torch.stack([m.to(dev) for m in self.on_the_image_mask]).to(torch.uint8).contiguous()
            mode = 2 if self._PP_MASKS else 1
        ops._call('di_loss_targets_f32', ops._ptr(gt_inds), ops._ptr(overlaps), ops._ptr(gt), ops._ptr(gl), gt.shape[1],
                  ops._ptr(mask), mode, B, L, P, nb, code, self.num_classes, float(tc['pos_weight']), _f(coder._scale()),
                  ops._ptr(labels), ops._ptr(label_w), ops._ptr(bbox_t), ops._ptr(bbox_w), ops._ptr(ious), ops._ptr(num_pos),
                  ops._ptr(iou_sum), ops._ptr(pos_cnt), ops._stream())
        grid, osf = tc['grid_size'], tc['out_size_factor']
        X, Y = grid[0] // osf, grid[1] // osf
        heatmap = torch.zeros(B, self.num_classes, Y, X, device=dev, dtype=torch.float32)
        ops._call('di_gaussian_heatmap_f32', ops._ptr(gt), nb, ops._ptr(gl), ops._ptr(n_gt), B, gt.shape[1], self.num_classes, Y, X,
                  _f([tc['voxel_size'][0], tc['voxel_size'][1], tc['point_cloud_range'][0], tc['point_cloud_range'][1], osf,
                      tc['min_radius'], tc['gaussian_overlap']]), ops._ptr(heatmap), ops._stream())
        return dict(labels=labels, label_weights=label_w, bbox_targets=bbox_t, bbox_weights=bbox_w, ious=ious, num_pos=num_pos,
                    iou_sum=iou_sum, pos_cnt=pos_cnt, heatmap=heatmap, gt_inds=gt_inds, L=L,
                    tensors=(heat, rot, dim, center, height, vel))

    def get_targets(self, gt_bboxes_3d, gt_labels_3d, preds_dict):
        """deepinteraction_decoder.py:315-353 -> (labels, label_weights, bbox_targets, bbox_weights, ious, num_pos,
        matched_ious, heatmap); num_pos / matched_ious are 0-dim device tensors (no host synchronisation)."""
        t = self._targets(gt_bboxes_3d, gt_labels_3d, preds_dict[0], use_masks=False)
        matched = (t['iou_sum'] / t['pos_cnt'].clamp(min=1).float()).mean()
        return (t['labels'], t['label_weights'], t['bbox_targets'], t['bbox_weights'], t['ious'], t['pos_cnt'].sum(), matched,
                t['heatmap'])

    def loss(self, gt_bboxes_3d, gt_labels_3d, preds_dicts, **kwargs):
        """deepinteraction_decoder.py:484-547 -> dict(loss_heatmap, layer_{l}_loss_cls, layer_{l}_loss_bbox, matched_ious)
        of 0-dim device tensors."""
        pd = preds_dicts[0][0]
        t = self._targets(gt_bboxes_3d, gt_labels_3d, pd, use_masks=True)
        heat, rot, dim, center, height, vel = t['tensors']
        B, K, LP = heat.shape
        L, P = t['L'], self.num_proposals
        dev = heat.device
        dense = pd['dense_heatmap'].contiguous().float()
        cw = self.train_cfg.get('code_weights', None)
        code = self.bbox_coder.code_size
        lc, lb, lh = self._loss_cfg['cls'], self._loss_cfg['bbox'], self._loss_cfg['heat']
        work = torch.empty(2 * 256 + L * 2 * 64, device=dev, dtype=torch.float64)
        out = torch.empty(2 + 2 * L, device=dev, dtype=torch.float32)
        ops._call('di_mmpi_losses_f32', ops._ptr(dense), ops._ptr(t['heatmap']), dense.numel(), ops._ptr(heat), ops._ptr(center),
                  ops._ptr(height), ops._ptr(dim), ops._ptr(rot), ops._ptr(vel), ops._ptr(t['labels']), ops._ptr(t['label_weights']),
                  ops._ptr(t['bbox_targets']), ops._ptr(t['bbox_weights']), ops._ptr(t['num_pos']), ops._ptr(t['iou_sum']),
                  ops._ptr(t['pos_cnt']), B, K, L, P, code, _f(list(cw) + [0.0] * (10 - len(cw))),
                  _f([lc.get('gamma', 2.0), lc.get('alpha', 0.25)]), _f([lh.get('alpha', 2.0), lh.get('gamma', 4.0)]),
                  _f([lh.get('loss_weight', 1.0), lc.get('loss_weight', 1.0), lb.get('loss_weight', 1.0)]), ops._ptr(work),
                  ops._ptr(out), ops._stream())
        res = dict(loss_heatmap=out[0])
        for l in range(L):
            res[f'layer_{l}_loss_cls'] = out[1 + 2 * l]
            res[f'layer_{l}_loss_bbox'] = out[2 + 2 * l]
        res['matched_ious'] = out[1 + 2 * L]
        self._last_targets = t
        self._last_dense = dense
        return res

    def loss_backward(self, grad=None):
        """Gradient of the losses of the last `loss` call (its targets and inputs; the assignment, targets and avg factors
        are constants) for the upstream gradient grad [2 + 2 L] of its outputs in their order (device; None = ones, the
        gradient of mmdet's sum of every loss key; the matched_ious entry takes none).
        -> (d dense heat-map logits [B, Y, X, 32] pixel-major, channels K..31 zero; d prediction rows [L, B*P, NP] in head
        order), on the device without a host round trip."""
        t, dense = self._last_targets, self._last_dense
        heat, rot, dim, center, height, vel = t['tensors']
        B, K, LP = heat.shape
        L, P = t['L'], self.num_proposals
        dev = heat.device
        _, _, Y, X = dense.shape
        if grad is None:
            grad = torch.ones(2 + 2 * L, device=dev, dtype=torch.float32)
        grad = grad.to(torch.float32).contiguous()
        assert grad.shape == (2 + 2 * L,) and grad.is_cuda
        cw = self.train_cfg.get('code_weights', None)
        code = self.bbox_coder.code_size
        lc, lb, lh = self._loss_cfg['cls'], self._loss_cfg['bbox'], self._loss_cfg['heat']
        work = torch.empty(2 * 256 + L * 2 * 64, device=dev, dtype=torch.float64)
        d_heat = torch.empty(B, Y, X, 32, device=dev, dtype=torch.float32)
        d_pred = torch.empty(L, B * P, code + K, device=dev, dtype=torch.float32)
        ops._call('di_mmpi_losses_bwd_f32', ops._ptr(dense), ops._ptr(t['heatmap']), dense.numel(), Y * X, ops._ptr(heat),
                  ops._ptr(center), ops._ptr(height), ops._ptr(dim), ops._ptr(rot), ops._ptr(vel), ops._ptr(t['labels']),
                  ops._ptr(t['label_weights']), ops._ptr(t['bbox_targets']), ops._ptr(t['bbox_weights']), ops._ptr(t['num_pos']),
                  B, K, L, P, code, _f(list(cw) + [0.0] * (10 - len(cw))), _f([lc.get('gamma', 2.0), lc.get('alpha', 0.25)]),
                  _f([lh.get('alpha', 2.0), lh.get('gamma', 4.0)]),
                  _f([lh.get('loss_weight', 1.0), lc.get('loss_weight', 1.0), lb.get('loss_weight', 1.0)]), ops._ptr(grad),
                  ops._ptr(work), ops._ptr(d_heat), ops._ptr(d_pred), ops._stream(), launches=4,
                  nbytes=losses_bwd_bytes(B, K, Y * X, L, P, code))
        return d_heat, d_pred
