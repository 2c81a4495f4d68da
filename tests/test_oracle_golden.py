"""CPU: the oracle restatement vs goldens produced by the reference's own Python
files (tools/make_goldens.py, stub-loaded in the build container)."""
import os
import sys

import numpy as np

import pytest
import torch

import oracle.mmri as ommri
import oracle.mmpi as ommpi
from deepinteraction_b200 import synth
from tools.make_goldens import small_frame, make_decoder, state_checksum
from conftest import rel_err
from golden_sample import golden_err, shape_of

G = os.path.join(os.path.dirname(__file__), "golden")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TOL = 5e-5   # fp32 re-association only; the goldens come from the reference's own torch code


def load(name):
    return torch.load(os.path.join(G, name + '.pt'), weights_only=False)


@pytest.mark.parametrize('tag', ['i2p_cfg1', 'i2p_cfg1_aug'])
def test_i2p_config1(tag):
    g = load(tag)
    torch.manual_seed(g['seed'])
    m = ommri.MMRI_I2P(64, 64, 0.1).eval()
    synth.randomize_norm_stats(m, g['seed'])
    assert state_checksum(m.state_dict()) == g['checksum']
    fr = synth.make_frame_batch(g['seed'], batch=2, num_views=1, in_hw=(256, 256), stride=4, c_img=64, c_pts=64,
                                bev_hw=(32, 32), n_points=20000, aug=g['aug'])
    pil, coors, npts = synth.pillarize([p.numpy() for p in fr['pts_metas']['pts']], pillar=108.0 / 32)
    fr['pts_metas'].update(pillars=torch.from_numpy(pil), pillar_coors=torch.from_numpy(coors),
                           pillars_num_points=torch.from_numpy(npts))
    with torch.no_grad():
        out = m(fr['pts_feats'], fr['img_feats'].view(2, 1, 64, 64, 64), fr['img_metas'], fr['pts_metas'])
    assert rel_err(out, g['out']) < TOL
    # empty pillars stay exactly zero
    occupied = torch.zeros(2, 32, 32, dtype=torch.bool)
    occupied[coors[:, 0], coors[:, 2], coors[:, 3]] = True
    assert float(out.permute(0, 2, 3, 1)[~occupied].abs().max()) == 0.0


def test_lcab():
    g = load('lcab')
    torch.manual_seed(g['seed'])
    m = ommri.LocalContextAttentionBlock(32, 32, 9).eval()
    synth.randomize_norm_stats(m, g['seed'])
    assert state_checksum(m.state_dict()) == g['checksum']
    gen = torch.Generator().manual_seed(g['seed'])
    tgt, src = torch.randn(2, 32, 13, 21, generator=gen), torch.randn(2, 32, 13, 21, generator=gen)
    with torch.no_grad():
        assert rel_err(m(tgt, src), g['out']) < TOL


@pytest.mark.parametrize('tag', ['bevwarp', 'bevwarp_aug'])
def test_bevwarp(tag):
    g = load(tag)
    fr = small_frame(g['seed'], aug=g['aug'], views=2, c_img=8, c_pts=8, bev=36)
    with torch.no_grad():
        out = ommri.BEVWarp()(fr['pts_feats'], fr['img_feats'].view(1, 2, 8, 28, 50), fr['img_metas'], fr['pts_metas'])
    assert rel_err(out, g['out']) < TOL


@pytest.mark.parametrize('tag', ['encoder_small', 'encoder_small_aug'])
def test_encoder_small(tag):
    g = load(tag)
    torch.manual_seed(g['seed'])
    m = ommri.DeepInteractionEncoder(2, 16, 24, 32).eval()
    synth.randomize_norm_stats(m, g['seed'])
    assert state_checksum(m.state_dict()) == g['checksum']
    fr = small_frame(g['seed'], aug=g['aug'], views=2, c_img=16, c_pts=24, bev=36, batch=2)
    with torch.no_grad():
        img, (p0, p1) = m(fr['img_feats'], fr['pts_feats'], fr['img_metas'], fr['pts_metas'])
    assert golden_err(img, g['img']) < TOL and golden_err(p0, g['pts_conv']) < TOL and golden_err(p1, g['pts']) < TOL


def test_encoder_c128():
    """Reference-generated golden at the base model's hidden width (C = 128), augmented frame."""
    g = load('encoder_c128')
    torch.manual_seed(g['seed'])
    m = ommri.DeepInteractionEncoder(2, 16, 24, 128).eval()
    synth.randomize_norm_stats(m, g['seed'])
    assert state_checksum(m.state_dict()) == g['checksum']
    fr = small_frame(g['seed'], aug=g['aug'], views=2, c_img=16, c_pts=24, bev=36, batch=1)
    with torch.no_grad():
        img, (p0, p1) = m(fr['img_feats'], fr['pts_feats'], fr['img_metas'], fr['pts_metas'])
    assert golden_err(img, g['img']) < TOL and golden_err(p0, g['pts_conv']) < TOL and golden_err(p1, g['pts']) < TOL


def _train_step(m, inputs, cots, call):
    with torch.enable_grad():
        xs = [x.clone().requires_grad_(True) for x in inputs]
        outs = call(m, xs)
        sum((o * c).sum() for o, c in zip(outs, cots)).backward()
    return [o.detach() for o in outs], [x.grad for x in xs]


def test_lcab_training_mode_matches_reference_golden():
    """TRAINING mode (BatchNorm batch statistics over the whole call, the reference's autograd Functions around the window
    ops): output, input / parameter gradients and the running statistics after the step equal the reference module's
    (tools/make_goldens.py G9).  This pins the oracle that the product's training step is compared with on the GPU."""
    g = load('lcab_train')
    torch.manual_seed(g['seed'])
    m = ommri.LocalContextAttentionBlock(32, 32, 9)
    synth.randomize_norm_stats(m, g['seed'])
    assert state_checksum(m.state_dict()) == g['checksum']
    m.train()
    gen = torch.Generator().manual_seed(g['seed'])
    tgt, src, cot = (torch.randn(2, 32, 9, 12, generator=gen) for _ in range(3))
    src[:, :, :2] = 0.0
    outs, d_in = _train_step(m, [tgt, src], [cot], lambda mm, xs: [mm(xs[0], xs[1])])
    assert rel_err(outs[0], g['outs'][0]) < 1e-6
    assert all(rel_err(a, b) < 1e-6 for a, b in zip(d_in, g['d_in']))
    for n, p in m.named_parameters():
        assert rel_err(p.grad, g['grads'][n]) < 1e-5, n
    for n, b in m.named_buffers():
        assert rel_err(b.float(), g['buffers'][n].float()) < 1e-6, n


def test_encoder_training_mode_matches_reference_golden():
    """Whole base encoder in TRAINING mode (batch of 2, augmented frame, I2P attention dropout set to 0): outputs, running
    statistics, input gradients and every parameter gradient vs the reference's own encoder."""
    g = load('encoder_train')
    torch.manual_seed(g['seed'])
    m = ommri.DeepInteractionEncoder(2, 16, 24, 32)
    synth.randomize_norm_stats(m, g['seed'])
    assert state_checksum(m.state_dict()) == g['checksum']
    m.train()
    for blk in m.fusion_blocks:
        blk.I2P_block.learnedAlign.dropout = 0.0
    fr = small_frame(g['seed'], aug=True, views=2, batch=2)
    gen = torch.Generator().manual_seed(g['seed'])
    cots = [torch.randn(shape_of(o), generator=gen) for o in g['outs']]
    call = lambda mm, xs: (lambda r: [r[0], r[1][0], r[1][1]])(mm(xs[0], xs[1], fr['img_metas'], fr['pts_metas']))
    outs, d_in = _train_step(m, [fr['img_feats'], fr['pts_feats']], cots, call)
    assert all(golden_err(a, b) < TOL for a, b in zip(outs, g['outs']))
    assert all(golden_err(a, b) < 1e-4 for a, b in zip(d_in, g['d_in']))
    for n, p in m.named_parameters():
        if n.endswith('out_proj.bn.bias'):          # analytically zero (cancelled by the next layer's batch mean): rounding noise
            assert float(p.grad.abs().max()) < 1e-3 and float(g['grads'][n].abs().max()) < 1e-3, n
            continue
        assert golden_err(p.grad, g['grads'][n]) < 1e-3, n
    for n, b in m.named_buffers():
        assert golden_err(b.float(), g['buffers'][n].float()) < 1e-5, n


@pytest.mark.parametrize('tag', ['encoder_pp_small', 'encoder_pp_nopolar'])
def test_encoder_plusplus(tag):
    """++ ("deformable") encoder, BASELINE config 4: oracle/mmri_pp.py vs the golden produced by the reference's own
    fusion_transformerv4.py (tools/make_goldens_pp.py).  The polar block runs flash-attn in fp16 in the reference
    (emulated in the golden); the oracle evaluates it in fp32, hence the looser bound on that case."""
    import oracle.mmri_pp as opp
    sys.path.insert(0, os.path.join(ROOT, 'tools'))
    import make_goldens_pp as mgp
    g = load(tag)
    img_l, pts_l = mgp.pp_layers(g['polar'])
    torch.manual_seed(g['seed'])
    m = opp.FusionTransformerv4(2, 2, 16, 24, 128, img_transformerlayers=img_l, pts_transformerlayers=pts_l).eval()
    mgp.randomize_pp(m, g['seed'])
    assert state_checksum(m.state_dict()) == g['checksum']
    fr = mgp.pp_frame(g['seed'], g['aug'])
    with torch.no_grad():
        img, (p0, p1) = m(list(fr['img_levels']), list(fr['pts_levels']), fr['img_metas'], fr['pts_metas'])
    st = g['channel_step']
    tol = 2e-4 if g['polar'] else 1e-5
    assert golden_err(img[:, ::st], g['img']) < tol and golden_err(p0[:, ::st], g['pts_conv']) < 1e-6
    assert golden_err(p1[:, ::st], g['pts']) < tol


@pytest.mark.parametrize('tag', ['decoder_small', 'decoder_small_aug'])
def test_decoder_small(tag):
    g = load(tag)
    torch.manual_seed(g['seed'])
    m = make_decoder(ommpi.DeepInteractionDecoder).eval()
    synth.randomize_norm_stats(m, g['seed'])
    assert state_checksum(m.state_dict()) == g['checksum']
    gen = torch.Generator().manual_seed(g['seed'])
    fr = small_frame(g['seed'], aug=g['aug'], views=2, batch=2)
    pts_in = [torch.randn(2, 128, 36, 36, generator=gen), torch.randn(2, 128, 36, 36, generator=gen)]
    img_in = torch.randn(4, 128, 28, 50, generator=gen)
    with torch.no_grad():
        out = m(pts_in, img_in, fr['img_metas'])[0][0]
    for k, ref in g['out'].items():
        assert rel_err(out[k], ref) < 2e-4, k
    assert bool((m.query_labels == g['query_labels']).all())
    for a, b in zip(m.on_the_image_mask, g['on_the_image_mask']):
        assert bool((a == b).all())


def pp_scales(m):
    """The generator's non-default branch scales (tools/make_goldens.py G7)."""
    with torch.no_grad():
        for i, blk in enumerate(m.decode_head):
            blk.scale.fill_(0.6 + 0.05 * i)
            blk.self_scale.fill_(0.35 - 0.03 * i)


@pytest.mark.parametrize('tag', ['decoder_pp_small', 'decoder_pp_small_aug'])
def test_decoder_pp_small(tag):
    """++ decoder oracle (V2 RCNN blocks incl. the literal self-branch broadcast, look-forward centres, cumulative
    on-image mask) against outputs of the reference's own deepinteractionplusplus_decoder.py."""
    from oracle import mmpi_pp
    g = load(tag)
    torch.manual_seed(g['seed'])
    m = make_decoder(mmpi_pp.DeepInteractionPlusPlusDecoder).eval()
    synth.randomize_norm_stats(m, g['seed'])
    pp_scales(m)
    assert state_checksum(m.state_dict()) == g['checksum']
    gen = torch.Generator().manual_seed(g['seed'])
    fr = small_frame(g['seed'], aug=g['aug'], views=2, batch=2)
    pts_in = [torch.randn(2, 128, 36, 36, generator=gen), torch.randn(2, 128, 36, 36, generator=gen)]
    img_in = torch.randn(4, 128, 28, 50, generator=gen)
    with torch.no_grad():
        out = m(pts_in, img_in, fr['img_metas'])[0][0]
    for k, ref in g['out'].items():
        assert rel_err(out[k], ref) < 2e-4, k
    assert bool((m.query_labels == g['query_labels']).all())
    assert len(m.on_the_image_mask) == len(g['on_the_image_mask']) == 4
    for a, b in zip(m.on_the_image_mask, g['on_the_image_mask']):
        assert bool((a == b).all())


@pytest.mark.parametrize('tag', ['decoder_loss', 'decoder_pp_loss'])
def test_loss_path(tag):
    """Targets (Hungarian assignment, encoded boxes, weights, gaussian heat maps) and the loss dict of oracle/loss.py
    part 1 against the outputs of the reference's own get_targets / loss / HungarianAssigner3D."""
    import oracle.loss as ol
    from tools.make_goldens import DEC_TRAIN_CFG, DEC_LOSSES, DEC_CODER
    g = load(tag)
    coder = ommpi.TransFusionBBoxCoder(**{k: v for k, v in DEC_CODER.items() if k != 'type'})
    lh = ol.LossHead(10, 24, 4, coder, DEC_TRAIN_CFG, plusplus=tag == 'decoder_pp_loss', **DEC_LOSSES)
    lh.query_labels, lh.on_the_image_mask = g['query_labels'], g['on_the_image_mask']
    out = lh.loss([ol.LiDARBoxes(b) for b in g['gt_boxes']], g['gt_labels'], [[{k: v.clone() for k, v in g['preds'].items()}]])
    for k, ref in g['losses'].items():
        assert rel_err(out[k], ref) < 1e-6, k
    # the goldens store get_targets' outputs (before loss() applies the on-image masks)
    tg = lh.get_targets([ol.LiDARBoxes(b) for b in g['gt_boxes']], g['gt_labels'], [{k: v.clone() for k, v in g['preds'].items()}])
    t = g['targets']
    assert torch.equal(tg[0], t['labels']) and torch.equal(tg[1], t['label_weights']) and torch.equal(tg[3], t['bbox_weights'])
    assert rel_err(tg[2], t['bbox_targets']) < 1e-6 and rel_err(tg[4], t['ious']) < 1e-6 and int(tg[5]) == t['num_pos']
    assert torch.equal(tg[7], t['heatmap'])


def test_heuristic_assigner_matches_reference_golden():
    """HeuristicAssigner3D (hungarian_assigner.py:50-91) run unmodified by tools/make_goldens.py (G10): assigned indices and labels
    bit-equal, matched IoUs to 1e-6 -- with and without the same-class constraint, incl. two boxes competing for one prediction."""
    import oracle.loss as ol
    g = load('heuristic_assign')
    for name, q in (('plain', None), ('same_class', g['query_labels'])):
        r = ol.HeuristicAssigner3D(dist_thre=g['dist_thre']).assign(g['pred'], g['gt'], None, g['gt_labels'], q)
        want = g['cases'][name]
        assert torch.equal(r.gt_inds, want['gt_inds']) and torch.equal(r.labels, want['labels']), name
        assert float((r.max_overlaps - want['max_overlaps']).abs().max()) < 1e-6 and int((r.gt_inds > 0).sum()) > 20, name


def test_rotated_iou_known_answers():
    import oracle.loss as ol
    a = torch.tensor([[0., 0., 0., 2., 2., 1., 0.], [0., 0., 0., 2., 2., 1., 0.7853981634], [5., 5., 0., 1., 1., 1., 0.3]])
    b = torch.tensor([[1., 0., 0., 2., 2., 1., 0.], [0., 0., 0.5, 2., 2., 1., 0.]])
    iou = ol.BboxOverlaps3D()(a, b)
    assert abs(float(iou[0, 0]) - (2 * 1 * 1) / (4 + 4 - 2)) < 1e-6                   # half overlap along x
    assert abs(float(iou[0, 1]) - (4 * 0.5) / (4 + 4 - 2)) < 1e-6                     # same footprint, half the height
    oct_area = 8 * (2 ** 0.5 - 1)                                                     # square vs the same square turned 45 deg
    assert abs(float(iou[1, 1]) - (oct_area * 0.5) / (8 - oct_area * 0.5)) < 1e-6
    assert float(iou[2].abs().max()) == 0.0


def test_depth_completion_numpy_matches_cv2():
    import numpy as np
    from oracle import depth_completion as dc
    rng = np.random.default_rng(3)
    d = np.zeros((112, 200), np.float32)
    ys, xs = rng.integers(30, 112, 3000), rng.integers(0, 200, 3000)
    d[ys, xs] = rng.uniform(1, 70, 3000).astype(np.float32)
    a, sa = dc.fill_in_multiscale(d, True)
    b, sb = dc.fill_in_multiscale_numpy(d, True)
    for k in ('s1', 's2', 's3', 's4', 's5', 's6', 's7m'):
        assert np.array_equal(sa[k], sb[k]), k       # morphology and medians are exact
    assert np.abs(a - b).max() < 1e-3                # bilateral: OpenCV LUT/SIMD rounding only


def test_roi_align_matches_torchvision():
    tvo = pytest.importorskip('torchvision.ops')
    from oracle.geometry import roi_align
    g = torch.Generator().manual_seed(0)
    feat = torch.randn(8, 20, 30, generator=g)
    boxes = torch.tensor([[2.0, 3.0, 17.5, 12.25], [-6.0, -4.0, 5.0, 8.0], [100.0, 60.0, 130.0, 90.0],
                          [10.0, 10.0, 10.0, 10.0], [110.0, 70.0, 125.0, 85.0]])
    for scale in (1.0, 0.25):
        a = roi_align(feat, boxes, 7, scale, 2)
        b = tvo.roi_align(feat[None], [boxes], 7, scale, 2, aligned=True)
        assert torch.allclose(a, b, atol=1e-5)


def test_oracle_get_bboxes_and_coder_match_reference_golden():
    """A16 + get_bboxes (SURVEY 8f): oracle restatement vs the stub-loaded reference (decoder.py:549-638,
    transfusion_bbox_coder.py:24-126), golden made by tools/make_goldens.py (G6)."""
    import oracle.mmpi as om
    from tools.make_goldens import make_decoder
    gold = torch.load(os.path.join(G, 'decoder_bboxes.pt'), weights_only=False)
    torch.manual_seed(gold['seed'])
    m = make_decoder(om.DeepInteractionDecoder).eval()
    m.bbox_coder.score_threshold = gold['score_threshold']
    m.query_labels = gold['query_labels']
    boxes, scores, labels = m.get_bboxes([[gold['preds']]], [dict()])[0]
    assert boxes.shape == gold['boxes'].shape and 0 < boxes.shape[0] < m.num_proposals      # the filter did filter
    assert torch.equal(labels, gold['labels'])
    assert rel_err(boxes, gold['boxes']) < 1e-6 and rel_err(scores, gold['scores']) < 1e-6
    assert rel_err(m.bbox_coder.encode(gold['boxes']), gold['encoded']) < 1e-6
    # encode(decode(x)) returns the regression targets (sin/cos normalised)
    full = m.bbox_coder.decode(torch.rand(1, 10, 24), *(gold['preds'][k][..., -24:] for k in ('rot', 'dim', 'center', 'height', 'vel')))
    enc = m.bbox_coder.encode(full[0]['bboxes'])
    assert rel_err(enc[:, :2], gold['preds']['center'][0, :, -24:].t()) < 1e-5


def test_oracle_circle_nms_semantics():
    import oracle.mmpi as om
    dets = np.array([[0, 0, .9], [.1, 0, .8], [1, 0, .7], [1, .05, .95], [5, 5, .1]], np.float32)
    assert om.circle_nms(dets, 0.05) == [3, 0, 4]            # 2 suppressed by 3, 1 by 0 (squared distance <= thresh)
    assert om.circle_nms(dets, 0.05, post_max_size=2) == [3, 0]
