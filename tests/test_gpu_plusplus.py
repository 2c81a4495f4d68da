"""GPU parity of the ++ ("deformable") encoder, BASELINE.json config 4: libdi_b200 kernels through the C ABI vs the
oracle (oracle/mmri_pp.py) and vs the goldens that tools/make_goldens_pp.py produced from the reference's own
fusion_transformerv4.py.  Tolerance 1e-3 (SURVEY.md 8(d)); the reference runs the polar block's attention in fp16."""
import os
import sys

import numpy as np
import pytest
import torch

from conftest import rel_err
from golden_sample import golden_err

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
G = os.path.join(ROOT, 'tests', 'golden')
TOL, TIGHT = 1e-3, 5e-5


def dev():
    return torch.device('cuda:0')


@pytest.mark.parametrize('L', [1, 2])
def test_msdeform_kernel_matches_oracle_core(L):
    import oracle.mmri_pp as opp
    from deepinteraction_b200 import ops
    g = torch.Generator().manual_seed(40 + L)
    B, hq, wq, heads, d, P = 3, 13, 21, 8, 16, 4
    shapes = [(13, 21), (7, 11)][:L]
    nq = hq * wq
    value = [torch.randn(B, h, w, heads * d, generator=g) for h, w in shapes]
    off = torch.randn(B, nq, heads, L, P, 2, generator=g) * 3.0            # up to ~10 px: exercises the zero padding
    logit = torch.randn(B, nq, heads, L * P, generator=g)
    ref_pts = opp.reference_points(hq, wq).unsqueeze(-2).repeat(1, 1, L, 1)
    norm = torch.tensor([[w, h] for h, w in shapes], dtype=torch.float32)
    loc = ref_pts[:, :, None, :, None, :] + off / norm[None, None, None, :, None, :]
    aw = logit.softmax(-1).view(B, nq, heads, L, P)
    v_flat = torch.cat([v.reshape(B, -1, heads, d) for v in value], 1)
    want = opp.ms_deform_attn_core(v_flat, shapes, loc, aw)                # (B, nq, C)
    raw = torch.cat([off.reshape(B * nq, -1), logit.reshape(B * nq, -1)], 1).contiguous().to(dev())
    got = ops.msdeform([v.to(dev()) for v in value], raw, B, hq, wq)
    assert rel_err(got.cpu().view(B, nq, -1), want) < 1e-5


def test_seq_attn_matches_softmax_attention():
    """di_seq_attn_f32 at G = 3, Wn = 7, Lq = 60, Lk = 28, 8 heads, through the float64 per-head check that
    test_gpu_polar_kernels.py runs over every other shape."""
    from test_gpu_polar_kernels import check_seq_attn
    check_seq_attn((3, 7, 60, 28, 8, False))


def _build_pair(polar, seed):
    sys.path.insert(0, os.path.join(ROOT, 'tools'))
    import make_goldens_pp as mgp
    import oracle.mmri_pp as opp
    from deepinteraction_b200 import mmri_pp
    img_l, pts_l = mgp.pp_layers(polar)
    torch.manual_seed(seed)
    o = opp.FusionTransformerv4(2, 2, 16, 24, 128, img_transformerlayers=img_l, pts_transformerlayers=pts_l).eval()
    mgp.randomize_pp(o, seed)
    m = mmri_pp.FusionTransformerv4(2, 2, 16, 24, 128, img_transformerlayers=img_l, pts_transformerlayers=pts_l)
    m.load_state_dict(o.state_dict(), strict=True)
    return o, m.to(dev()).eval(), mgp


@pytest.mark.parametrize('tag', ['encoder_pp_nopolar', 'encoder_pp_small'])
def test_plusplus_encoder_matches_reference_golden_and_oracle(tag):
    from deepinteraction_b200 import synth
    gold = torch.load(os.path.join(G, tag + '.pt'), weights_only=False)
    torch.set_grad_enabled(False)
    o, m, mgp = _build_pair(gold['polar'], gold['seed'])
    fr = mgp.pp_frame(gold['seed'], gold['aug'])
    r_img, (r_p0, r_p1) = o(list(fr['img_levels']), list(fr['pts_levels']), fr['img_metas'], fr['pts_metas'])
    frd = synth.to_device(fr, dev())
    img, (p0, p1) = m([t.to(dev()) for t in fr['img_levels']], [t.to(dev()) for t in fr['pts_levels']], frd['img_metas'],
                      frd['pts_metas'])
    errs = (rel_err(img.cpu(), r_img), rel_err(p0.cpu(), r_p0), rel_err(p1.cpu(), r_p1))
    print(tag, 'vs oracle: img %.2e pts_conv %.2e pts %.2e' % errs)
    assert errs[1] < TIGHT and max(errs) < TOL
    st = gold['channel_step']
    gerr = (golden_err(img.cpu()[:, ::st], gold['img']), golden_err(p0.cpu()[:, ::st], gold['pts_conv']),
            golden_err(p1.cpu()[:, ::st], gold['pts']))
    print(tag, 'vs reference golden: img %.2e pts_conv %.2e pts %.2e' % gerr)
    assert max(gerr) < TOL


def test_plusplus_encoder_batch2_no_aug_matches_oracle():
    """Two samples, three cameras, un-augmented frame (identity affine), polar block included."""
    from deepinteraction_b200 import synth
    torch.set_grad_enabled(False)
    o, m, mgp = _build_pair(True, 2207)
    fr = mgp.pp_frame(2207, False, views=3, batch=2)
    r_img, (r_p0, r_p1) = o(list(fr['img_levels']), list(fr['pts_levels']), fr['img_metas'], fr['pts_metas'])
    frd = synth.to_device(fr, dev())
    img, (p0, p1) = m([t.to(dev()) for t in fr['img_levels']], [t.to(dev()) for t in fr['pts_levels']], frd['img_metas'],
                      frd['pts_metas'])
    assert rel_err(img.cpu(), r_img) < TOL and rel_err(p1.cpu(), r_p1) < TOL
