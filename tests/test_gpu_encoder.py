"""GPU parity: libdi_b200 encoder kernels (called through the C ABI) vs the CPU oracle.

Tolerance (SURVEY.md 8(d)): per output tensor max|a-b| / max|b| <= 1e-3; the fp32 FFMA kernels are
expected to be ~1e-5, so most checks use a tighter bound to catch real bugs."""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from conftest import rel_err
from golden_sample import golden_err, shape_of

pytestmark = pytest.mark.gpu
TOL = 1e-3
TIGHT = 5e-5
G = os.path.join(os.path.dirname(__file__), 'golden')


def dev():
    return torch.device('cuda:0')


# ---------------------------------------------------------------------------------------------
def test_linear_matches_torch():
    from deepinteraction_b200 import ops
    g = torch.Generator().manual_seed(0)
    for (M, N, Ks, act, use_res) in [(300, 128, [128], ops.ACT_RELU, False), (1000, 96, [64, 32], ops.ACT_NONE, True),
                                     (257, 130, [128, 128, 128], ops.ACT_GELU, False), (77, 20, [50], ops.ACT_NONE, False),
                                     (200, 384, [2], ops.ACT_RELU, False), (513, 128, [36, 128], ops.ACT_NONE, True)]:
        srcs = [torch.randn(M, k, generator=g) for k in Ks]
        W = torch.randn(N, sum(Ks), generator=g) / np.sqrt(sum(Ks))
        b = torch.randn(N, generator=g)
        res = torch.randn(50, N, generator=g) if use_res else None
        ref = torch.cat(srcs, 1).double() @ W.double().t() + b.double()
        if use_res:
            ref = ref + res.double()[torch.arange(M) % 50]
        ref = {ops.ACT_NONE: lambda x: x, ops.ACT_RELU: F.relu, ops.ACT_GELU: F.gelu}[act](ref).float()
        out = ops.linear([s.to(dev()) for s in srcs], W.to(dev()), b.to(dev()), act,
                         res=None if res is None else res.to(dev()), res_mod=50 if use_res else 0)
        assert rel_err(out.cpu(), ref) < TIGHT, (M, N, Ks)


def test_linear_strided_views_and_splitk():
    from deepinteraction_b200 import ops
    g = torch.Generator().manual_seed(1)
    big = torch.randn(400, 384, generator=g).to(dev())
    W = (torch.randn(128, 128, generator=g) / 11).to(dev())
    out = ops.linear([big[:, 128:256]], W)
    assert rel_err(out.cpu(), (big[:, 128:256].cpu().double() @ W.cpu().double().t()).float()) < TIGHT
    A = torch.randn(200, 6272, generator=g).to(dev())
    W2 = (torch.randn(128, 6272, generator=g) / 80).to(dev())
    part = ops.linear([A], W2, splits=16)
    assert part.shape[0] > 1
    bias = torch.randn(128, generator=g).to(dev())
    y = ops.rows_finish(part, bias=bias)
    ref = (A.cpu().double() @ W2.cpu().double().t() + bias.cpu().double()).float()
    assert rel_err(y.cpu(), ref) < TIGHT
    # bitwise deterministic
    y2 = ops.rows_finish(ops.linear([A], W2, splits=16), bias=bias)
    assert torch.equal(y, y2)


def test_conv3x3_matches_torch():
    from deepinteraction_b200 import ops, fold
    g = torch.Generator().manual_seed(2)
    for (N, Cin, H, W, Cout, nhwc_in, nchw_out, act) in [(2, 24, 13, 17, 32, False, False, ops.ACT_NONE),
                                                         (1, 16, 20, 9, 10, True, True, ops.ACT_NONE),
                                                         (3, 64, 15, 31, 128, True, False, ops.ACT_RELU),
                                                         (1, 40, 36, 36, 128, False, False, ops.ACT_NONE)]:
        x = torch.randn(N, Cin, H, W, generator=g)
        w = torch.randn(Cout, Cin, 3, 3, generator=g) / np.sqrt(9 * Cin)
        b = torch.randn(Cout, generator=g)
        ref = F.conv2d(x.double(), w.double(), b.double(), padding=1)
        if act == ops.ACT_RELU:
            ref = F.relu(ref)
        xin = x.permute(0, 2, 3, 1).contiguous() if nhwc_in else x
        y = ops.conv3x3(xin.to(dev()), fold.pack_conv3x3(w).contiguous().to(dev()), b.to(dev()), Cout, nhwc_in,
                        nchw_out, act)
        y = y.cpu() if nchw_out else y.cpu().permute(0, 3, 1, 2)
        assert rel_err(y, ref.float()) < TIGHT


def test_layout_converters_roundtrip():
    from deepinteraction_b200 import ops
    x = torch.randn(2, 37, 5, 41, device=dev())
    y = ops.nchw_to_nhwc(x)
    assert torch.equal(y, x.permute(0, 2, 3, 1).contiguous())
    assert torch.equal(ops.nhwc_to_nchw(y), x)


@pytest.mark.parametrize('kernel', [0, 1], ids=['mma-bf16split', 'ffma'])
@pytest.mark.parametrize('ks,C,H,W', [(9, 32, 13, 21), (9, 128, 40, 33), (3, 16, 7, 5), (9, 64, 16, 16), (9, 128, 9, 50),
                                      (9, 96, 11, 19), (9, 256, 12, 20), (9, 48, 10, 12)])
def test_window_attention_matches_oracle(ks, C, H, W, kernel):
    """Both kernels of di_lcab_window_f32: mma.sync bf16-split (default for ks=9, C%32==0) and FFMA (ks=3, C%32!=0, or
    forced)."""
    import oracle.mmri as om
    from deepinteraction_b200 import ops, _lib
    _lib.lib().di_set_window_ffma(kernel)
    g = torch.Generator().manual_seed(3)
    N = 2
    q, k, v = (torch.randn(N, C, H, W, generator=g) for _ in range(3))
    w = F.softmax(om.window_similarity(q, k, ks) / np.sqrt(C), -1)
    ref = om.window_weighting(v, w, ks)
    rows = lambda t: t.permute(0, 2, 3, 1).reshape(-1, C).contiguous().to(dev())
    try:
        out = ops.lcab_window(rows(q), rows(k), rows(v), N, H, W, C, ks)
        out = out.view(N, H, W, C).permute(0, 3, 1, 2).cpu()
    finally:
        _lib.lib().di_set_window_ffma(0)
    assert rel_err(out, ref) < TIGHT


@pytest.mark.parametrize('C,H,W', [(64, 16, 16), (128, 40, 33), (128, 9, 50)])
def test_window_attention_presplit_operands(C, H, W):
    """The pre-split operand path: host-side model of the format -> di_lcab_window_pre_f32 vs the oracle, and
    di_linear_tcb_split_f32 emits exactly that format."""
    import oracle.mmri as om
    from deepinteraction_b200 import ops, fold
    g = torch.Generator().manual_seed(11)
    N = 2
    q, k, v = (torch.randn(N, C, H, W, generator=g) for _ in range(3))
    w = F.softmax(om.window_similarity(q, k, 9) / np.sqrt(C), -1)
    ref = om.window_weighting(v, w, 9)
    rows = lambda t: t.permute(0, 2, 3, 1).reshape(-1, C).contiguous().to(dev())
    out = ops.lcab_window_pre(fold.split_rows(rows(q), 1), fold.split_rows(rows(k), 1), fold.split_rows(rows(v), 2),
                              N, H, W, C)
    assert rel_err(out.view(N, H, W, C).permute(0, 3, 1, 2).cpu(), ref) < TIGHT
    # the dense layer's split epilogue == split_rows(plain output), bit for bit
    M = 1000
    x = torch.randn(M, 128, generator=g).to(dev())
    Wt = fold.Weight(torch.randn(3 * C, 128, generator=g) / 11, dev())
    b = torch.randn(3 * C, generator=g).to(dev())
    plain = ops.linear([x], Wt, b, ops.ACT_RELU)
    mixed = ops.linear_split([x], Wt, b, ops.ACT_RELU, 2 * C, 2)
    assert torch.equal(mixed[:, :2 * C], plain[:, :2 * C])
    assert torch.equal(mixed[:, 2 * C:].contiguous().view(torch.int32),
                       fold.split_rows(plain[:, 2 * C:].contiguous(), 2).view(torch.int32))
    k1 = ops.linear_split([x], Wt, b, ops.ACT_RELU, 0, 1)
    assert torch.equal(k1.view(torch.int32), fold.split_rows(plain, 1).view(torch.int32))


@pytest.mark.parametrize('N,H,W', [(2, 16, 8), (1, 40, 33), (2, 9, 50), (3, 37, 21), (1, 112, 200)])
def test_window_attention_planar_operands(N, H, W):
    """Planar window kernel (lcab.cu, C = 128): host-side model of the planar operand format ->
    di_lcab_window_tc_f32 vs the oracle (edge tiles, several images, the base image-map shape), and
    di_linear_tcb_split_f32 kind 3 emits exactly that format."""
    import oracle.mmri as om
    from deepinteraction_b200 import ops, fold
    C = 128
    g = torch.Generator().manual_seed(17 + H)
    q, k, v = (torch.randn(N, C, H, W, generator=g) for _ in range(3))
    q = q * 1.7                                         # logits with a spread of a few units after the 1/sqrt(C) scale
    w = F.softmax(om.window_similarity(q, k, 9) / np.sqrt(C), -1)
    ref = om.window_weighting(v, w, 9)
    rows = lambda t: t.permute(0, 2, 3, 1).reshape(-1, C).contiguous().to(dev())
    out = ops.lcab_window_tc(fold.split_rows(rows(q), 3), fold.split_rows(rows(k), 3), fold.split_rows(rows(v), 3),
                             N, H, W, C)
    assert rel_err(out.view(N, H, W, C).permute(0, 3, 1, 2).cpu(), ref) < TIGHT
    # a second launch on the same stream must reproduce the result bit for bit
    out2 = ops.lcab_window_tc(fold.split_rows(rows(q), 3), fold.split_rows(rows(k), 3), fold.split_rows(rows(v), 3),
                              N, H, W, C)
    assert torch.equal(out, out2)


@pytest.mark.parametrize('M,self_attn', [(1000, True), (134400, False), (128, True), (32400, True)])
def test_lcab_projection_chain_equals_unfused_layers(M, self_attn):
    """di_lcab_proj_f32 (second stage in place over q1 / k1 in the q / k buffers) == the unfused chain through separate
    buffers (q1 / k1 in their own tensors, then di_linear_tcb_split_f32), bit for bit."""
    from deepinteraction_b200 import ops, fold
    g = torch.Generator().manual_seed(29)
    C = 128
    xt = torch.randn(M, C, generator=g).to(dev())
    xs = xt if self_attn else torch.randn(M, C, generator=g).to(dev())
    w1 = fold.Weight(torch.randn(3 * C, C, generator=g) / 11, dev())
    w2 = fold.Weight(torch.randn(2 * C, C, generator=g) / 11, dev())
    b1, b2 = torch.randn(3 * C, generator=g).to(dev()), torch.randn(2 * C, generator=g).to(dev())
    q, k, v = ops.lcab_proj(xt, xs, w1, b1, w2, b2)
    wq1, wk1, wv = (fold.Weight(w1.w[i * C:(i + 1) * C].cpu().double(), dev()) for i in range(3))
    wq2, wk2 = (fold.Weight(w2.w[i * C:(i + 1) * C].cpu().double(), dev()) for i in range(2))
    q1 = ops.linear([xt], wq1, b1[:C].contiguous(), ops.ACT_RELU)
    k1 = ops.linear([xs], wk1, b1[C:2 * C].contiguous(), ops.ACT_RELU)
    want_q = ops.linear_split([q1], wq2, b2[:C].contiguous(), ops.ACT_RELU, 0, 3)
    want_k = ops.linear_split([k1], wk2, b2[C:].contiguous(), ops.ACT_RELU, 0, 3)
    want_v = ops.linear_split([xs], wv, b1[2 * C:].contiguous(), ops.ACT_RELU, 0, 3)
    i32 = lambda t: t.contiguous().view(torch.int32)
    assert torch.equal(i32(q), i32(want_q)) and torch.equal(i32(k), i32(want_k)) and torch.equal(i32(v), i32(want_v))


def test_linear_split_planar_format():
    """The dense layer's planar split epilogue (kind 3) == fold.split_rows(plain output, 3), bit for bit, also when
    only the trailing 128 columns of a wider output are split (q1 | k1 | v)."""
    from deepinteraction_b200 import ops, fold
    g = torch.Generator().manual_seed(23)
    M, C = 1000, 128
    x = torch.randn(M, 128, generator=g).to(dev())
    Wt = fold.Weight(torch.randn(3 * C, 128, generator=g) / 11, dev())
    b = torch.randn(3 * C, generator=g).to(dev())
    plain = ops.linear([x], Wt, b, ops.ACT_RELU)
    mixed = ops.linear_split([x], Wt, b, ops.ACT_RELU, 2 * C, 3)
    assert torch.equal(mixed[:, :2 * C], plain[:, :2 * C])
    assert torch.equal(mixed[:, 2 * C:].contiguous().view(torch.int32),
                       fold.split_rows(plain[:, 2 * C:].contiguous(), 3).view(torch.int32))
    allp = ops.linear_split([x], Wt, b, ops.ACT_RELU, 0, 3)
    assert torch.equal(allp.view(torch.int32), fold.split_rows(plain, 3).view(torch.int32))


def _mk_lcab(C, seed):
    import oracle.mmri as om
    from deepinteraction_b200 import synth
    torch.manual_seed(seed)
    m = om.LocalContextAttentionBlock(C, C, 9).eval()
    synth.randomize_norm_stats(m, seed)
    return m


@pytest.mark.parametrize('self_attn', [True, False])
def test_lcab_block_matches_oracle(self_attn):
    from deepinteraction_b200 import mmri
    C, N, H, W = 32, 2, 13, 21
    m = _mk_lcab(C, 1300)
    holder = mmri.LocalContextAttentionBlock(C, C, 9)
    holder.load_state_dict(m.state_dict(), strict=True)
    g = torch.Generator().manual_seed(1300)
    tgt, src = torch.randn(N, C, H, W, generator=g), torch.randn(N, C, H, W, generator=g)
    if self_attn:
        src = tgt
    with torch.no_grad():
        ref = m(tgt, src)
    pk = mmri._pack_lcab(holder, dev())
    rows = lambda t: t.permute(0, 2, 3, 1).reshape(-1, C).contiguous().to(dev())
    t_r = rows(tgt)
    s_r = t_r if self_attn else rows(src)
    out = mmri.lcab_forward(pk, t_r, s_r, N, H, W).view(N, H, W, C).permute(0, 3, 1, 2).cpu()
    assert rel_err(out, ref) < TIGHT
    if not self_attn:      # golden from the reference's own code
        gold = torch.load(os.path.join(G, 'lcab.pt'), weights_only=False)
        assert rel_err(out, gold['out']) < TIGHT


def _cfg1_frame(seed, aug):
    from deepinteraction_b200 import synth
    fr = synth.make_frame_batch(seed, batch=2, num_views=1, in_hw=(256, 256), stride=4, c_img=64, c_pts=64,
                                bev_hw=(32, 32), n_points=20000, aug=aug)
    pil, coors, npts = synth.pillarize([p.numpy() for p in fr['pts_metas']['pts']], pillar=108.0 / 32)
    fr['pts_metas'].update(pillars=torch.from_numpy(pil), pillar_coors=torch.from_numpy(coors),
                           pillars_num_points=torch.from_numpy(npts))
    return fr


@pytest.mark.parametrize('tag', ['i2p_cfg1', 'i2p_cfg1_aug'])
def test_i2p_config1_matches_golden_and_oracle(tag):
    """BASELINE.json configs[0]: single MMRI img->pts cross-attention, 32x32 BEV, C=64, 1 cam 64x64."""
    import oracle.mmri as om
    from deepinteraction_b200 import mmri, synth, fold, ops, geom
    gold = torch.load(os.path.join(G, tag + '.pt'), weights_only=False)
    torch.manual_seed(gold['seed'])
    m = om.MMRI_I2P(64, 64, 0.1).eval()
    synth.randomize_norm_stats(m, gold['seed'])
    fr = _cfg1_frame(gold['seed'], gold['aug'])
    enc = mmri.DeepInteractionEncoder(1, 64, 64, 64).to(dev()).eval()
    enc.fusion_blocks[0].I2P_block.load_state_dict(m.state_dict(), strict=True)
    lp = dict(i2p=tuple(fold.dev(t, dev()) for t in fold.i2p_fold(enc.fusion_blocks[0].I2P_block.learnedAlign)))
    pm = enc._canon_pts_metas(fr['pts_metas'], dev())
    pts_nhwc = fr['pts_feats'].permute(0, 2, 3, 1).contiguous().to(dev())
    img_nhwc = fr['img_feats'].permute(0, 2, 3, 1).contiguous().to(dev())

    class Gm:
        pass
    g = Gm()
    g.proj, g.i2l = geom.camera_rows(fr['img_metas'], dev())
    g.V, g.in_hw = 1, (256, 256)
    out = enc.i2p(lp, pts_nhwc, img_nhwc, pm, g).permute(0, 3, 1, 2).cpu()
    assert rel_err(out, gold['out']) < TIGHT
    occupied = torch.zeros(2, 32, 32, dtype=torch.bool)
    c = fr['pts_metas']['pillar_coors'].long()
    occupied[c[:, 0], c[:, 2], c[:, 3]] = True
    assert float(out.permute(0, 2, 3, 1)[~occupied].abs().max()) == 0.0     # empty pillars are exactly 0


@pytest.mark.parametrize('aug', [False, True])
def test_bevwarp_stages_match_oracle(aug):
    import oracle.mmri as om
    from deepinteraction_b200 import mmri, ops
    from tools.make_goldens import small_frame
    fr = small_frame(1400, aug=aug, views=2, c_img=8, c_pts=8, bev=36)
    with torch.no_grad():
        ref, aux = om.BEVWarp()(fr['pts_feats'], fr['img_feats'].view(1, 2, 8, 28, 50), fr['img_metas'],
                                fr['pts_metas'], return_aux=True)
    pm = {k: v for k, v in fr['pts_metas'].items()}
    pm['pts'] = [p.to(dev()) for p in pm['pts']]
    g = mmri.Geometry(fr['img_metas'], pm, (28, 50), (36, 36), dev(), want_debug=True)
    g.wait()
    sparse = g.sparse.cpu()
    assert torch.equal(sparse > 0, aux[0]['sparse'] > 0), 'sparse depth maps must have identical support'
    if aug:    # the augmentation is folded into the projection matrix: depths agree to fp32 rounding only
        assert float((sparse - aux[0]['sparse']).abs().max()) < 1e-4
    else:
        assert torch.equal(sparse, aux[0]['sparse']), 'sparse depth maps must match bit-for-bit'
    dense = g.dense.cpu()
    assert float((dense - aux[0]['dense']).abs().max()) < 2e-3      # bilateral LUT rounding only
    bev = fr['pts_feats'].permute(0, 2, 3, 1).contiguous().to(dev())
    warped = ops.bev_sample(bev, g.grid, 2).permute(0, 3, 1, 2).cpu()
    assert rel_err(warped, ref[0]) < 2e-4
    gold = torch.load(os.path.join(G, 'bevwarp_aug.pt' if aug else 'bevwarp.pt'), weights_only=False)
    assert rel_err(warped, gold['out'][0]) < 2e-4


def test_depth_completion_matches_opencv_on_random_maps():
    """Stage-exactness of the GPU ip_basic restatement on denser/sparser random maps (112x200)."""
    from oracle import depth_completion as dc
    from deepinteraction_b200 import ops
    rng = np.random.default_rng(5)
    maps = []
    for n in (300, 3000, 12000):
        d = np.zeros((112, 200), np.float32)
        ys, xs = rng.integers(20, 112, n), rng.integers(0, 200, n)
        d[ys, xs] = rng.uniform(0.5, 75, n).astype(np.float32)
        maps.append(d)
    maps.append(np.zeros((112, 200), np.float32))                      # empty map stays empty
    keys = torch.zeros(len(maps), 112, 200, dtype=torch.int64)
    for i, d in enumerate(maps):
        bits = torch.from_numpy(d.view(np.int32).astype(np.int64))
        keys[i] = torch.where(torch.from_numpy(d) > 0, bits | (1 << 32), torch.zeros_like(bits))
    dense = ops.depth_complete(keys.to(dev())).cpu().numpy()
    for i, d in enumerate(maps):
        ref = dc.fill_in_multiscale(d)
        assert np.abs(dense[i] - ref).max() < 2e-3, i


@pytest.mark.parametrize('tag', ['encoder_small', 'encoder_small_aug'])
def test_encoder_small_matches_reference_golden(tag):
    from deepinteraction_b200 import mmri, synth
    from tools.make_goldens import small_frame
    import oracle.mmri as om
    gold = torch.load(os.path.join(G, tag + '.pt'), weights_only=False)
    torch.manual_seed(gold['seed'])
    m = om.DeepInteractionEncoder(2, 16, 24, 32).eval()
    synth.randomize_norm_stats(m, gold['seed'])
    enc = mmri.DeepInteractionEncoder(2, 16, 24, 32)
    enc.load_state_dict(m.state_dict(), strict=True)
    enc = enc.to(dev()).eval()
    fr = synth.to_device(small_frame(gold['seed'], aug=gold['aug'], views=2, c_img=16, c_pts=24, bev=36, batch=2), dev())
    img, (p0, p1) = enc(fr['img_feats'], fr['pts_feats'], fr['img_metas'], fr['pts_metas'])
    assert tuple(img.shape) == shape_of(gold['img']) and tuple(p1.shape) == shape_of(gold['pts'])
    assert golden_err(p0.cpu(), gold['pts_conv']) < TIGHT
    assert golden_err(p1.cpu(), gold['pts']) < TOL
    assert golden_err(img.cpu(), gold['img']) < TOL
    print(tag, 'rel err img %.2e pts %.2e' % (golden_err(img.cpu(), gold['img']), golden_err(p1.cpu(), gold['pts'])))


@pytest.mark.parametrize('cloud,n', [('lidar', 60000), ('dense', 9000)])
def test_gpu_pillarisation_is_bit_exact(cloud, n):
    """(f1) di_pillarize_f32 == synth.pillarize (lowest-index points first, pillars sorted by (b, y, x)), bit for bit,
    for exact-size inputs and for capacity buffers with device-side counts; points on cell borders included."""
    from deepinteraction_b200 import ops, synth
    rng = np.random.default_rng(77)
    pts = [synth.make_points(n, rng, cloud), synth.make_points(n // 3, rng, cloud)]
    for p in pts:                                   # plant points exactly on pillar borders and on the range limits
        p[:50, 0] = np.round(p[:50, 0] / 0.6) * 0.6
        p[50:60, 2] = -5.0
        p[60:70, 0] = 54.0
    Y = X = 180
    pil, coors, cnt = synth.pillarize(pts, pillar=108.0 / X)
    dpts = [torch.from_numpy(p).to(dev()) for p in pts]
    g_pil, g_coors, g_cnt, g_n = ops.pillarize(dpts, (Y, X), synth.PC_RANGE, 20)
    P = int(g_n.item())
    assert P == len(cnt)
    assert torch.equal(g_coors[:P].cpu(), torch.from_numpy(coors)) and torch.equal(g_cnt[:P].cpu(), torch.from_numpy(cnt))
    assert torch.equal(g_pil[:P].cpu(), torch.from_numpy(pil))
    # capacity buffers (stale rows behind the live count) + device-side counts
    cap = 1 << 17
    bufs = [torch.randn(cap, 5, device=dev()) for _ in pts]
    for b, p in zip(bufs, dpts):
        b[:p.shape[0]] = p
    n_dev = torch.tensor([p.shape[0] for p in dpts], dtype=torch.int32, device=dev())
    c_pil, c_coors, c_cnt, c_n = ops.pillarize(bufs, (Y, X), synth.PC_RANGE, 20, n_dev=n_dev)
    assert int(c_n.item()) == P and torch.equal(c_pil[:P], g_pil[:P]) and torch.equal(c_coors[:P], g_coors[:P])


def test_encoder_generates_pillars_when_not_given():
    """pts_metas without 'pillars': the encoder pillarises on the GPU and reproduces the run with host-built pillars."""
    from deepinteraction_b200 import mmri, synth
    import oracle.mmri as om
    seed = 1950
    torch.manual_seed(seed)
    m = om.DeepInteractionEncoder(2, 16, 24, 128).eval()
    synth.randomize_norm_stats(m, seed)
    enc = mmri.DeepInteractionEncoder(2, 16, 24, 128)
    enc.load_state_dict(m.state_dict(), strict=True)
    enc = enc.to(dev()).eval()
    from tools.make_goldens import small_frame
    fr = synth.to_device(small_frame(seed, aug=True, views=2, c_img=16, c_pts=24, bev=36, batch=2), dev())
    want = [t.clone() for t in enc.forward_nhwc(fr['img_feats'], fr['pts_feats'], fr['img_metas'], fr['pts_metas'])]
    got = enc.forward_nhwc(fr['img_feats'], fr['pts_feats'], fr['img_metas'], dict(pts=fr['pts_metas']['pts']))
    for a, b in zip(got, want):
        assert torch.equal(a, b)


def test_encoder_c128_matches_reference_golden():
    """C = 128 (planar window kernel) against a golden produced by the reference's own files."""
    from deepinteraction_b200 import mmri, synth
    from tools.make_goldens import small_frame
    import oracle.mmri as om
    gold = torch.load(os.path.join(G, 'encoder_c128.pt'), weights_only=False)
    torch.manual_seed(gold['seed'])
    m = om.DeepInteractionEncoder(2, 16, 24, 128).eval()
    synth.randomize_norm_stats(m, gold['seed'])
    enc = mmri.DeepInteractionEncoder(2, 16, 24, 128)
    enc.load_state_dict(m.state_dict(), strict=True)
    enc = enc.to(dev()).eval()
    fr = synth.to_device(small_frame(gold['seed'], aug=gold['aug'], views=2, c_img=16, c_pts=24, bev=36, batch=1), dev())
    img, (p0, p1) = enc(fr['img_feats'], fr['pts_feats'], fr['img_metas'], fr['pts_metas'])
    assert golden_err(p0.cpu(), gold['pts_conv']) < TIGHT
    assert golden_err(p1.cpu(), gold['pts']) < TOL
    assert golden_err(img.cpu(), gold['img']) < TOL


def test_encoder_medium_c128_matches_oracle():
    """C=128 (the production width), 3 cameras 56x100, 90x90 BEV, dense cloud: every module vs the oracle."""
    from deepinteraction_b200 import mmri, synth
    import oracle.mmri as om
    seed = 1700
    torch.manual_seed(seed)
    m = om.DeepInteractionEncoder(2, 32, 48, 128).eval()
    synth.randomize_norm_stats(m, seed)
    fr = synth.make_frame_batch(seed, batch=1, num_views=3, in_hw=(224, 400), stride=4, c_img=32, c_pts=48,
                                bev_hw=(90, 90), n_points=60000, cloud='dense')
    pil, coors, npts = synth.pillarize([p.numpy() for p in fr['pts_metas']['pts']], pillar=108.0 / 90)
    fr['pts_metas'].update(pillars=torch.from_numpy(pil), pillar_coors=torch.from_numpy(coors),
                           pillars_num_points=torch.from_numpy(npts))
    with torch.no_grad():
        r_img, (r_p0, r_p1) = m(fr['img_feats'], fr['pts_feats'], fr['img_metas'], fr['pts_metas'])
    enc = mmri.DeepInteractionEncoder(2, 32, 48, 128)
    enc.load_state_dict(m.state_dict(), strict=True)
    enc = enc.to(dev()).eval()
    frd = synth.to_device(fr, dev())
    img, (p0, p1) = enc(frd['img_feats'], frd['pts_feats'], frd['img_metas'], frd['pts_metas'])
    e = (rel_err(img.cpu(), r_img), rel_err(p0.cpu(), r_p0), rel_err(p1.cpu(), r_p1))
    print('medium encoder rel err img %.2e pts_conv %.2e pts %.2e' % e)
    assert max(e) < TOL


def test_encoder_refuses_training_mode_and_cpu():
    from deepinteraction_b200 import mmri
    enc = mmri.DeepInteractionEncoder(1, 8, 8, 16)
    with pytest.raises(RuntimeError):
        enc.eval().pack()
    enc = enc.to(dev()).train()
    with pytest.raises(NotImplementedError):
        enc.forward_nhwc(torch.zeros(1, 8, 8, 8, device=dev()), torch.zeros(1, 8, 8, 8, device=dev()), [], {})


def _edge_models(seed=5):
    from deepinteraction_b200 import mmri, synth
    import oracle.mmri as om
    torch.manual_seed(seed)
    m = om.DeepInteractionEncoder(1, 16, 24, 32).eval()
    synth.randomize_norm_stats(m, seed)
    enc = mmri.DeepInteractionEncoder(1, 16, 24, 32)
    enc.load_state_dict(m.state_dict(), strict=True)
    return m, enc.to(dev()).eval()


@pytest.mark.parametrize('case', ['empty_cloud', 'three_points', 'no_valid_keys', 'max_points_per_pillar'])
def test_encoder_edge_inputs_match_oracle(case):
    """Degenerate geometry the reference tolerates: a sample without lidar points (all-zero depth maps -> nothing
    lifted), a 3-point cloud, pillars whose points project into no camera (0 valid keys -> zero row, eu.py:314-316),
    pillars filled to the 20-point cap."""
    from deepinteraction_b200 import synth
    from tools.make_goldens import small_frame
    m, enc = _edge_models()
    fr = small_frame(21, aug=False, views=2, c_img=16, c_pts=24, bev=36, batch=2)
    pm = dict(fr['pts_metas'])
    if case == 'empty_cloud':
        pm['pts'] = [pm['pts'][0], pm['pts'][1][:0]]
    elif case == 'three_points':
        pm['pts'] = [pm['pts'][0], pm['pts'][1][:3]]
    elif case == 'no_valid_keys':
        pil = pm['pillars'].clone()
        pil[pm['pillar_coors'][:, 0] == 1, :, 2] = -500.0
        pm['pillars'] = pil
    else:
        pm['pillars_num_points'] = torch.full_like(pm['pillars_num_points'], 20)
        pm['pillars'] = pm['pillars'] + (pm['pillars'] == 0) * pm['pillars'][:, :1]      # padded slots become real points
    with torch.no_grad():
        r_img, (r_p0, r_p1) = m(fr['img_feats'], fr['pts_feats'], fr['img_metas'], pm)
    frd = synth.to_device(dict(fr, pts_metas=pm), dev())
    img, (p0, p1) = enc(frd['img_feats'], frd['pts_feats'], frd['img_metas'], frd['pts_metas'])
    e = (rel_err(img.cpu(), r_img), rel_err(p0.cpu(), r_p0), rel_err(p1.cpu(), r_p1))
    print(case, 'rel err img %.2e pts_conv %.2e pts %.2e' % e)
    assert max(e) < TOL


def test_encoder_without_pillars_is_defined():
    """No pillars at all: the reference crashes on the empty reshape (eu.py:313); this path defines the I2P term as
    zero, i.e. the result equals the one obtained from pillars that see no camera."""
    from deepinteraction_b200 import synth
    from tools.make_goldens import small_frame
    m, enc = _edge_models()
    fr = small_frame(21, aug=False, views=2, c_img=16, c_pts=24, bev=36, batch=2)
    pm = dict(fr['pts_metas'])
    blind = pm['pillars'].clone()
    blind[:, :, 2] = -500.0
    with torch.no_grad():
        r_img, (r_p0, r_p1) = m(fr['img_feats'], fr['pts_feats'], fr['img_metas'], dict(pm, pillars=blind))
    pm0 = dict(pm, pillars=pm['pillars'][:0], pillar_coors=pm['pillar_coors'][:0],
               pillars_num_points=pm['pillars_num_points'][:0])
    frd = synth.to_device(dict(fr, pts_metas=pm0), dev())
    img, (p0, p1) = enc(frd['img_feats'], frd['pts_feats'], frd['img_metas'], frd['pts_metas'])
    assert rel_err(img.cpu(), r_img) < TOL and rel_err(p1.cpu(), r_p1) < TOL


@pytest.mark.parametrize('C', [256, 512])
def test_encoder_hidden_256_512_matches_oracle(C):
    """SURVEY config 5 varies the encoder width: C = 256 / 512 (window kernel with 8 / 16 channel chunks, K = C / 3C
    dense layers on the tensor-core path, I2P fold at C)."""
    from deepinteraction_b200 import mmri, synth
    import oracle.mmri as om
    seed = 1720
    torch.manual_seed(seed)
    m = om.DeepInteractionEncoder(1, 64, 64, C).eval()
    synth.randomize_norm_stats(m, seed)
    fr = synth.make_frame_batch(seed, batch=1, num_views=2, in_hw=(128, 224), stride=4, c_img=64, c_pts=64,
                                bev_hw=(48, 48), n_points=20000, cloud='dense')
    pil, coors, npts = synth.pillarize([p.numpy() for p in fr['pts_metas']['pts']], pillar=108.0 / 48)
    fr['pts_metas'].update(pillars=torch.from_numpy(pil), pillar_coors=torch.from_numpy(coors),
                           pillars_num_points=torch.from_numpy(npts))
    with torch.no_grad():
        r_img, (r_p0, r_p1) = m(fr['img_feats'], fr['pts_feats'], fr['img_metas'], fr['pts_metas'])
    enc = mmri.DeepInteractionEncoder(1, 64, 64, C)
    enc.load_state_dict(m.state_dict(), strict=True)
    enc = enc.to(dev()).eval()
    frd = synth.to_device(fr, dev())
    img, (p0, p1) = enc(frd['img_feats'], frd['pts_feats'], frd['img_metas'], frd['pts_metas'])
    e = (rel_err(img.cpu(), r_img), rel_err(p0.cpu(), r_p0), rel_err(p1.cpu(), r_p1))
    print('C=%d encoder rel err img %.2e pts_conv %.2e pts %.2e' % ((C,) + e))
    assert max(e) < TOL
