"""Backward of the decoder's query x BEV TransformerDecoderLayer (backward.decoder_layer_backward, csrc/xattn_bwd.cu and the
small row kernels di_mha_small_bwd_f32 / di_ln_bwd_f32) against float64 autograd.

The attention-gradient kernel is held to rel_err <= 1e-4 and, per (key or query, head) row of 16 channels, to row_err <=
1e-4 with each row scaled by the magnitude of the terms summed into it (test_gpu_geometry_kernels.row_err), so a wrong
gradient of a key that receives little attention cannot hide behind the global maximum.  For dK_j = sum_i dS_ij Q_i with
dS_ij = A_ij (dA_ij - sum_j' A_ij' dA_ij') and dA_ij = sum_c dO_ic v_jc, the scale is sum_i |dS|_ij |Q_i| with
|dS|_ij = A_ij (t_ij + sum_j' A_ij' t_ij'), t_ij = sum_c |dO_ic| |v_jc|: rounding is relative to these terms, not to
their sums, which cancel (most of all under a sharp softmax, where dA_ij of the dominant key is close to D_i).  The whole layer is compared with autograd through
oracle.mmpi.TransformerDecoderLayer at 1e-4, or 5x the error fp32 autograd through the same oracle makes.
"""
import pytest
import torch

from conftest import rel_err
from test_gpu_geometry_kernels import row_err, same_bits

pytestmark = pytest.mark.gpu

SENT = -1234.5
TOL = 1e-4


def dev():
    return torch.device('cuda:0')


def _ops():
    from deepinteraction_b200 import ops
    return ops


# ---------------------------------------------------------------------------------------------------------------------
# 1. attention-gradient kernel
# ---------------------------------------------------------------------------------------------------------------------
def _attn_inputs(B, P, HW, sharp, seed):
    from deepinteraction_b200 import fold
    ops = _ops()
    g = torch.Generator().manual_seed(seed)
    C, d = 128, dev()
    x = torch.randn(B * HW, C, generator=g)
    W = torch.randn(2 * C, C, generator=g) / C ** 0.5
    bias = torch.randn(2 * C, generator=g) * 0.1
    pos = torch.randn(HW, 2 * C, generator=g) * 0.3
    with _precise_tc():
        kv = ops.linear([x.to(d)], fold.Weight(W, d), bias.to(d), res=pos.to(d), res_mod=HW)     # 3xTF32 GEMM
    q = torch.randn(B * P, C, generator=g).to(d)
    k64 = kv[:, :C].double().view(B, HW, 8, 16)
    s = torch.einsum('bphd,bkhd->bhpk', q.double().view(B, P, 8, 16), k64)
    spread = (s.amax(-1) - s.amin(-1)).mean() if HW > 1 else s.abs().mean() * 2 + 1
    q = q * float((30.0 if sharp else 0.5) / spread)
    dout = torch.randn(B * P, C, generator=g).to(d)
    return q.contiguous(), kv.contiguous(), dout


class _precise_tc:
    def __enter__(self):
        ops = _ops()
        self.saved, ops.TC_BF16[0] = ops.TC_BF16[0], False

    def __exit__(self, *a):
        _ops().TC_BF16[0] = self.saved


def _attn_reference(q, kv, dout, B, P, HW):
    """float64 autograd of dense attention -> (dq, dk, dv, their term-magnitude scales, lse)."""
    C = 128
    q64 = q.double().view(B, P, 8, 16).requires_grad_(True)
    k64 = kv[:, :C].double().view(B, HW, 8, 16).requires_grad_(True)
    v64 = kv[:, C:].double().view(B, HW, 8, 16).requires_grad_(True)
    go = dout.double().view(B, P, 8, 16)
    with torch.enable_grad():
        s = torch.einsum('bphd,bkhd->bhpk', q64, k64)
        a = s.softmax(-1)
        o = torch.einsum('bhpk,bkhd->bphd', a, v64)
        (o * go).sum().backward()
    with torch.no_grad():
        lse = torch.logsumexp(s, -1)                                            # [B, 8, P]
        da_t = torch.einsum('bphd,bkhd->bhpk', go.abs(), v64.abs())              # |terms| of dA_ij = dO_i . v_j
        w = a * (da_t + (a * da_t).sum(-1, keepdim=True))                       # |terms| of dS = A (dA - sum_j A dA)
        sq = torch.einsum('bhpk,bkhd->bphd', w, k64.abs())
        sk = torch.einsum('bhpk,bphd->bkhd', w, q64.abs())
        sv = torch.einsum('bhpk,bphd->bkhd', a, go.abs())
    rows = lambda t, n: t.reshape(B * n, C)
    return (rows(q64.grad, P), rows(k64.grad, HW), rows(v64.grad, HW), rows(sq, P), rows(sk, HW), rows(sv, HW),
            lse.detach())


def _run_bwd(q, kv, dout, B, P, HW, pad=64):
    """Planes in buffers whose rows past B*HW hold NaN, forward with lse, backward into a sentinel-filled dK | dV buffer."""
    from deepinteraction_b200 import _lib
    ops = _ops()
    d = dev()
    nan = float('nan')
    qp = torch.empty(B * P, 192, device=d)
    kp = torch.full((B * HW + pad, 192), nan, device=d)
    vp = torch.full((B * HW + pad, 128), nan, device=d)
    ops._call('di_attn_planes_f32', ops._ptr(q), 128, ops._ptr(qp), B * P, ops._ptr(kv), 256, ops._ptr(kp), ops._ptr(vp),
              B * HW, ops._stream())
    nsplit = _lib.lib().di_xattn_tc_splits(B, HW)
    part = torch.empty(B * 8 * nsplit * 18 * P, device=d)
    out = torch.empty(B * P, 128, device=d)
    lse = torch.empty(B, 8, P, device=d)
    ops._call('di_xattn_tc_lse_f32', ops._ptr(qp), ops._ptr(kp), ops._ptr(vp), ops._ptr(part), ops._ptr(out), ops._ptr(lse),
              B, P, HW, 8, ops._stream())
    dkv = torch.full((B * HW + pad, 256), SENT, device=d)
    dq, _ = ops.xattn_bwd((qp, kp, vp), out, lse, dout, B, P, HW, 8, dkv=dkv[:B * HW])
    torch.cuda.synchronize()
    return dq, dkv, out, lse


ATTN_SHAPES = [(1, 200, 32400), (2, 200, 32400), (3, 1, 1), (1, 15, 63), (2, 64, 64), (3, 65, 65), (1, 256, 1000),
               (2, 1, 32400), (3, 256, 63), (1, 65, 1), (2, 15, 1000), (1, 64, 65), (3, 200, 1000), (1, 256, 32400)]


@pytest.mark.parametrize('sharp', [False, True], ids=['flat', 'sharp'])
@pytest.mark.parametrize('B,P,HW', ATTN_SHAPES)
def test_xattn_bwd_matches_float64_autograd(B, P, HW, sharp):
    q, kv, dout = _attn_inputs(B, P, HW, sharp, 7 * B + P + HW)
    dq, dkv, _, _ = _run_bwd(q, kv, dout, B, P, HW)
    rq, rk, rv, sq, sk, sv, _ = _attn_reference(q, kv, dout, B, P, HW)
    dk, dv = dkv[:B * HW, :128], dkv[:B * HW, 128:]
    assert bool(torch.isfinite(dq).all()) and bool(torch.isfinite(dkv).all())
    errs = dict(dq=(rel_err(dq.double(), rq), row_err(dq, rq, sq, 16)),
                dk=(rel_err(dk.double(), rk), row_err(dk, rk, sk, 16)),
                dv=(rel_err(dv.double(), rv), row_err(dv, rv, sv, 16)))
    print({k: '%.1e / %.1e' % v for k, v in errs.items()})
    for k, (e, r) in errs.items():
        # one key: A = 1 and dS = dA - D is exactly zero, so the references of dQ and dK are float64 rounding and only
        # the scaled per-row error is meaningful
        assert (e <= TOL or (k != 'dv' and HW == 1)) and r <= TOL, (k, e, r)
    assert bool((dkv[B * HW:] == SENT).all()), 'rows past HW were written'
    dq2, dkv2, _, _ = _run_bwd(q, kv, dout, B, P, HW)
    assert same_bits(dq, dq2) and same_bits(dkv, dkv2), 'two calls differ'


@pytest.mark.parametrize('B,P,HW', [(1, 200, 32400), (2, 65, 1000), (3, 1, 63), (1, 256, 1)])
def test_xattn_tc_lse_matches_plain_entry_and_float64(B, P, HW):
    ops = _ops()
    q, kv, dout = _attn_inputs(B, P, HW, True, 11 + P + HW)
    out, lse, _ = ops.xattn_tc_lse(q, kv, B, P, HW, 8)
    assert same_bits(out, ops.xattn_tc(q, kv, B, P, HW, 8))
    want = _attn_reference(q, kv, dout, B, P, HW)[-1]
    assert rel_err(lse.double(), want) <= 1e-6


def test_xattn_bwd_rejects_unsupported_configurations():
    ops = _ops()
    q, kv, dout = _attn_inputs(1, 20, 100, False, 3)
    out, lse, planes = ops.xattn_tc_lse(q, kv, 1, 20, 100, 8)
    with pytest.raises(RuntimeError, match='8 heads'):
        ops.xattn_bwd(planes, out, lse, dout, 1, 20, 100, 4)


# ---------------------------------------------------------------------------------------------------------------------
# 2. self-attention and LayerNorm backward
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('B,P', [(1, 1), (2, 200), (1, 512)])
def test_mha_small_bwd_matches_float64_autograd(B, P):
    ops = _ops()
    g = torch.Generator().manual_seed(P)
    C, H = 128, 8
    qkv = torch.randn(B * P, 3 * C, generator=g)
    qkv[:, :C] *= 0.5
    dout = torch.randn(B * P, C, generator=g)
    x = qkv.double().requires_grad_(True)
    with torch.enable_grad():
        qh, kh, vh = (x[:, i * C:(i + 1) * C].reshape(B, P, H, 16) for i in range(3))
        a = torch.einsum('bphd,bkhd->bhpk', qh, kh).softmax(-1)
        o = torch.einsum('bhpk,bkhd->bphd', a, vh).reshape(B * P, C)
        (o * dout.double()).sum().backward()
    qd = qkv.to(dev())
    got = ops.mha_small_bwd(qd[:, :C], qd[:, C:2 * C], qd[:, 2 * C:], dout.to(dev()), B, P, H)
    assert rel_err(got.double().cpu(), x.grad) < 1e-5
    again = ops.mha_small_bwd(qd[:, :C], qd[:, C:2 * C], qd[:, 2 * C:], dout.to(dev()), B, P, H)
    assert same_bits(got, again)


@pytest.mark.parametrize('M', [1, 200, 512])
def test_ln_bwd_matches_float64_autograd(M):
    ops = _ops()
    g = torch.Generator().manual_seed(M + 1)
    C = 128
    z = torch.randn(M, C, generator=g) * 2
    z[::3] = 500.0 + torch.randn((M + 2) // 3, C, generator=g)           # mean / spread ~ 500
    gamma, beta = torch.rand(C, generator=g) + 0.5, torch.randn(C, generator=g)
    dy = torch.randn(M, C, generator=g)
    zz, gg, bb = (t.double().requires_grad_(True) for t in (z, gamma, beta))
    with torch.enable_grad():
        torch.nn.functional.layer_norm(zz, (C,), gg, bb, 1e-5).mul(dy.double()).sum().backward()
    dz, dg, db = ops.ln_bwd(dy.to(dev()), z.to(dev()), gamma.to(dev()))
    assert rel_err(dz.double().cpu(), zz.grad) < 2e-5
    assert rel_err(dg.double().cpu(), gg.grad) < 2e-5
    assert rel_err(db.double().cpu(), bb.grad) < 2e-6


# ---------------------------------------------------------------------------------------------------------------------
# 3. the whole layer
# ---------------------------------------------------------------------------------------------------------------------
def _decoder(base_shape, plusplus):
    from test_gpu_decoder import _build
    if base_shape:
        test_cfg = dict(dataset='nuScenes', grid_size=[1440, 1440, 40], out_size_factor=8, pc_range=[-54.0, -54.0],
                        voxel_size=[0.075, 0.075], nms_type=None)
        coder = dict(type='TransFusionBBoxCoder', pc_range=[-54.0, -54.0], voxel_size=[0.075, 0.075], out_size_factor=8,
                     post_center_range=[-61.2, -61.2, -10.0, 61.2, 61.2, 10.0], score_threshold=0.0, code_size=10)
        return _build(1700 + plusplus, 6, 200, test_cfg, coder, plusplus=plusplus)[1]
    return _build(1710 + plusplus, 2, 40, plusplus=plusplus)[1]


def _layer_inputs(m, B, seed):
    g = torch.Generator().manual_seed(seed)
    Y, X, C, P = m.y_size, m.x_size, 128, m.num_proposals
    bev = torch.randn(B, Y, X, C, generator=g)
    query = torch.randn(B * P, C, generator=g)
    pix = torch.randint(0, Y * X, (B * P,), generator=g)
    qpos = torch.stack([(pix % X).float() + 0.5, (pix // X).float() + 0.5], 1)
    grad = torch.randn(B * P, C, generator=g)
    return query, qpos, bev, grad


def _oracle_grads(m, query, qpos, bev, grad, dtype, device):
    import oracle.mmpi as om
    B, Y, X, C = bev.shape
    P = query.shape[0] // B
    lay = om.TransformerDecoderLayer(C, 8, 256, om.PositionEmbeddingLearned(2, C), om.PositionEmbeddingLearned(2, C))
    lay.load_state_dict(m.decoder[0].state_dict(), strict=True)
    lay = lay.to(device=device, dtype=dtype).eval()
    ys, xs = torch.meshgrid(torch.arange(Y, dtype=dtype), torch.arange(X, dtype=dtype), indexing='ij')
    bev_pos = torch.stack([xs + 0.5, ys + 0.5], -1).view(1, -1, 2).expand(B, -1, -1).to(device)
    qf = query.to(device, dtype).view(B, P, C).permute(0, 2, 1).contiguous().requires_grad_(True)
    kf = bev.to(device, dtype).view(B, Y * X, C).permute(0, 2, 1).contiguous().requires_grad_(True)
    with torch.enable_grad():
        out = lay(qf, kf, qpos.to(device, dtype).view(B, P, 2), bev_pos)
        (out * grad.to(device, dtype).view(B, P, C).permute(0, 2, 1)).sum().backward()
    res = dict(d_query=qf.grad.permute(0, 2, 1).reshape(B * P, C), d_bev=kf.grad.permute(0, 2, 1).reshape(B, Y, X, C))
    res.update({'grads.' + n: p.grad for n, p in lay.named_parameters()})
    return res


@pytest.mark.parametrize('plusplus', [False, True], ids=['base', 'plusplus'])
@pytest.mark.parametrize('base_shape', [False, True], ids=['small', 'base_shape'])
def test_decoder_layer_backward_matches_oracle_autograd(base_shape, plusplus):
    from deepinteraction_b200 import backward
    m = _decoder(base_shape, plusplus)
    B = 1 if base_shape else 2
    query, qpos, bev, grad = _layer_inputs(m, B, 90 + base_shape + 2 * plusplus)
    d = dev()
    r = backward.decoder_layer_backward(m, query.to(d), qpos.to(d), bev.to(d), grad.to(d))
    got = dict(d_query=r['d_query'], d_bev=r['d_bev'])
    got.update({'grads.' + n: t for n, t in r['grads'].items()})
    want = _oracle_grads(m, query, qpos, bev, grad, torch.float64, d)
    f32 = _oracle_grads(m, query, qpos, bev, grad, torch.float32, d)
    assert set(got) == set(want) and len(r['grads']) == 30
    sd = m.decoder[0].state_dict()
    for k, w in want.items():
        if k.startswith('grads.'):
            assert got[k].shape == sd[k[6:]].shape, k
        bar = max(TOL, 5 * rel_err(f32[k].double(), w))
        e = rel_err(got[k].double(), w)
        print('%-60s %.1e (bar %.1e)' % (k, e, bar))
        assert e <= bar, (k, e, bar)


def test_decoder_layer_function_forward_is_the_layer_and_backward_matches():
    from deepinteraction_b200 import backward
    from tools.make_goldens import small_frame
    from test_gpu_decoder import _build
    _, m = _build(1600, 2, 24)
    gen = torch.Generator().manual_seed(1600)
    fr = small_frame(1600, aug=True, views=2, batch=2)
    pts_in = [torch.randn(2, 128, 36, 36, generator=gen), torch.randn(2, 128, 36, 36, generator=gen)]
    img_in = torch.randn(4, 128, 28, 50, generator=gen)
    nhwc = lambda t: t.permute(0, 2, 3, 1).contiguous().to(dev())
    dbg = {}
    bev = nhwc(pts_in[0])
    m.forward_nhwc(bev, nhwc(pts_in[1]), nhwc(img_in), fr['img_metas'], debug=dbg)
    q0 = dbg['query_feat0'].clone().requires_grad_(True)
    b0 = bev.clone().requires_grad_(True)
    with torch.enable_grad():
        out = backward.DecoderLayerFunction.apply(m, q0, dbg['query_pos0'], b0)
        assert same_bits(out.detach(), dbg['query_feat1'])
        grad = torch.randn(out.shape, generator=gen).to(dev())
        (out * grad).sum().backward()
    r = backward.decoder_layer_backward(m, dbg['query_feat0'], dbg['query_pos0'], bev, grad)
    assert same_bits(q0.grad, r['d_query']) and same_bits(b0.grad, r['d_bev'])


def test_decoder_layer_backward_does_not_synchronise():
    from deepinteraction_b200 import backward
    m = _decoder(False, False)
    d = dev()
    query, qpos, bev, grad = (t.to(d) for t in _layer_inputs(m, 2, 5))
    backward.decoder_layer_backward(m, query, qpos, bev, grad)          # warm-up: builds the per-pack tensors
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode('error')
    try:
        r = backward.decoder_layer_backward(m, query, qpos, bev, grad)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
    assert bool(torch.isfinite(r['d_bev']).all())


def test_decoder_layer_backward_rejects_unsupported_query_count():
    from deepinteraction_b200 import backward
    m = _decoder(False, False)
    d = dev()
    query, qpos, bev, grad = (t.to(d) for t in _layer_inputs(m, 2, 6))
    with pytest.raises(NotImplementedError, match='P <= 256'):
        backward.decoder_layer_backward(m, query.repeat(8, 1), qpos.repeat(8, 1), bev, grad.repeat(8, 1))
