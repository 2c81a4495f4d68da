"""Kernel-level tests of the ++ encoder's gradient kernels (csrc/deform.cu) against float64: di_msdeform_bwd_f32,
di_seq_attn_bwd_f32, di_polar_gather_bwd_f32 and di_axpy_bwd_f32.

Bars.
* msdeform backward: float64 autograd through the oracle's core (oracle.mmri_pp.ms_deform_attn_core, the softmax and
  ref + off / (W, H)).  Every gradient is a short fp32 chain: a softmax (one exp and a division per weight), a 4-term
  bilinear blend of 4-channel dot products reduced over the head's 4 lanes, and one product with the weight.  Each
  step rounds at u = 2^-24 relative to its terms, so about 30u ~ 2e-6 of the terms; the logit gradient
  a_i (dw_i - sum_j a_j dw_j) may cancel, and the value gradient is a sum over queries in any order.  TOL = 1e-5 of the
  largest gradient (conftest.rel_err).  Outside the map every gradient is exactly 0.  The dyadic case puts every
  location on integer pixels (power-of-two maps, offsets in multiples of 1/4) so that floor() agrees in fp32 and float64:
  there the bilinear derivative is one-sided in both.
* seq_attn backward: float64 autograd of softmax(q k^T / 4) v.  dq and dk sum Lk resp. Lq terms P (dP - D) of 16-channel
  dot products; dv sums Lq terms.  The fp32 sums over at most 112 terms round at ~ sqrt(112) u of the terms, and D_t is
  taken from the saved fp32 output.  TOL = 1e-5 (rel_err per tensor), as the forward's.
* polar gather backward: the adjoint identity <gather(rays), g> = <rays, gather_bwd(g)>, both sides in float64, the
  left one from _gather_ref of test_gpu_polar_kernels.py, the right one from the kernel's d rays.  The kernel's weights
  are fp32 products w_corner / count (2u), and its position rounds as the forward's (the dyadic rigs: exactly), so the
  two sides agree to 1e-5 of sum |rays| |g| w.
* axpy backward: d s against float64 to 1e-6 relative to sum |dout b| (double partials: the only rounding is the final
  cast to fp32); db = s dout exactly.
"""
import ctypes
import math
import zlib

import pytest
import torch

from conftest import rel_err
from kernel_check import _status, same_bits

gpu = pytest.mark.gpu
DI_ERR_ARG, DI_ERR_UNSUPPORTED = -1, -3
TOL = 1e-5


def dev():
    return torch.device('cuda:0')


# ---------------------------------------------------------------------------------------------------------------------
# 1. di_msdeform_bwd_f32
# ---------------------------------------------------------------------------------------------------------------------
def _msda_ref(values, raw, dout, B, hq, wq):
    """float64 autograd through ms_deform_attn_core: -> (d raw, [d value_l])."""
    import oracle.mmri_pp as opp
    L = len(values)
    nq = hq * wq
    shapes = [tuple(v.shape[1:3]) for v in values]
    vals = [v.double().cpu().requires_grad_(True) for v in values]
    r = raw.double().cpu().requires_grad_(True)
    off = r[:, :8 * L * 4 * 2].reshape(B, nq, 8, L, 4, 2)
    logit = r[:, 8 * L * 4 * 2:8 * L * 4 * 3].reshape(B, nq, 8, L * 4)
    ry, rx = torch.meshgrid(torch.arange(hq, dtype=torch.float64) + 0.5, torch.arange(wq, dtype=torch.float64) + 0.5,
                            indexing='ij')
    ref = torch.stack([rx.reshape(-1) / wq, ry.reshape(-1) / hq], -1)[None].unsqueeze(-2).repeat(1, 1, L, 1)
    norm = torch.tensor([[w, h] for h, w in shapes], dtype=torch.float64)
    loc = ref[:, :, None, :, None, :] + off / norm[None, None, None, :, None, :]
    aw = logit.softmax(-1).view(B, nq, 8, L, 4)
    v_flat = torch.cat([v.reshape(B, -1, 8, 16) for v in vals], 1)
    out = opp.ms_deform_attn_core(v_flat, shapes, loc, aw)
    out.backward(dout.double().cpu().view(B, nq, 128))
    return r.grad, [v.grad for v in vals]


# id: (B, hq, wq, level shapes, offset kind, logit scale)
MSDA_CASES = {
    'L1_random': (2, 13, 21, [(13, 21)], 'random', 1.0),
    'L2_random': (2, 13, 21, [(13, 21), (7, 11)], 'random', 1.0),
    'L2_border_band': (1, 12, 20, [(12, 20), (6, 10)], 'border', 1.0),
    'L1_outside': (1, 9, 15, [(9, 15)], 'outside', 1.0),
    'L2_dyadic': (2, 8, 16, [(8, 16), (4, 8)], 'dyadic', 1.0),
    'L2_saturated': (1, 13, 21, [(13, 21), (7, 11)], 'random', 40.0),
    'L1_nq_tail': (3, 5, 7, [(5, 7)], 'random', 1.0),             # 105 queries: not a multiple of 8 warps
}


def _msda_inputs(case):
    B, hq, wq, shapes, kind, lscale = MSDA_CASES[case]
    L, nq = len(shapes), hq * wq
    g = torch.Generator().manual_seed(zlib.crc32(case.encode()))
    values = [torch.randn(B, h, w, 128, generator=g) for h, w in shapes]
    logit = torch.randn(B * nq, 8 * L * 4, generator=g) * lscale
    if kind == 'random':                           # up to ~10 px: zero padding at the map edges
        off = torch.randn(B * nq, 8, L, 4, 2, generator=g) * 3.0
    elif kind == 'border':                          # every location in the band -1 < x < 0 or W-1 < x < W (and in y)
        ry, rx = torch.meshgrid(torch.arange(hq) + 0.5, torch.arange(wq) + 0.5, indexing='ij')
        off = torch.empty(B * nq, 8, L, 4, 2)
        for l, (h, w) in enumerate(shapes):
            px, py = rx.reshape(-1) / wq * w - 0.5, ry.reshape(-1) / hq * h - 0.5      # pixel of the reference point
            frac = torch.rand(B * nq, 8, 4, 2, generator=g) * 0.8 + 0.1
            left = torch.rand(B * nq, 8, 4, 2, generator=g) < 0.5
            tx = torch.where(left[..., 0], -frac[..., 0], w - 1 + frac[..., 0])
            ty = torch.where(left[..., 1], -frac[..., 1], h - 1 + frac[..., 1])
            off[:, :, l, :, 0] = tx - px.repeat(B)[:, None, None]
            off[:, :, l, :, 1] = ty - py.repeat(B)[:, None, None]
    elif kind == 'outside':                         # every corner outside the map: all gradients exactly 0
        off = (torch.rand(B * nq, 8, L, 4, 2, generator=g) + 1.0) * 40.0 * torch.where(
            torch.rand(B * nq, 8, L, 4, 2, generator=g) < 0.5, -1.0, 1.0)
    else:                                           # integer pixel positions: offsets in multiples of 1/2 (level 1: +1/4)
        off = torch.randint(-6, 7, (B * nq, 8, L, 4, 2), generator=g).float()
        if L > 1:
            off[:, :, 1] += 0.25                    # (i + 0.5) / 2 - 0.5 + 0.25 = i / 2: integer or half pixels
    raw = torch.cat([off.reshape(B * nq, -1), logit], 1)
    dout = torch.randn(B * nq, 128, generator=g)
    return B, hq, wq, values, raw, dout


def _msda_run(values, raw, dout, B, hq, wq):
    from deepinteraction_b200 import ops
    d = lambda t: t.to(dev()).contiguous()
    return ops.msdeform_bwd([d(v) for v in values], d(raw), d(dout), B, hq, wq)


@gpu
@pytest.mark.parametrize('case', list(MSDA_CASES))
def test_msdeform_bwd_matches_float64(case):
    B, hq, wq, values, raw, dout = _msda_inputs(case)
    want_raw, want_vals = _msda_ref(values, raw, dout, B, hq, wq)
    d_raw, d_vals = _msda_run(values, raw, dout, B, hq, wq)
    d_raw2, _ = _msda_run(values, raw, dout, B, hq, wq)
    assert same_bits(d_raw, d_raw2), 'd_raw must not depend on the call'
    if MSDA_CASES[case][4] == 'outside':
        n_off = raw.shape[1] // 3 * 2
        assert bool((d_raw[:, :n_off] == 0).all()) and all(bool((v == 0).all()) for v in d_vals)
        # the logits still get a_i (dw_i - sum a_j dw_j) = 0 exactly, dw being 0
        assert bool((d_raw == 0).all())
        return
    n_off = raw.shape[1] // 3 * 2
    e_off = rel_err(d_raw[:, :n_off].cpu().double(), want_raw[:, :n_off])
    e_log = rel_err(d_raw[:, n_off:].cpu().double(), want_raw[:, n_off:])
    e_val = max(rel_err(g.cpu().double(), w) for g, w in zip(d_vals, want_vals))
    print(f'msdeform_bwd {case}: d offsets {e_off:.2e} d logits {e_log:.2e} d values {e_val:.2e}')
    assert max(e_off, e_log, e_val) < TOL


@gpu
def test_msdeform_bwd_rejects_before_any_launch():
    """Unsupported configurations are DI_ERR_UNSUPPORTED and bad strides DI_ERR_ARG, before anything is written."""
    from deepinteraction_b200 import ops
    B, hq, wq, values, raw, dout = _msda_inputs('L1_nq_tail')
    v = values[0].to(dev())
    r, g = raw.to(dev()), dout.to(dev())
    d_raw = torch.full_like(r, 7.0)
    d_v = torch.zeros_like(v)
    sh = (ctypes.c_int * 4)(hq, wq, hq, wq)
    p = ops._ptr

    def call(heads=8, dim=16, L=1, P=4, ld_draw=None):
        return _status('di_msdeform_bwd_f32', p(v), p(v), p(r), r.stride(0), p(g), g.stride(0), p(d_raw),
                       d_raw.stride(0) if ld_draw is None else ld_draw, p(d_v), p(d_v), B, hq * wq, hq, wq, heads, dim, L,
                       P, sh)
    assert call(heads=4) == DI_ERR_UNSUPPORTED
    assert call(dim=32) == DI_ERR_UNSUPPORTED
    assert call(P=8) == DI_ERR_UNSUPPORTED
    assert call(L=3) == DI_ERR_UNSUPPORTED
    assert call(ld_draw=95) == DI_ERR_ARG
    assert bool((d_raw == 7.0).all()) and bool((d_v == 0).all()), 'a rejected call wrote its outputs'


# ---------------------------------------------------------------------------------------------------------------------
# 2. di_seq_attn_bwd_f32
# ---------------------------------------------------------------------------------------------------------------------
SEQ_CASES = [(12, 200, 60, 60, False), (12, 200, 60, 112, False), (12, 200, 60, 60, True), (12, 200, 60, 112, True),
             (3, 7, 60, 33, False), (5, 3, 60, 1, False), (1, 5, 60, 257, True), (3, 5, 97, 112, False),
             (2, 3, 33, 65, True)]


def _seq_id(c):
    return 'G%d_Wn%d_Lq%d_Lk%d_%s' % (c[0], c[1], c[2], c[3], 'sharp' if c[4] else 'flat')


@gpu
@pytest.mark.parametrize('case', SEQ_CASES, ids=_seq_id)
def test_seq_attn_bwd_matches_float64(case):
    """q, k, v as the polar block passes them: one packed [M, 3C] buffer for the self attention (Lq == Lk), q of a
    [Mq, C] buffer and k | v of a [Mk, 2C] buffer otherwise; dq | dk | dv written into the same packing.  The sharp
    cases use q and k in multiples of 1/4 (exact logits with a spread of ~60, as check_seq_attn)."""
    from deepinteraction_b200 import ops
    G, Wn, Lq, Lk, sharp = case
    H, C = 8, 128
    g = torch.Generator().manual_seed(zlib.crc32(_seq_id(case).encode()))
    Mq, Mk = G * Lq * Wn, G * Lk * Wn
    packed = Lq == Lk
    qb = torch.randn(Mq, 3 * C, generator=g)
    kvb = qb[:, C:] if packed else torch.randn(Mk, 2 * C, generator=g)
    if sharp:
        qb[:, :C] = torch.randint(-24, 25, (Mq, C), generator=g).float() / 4
        kvb[:, :C] = torch.randint(-24, 25, (Mk, C), generator=g).float() / 4
    dout = torch.randn(Mq, C, generator=g)
    qb = qb.to(dev())
    kvb = qb[:, C:] if packed else kvb.to(dev())
    q, k, v = qb[:, :C], kvb[:, :C], kvb[:, C:2 * C]
    out = ops.seq_attn(q, k, v, G, Wn, Lq, Lk, H)
    res = []
    for _ in range(2):
        if packed:
            buf = torch.full((Mq, 3 * C), float('nan'), device=dev())
            dq, dk, dv = buf[:, :C], buf[:, C:2 * C], buf[:, 2 * C:]
        else:
            dq = torch.full((Mq, C), float('nan'), device=dev())
            dkv = torch.full((Mk, 2 * C), float('nan'), device=dev())
            dk, dv = dkv[:, :C], dkv[:, C:]
        ops.seq_attn_bwd(q, k, v, out, dout.to(dev()), G, Wn, Lq, Lk, H, dq, dk, dv)
        res.append([t.clone() for t in (dq, dk, dv)])
    assert all(same_bits(a, b) for a, b in zip(*res)), 'gradients must not depend on the call'
    sp = lambda t, L: t.double().cpu().reshape(G, L, Wn, H, 16).permute(0, 2, 3, 1, 4).requires_grad_(True)
    q6, k6, v6 = sp(q, Lq), sp(k, Lk), sp(v, Lk)
    a = torch.softmax(q6 @ k6.transpose(-1, -2) * 0.25, -1) @ v6
    a.backward(dout.double().reshape(G, Lq, Wn, H, 16).permute(0, 2, 3, 1, 4))
    back = lambda t, L: t.permute(0, 3, 1, 2, 4).reshape(G * L * Wn, C)
    errs = [rel_err(got.cpu().double(), back(w.grad, L)) for got, w, L in zip(res[0], (q6, k6, v6), (Lq, Lk, Lk))]
    print('seq_attn_bwd %s: dq %.2e dk %.2e dv %.2e' % ((_seq_id(case),) + tuple(errs)))
    assert max(errs) < TOL


@gpu
def test_seq_attn_bwd_rejects_long_queries_and_head_dim():
    from deepinteraction_b200 import ops
    G, Wn, L, C = 1, 2, 4, 128
    x = torch.randn(G * L * Wn, C, device=dev())
    p = ops._ptr
    call = lambda Lq, dim: _status('di_seq_attn_bwd_f32', *([p(x), C] * 8), G, Wn, Lq, L, 8, dim)
    assert call(L, 8) == DI_ERR_UNSUPPORTED
    assert call(129, 16) == DI_ERR_UNSUPPORTED


# ---------------------------------------------------------------------------------------------------------------------
# 3. di_polar_gather_bwd_f32: the adjoint of the gather
# ---------------------------------------------------------------------------------------------------------------------
def _adjoint_check(rays, lidar, proj, undo, camc, V, in_hw, pc, r0, r_cnt, seed):
    from deepinteraction_b200 import ops
    from test_gpu_polar_kernels import _gather_ref
    d64 = lambda t: t.double().to(dev())
    out, _, count = _gather_ref(d64(rays), d64(lidar) * 0, d64(proj), d64(undo), d64(camc), V, in_hw, pc, r0, r_cnt)
    g = torch.randn(lidar.shape, generator=torch.Generator().manual_seed(seed))
    d = lambda t: t.to(dev()).contiguous()
    d_rays = [ops.polar_gather_bwd(d(g), tuple(rays.shape), d(proj), d(undo), d(camc), V, in_hw, pc, r0, r_cnt)
              for _ in range(2)]
    lhs = float((out * d64(g)).sum())
    rhs = float((d64(rays) * d_rays[0].double()).sum())
    # the same weights applied to |rays| and |g|: the scale of the terms of both inner products
    scale = float((d64(rays).abs() * d_rays[0].double().abs()).sum()) + 1e-300
    e = abs(lhs - rhs) / scale
    # cells no camera sees take no gradient; every d ray is finite
    assert bool(torch.isfinite(d_rays[0]).all())
    return e, count, d_rays


@gpu
@pytest.mark.parametrize('case', ['b1_v1', 'b2_v2', 'b2_v6', 'b1_v7_depth', 'b2_v3_y16_x32'])
def test_polar_gather_bwd_is_the_adjoint_dyadic(case):
    """The dyadic rigs of test_gpu_polar_kernels.py: borders on cell centres, cells no camera sees (b1_v7_depth has a
    camera that sees none), and the radius clamped below r0 and above r0 + R."""
    from test_gpu_polar_kernels import GATHER_CASES, IN_D, PC_D, R0_D, R_D, W_D, _dyadic, _radius_clamped
    B, names, Y, X = GATHER_CASES[case]
    V = len(names)
    proj, undo, camc = _dyadic(names, B)
    g = torch.Generator().manual_seed(sum(map(ord, case)) + 5)
    rays = torch.randn(B * V, R_D, W_D, 128, generator=g)
    lidar = torch.zeros(B, Y, X, 128)
    e, count, _ = _adjoint_check(rays, lidar, proj, undo, camc, V, IN_D, PC_D, R0_D, float(R_D), 99)
    below, above = _radius_clamped(B, names, Y, X)
    print(f'polar_gather_bwd {case}: adjoint {e:.2e}; unseen cells {int((count == 0).sum())}; clamped {below}/{above}')
    if 'Z' not in names:
        assert bool((count == 0).any())
    assert e < TOL


@gpu
def test_polar_gather_bwd_is_the_adjoint_config4_rig():
    """B = 2, V = 6, R = 60, W = 200, 180 x 180 on the synthetic rig (un-augmented, as the forward's test)."""
    from deepinteraction_b200 import geom, polar
    from test_gpu_polar_kernels import PC, _metas
    B, V, R, W, Y, X = 2, 6, 60, 200, 180, 180
    metas = _metas(B, V, (448, 800), False)
    proj, _ = geom.camera_rows_host(metas)
    _, undo, camc = polar.polar_consts_host(metas)
    g = torch.Generator().manual_seed(405)
    rays = torch.randn(B * V, R, W, 128, generator=g)
    e, count, d_rays = _adjoint_check(rays, torch.zeros(B, Y, X, 128), proj, undo, camc, V, geom.input_hw(metas), PC, 1.0,
                                      float(R), 406)
    print(f'polar_gather_bwd config4: adjoint {e:.2e}; cells seen by 0 cameras {int((count == 0).sum())}')
    assert e < TOL


# ---------------------------------------------------------------------------------------------------------------------
# 4. di_axpy_bwd_f32
# ---------------------------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize('n', [4, 1028, 128 * 180 * 180, 6 * 112 * 200 * 128])
def test_axpy_bwd_matches_float64(n):
    from deepinteraction_b200 import ops
    g = torch.Generator().manual_seed(n)
    dout, b = torch.randn(n, generator=g), torch.randn(n, generator=g)
    s = torch.tensor([0.7])
    outs = [ops.axpy_bwd(dout.to(dev()), b.to(dev()), s.to(dev())) for _ in range(2)]
    (db, ds), (db2, ds2) = outs
    assert same_bits(ds, ds2) and same_bits(db, db2)
    assert torch.equal(db.cpu(), dout * s)
    want = float((dout.double() * b.double()).sum())
    scale = float((dout.double() * b.double()).abs().sum())
    e = abs(float(ds) - want) / scale
    print(f'axpy_bwd n={n}: d s {e:.2e}')
    assert e < 1e-6
