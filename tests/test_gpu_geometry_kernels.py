"""Kernel-level tests of the plain-CUDA sampling, attention and row kernels of the MMRI encoders (csrc/geometry.cu,
csrc/deform.cu and the shift kernel of csrc/lcab_bwd.cu) against float64 references written from each operation's
definition.  They cover every channel-width instantiation (NJ = 1, 2, 4 lane slices, and widths that fill a later slice
only partly), the map borders and non-finite coordinates, the strict validity tests, the live-count (n_dev) contract of
the capacity-sized arrays, outputs that are accumulated into, and atomics that collide.

Error metric.  Beside conftest.rel_err (max|a-b| / max|b|), row_err takes the max over output rows of
max|a-b| / scale_row, where scale_row is the magnitude of the terms summed into that row (>= max|b_row|).  A global max
hides a wrong row whose values are small, such as a pillar whose one valid key sits at a border; and fp32 rounding is
relative to the summed terms, not to their sum, which may cancel.  A row whose terms are all zero must be exactly zero.

Bars.  These kernels use fp32 FFMA only.  The geometry fed to them is exactly representable (power-of-two camera
scales and depths, dyadic points and offsets), so the sampling positions of kernel and reference agree exactly and what
remains is fp32 rounding of the sums: a few units of 2^-24 times a sqrt of the term count, about 1e-6 of the row scale.
TOL = 1e-5 leaves a 10x margin.  Kernels that only move data are held to bit equality.
"""
import ctypes
import math

import pytest
import torch
import torch.nn.functional as F

from conftest import rel_err
from kernel_check import _capi, row_err, same_bits

pytestmark = pytest.mark.gpu

TOL = 1e-5
SENT = -1234.5          # sentinel of the cells a kernel must leave alone
U = 2.0 ** -24          # fp32 unit roundoff


def dev():
    return torch.device('cuda:0')


def _ops():
    from deepinteraction_b200 import ops
    return ops


def _p(t):
    return _ops()._ptr(t)


# ---------------------------------------------------------------------------------------------------------------------
# 1. bev_sample / bev_sample_bwd
# ---------------------------------------------------------------------------------------------------------------------
def _edge_coords(n):
    """Pixel-space coordinates (align_corners=False) along an axis of n pixels: the zero-padding borders, exact integers
    and half-integers, just inside / outside the map, and values the kernel's guard must reject."""
    return [-1.0, -1.0 + 1e-3, -0.5, 0.0, 1.0, 0.5, 2.5, n - 1.0, n - 0.5, n - 1e-3, float(n), n + 0.9,
            1e30, float('nan'), float('inf'), float('-inf'), -1e30]


def _bev_grid(B, V, Yb, Xb, gen, hot=(7.0, 5.0), n_hot=768):
    """[B*V, N, 2] sampling coordinates: every x edge with every y edge, random points in and around the map, and
    n_hot points per image inside one 3x3 patch (its atomics collide in the backward)."""
    ex, ey = torch.tensor(_edge_coords(Xb)), torch.tensor(_edge_coords(Yb))
    gx, gy = torch.meshgrid(ex, ey, indexing='ij')
    edge = torch.stack([gx.flatten(), gy.flatten()], -1).expand(B * V, -1, -1)
    rand = torch.rand(B * V, 64, 2, generator=gen, dtype=torch.float64) * torch.tensor([Xb + 3.0, Yb + 3.0]) - 2.0
    hotp = torch.tensor(hot) + (torch.rand(B * V, n_hot, 2, generator=gen, dtype=torch.float64) * 2 - 1)
    return torch.cat([edge.float(), rand.float(), hotp.float()], 1).contiguous()


def _bev_ref(bev64, grid, B, V):
    """F.grid_sample(float64, bilinear, zeros, align_corners=False) of bev[b] for image b*V+v at pixel coordinates
    grid[b*V+v] -> [B*V, N, C], and the mask of the samples whose coordinates are non-finite or huge (zero rows)."""
    Yb, Xb = bev64.shape[1:3]
    g = grid.double()
    bad = ~(torch.isfinite(g).all(-1) & (g.abs() < 1e4).all(-1))
    g = torch.where(bad[..., None], torch.full_like(g, -10.0), g)          # far outside: grid_sample gives 0
    norm = torch.stack([(2 * g[..., 0] + 1) / Xb - 1, (2 * g[..., 1] + 1) / Yb - 1], -1)
    src = bev64.permute(0, 3, 1, 2)[torch.arange(B).repeat_interleave(V)]
    out = F.grid_sample(src, norm[:, None], mode='bilinear', padding_mode='zeros', align_corners=False)
    return out[:, :, 0].transpose(1, 2), bad


@pytest.mark.parametrize('C', [4, 64, 128, 132, 256, 260, 384, 512])
def test_bev_sample_fwd_bwd_matches_grid_sample(C):
    ops = _ops()
    gen = torch.Generator().manual_seed(100 + C)
    B, V, Yb, Xb = 2, 3, 8, 16          # non-square; powers of two keep the reference's normalised grid exact
    bev = torch.randn(B, Yb, Xb, C, generator=gen)
    grid = _bev_grid(B, V, Yb, Xb, gen)
    N = grid.shape[1]
    bev64 = bev.double().requires_grad_(True)
    want, bad = _bev_ref(bev64, grid, B, V)
    scale, _ = _bev_ref(bev.double().abs(), grid, B, V)                    # sum of |w v| per output element
    got = ops.bev_sample(bev.to(dev()), grid.view(B * V, 1, N, 2).to(dev()), V).view(B * V, N, C).cpu()
    e_row, e_glob = row_err(got, want, scale), rel_err(got.double(), want.detach())
    print(f'bev_sample C={C}: row {e_row:.2e} global {e_glob:.2e}')
    assert bool((got[bad] == 0).all()), 'non-finite / huge coordinates must give an exactly zero row'
    assert e_row < TOL and e_glob < TOL

    # backward: d_bev is pre-filled and must be accumulated into
    d_out = torch.randn(B * V, N, C, generator=gen)
    prefill = torch.randn(B, Yb, Xb, C, generator=gen)
    grad, = torch.autograd.grad(want, bev64, d_out.double(), retain_graph=True)
    gscale, = torch.autograd.grad(want, bev64, d_out.double().abs())
    d_bev, d_out_d, grid_d = prefill.to(dev()), d_out.to(dev()), grid.to(dev())
    _capi('di_bev_sample_bwd_f32', _p(d_out_d), _p(grid_d), _p(d_bev), B, V, N, Yb, Xb, C)
    d_want = prefill.double() + grad
    # 3 x 768 samples per batch element land in one 3x3 patch: the fp32 atomics, in whatever order they run, round
    # each partial sum once, about 2^-24 sqrt(n) ~ 3e-6 of the summed |terms| (the row scale); TOL holds that
    e_row, e_glob =row_err(d_bev, d_want, prefill.double().abs() + gscale), rel_err(d_bev.cpu().double(), d_want)
    print(f'bev_sample_bwd C={C}: row {e_row:.2e} global {e_glob:.2e}')
    assert e_row < TOL and e_glob < TOL
    # samples the guard rejects scatter nothing: d_bev stays bit-identical
    gb = grid[:, bad[0]].contiguous().to(dev())
    d_bad = torch.randn(B * V, gb.shape[1], C, generator=gen).to(dev())
    d_bev = prefill.to(dev())
    _capi('di_bev_sample_bwd_f32', _p(d_bad), _p(gb), _p(d_bev), B, V, gb.shape[1], Yb, Xb, C)
    assert same_bits(d_bev, prefill)


# ---------------------------------------------------------------------------------------------------------------------
# 2. i2p_attend / i2p_attend_bwd and the dropout variants
# ---------------------------------------------------------------------------------------------------------------------
H_IN, W_IN, H_F, W_F = 32, 64, 8, 16           # powers of two: u / W_IN and the un-normalisation stay exact
EPS32 = float(torch.tensor(1e-5, dtype=torch.float32))


def _cam(b, v):
    """Camera b, v: u = f x / z + W_IN / 2 + ox, v = f y / z + H_IN / 2 + oy, depth z.  Power-of-two f and integer
    offsets keep every projection, division and un-normalisation of dyadic points exact in fp32.  The one inexact
    projection, of the points at depth ~1e-5, lands at (6.5 | 7.5 | 8.5, 3.25 | 3.5 | 3.75): inside a pixel cell, so its
    one-ulp rounding moves weight between the same four pixels the float64 reference uses."""
    f = (4.0, 8.0, 16.0)[(b + v) % 3]
    return f, 4.0 * ((v + 2 * b) % 3 - 1), 1.0 * ((v + b) % 3 - 1)


def _proj(B, V):
    proj = torch.zeros(B, V, 12)
    for b in range(B):
        for v in range(V):
            f, ox, oy = _cam(b, v)
            proj[b, v] = torch.tensor([f, 0, W_IN / 2 + ox, 0, 0, f, H_IN / 2 + oy, 0, 0, 0, 1, 0])
    return proj


def _edge_points(b, v):
    """Points on and next to the thresholds of camera (b, v): u = 0 and u = W_IN (nx = -1, 1: invalid), u just inside
    both, the same for v, and depth exactly at (invalid) and one ulp above (valid) the 1e-5 guard."""
    f, ox, oy = _cam(b, v)
    cu, cv, d = W_IN / 2 + ox, H_IN / 2 + oy, 2.0 ** -4
    above = float(torch.nextafter(torch.tensor(EPS32), torch.tensor(1.0)))
    return [(-cu / f, 0, 1), ((W_IN - cu) / f, 0, 1), ((d - cu) / f, 0, 1), ((W_IN - d - cu) / f, 0, 1),
            (0, -cv / f, 1), (0, (H_IN - cv) / f, 1), (0, (d - cv) / f, 1), (0, (H_IN - d - cv) / f, 1),
            (0, 0, EPS32), (0, 0, above)]


def _i2p_case(C, T, V, seed, B=2, pdim=5):
    """Pillars of every kind: random points (some behind the camera or at depth 0, some outside the image), npts = 0,
    npts > T, pillars that see nothing, threshold points, and duplicated pillars that sample the same pixels.  Slots
    past npts hold points that would be valid, so a kernel that ignores npts fails."""
    g = torch.Generator().manual_seed(seed)
    rnd = lambda *s: torch.rand(*s, generator=g)

    def rand_points(n):
        xy = torch.randint(-12 * 16, 12 * 16 + 1, (n, 2), generator=g).float() / 16
        z = torch.tensor([0.5, 1.0, 2.0, 4.0])[torch.randint(0, 4, (n,), generator=g)]
        r = rnd(n)
        z = torch.where(r < 0.1, -z, torch.where(r < 0.15, torch.zeros_like(z), z))
        return torch.cat([xy, z[:, None]], 1)

    pts, npts, bs = [], [], []

    def add(p3, n, b):
        full = torch.cat([p3, rnd(T, pdim - 3) * 100], 1)
        pts.append(full)
        npts.append(n)
        bs.append(b)

    for i in range(24):
        add(rand_points(T), int(torch.randint(1, T + 1, (1,), generator=g)), i % B)
    for b in range(B):
        add(rand_points(T), 0, b)                                               # npts = 0
        add(rand_points(T), T + 7, b)                                           # npts > T: clamped
        blind = rand_points(T)
        blind[:, 2] = -blind[:, 2].abs() - 0.5                                  # all behind the camera
        add(blind, T, b)
        far = rand_points(T)
        far[:, 0] = 1000.0                                                      # all right of every image
        far[:, 2] = 1.0
        add(far, T, b)
        for v in range(V):                                                      # threshold points, T per pillar
            e = torch.tensor(_edge_points(b, v), dtype=torch.float32)
            for s in range(0, e.shape[0], T):
                chunk = e[s:s + T]
                fill = rand_points(T)
                fill[:chunk.shape[0]] = chunk
                add(fill, chunk.shape[0], b)
    for i in range(4):                                                          # 3 copies each: same pixels
        for _ in range(3):
            add(pts[i].clone()[:, :3], npts[i], bs[i])
    perm = torch.randperm(len(pts), generator=g)
    pillars = torch.stack(pts)[perm].contiguous()
    npts = torch.tensor(npts, dtype=torch.int32)[perm]
    coors = torch.zeros(len(pts), 4, dtype=torch.int32)
    coors[:, 0] = torch.tensor(bs, dtype=torch.int32)[perm]
    coors[:, 2:] = torch.randint(0, 50, (len(pts), 2), generator=g, dtype=torch.int32)
    P = len(pts)
    return dict(pillars=pillars, npts=npts, coors=coors, proj=_proj(B, V), B=B, V=V, T=T, C=C,
                qk=torch.randn(P, C, generator=g) * (2.0 / math.sqrt(C)),
                img=torch.randn(B * V, H_F, W_F, C, generator=g),
                ds=torch.randn(P, C + 4, generator=g), d_img0=torch.randn(B * V, H_F, W_F, C, generator=g))


def _i2p_ref(cs, mask=None):
    """float64 I2P attention from its definition.  Key j = t*V + v of pillar p: point t projected by proj[b, v]; valid
    when t < min(npts, T), cz > 1e-5 and both normalised coordinates lie strictly inside (-1, 1) -- evaluated in fp32
    with the kernel's formula, the contract.  k_j = grid_sample(img[b*V + v]) at the normalised coordinates;
    s = sum_j a_j m_j k_j with a = softmax over the valid keys of qk . k_j, m the dropout factors (1 without);
    rho = sum_j a_j m_j.  Returns leaves (qk, img) for autograd and the per-key tensors for the error scales."""
    pl, proj, V, T = cs['pillars'], cs['proj'], cs['V'], cs['T']
    P, C = cs['qk'].shape
    b = cs['coors'][:, 0].long()
    M = proj[b]                                                                   # [P, V, 12] fp32
    x, y, z = (pl[:, :, i, None] for i in range(3))                               # [P, T, 1]
    m = lambda i: M[:, None, :, i]
    cx = m(0) * x + m(1) * y + m(2) * z + m(3)
    cy = m(4) * x + m(5) * y + m(6) * z + m(7)
    cz = m(8) * x + m(9) * y + m(10) * z + m(11)
    eps = torch.tensor(1e-5, dtype=torch.float32)
    zz = torch.maximum(cz, eps)
    nx, ny = (cx / zz / W_IN - 0.5) * 2, (cy / zz / H_IN - 0.5) * 2
    live = torch.arange(T)[None, :, None] < torch.clamp(cs['npts'].long(), max=T)[:, None, None]
    valid = live & (cz > eps) & (nx > -1) & (nx < 1) & (ny > -1) & (ny < 1)       # [P, T, V]
    # sampling positions in float64
    M64, x, y, z = M.double(), x.double(), y.double(), z.double()
    m = lambda i: M64[:, None, :, i]
    u = (m(0) * x + m(1) * y + m(2) * z + m(3)) / (m(8) * x + m(9) * y + m(10) * z + m(11))
    w = (m(4) * x + m(5) * y + m(6) * z + m(7)) / (m(8) * x + m(9) * y + m(10) * z + m(11))
    grid = torch.stack([2 * u / W_IN - 1, 2 * w / H_IN - 1], -1)
    grid = torch.where(valid[..., None], grid, torch.full_like(grid, -3.0))       # invalid keys: outside, masked anyway
    qk = cs['qk'].double().requires_grad_(True)
    img = cs['img'].double().requires_grad_(True)
    src = img.permute(0, 3, 1, 2)
    K = torch.zeros(P, T, V, C, dtype=torch.float64)
    for bb in range(cs['B']):
        pb = (b == bb).nonzero().squeeze(1)
        for v in range(V):
            smp = F.grid_sample(src[bb * V + v:bb * V + v + 1], grid[pb, :, v].reshape(1, 1, -1, 2), mode='bilinear',
                                padding_mode='zeros', align_corners=False)[0, :, 0]
            K = K.index_put((pb[:, None], torch.arange(T)[None, :], torch.tensor(v)), smp.t().reshape(-1, T, C))
    K, valid = K.reshape(P, T * V, C), valid.reshape(P, T * V)
    lg = torch.einsum('pc,psc->ps', qk, K).masked_fill(~valid, -math.inf)
    mx = lg.detach().amax(1, keepdim=True)
    e = torch.exp(lg - torch.where(torch.isfinite(mx), mx, torch.zeros_like(mx)))
    L = e.sum(1, keepdim=True)
    a = e / torch.where(L > 0, L, torch.ones_like(L))
    am = a if mask is None else a * mask.double()
    s = torch.einsum('ps,psc->pc', am, K)
    return dict(qk=qk, img=img, K=K, a=a, am=am, s=s, rho=am.sum(1), cnt=valid.sum(1).int(), valid=valid)


def _i2p_scales(r, ds, drho, mask=None):
    """Term magnitudes: forward sum_j a_j m_j |k_j|; dqk sum_j a_j (|m_j (t_j + drho)| + |D|) |k_j| with t_j = ds . k_j."""
    K, a, am = r['K'].detach(), r['a'].detach(), r['am'].detach()
    tv = torch.einsum('pc,psc->ps', ds, K) + drho[:, None]
    if mask is not None:
        tv = tv * mask.double()
    D = (a * tv).sum(1, keepdim=True)
    fwd = torch.einsum('ps,psc->pc', am.abs(), K.abs())
    bwd = torch.einsum('ps,psc->pc', a * (tv.abs() + D.abs()), K.abs())
    return fwd, bwd


def _to(cs, d):
    """The case's tensors on the device (held here: the C entry points get raw pointers)."""
    return {k: v.to(d) if torch.is_tensor(v) else v for k, v in cs.items()}


def _i2p_args(g):
    return [_p(g[k]) for k in ('qk', 'pillars', 'npts', 'coors', 'proj', 'img')]


TV_CASES = [(1, 1), (31, 1), (11, 3), (64, 4)]           # T*V = 1, 31, 33, 256 keys per pillar (256: all 8 ballot slices)


@pytest.mark.parametrize('TV', TV_CASES, ids=lambda tv: 'T%dV%d' % tv)
@pytest.mark.parametrize('C', [64, 128, 192, 256, 320, 512])
def test_i2p_attend_fwd_bwd_matches_float64(C, TV):
    ops = _ops()
    d = dev()
    T, V = TV
    cs = _i2p_case(C, T, V, seed=C * 7 + T)
    P, B, pdim = cs['qk'].shape[0], cs['B'], cs['pillars'].shape[2]
    r = _i2p_ref(cs)
    ds = cs['ds'][:, :C].contiguous()
    fs, bs = _i2p_scales(r, ds.double(), torch.zeros(P, dtype=torch.float64))
    n_live = P - 7
    assert int((r['cnt'] == 0).sum()) >= 3 * B and int((r['cnt'] > 0).sum()) >= 8
    g = _to(cs, d)
    ds_d = ds.to(d)
    n_dev = torch.tensor([n_live], dtype=torch.int32, device=d)

    # forward through the wrapper
    s, cnt = ops.i2p_attend(g['qk'], g['pillars'], g['npts'], g['coors'], g['proj'], g['img'], V, (H_IN, W_IN))
    e_row, e_glob = row_err(s, r['s'], fs), rel_err(s.cpu().double(), r['s'].detach())
    print(f'i2p_attend C={C} T={T} V={V}: P={P}, row {e_row:.2e} global {e_glob:.2e}')
    assert torch.equal(cnt.cpu(), r['cnt'])
    assert bool((s.cpu()[r['cnt'] == 0] == 0).all())
    assert e_row < TOL and e_glob < TOL

    # forward with a live count below the capacity: rows past it keep the sentinel bit for bit
    s2 = torch.full((P, C), SENT, device=d)
    cnt2 = torch.full((P,), -3, dtype=torch.int32, device=d)
    _capi('di_i2p_attend_f32', *_i2p_args(g), _p(s2), _p(cnt2), P, T, pdim, V, H_F, W_F, C, H_IN, W_IN, _p(n_dev))
    assert same_bits(s2[:n_live], s[:n_live]) and torch.equal(cnt2[:n_live].cpu(), r['cnt'][:n_live])
    assert bool((s2[n_live:] == SENT).all()) and bool((cnt2[n_live:] == -3).all())

    # backward (the C entry point: the wrapper passes no live count): dqk written, d_img pre-filled and accumulated into
    grads = torch.autograd.grad(r['s'], (r['qk'], r['img']), ds.double(), retain_graph=True)
    a = _i2p_args(g)
    dqk = torch.full((P, C), SENT, device=d)
    d_img = cs['d_img0'].to(d)
    _capi('di_i2p_attend_bwd_f32', a[0], _p(ds_d), *a[1:], _p(d_img), _p(dqk), P, T, pdim, V, H_F, W_F, C, H_IN, W_IN,
          None)
    want_img = cs['d_img0'].double() + grads[1]
    e_q, e_qg = row_err(dqk, grads[0], bs), rel_err(dqk.cpu().double(), grads[0])
    e_i, e_ig = row_err(d_img, want_img, torch.zeros(1)), rel_err(d_img.cpu().double(), want_img)
    print(f'i2p_attend_bwd: dqk row {e_q:.2e} global {e_qg:.2e}; d_img row {e_i:.2e} global {e_ig:.2e}')
    assert e_q < TOL and e_qg < TOL and e_i < TOL and e_ig < TOL
    assert bool((dqk.cpu()[r['cnt'] == 0] == 0).all())
    untouched = grads[1].abs().amax(-1) == 0                                      # pixels no valid key reaches
    assert same_bits(d_img.cpu()[untouched], cs['d_img0'][untouched])

    # backward with the live count: dqk rows past it keep the sentinel, d_img gets the live pillars only
    ds_live = ds.double().clone()
    ds_live[n_live:] = 0
    g_live = torch.autograd.grad(r['s'], r['img'], ds_live)[0]
    dqk = torch.full((P, C), SENT, device=d)
    d_img = cs['d_img0'].to(d)
    _capi('di_i2p_attend_bwd_f32', a[0], _p(ds_d), *a[1:], _p(d_img), _p(dqk), P, T, pdim, V, H_F, W_F, C, H_IN, W_IN,
          _p(n_dev))
    want_img = cs['d_img0'].double() + g_live
    assert bool((dqk[n_live:] == SENT).all())
    assert row_err(dqk[:n_live], grads[0][:n_live], bs[:n_live]) < TOL
    assert row_err(d_img, want_img, torch.zeros(1)) < TOL and rel_err(d_img.cpu().double(), want_img) < TOL


@pytest.mark.parametrize('TV', [(11, 3), (64, 4)], ids=lambda tv: 'T%dV%d' % tv)
@pytest.mark.parametrize('C', [64, 128, 192, 256, 320, 512])
def test_i2p_attend_dropout_fwd_bwd_matches_float64(C, TV):
    ops = _ops()
    d = dev()
    T, V = TV
    pdrop, seed = 0.3, 977 + C
    cs = _i2p_case(C, T, V, seed=C * 5 + T + 1)
    P = cs['qk'].shape[0]
    mask = ops.i2p_dropout_mask(P, T * V, pdrop, seed, d).cpu()                  # key layout t*V + v
    vals = mask.unique().tolist()
    assert len(vals) == 2 and vals[0] == 0.0 and abs(vals[1] - 1 / (1 - pdrop)) < 1e-6
    r = _i2p_ref(cs, mask)
    ds, drho = cs['ds'], cs['ds'][:, C]
    fs, bs = _i2p_scales(r, ds[:, :C].double(), drho.double(), mask)
    g = _to(cs, d)
    args = (g['qk'], g['pillars'], g['npts'], g['coors'], g['proj'], g['img'], V, (H_IN, W_IN))
    s, cnt = ops.i2p_attend(*args, dropout=(pdrop, seed))
    s = s.cpu()
    e_s, e_rho = row_err(s[:, :C], r['s'], fs), row_err(s[:, C:C + 1], r['rho'][:, None], r['rho'][:, None])
    print(f'i2p_attend dropout C={C} T={T} V={V}: s row {e_s:.2e}, rho {e_rho:.2e}')
    assert torch.equal(cnt.cpu(), r['cnt'])
    assert e_s < TOL and e_rho < TOL and rel_err(s[:, :C].double(), r['s'].detach()) < TOL
    assert bool((s[:, C + 1:] == 0).all())

    # backward through autograd of the same masked function: loss = sum(ds[:, :C] * s) + sum(ds[:, C] * rho)
    out = torch.cat([r['s'], r['rho'][:, None]], 1)
    g_qk, g_img = torch.autograd.grad(out, (r['qk'], r['img']), ds[:, :C + 1].double())
    d_img = cs['d_img0'].to(d)
    dqk = ops.i2p_attend_bwd(g['qk'], g['ds'], g['pillars'], g['npts'], g['coors'], g['proj'], g['img'], d_img, V,
                             (H_IN, W_IN), dropout=(pdrop, seed))
    want_img = cs['d_img0'].double() + g_img
    e_q, e_i = row_err(dqk, g_qk, bs), row_err(d_img, want_img, torch.zeros(1))
    print(f'i2p_attend_bwd dropout: dqk row {e_q:.2e}, d_img row {e_i:.2e}')
    assert e_q < TOL and e_i < TOL
    assert rel_err(dqk.cpu().double(), g_qk) < TOL and rel_err(d_img.cpu().double(), want_img) < TOL

    # the wrapper's rows past the live count feed a dense layer: zero, with and without dropout
    n_live = P - 5
    n_dev = torch.tensor([n_live], dtype=torch.int32, device=d)
    for drop in (None, (pdrop, seed)):
        s3, _ = ops.i2p_attend(*args, n_dev=n_dev, dropout=drop)
        ref = s if drop else ops.i2p_attend(*args)[0].cpu()
        assert same_bits(s3[:n_live], ref[:n_live]) and bool((s3[n_live:] == 0).all()), drop


def test_i2p_attend_empty_and_single_key_rows():
    """T*V = 1: every pillar has at most one key, so s is that key's sample (or 0) and dqk is exactly 0."""
    ops = _ops()
    d = dev()
    cs = _i2p_case(260, 1, 1, seed=5)
    r = _i2p_ref(cs)
    g = _to(cs, d)
    s, cnt = ops.i2p_attend(g['qk'], g['pillars'], g['npts'], g['coors'], g['proj'], g['img'], 1, (H_IN, W_IN))
    assert torch.equal(cnt.cpu(), r['cnt']) and int(cnt.max()) == 1
    k0 = r['K'][:, 0].detach()
    assert row_err(s, k0 * r['valid'][:, :1], k0.abs()) < TOL
    d_img = torch.zeros_like(g['img'])
    dqk = ops.i2p_attend_bwd(g['qk'], g['ds'][:, :260].contiguous(), g['pillars'], g['npts'], g['coors'], g['proj'],
                             g['img'], d_img, 1, (H_IN, W_IN))
    assert bool((dqk == 0).all())


# ---------------------------------------------------------------------------------------------------------------------
# 3. lift_grid
# ---------------------------------------------------------------------------------------------------------------------
def _img2lidar(n_img, H_in, W_in):
    """[n_img, 4, 4] inverse lidar2img of forward-looking pinhole cameras at different yaws, rounded to fp32."""
    out = []
    for i in range(n_img):
        yaw = 0.3 + 1.7 * i
        c, s = math.cos(yaw), math.sin(yaw)
        Rz = torch.tensor([[c, -s, 0], [s, c, 0], [0, 0, 1]], dtype=torch.float64)
        axes = torch.tensor([[0, -1, 0], [0, 0, -1], [1, 0, 0]], dtype=torch.float64)   # lidar -> camera axes
        R = axes @ Rz.t()
        pos = torch.tensor([0.7 * c, 0.7 * s, 1.6], dtype=torch.float64)
        K = torch.tensor([[0.8 * W_in, 0, W_in / 2], [0, 0.8 * W_in, H_in / 2], [0, 0, 1]], dtype=torch.float64)
        l2i = torch.eye(4, dtype=torch.float64)
        l2i[:3, :3], l2i[:3, 3] = K @ R, -(K @ R @ pos)
        out.append(torch.inverse(l2i))
    m = torch.stack(out).float().double()
    m[:, 3] = torch.tensor([0, 0, 0, 1.0])
    return m


@pytest.mark.parametrize('w', [1, 2, 63, 64, 176])
@pytest.mark.parametrize('h', [1, 2, 63, 64, 176])
def test_lift_grid_matches_oracle_lift_pixels(h, w):
    import oracle.mmri as om
    ops = _ops()
    gen = torch.Generator().manual_seed(h * 1000 + w)
    n_img, (H_in, W_in), (Yb, Xb) = 2, (256, 704), (180, 200)
    lo, hi = torch.tensor(om.PC_RANGE[:3], dtype=torch.float64), torch.tensor(om.PC_RANGE[3:], dtype=torch.float64)
    i2l = _img2lidar(n_img, H_in, W_in)
    near_cam = torch.rand(n_img, h, w, generator=gen) < 0.3                      # short depths: inside at every row
    depth = torch.where(near_cam, torch.rand(n_img, h, w, generator=gen) * 5, torch.rand(n_img, h, w, generator=gen) * 90)
    depth = (depth + 0.5).float()
    for _ in range(20):                     # keep every point clear of the pc_range faces (fp32 vs float64 rounding)
        _, _, xyz = om.lift_pixels(depth.double(), i2l, (H_in, W_in), {})
        near = (torch.minimum((xyz - lo).abs(), (xyz - hi).abs()) < 1e-2).any(-1)
        if not bool(near.any()):
            break
        depth = torch.where(near, depth * 1.037, depth)
    assert not bool(near.any())
    g, mask, xyz = om.lift_pixels(depth.double(), i2l, (H_in, W_in), {})
    want = torch.stack([((g[..., 0] + 1) * Xb - 1) / 2, ((g[..., 1] + 1) * Yb - 1) / 2], -1)
    got = ops.lift_grid(depth.to(dev()), i2l[:, :3].float().reshape(n_img, 12).contiguous().to(dev()), (H_in, W_in),
                        (Yb, Xb), om.PC_RANGE).cpu()
    assert bool((got[~mask] == -1e30).all()), 'points outside pc_range must get exactly -1e30'
    assert bool((got[mask] > -1).all())
    # fp32 rounding of the coordinates: the sum of |M_ij X_j| terms in metres, scaled to BEV pixels, plus the
    # un-normalisation's own rounding
    xs = torch.linspace(0, W_in - 1, w, dtype=torch.float32).double().view(1, 1, w)
    ys = torch.linspace(0, H_in - 1, h, dtype=torch.float32).double().view(1, h, 1)
    d64 = depth.double()
    terms = torch.stack([(xs * d64).expand(n_img, h, w), (ys * d64).expand(n_img, h, w), d64, torch.ones_like(d64)], -1)
    mag = torch.einsum('nij,nhwj->nhwi', i2l[:, :2].abs(), terms.abs())
    px = torch.tensor([Xb, Yb], dtype=torch.float64) / (hi[:2] - lo[:2])
    tol = 8 * U * (mag * px + torch.tensor([Xb, Yb], dtype=torch.float64) + 1)
    err = (got.double() - want).abs()
    print(f'lift_grid h={h} w={w}: {int(mask.sum())} of {mask.numel()} valid, max err {float(err[mask].max()) if mask.any() else 0:.2e} px')
    assert int(mask.sum()) > 0 and int((~mask).sum()) > 0 or h * w <= 2
    assert bool((err[mask] <= tol[mask]).all())


# ---------------------------------------------------------------------------------------------------------------------
# 4. msdeform
# ---------------------------------------------------------------------------------------------------------------------
MSD_SHAPES = [[(8, 16)], [(1, 1)], [(13, 21)], [(4, 8), (8, 16)], [(1, 1), (4, 8)], [(13, 21), (7, 11)]]


def _msd_offsets(B, nq, hq, wq, shapes, gen, heads=8, P=4):
    """Offsets [B, nq, heads, L, P, 2] in level pixels (location = reference + offset / (W_l, H_l)) of several kinds:
    random +-3 px, exactly on a pixel centre, exactly on the zero-padding border x or y = -0.5 or W_l - 0.5, both, and
    +-1e4 px.  Offsets are dyadic and the query grid is a power of two, so on power-of-two levels every location is
    exact in fp32.  On other levels offset / W_l rounds; random samples are kept 2^-8 px clear of the pixel grid lines
    there, where a corner weight near 0 would carry that rounding as a large relative error."""
    L = len(shapes)
    qi = torch.arange(nq)
    refx = ((qi % wq).double() + 0.5) / wq
    refy = ((qi // wq).double() + 0.5) / hq
    off = torch.zeros(B, nq, heads, L, P, 2, dtype=torch.float64)
    for l, (H, W) in enumerate(shapes):
        kind = torch.randint(0, 7, (B, nq, heads, P), generator=gen)
        rx, ry = refx.view(1, nq, 1, 1) * W, refy.view(1, nq, 1, 1) * H
        cx = torch.randint(0, W, kind.shape, generator=gen).double() + 0.5 - rx      # pixel centres
        cy = torch.randint(0, H, kind.shape, generator=gen).double() + 0.5 - ry
        side = torch.randint(0, 2, kind.shape, generator=gen).double()
        bx, by = side * W - rx, (1 - side) * H - ry                                 # x or y = -0.5 / size - 0.5
        far = (torch.randint(0, 2, kind.shape, generator=gen).double() * 2 - 1) * 1e4
        rnd = torch.round(torch.randn(B, nq, heads, P, 2, generator=gen, dtype=torch.float64) * 3 * 1024) / 1024
        for i, r0 in ((0, rx), (1, ry)):
            c = r0 + rnd[..., i] - 0.5                                               # pixel coordinate
            near = (c - torch.round(c)).abs() < 2.0 ** -8
            rnd[..., i] = torch.where(near, rnd[..., i] + 2.0 ** -7, rnd[..., i])
        ox = torch.stack([rnd[..., 0], cx, bx, cx, bx, far, cx], 0).gather(0, kind[None]).squeeze(0)
        oy = torch.stack([rnd[..., 1], cy, cy, by, by, cy, far], 0).gather(0, kind[None]).squeeze(0)
        off[:, :, :, l, :, 0], off[:, :, :, l, :, 1] = ox, oy
    return off.float()


@pytest.mark.parametrize('B', [1, 3])
@pytest.mark.parametrize('shapes', MSD_SHAPES, ids=lambda s: 'x'.join('%d_%d' % hw for hw in s))
def test_msdeform_matches_oracle_core(shapes, B):
    import oracle.mmri_pp as opp
    ops = _ops()
    d = dev()
    L, heads, dh, P, hq, wq = len(shapes), 8, 16, 4, 4, 8
    nq = hq * wq
    gen = torch.Generator().manual_seed(31 * B + sum(h * w for h, w in shapes))
    value = [torch.randn(B, h, w, heads * dh, generator=gen) for h, w in shapes]
    off = _msd_offsets(B, nq, hq, wq, shapes, gen)
    logit = torch.randn(B, nq, heads, L * P, generator=gen)
    # spreads of ~80 around +60 (exp overflows without the max subtraction); multiples of 2^-8, so logit - max is exact
    wide = torch.rand(B, nq, heads, 1, generator=gen) < 0.5
    spread = torch.round((torch.rand(B, nq, heads, L * P, generator=gen) * 80 - 40) * 256) / 256
    logit = torch.where(wide, 60 + spread, logit)
    norm = torch.tensor([[w, h] for h, w in shapes], dtype=torch.float64)
    ref_pts = opp.reference_points(hq, wq).double().unsqueeze(-2).repeat(1, 1, L, 1)
    loc = ref_pts[:, :, None, :, None, :] + off.double() / norm[None, None, None, :, None, :]
    aw = logit.double().softmax(-1).view(B, nq, heads, L, P)
    flat = lambda vs: torch.cat([v.reshape(B, -1, heads, dh) for v in vs], 1)
    want = opp.ms_deform_attn_core(flat([v.double() for v in value]), shapes, loc, aw)
    scale = opp.ms_deform_attn_core(flat([v.double().abs() for v in value]), shapes, loc, aw)
    width = heads * L * P * 3
    raw = torch.full((B * nq, width + 12), float('nan'))                          # ld_raw > 8*L*P*3, padding never read
    raw[:, :width] = torch.cat([off.reshape(B * nq, -1), logit.reshape(B * nq, -1)], 1)
    raw = raw.to(d)
    vd = [v.to(d) for v in value]
    got = ops.msdeform(vd, raw[:, :width], B, hq, wq).cpu().view(B, nq, -1)
    e_row, e_glob = row_err(got, want, scale, width=dh), rel_err(got.double(), want)
    print(f'msdeform L={L} {shapes} B={B}: row {e_row:.2e} global {e_glob:.2e}')
    assert e_row < TOL and e_glob < TOL
    # output wider than 128 columns: the kernel writes columns 0..127 only
    ldo = 136
    out = torch.full((B * nq, ldo), SENT, device=d)
    sh = (ctypes.c_int * (2 * L))(*[s for hw in shapes for s in hw])
    _capi('di_msdeform_f32', _p(vd[0]), _p(vd[1]) if L > 1 else None, _p(raw), raw.stride(0), _p(out), ldo, B, nq, hq, wq,
          heads, dh, L, P, sh)
    assert same_bits(out[:, :128], got.view(B * nq, 128)) and bool((out[:, 128:] == SENT).all())


# ---------------------------------------------------------------------------------------------------------------------
# 5. row kernels: bit-exact against torch indexing
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('C', [4, 132, 512, 640])
def test_row_gather_scatter_kernels_bit_exact(C):
    """Pillar cells are unique by construction (one pillar per BEV cell), and scatter_rows_add is a plain
    read-modify-write that relies on it: the test uses unique cells only."""
    ops = _ops()
    d = dev()
    gen = torch.Generator().manual_seed(C)
    B, Y, X, P = 2, 7, 9, 40
    cells = torch.randperm(B * Y * X, generator=gen)[:P]
    b, y, x = cells // (Y * X), (cells // X) % Y, cells % X
    coors = torch.stack([b, torch.zeros_like(b), y, x], 1).int().to(d)
    cnt = torch.randint(0, 3, (P,), generator=gen, dtype=torch.int32)
    cnt[:3] = 0
    cnt_d = cnt.to(d)
    on = (cnt > 0)[:, None]
    n_live = P - 9
    n_dev = torch.tensor([n_live], dtype=torch.int32, device=d)
    m = torch.randn(B, Y, X, C, generator=gen)
    md = m.to(d)
    rows_want = m[b, y, x]

    rows = torch.full((P, C), SENT, device=d)
    _capi('di_gather_rows_f32', _p(md), _p(coors), _p(rows), P, Y, X, C, None)
    assert same_bits(rows, rows_want)
    rows = torch.full((P, C), SENT, device=d)
    _capi('di_gather_rows_f32', _p(md), _p(coors), _p(rows), P, Y, X, C, _p(n_dev))
    assert same_bits(rows[:n_live], rows_want[:n_live]) and bool((rows[n_live:] == SENT).all())
    rows = ops.gather_rows(md, coors, n_dev)
    assert same_bits(rows[:n_live], rows_want[:n_live]) and bool((rows[n_live:] == 0).all())
    assert same_bits(ops.gather_rows_masked(md, cnt_d, coors), torch.where(on, rows_want, torch.zeros(())))

    src = torch.randn(P, C, generator=gen)
    base = torch.randn(B, Y, X, C, generator=gen)
    for live in (P, n_live):
        nd = None if live == P else n_dev
        want = base.clone()
        want[b[:live], y[:live], x[:live]] = torch.where(on, src, torch.zeros(()))[:live]
        got = ops.scatter_rows(src.to(d), cnt_d, coors, base.to(d), nd)
        assert same_bits(got, want)
        want = base.clone()
        want[b[:live], y[:live], x[:live]] += torch.where(on, src, torch.zeros(()))[:live]   # fp32 add, as the kernel
        got = ops.scatter_rows_add(src.to(d), cnt_d, coors, base.to(d), nd)
        assert same_bits(got, want)

    # P = 0: nothing to do, and nothing touched
    e_c, e_i = torch.zeros(0, 4, dtype=torch.int32, device=d), torch.zeros(0, dtype=torch.int32, device=d)
    e_r = torch.zeros(0, C, device=d)
    assert ops.gather_rows(md, e_c).shape == (0, C) and ops.gather_rows_masked(md, e_i, e_c).shape == (0, C)
    assert same_bits(ops.scatter_rows(e_r, e_i, e_c, md.clone()), m)
    assert same_bits(ops.scatter_rows_add(e_r, e_i, e_c, md.clone()), m)


def _shift_ref(x, dy, dx):
    N, H, W, C = x.shape
    out = torch.zeros_like(x)
    y0, y1, x0, x1 = max(0, -dy), min(H, H - dy), max(0, -dx), min(W, W - dx)
    if y0 < y1 and x0 < x1:
        out[:, y0:y1, x0:x1] = x[:, y0 + dy:y1 + dy, x0 + dx:x1 + dx]
    return out


@pytest.mark.parametrize('C', [4, 132])
def test_shift_map_bit_exact(C):
    ops = _ops()
    gen = torch.Generator().manual_seed(3 + C)
    N, H, W = 3, 5, 7
    x = torch.randn(N, H, W, C, generator=gen)
    xd = x.to(dev())
    for dy in (-1, 0, 1, H, -H - 2):
        for dx in (-1, 0, 1, W + 3, -W):
            assert same_bits(ops.shift_map(xd, dy, dx), _shift_ref(x, dy, dx)), (dy, dx)


def test_add_rows_mod_and_axpy_bit_exact():
    ops = _ops()
    gen = torch.Generator().manual_seed(11)
    for M, mod, C in ((50, 7, 12), (13, 13, 4), (9, 4, 132)):                    # M not a multiple of mod
        x, pos = torch.randn(M, C, generator=gen), torch.randn(mod, C, generator=gen)
        got = ops.add_rows_mod(x.to(dev()), pos.to(dev()))
        assert same_bits(got, x + pos[torch.arange(M) % mod]), (M, mod, C)
    for n in (4, 4100):
        # dyadic operands with few bits: a + s b is exact in fp32 whether or not the kernel fuses it into an FMA
        a = torch.randint(-512, 512, (n,), generator=gen).float() / 64
        b_ = torch.randint(-512, 512, (n,), generator=gen).float() / 64
        s = torch.tensor([-0.75])
        got = ops.axpy(a.to(dev()), b_.to(dev()), s.to(dev()))
        assert same_bits(got, (a.double() + s.double() * b_.double()).float()), n
