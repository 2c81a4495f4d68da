"""Kernel-level tests of the ++ encoder's polar-ray block (MMRI_I2P_Polar, deepinteraction_b200/polar.py) against float64
references written from the reference's definition (fusion_transformerv4.py:551-638, restated in
oracle/mmri_pp.py::MMRI_I2P_Polar.forward): the ray grid di_polar_grid_f32, the column attention di_seq_attn_f32, the
ray-to-BEV gather di_polar_gather_f32 (csrc/deform.cu), and the block composed.  The CPU-only tests pin the float64
grid and gather references, and polar_consts_host, to the oracle module itself, so the GPU tests compare the kernels
with the reference's formula and not with a restatement of the kernels.

Bars.
* polar grid: per coordinate |got - want| / (|want| + map size of that axis).  The kernel's fp32 chain is about ten
  operations (a 4-term dot product, the subtraction of the camera centre, a sqrt and a division for the ray direction,
  the depth product, the 3-term augmentation row, the normalisation and the scale to pixels).  Each rounds once at
  u = 2^-24 relative to its operands.  The one cancellation, ray point minus camera centre, amplifies by
  sum|terms| / |direction| <= 4 on these rigs.  The other operands are bounded by |coord| + map size, since the
  augmentation's translation and x_min lie inside the map's range.  That gives about 20u = 1.2e-6; GRID_TOL = 4e-6.
* seq_attn: row_err per 16-channel head row, scaled by sum_j A_ij |v_j|: fp32 FFMA over at most 257 keys and 16
  channels, TOL = 1e-5 as for the other FFMA kernels.  The sharp-logit cases (logit spread about 60, so the online
  softmax rescales its running sums many times) use q and k in multiples of 1/4: every logit is exact in fp32, and
  only the exponentials and sums round.
* polar gather: row_err per cell, scaled by (sum over the seeing cameras of the bilinear weights times |ray|) / count
  + |lidar|, TOL = 1e-5.  The radius passes through a sqrt and is never exact, and on the synthetic camera rig the
  projected pixel is not exact either.  So the allowed error adds the fp32 rounding bound of the sample position
  (dgx, dgy, from the magnitudes of the terms that form it) times the bilinear slope there.  The dyadic cases make
  every strict comparison exact in fp32 and float64 alike (power-of-two scales, height-free rows), so the
  visibility masks agree bit for bit.
* block: conftest.rel_err against the oracle module in float64.  The block runs seven dense layers on the bf16-split
  GEMM, whose bar is 1.5e-5 relative to the terms (test_gpu_dense_kernels.py).  Each is followed by a LayerNorm that
  brings the rows back to unit scale, so the errors add at about unit gain: 7 x 1.5e-5 ~ 1e-4.  The two attentions
  (1e-5 each) and the samplings stay below that.  BLOCK_TOL = 1e-4.  The reference inverts lidar2img in fp32 (:555),
  and so does polar_consts_host; the float64 oracle keeps that one step in fp32.
"""
import copy
import ctypes
import math
import os
import sys
import zlib
from types import SimpleNamespace

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from conftest import rel_err
from kernel_check import SENT, _capi, _status, canvas, outside_intact, row_err, same_bits

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
gpu = pytest.mark.gpu

DI_ERR_ARG, DI_ERR_UNSUPPORTED = -1, -3
U = 2.0 ** -24                                      # fp32 unit roundoff
EPS32 = float(torch.tensor(1e-5, dtype=torch.float32))   # the reference compares fp32 depths with 1e-5 (:609-612)
PC = (-54.0, -54.0, -5.0, 54.0, 54.0, 3.0)
TOL = 1e-5
GRID_TOL = 4e-6
BLOCK_TOL = 1e-4
Z = 10                                              # height samples per BEV cell (:591)

# a second augmentation, different from synth.AUG_META in every op: rotation, scale, translation and a vertical flip
AUG_B = dict(pcd_rotation=[[math.cos(-0.45), -math.sin(-0.45), 0.0], [math.sin(-0.45), math.cos(-0.45), 0.0],
                           [0.0, 0.0, 1.0]],
             pcd_scale_factor=0.9, pcd_trans=[-0.4, 0.3, 0.1], pcd_horizontal_flip=False, pcd_vertical_flip=True,
             transformation_3d_flow=['R', 'S', 'T', 'HF', 'VF'])


def dev():
    return torch.device('cuda:0')


def _p(t):
    from deepinteraction_b200 import ops
    return ops._ptr(t)


def _rng6(pc):
    return (ctypes.c_float * 6)(*[float(v) for v in pc])


def _metas(B, V, in_hw, aug):
    """img_metas of B samples on the synthetic V-camera rig; with aug, sample 0 carries synth.AUG_META and sample 1
    AUG_B."""
    from deepinteraction_b200 import synth
    rig = synth.camera_rig(V, in_hw)
    c2l, intr = synth.camera_extras(V, in_hw)
    metas = []
    for b in range(B):
        m = dict(lidar2img=[x.astype(np.float32) for x in rig], cam2lidar=[x.astype(np.float32) for x in c2l],
                 cam_intrinsic=[x.astype(np.float32) for x in intr], input_shape=in_hw)
        if aug:
            m.update(copy.deepcopy((synth.AUG_META, AUG_B)[b % 2]))
        metas.append(m)
    return metas


# ---------------------------------------------------------------------------------------------------------------------
# float64 references
# ---------------------------------------------------------------------------------------------------------------------
def _grid_ref(cam, R, W, h, im_scale, radius_range, pc, Yb, Xb):
    """BEV pixel coordinates [BV, R, W, 2] of the ray queries (:551-579), float64, from the block's camera constants
    cam [BV, 26] (rows 0-1 of inverse(lidar2img), camera centre xy, rows 0-1 of the forward augmentation).
    Pixel (u, v) = ((w + 0.5) * im_scale, (h // 2) * im_scale) is lifted with the inverse to its lidar point, the
    direction from the camera centre is normalised, each depth arange(r0, r1, step) + step / 2 is placed along it at
    z = 0, augmented, normalised to [0, 1] over the range, and mapped through grid_sample's align_corners=False
    un-normalisation ((2n - 1) + 1) * size / 2 - 0.5."""
    c = cam.double().cpu()
    inv, centre, aug = c[:, 0:8].view(-1, 2, 4), c[:, 8:10], c[:, 10:18].view(-1, 2, 4)
    u = (torch.arange(W, dtype=torch.float64) + 0.5) * im_scale
    cam_coors = torch.stack([u, torch.full_like(u, float(h // 2)) * im_scale, torch.ones_like(u), torch.ones_like(u)])
    d = inv @ cam_coors - centre[:, :, None]                                   # [BV, 2, W]
    d = d / d.norm(dim=1, keepdim=True)
    depths = torch.arange(radius_range[0], radius_range[1], radius_range[2], dtype=torch.float64) + radius_range[2] / 2
    assert depths.numel() == R
    xy = depths[None, :, None, None] * d.transpose(1, 2)[:, None]              # [BV, R, W, 2]
    p4 = torch.cat([xy, torch.zeros_like(xy[..., :1]), torch.ones_like(xy[..., :1])], -1)
    a = p4 @ aug.transpose(1, 2)[:, None]                                      # [BV, R, W, 2]
    n = torch.stack([(a[..., 0] - pc[0]) / (pc[3] - pc[0]), (a[..., 1] - pc[1]) / (pc[4] - pc[1])], -1)
    size = torch.tensor([float(Xb), float(Yb)], dtype=torch.float64)
    return ((n * 2 - 1) + 1) * size / 2 - 0.5


def _cell_points(Y, X, pc, device):
    """[Y, X, Z, 4] homogeneous height samples of every cell, indexed explicitly as (iy, ix, iz) (:591-596)."""
    f64 = dict(dtype=torch.float64, device=device)
    px = (torch.arange(X, **f64) + 0.5) / X * (pc[3] - pc[0]) + pc[0]
    py = (torch.arange(Y, **f64) + 0.5) / Y * (pc[4] - pc[1]) + pc[1]
    pz = (torch.arange(Z, **f64) + 0.5) / Z * (pc[5] - pc[2]) + pc[2]
    P = torch.stack(torch.broadcast_tensors(px[None, :, None], py[:, None, None], pz[None, None, :]), -1)
    return torch.cat([P, torch.ones_like(P[..., :1])], -1)


def _cell_magnitudes(Y, X, pc):
    """[4] magnitudes of the terms that form a cell's coordinates ((i + 0.5) / n * range + min, then 1): the fp32
    rounding of a coordinate is relative to these, not to the coordinate, which cancels near the map's centre."""
    return torch.tensor([pc[3] - pc[0] + abs(pc[0]), pc[4] - pc[1] + abs(pc[1]), pc[5] - pc[2] + abs(pc[2]), 1.0],
                        dtype=torch.float64)


def _project(hom, m, in_hw):
    """Per height sample: cz, normalised pixel (nx, ny) and the strict mask of :609-620, float64."""
    xyz = hom @ m.view(3, 4).T
    cz = xyz[..., 2]
    zz = cz.clamp_min(EPS32)
    nx = 2 * (xyz[..., 0] / zz / in_hw[1]) - 1
    ny = 2 * (xyz[..., 1] / zz / in_hw[0]) - 1
    ok = (cz > EPS32) & (nx > -1) & (nx < 1) & (ny > -1) & (ny < 1)
    return xyz, cz, nx, ny, ok


def _bilinear(src, gx, gy):
    """F.grid_sample (float64, bilinear, zero padding, align_corners=False) of src [C, R, W] at pixel coordinates
    gx, gy [Y, X] -> [Y, X, C]."""
    R, W = src.shape[1:]
    loc = torch.stack([(2 * gx + 1) / W - 1, (2 * gy + 1) / R - 1], -1)
    return F.grid_sample(src[None], loc[None], mode='bilinear', padding_mode='zeros', align_corners=False)[0].permute(1, 2, 0)


def _gather_ref(rays, lidar, proj, undo, camc, V, in_hw, pc, r0, r_cnt):
    """di_polar_gather_f32's operation from :586-640, float64, on the kernel's inputs.  Per sample b, camera v and cell:
    the Z height samples are projected with proj[b, v] (lidar2img with the augmentation undone); the cell is seen when
    any sample passes the strict depth / in-image test; the sampling location is the mean over ALL Z samples of the
    normalised pixel x and of the clamped normalised radius (radius from the un-augmented xy, undo[b], to the camera
    centre camc); the ray map is grid-sampled there; the seeing cameras are averaged (count 0 -> 1) and lidar added.

    Returns (out, allowed, count): allowed = TOL * (sum_seen bilinear |ray| / count + |lidar|) + dgx * Sx + dgy * Sy,
    where dgx, dgy bound the fp32 rounding of the sample position (4u of the magnitude of every dot product and the
    relative rounding of each later step) and Sx, Sy are the bilinear slopes there (sum of |ray| at the corner pairs)."""
    B, Y, X, C = lidar.shape
    _, R, W, _ = rays.shape
    hom = _cell_points(Y, X, pc, rays.device)
    mag = torch.maximum(hom.abs(), _cell_magnitudes(Y, X, pc).to(rays.device))
    out = torch.zeros(B, Y, X, C, dtype=torch.float64, device=rays.device)
    scale, slack = torch.zeros_like(out), torch.zeros_like(out)
    count = torch.zeros(B, Y, X, dtype=torch.float64, device=rays.device)
    for b in range(B):
        ua = undo[b].view(3, 4)[:2]
        rxy = hom @ ua.T
        t_r = (mag @ ua.abs().T).sum(-1)
        for v in range(V):
            m = proj[b, v]
            xyz, cz, nx, ny, ok = _project(hom, m, in_hw)
            seen = ok.any(-1)
            r = (rxy - camc[b * V + v]).norm(dim=-1)
            nr = (2 * (r - r0) / r_cnt - 1).clamp(-1, 1)
            sx, sr = nx.mean(-1), nr.mean(-1)
            gx, gy = (sx + 1) / 2 * W - 0.5, (sr + 1) / 2 * R - 0.5
            src = rays[b * V + v].permute(2, 0, 1)
            s, a = _bilinear(src, gx, gy), _bilinear(src.abs(), gx, gy)
            # position rounding bound
            t = mag @ m.view(3, 4).abs().T                                   # magnitudes of the dot products
            zz = cz.clamp_min(EPS32)
            pu = xyz[..., 0] / zz
            d_nx = 2 * (4 * U * (t[..., 0] + pu.abs() * t[..., 2]) / zz + 2 * U * pu.abs()) / in_hw[1] + 2 * U
            d_gx = W / 2 * (d_nx.mean(-1) + 6 * U * nx.abs().mean(-1)) + U * W
            d_r = 4 * U * (t_r + camc[b * V + v].abs().sum()) + 4 * U * r
            d_nr = 2 * d_r / r_cnt + 4 * U * (nr.abs() + 1)
            d_gy = R / 2 * (d_nr.mean(-1) + 6 * U * nr.abs().mean(-1)) + U * R
            fx, fy = gx.floor(), gy.floor()
            s_x = _bilinear(src.abs(), fx, gy) + _bilinear(src.abs(), fx + 1, gy)
            s_y = _bilinear(src.abs(), gx, fy) + _bilinear(src.abs(), gx, fy + 1)
            w = seen[..., None].double()
            out[b] += s * w
            scale[b] += a * w
            slack[b] += (d_gx[..., None] * s_x + d_gy[..., None] * s_y) * w
            count[b] += seen.double()
    n = count.clamp_min(1)[..., None]
    return out / n + lidar, TOL * (scale / n + lidar.abs()) + slack / n, count


def _well_posed(proj, in_hw, pc, Y, X):
    """True when no height sample of any camera lies near a strict border: the normalised pixel (nx, ny) of every
    sample in front of the camera is at least 1e-5 from -1 and 1, and every depth cz is at least 64u of the magnitude of
    its terms from eps (16 times its fp32 rounding bound).  Then fp32 and float64 agree on every mask."""
    hom = _cell_points(Y, X, pc, proj.device)
    pix, depth = float('inf'), float('inf')
    for b in range(proj.shape[0]):
        for v in range(proj.shape[1]):
            m = proj[b, v].double()
            _, cz, nx, ny, _ = _project(hom, m, in_hw)
            tz = hom.abs() @ m.view(3, 4)[2].abs()
            front = cz > EPS32 + 64 * U * tz
            d = torch.stack([(nx - 1).abs(), (nx + 1).abs(), (ny - 1).abs(), (ny + 1).abs()], -1).amin(-1)[front]
            pix = min(pix, float(d.min()) if d.numel() else pix)
            depth = min(depth, float(((cz - EPS32).abs() / tz).min()))
    print(f'strict borders: pixel margin {pix:.2e}, depth margin {depth / U:.0f}u of its terms')
    return pix > 1e-5 and depth > 64 * U


# ---------------------------------------------------------------------------------------------------------------------
# CPU: the references and polar_consts_host against the oracle module
# ---------------------------------------------------------------------------------------------------------------------
class _RecordGridSample:
    """Stand-in for torch.nn.functional inside oracle.mmri_pp that records every grid_sample call (input, grid)."""

    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        return getattr(F, name)

    def grid_sample(self, inp, grid, **kw):
        self.calls.append((inp, grid))
        return F.grid_sample(inp, grid, **kw)


@pytest.fixture(scope='module')
def oracle_run():
    """The oracle MMRI_I2P_Polar in float64 on an augmented two-sample, three-camera frame (36 x 36 BEV, 28 x 50 image
    features); its grid_sample calls are recorded: per camera the ray-query grid, then (decoded rays, gather grid)."""
    import oracle.mmri_pp as opp
    B, V, h, w, Y, X, C = 2, 3, 28, 50, 36, 36, 128
    metas = _metas(B, V, (4 * h, 4 * w), True)
    g = torch.Generator().manual_seed(77)
    lidar = torch.randn(B, C, Y, X, generator=g, dtype=torch.float64)
    img = torch.randn(B * V, C, h, w, generator=g, dtype=torch.float64)
    torch.manual_seed(77)
    blk = opp.MMRI_I2P_Polar(C, 0.1).double().eval()
    rec, saved, prev = _RecordGridSample(), opp.F, torch.get_default_dtype()
    opp.F = rec
    torch.set_default_dtype(torch.float64)
    try:
        with torch.no_grad():
            out = blk(lidar, img, metas, None)
    finally:
        opp.F = saved
        torch.set_default_dtype(prev)
    assert len(rec.calls) == 2 * V
    return dict(metas=metas, lidar=lidar, out=out, calls=rec.calls, B=B, V=V, h=h, w=w, Y=Y, X=X, R=blk.radius,
                radius_range=blk.radius_range, pc=blk.pc_range)


def test_polar_consts_host_match_oracle_geometry(oracle_run):
    """cam = rows 0-1 of the inverse of lidar2img, the camera centre (cam2lidar[:2, 3]) and rows 0-1 of the forward
    augmentation; undo = rows 0-2 of the reverse augmentation; camc = the centre -- as the oracle applies them."""
    from deepinteraction_b200 import geom, polar
    from oracle.geometry import affine_of_transformation
    metas, B, V = oracle_run['metas'], oracle_run['B'], oracle_run['V']
    cam, undo, camc = polar.polar_consts_host(metas)
    l2i = torch.from_numpy(geom.lidar2img_array(metas)).double()
    inv64 = torch.linalg.inv(l2i)[:, :, :2].reshape(B * V, 8)
    e_inv = row_err(cam[:, 0:8], inv64, inv64.abs(), width=4)
    print(f'img2lidar rows: fp32 inverse vs float64 {e_inv:.2e}')
    assert e_inv < 1e-5
    c2l = torch.tensor(np.asarray([m['cam2lidar'] for m in metas]), dtype=torch.float32)
    assert torch.equal(cam[:, 8:10], c2l[:, :, :2, 3].reshape(B * V, 2))
    assert torch.equal(camc, cam[:, 8:10])
    for b, meta in enumerate(metas):
        fwd, rev = affine_of_transformation(meta, False), affine_of_transformation(meta, True)
        for v in range(V):
            assert torch.allclose(cam[b * V + v, 10:18].double(), fwd[:2].reshape(8), rtol=0, atol=2 * U * 4)
        assert torch.allclose(undo[b].double(), rev[:3].reshape(12), rtol=0, atol=2 * U * 4)


def test_grid_reference_matches_oracle_ray_grid(oracle_run):
    """_grid_ref on polar_consts_host's constants equals the oracle's norm_xy * size - 0.5, camera by camera."""
    from deepinteraction_b200 import polar
    o = oracle_run
    cam, _, _ = polar.polar_consts_host(o['metas'])
    want = _grid_ref(cam, o['R'], o['w'], o['h'], 4.0, o['radius_range'], o['pc'], o['Y'], o['X'])
    size = torch.tensor([float(o['X']), float(o['Y'])], dtype=torch.float64)
    worst = 0.0
    for v in range(o['V']):
        inp, grid = o['calls'][2 * v]
        assert inp is o['lidar'] and grid.shape == (o['B'], o['R'], o['w'], 2)
        pix = (grid + 1) / 2 * size - 0.5
        for b in range(o['B']):
            worst = max(worst, float(((want[b * o['V'] + v] - pix[b]).abs() / (pix[b].abs() + size)).max()))
    print(f'ray grid: reference vs oracle {worst:.2e}')
    assert worst < 1e-5        # the fp32 inverse and augmentation rows of the constants, ~1e-7 of the terms


def test_gather_reference_matches_oracle(oracle_run):
    """_gather_ref on the oracle's own decoded rays and the folded camera rows equals the oracle's block output."""
    from deepinteraction_b200 import geom, polar
    o = oracle_run
    B, V = o['B'], o['V']
    rays = torch.stack([o['calls'][2 * v + 1][0][b].permute(1, 2, 0) for b in range(B) for v in range(V)])
    proj, _ = geom.camera_rows_host(o['metas'])
    _, undo, camc = polar.polar_consts_host(o['metas'])
    lidar = o['lidar'].permute(0, 2, 3, 1)
    in_hw = geom.input_hw(o['metas'])
    assert _well_posed(proj, in_hw, o['pc'], o['Y'], o['X'])
    want, _, count = _gather_ref(rays, lidar, proj.double(), undo.double(), camc.double(), V, in_hw, o['pc'],
                                 o['radius_range'][0], float(o['R']))
    got = o['out'].permute(0, 2, 3, 1)
    e = row_err(want, got, (want - lidar).abs() + lidar.abs())
    print(f'gather: reference vs oracle {e:.2e}; cells seen by 0/1/2+ cameras:',
          [int((count == k).sum()) for k in (0, 1)], int((count >= 2).sum()))
    assert bool((count == 0).any()) and bool((count == 1).any())
    assert e < 1e-5


# ---------------------------------------------------------------------------------------------------------------------
# 1. di_polar_grid_f32
# ---------------------------------------------------------------------------------------------------------------------
# id: (B, V, R, W, h_feat, (Yb, Xb), radius_range, pc_range, augmented)
GRID_CASES = {
    'config4': (2, 6, 60, 200, 112, (180, 180), (1.0, 61.0, 1.0), PC, False),
    'config4_aug': (2, 6, 60, 200, 112, (180, 180), (1.0, 61.0, 1.0), PC, True),
    'r_step_half': (1, 6, 40, 50, 28, (36, 36), (2.0, 22.0, 0.5), PC, True),
    'y96_x160': (2, 3, 60, 50, 28, (96, 160), (1.0, 61.0, 1.0), (-51.2, -30.0, -5.0, 51.2, 30.0, 3.0), True),
    'tail_273': (1, 3, 7, 13, 9, (40, 24), (1.0, 8.0, 1.0), PC, True),      # 3 * 7 * 13 = 273 threads
}


@gpu
@pytest.mark.parametrize('case', list(GRID_CASES))
def test_polar_grid_matches_float64(case):
    """Every (camera, radius bin, column) of the grid, bins 0 and R-1 and columns 0 and W-1 included; nothing is
    written past the grid."""
    from deepinteraction_b200 import polar
    B, V, R, W, h, (Yb, Xb), rr, pc, aug = GRID_CASES[case]
    cam, _, _ = polar.polar_consts_host(_metas(B, V, (4 * h, 4 * W), aug))
    want = _grid_ref(cam, R, W, h, 4.0, rr, pc, Yb, Xb)
    n = B * V * R * W * 2
    buf = torch.full((n + 67,), SENT, dtype=torch.int32, device=dev())
    cam_d = cam.to(dev())
    _capi('di_polar_grid_f32', _p(cam_d), _p(buf), B * V, R, W, h, 4.0, rr[0], rr[2], _rng6(pc), Yb, Xb)
    assert bool((buf[n:] == SENT).all()), 'written past the grid'
    got = buf[:n].view(torch.float32).view(B * V, R, W, 2).cpu().double()
    size = torch.tensor([float(Xb), float(Yb)], dtype=torch.float64)
    err = (got - want).abs() / (want.abs() + size)
    edge = max(float(err[:, [0, -1]].max()), float(err[:, :, [0, -1]].max()))
    inside = ((want > -0.5) & (want < size - 0.5)).all(-1).float().mean()
    print(f'polar_grid {case}: {float(err.max()):.2e} (edge bins / columns {edge:.2e}); {float(inside):.0%} inside the map')
    assert float(err.max()) < GRID_TOL


# ---------------------------------------------------------------------------------------------------------------------
# 2. di_seq_attn_f32
# ---------------------------------------------------------------------------------------------------------------------
LQ = (1, 31, 32, 33, 60, 64, 65, 97)
LK = (1, 2, 28, 60, 112, 257)
SEQ_CASES = ([(2, 5, lq, lk, 8, False) for lq in LQ for lk in LK]
             + [(2, 5, lq, lk, 8, True) for lq in (33, 97) for lk in (2, 112, 257)]
             + [(1, 5, 33, 60, 1, False), (1, 5, 97, 112, 1, True),          # 5 and 252 warps: not multiples of 8
                (3, 7, 65, 28, 12, False), (3, 7, 33, 257, 12, True)]
             + [(12, 200, 60, lk, 8, sharp) for lk in (60, 112) for sharp in (False, True)])   # the block's two calls


def _seq_id(c):
    G, Wn, Lq, Lk, H, sharp = c
    return f'G{G}_Wn{Wn}_Lq{Lq}_Lk{Lk}_h{H}_' + ('sharp' if sharp else 'flat')


def _seq_ref(q, k, v, G, Wn, Lq, Lk, heads):
    """float64 softmax(q k^T / 4) v per (sequence, head); token t of sequence (g, w) is row (g * L + t) * Wn + w.
    Returns the output and sum_j A_ij |v_j|, both [G * Lq * Wn, heads * 16]."""
    sp = lambda t, L: t.double().reshape(G, L, Wn, heads, 16).permute(0, 2, 3, 1, 4)     # (G, Wn, H, L, 16)
    a = torch.softmax(sp(q, Lq) @ sp(k, Lk).transpose(-1, -2) * 0.25, -1)
    back = lambda t: t.permute(0, 3, 1, 2, 4).reshape(G * Lq * Wn, heads * 16)
    return back(a @ sp(v, Lk)), back(a @ sp(v, Lk).abs())


def check_seq_attn(case):
    """di_seq_attn_f32 against float64 at one (G, Wn, Lq, Lk, heads, sharp) case.  q, k, v are the strided views
    polar.py passes (q, k, v of one [M, 3C] buffer when Lq == Lk as in the self attention; else q from a [Mq, 3C]
    buffer and k, v of a [Mk, 2C] buffer, as the cross attention's kv), the output a view with ldo > C in a sentinel
    canvas; two calls give the same bits; row_err per head row and the global rel_err both stay under TOL.
    (test_gpu_plusplus.py::test_seq_attn_matches_softmax_attention runs it at G = 3, Wn = 7, Lq = 60, Lk = 28.)"""
    G, Wn, Lq, Lk, H, sharp = case
    C = 16 * H
    g = torch.Generator().manual_seed(zlib.crc32(_seq_id(case).encode()))
    Mq, Mk = G * Lq * Wn, G * Lk * Wn
    if Lq == Lk:
        qkv = torch.randn(Mq, 3 * C, generator=g)
        qb, kvb = qkv, qkv[:, C:]
    else:
        qb, kvb = torch.randn(Mq, 3 * C, generator=g), torch.randn(Mk, 2 * C, generator=g)
    if sharp:                  # multiples of 1/4 up to 6: logits exact in fp32, std ~12, spread ~60 over the keys
        qb[:, :C] = torch.randint(-24, 25, (Mq, C), generator=g).float() / 4
        kvb[:, :C] = torch.randint(-24, 25, (Mk, C), generator=g).float() / 4
    qb = qb.to(dev())
    kvb = qb[:, C:] if Lq == Lk else kvb.to(dev())
    q, k, v = qb[:, :C], kvb[:, :C], kvb[:, C:2 * C]
    want, scale = _seq_ref(q, k, v, G, Wn, Lq, Lk, H)
    if sharp:
        logits = (q.double().reshape(G, Lq, Wn, H, 16).permute(0, 2, 3, 1, 4)
                  @ k.double().reshape(G, Lk, Wn, H, 16).permute(0, 2, 3, 4, 1)) * 0.25
        spread = float((logits.amax(-1) - logits.amin(-1)).median())
        assert Lk < 28 or spread > 40, spread
    outs = []
    for _ in range(2):
        buf, out = canvas(Mq, C)
        _capi('di_seq_attn_f32', _p(q), q.stride(0), _p(k), k.stride(0), _p(v), v.stride(0), _p(out), out.stride(0),
              G, Wn, Lq, Lk, H, 16)
        assert outside_intact(buf, Mq, C), 'written outside the output view'
        outs.append(out.clone())
    assert same_bits(outs[0], outs[1])
    got = outs[0]
    assert bool(torch.isfinite(got).all()), 'rows left unwritten'
    e, e_glob = row_err(got, want, scale, width=16), rel_err(got.double(), want)
    print(f'seq_attn {_seq_id(case)}: row {e:.2e} global {e_glob:.2e}')
    assert e < TOL and e_glob < TOL


@gpu
@pytest.mark.parametrize('case', SEQ_CASES, ids=_seq_id)
def test_seq_attn_matches_float64(case):
    check_seq_attn(case)


@gpu
def test_seq_attn_rejects_head_dim_and_misaligned_strides():
    """dim != 16 is DI_ERR_UNSUPPORTED; a leading dimension or a pointer off the 16-byte grid is a bad argument; a
    rejected call writes nothing."""
    G, Wn, L, H, C = 2, 3, 4, 8, 128
    M = G * L * Wn
    qkv = torch.randn(M, 3 * C + 4, device=dev())
    q, k, v = qkv[:, :C], qkv[:, C:2 * C], qkv[:, 2 * C:3 * C]
    buf, out = canvas(M, C)
    ld = qkv.stride(0)
    call = lambda q_, ldq, ldo, dim: _status('di_seq_attn_f32', _p(q_), ldq, _p(k), ld, _p(v), ld, _p(out), ldo,
                                             G, Wn, L, L, H, dim)
    assert call(q, ld, out.stride(0), 8) == DI_ERR_UNSUPPORTED
    assert call(q, ld, out.stride(0), 32) == DI_ERR_UNSUPPORTED
    assert call(q, ld - 2, out.stride(0), 16) == DI_ERR_ARG                     # ldq % 4 != 0
    assert call(q, ld, out.stride(0) - 2, 16) == DI_ERR_ARG                     # ldo % 4 != 0
    assert call(qkv[:, 1:C + 1], ld, out.stride(0), 16) == DI_ERR_ARG           # q 4 bytes off the 16-byte grid
    assert outside_intact(buf, 0, 0), 'a rejected call wrote its output'
    assert call(q, ld, out.stride(0), 16) == 0


# ---------------------------------------------------------------------------------------------------------------------
# 3. di_polar_gather_f32
# ---------------------------------------------------------------------------------------------------------------------
# Dyadic cases: BEV range +-64 m (z from -2 to 6), Y, X powers of two, so cell centres are integers (px = 4 ix - 62 at
# X = 32) and height sample 2 sits at z = 0 exactly; input image 32 x 64, ray maps R = 12 bins x W = 16 columns,
# r0 = 6.  An affine camera (a, b, u0, c, d, v0, cz) projects to u = a px + b py + u0, v = c px + d py + v0 at depth
# cz (a power of two), independent of the height: all ten samples of a cell agree, every product is exact, and the
# borders u = 0, u = 64, v = 0, v = 32 fall on cell centres.
PC_D = (-64.0, -64.0, -2.0, 64.0, 64.0, 6.0)
IN_D, R_D, W_D, R0_D = (32, 64), 12, 16, 6.0
AFFINE = dict(
    A=(1.0, 0.0, 30.0, 0.0, 0.5, 15.0, 1.0),          # u = 0 at ix 8, u = 64 at ix 24; v = 0 at iy 8, v = 32 at iy 24
    B=(-0.5, 0.0, 33.0, 0.0, 0.25, 16.5, 2.0),        # flipped; u = 64 at ix 0, v = 32 at iy 31
    C=(0.0, 1.0, 2.0, -0.5, 0.0, 15.0, 0.5),          # transposed: u from py, v from -px
    D=(0.5, 0.25, 32.0, 0.0, 0.5, 16.0, 1.0),         # sheared
    E=(2.0, 0.0, 60.0, 0.0, -2.0, 20.0, 4.0),         # small window: ix 9..15, iy 15..17
    F=(0.25, 0.25, 32.0, 0.25, -0.25, 16.0, 1.0),     # wide diamond
)
CAMC = dict(A=(2.0, 2.0), B=(-10.0, 6.0), C=(-4.0, 30.0), D=(6.0, -6.0), E=(-22.0, 18.0), F=(14.0, -14.0),
            Z=(0.0, 0.0), S=(0.0, 0.0))


def _affine_row(a, b, u0, c, d, v0, cz, shift):
    """proj rows of an affine camera moved by `shift` metres along x (u0 - a * shift keeps its borders on centres)."""
    return [cz * a, cz * b, 0.0, cz * (u0 - a * shift), cz * c, cz * d, 0.0, cz * (v0 - c * shift), 0.0, 0.0, 0.0, cz]


def _special_row(name):
    """Z: depth = z + eps with the pixel at the image centre: heights 0 and 1 lie behind the camera (their pixel x is
    divided by eps: |nx| ~ 1e5), height 2 sits at depth == eps exactly (rejected), heights 3..9 are in view -- the cell is
    seen, but its mean pixel x lies far outside the ray map.  S: depth = z - 6.8: only heights above the top sample
    (z = 5.6) would be in front; no cell is seen."""
    h, w = IN_D
    if name == 'Z':
        return [0.0, 0.0, w / 2, w / 2 * EPS32, 0.0, 0.0, h / 2, h / 2 * EPS32, 0.0, 0.0, 1.0, EPS32]
    return [0.0, 0.0, w / 2, -w / 2 * 6.8, 0.0, 0.0, h / 2, -h / 2 * 6.8, 0.0, 0.0, 1.0, -6.8]


def _dyadic(names, B):
    """proj [B, V, 12], undo [B, 12] (identity; then a 90-degree turn with a flip and a shift), camc [B*V, 2]; sample 1
    sees the scene moved by one cell."""
    proj = torch.tensor([[_affine_row(*AFFINE[n], shift=4.0 * b) if n in AFFINE else _special_row(n) for n in names]
                         for b in range(B)], dtype=torch.float32)
    undos = ([1.0, 0, 0, 0, 0, 1.0, 0, 0, 0, 0, 1.0, 0], [0, -1.0, 0, 4.0, -1.0, 0, 0, -8.0, 0, 0, 1.0, 0])
    undo = torch.tensor([undos[b % 2] for b in range(B)], dtype=torch.float32)
    camc = torch.tensor([[CAMC[n][0] + 4.0 * b, CAMC[n][1]] for b in range(B) for n in names], dtype=torch.float32)
    return proj, undo, camc


# id: (B, camera names, Y, X)
GATHER_CASES = {
    'b1_v1': (1, 'A', 32, 32),
    'b2_v2': (2, 'AB', 32, 32),
    'b2_v6': (2, 'ABCDEF', 32, 32),
    'b1_v7_depth': (1, 'ABCDEZS', 32, 32),
    'b2_v3_y16_x32': (2, 'ADF', 16, 32),
}


def _run_gather(rays, lidar, proj, undo, camc, V, in_hw, pc, r0, r_cnt):
    from deepinteraction_b200 import ops
    d = lambda t: t.to(dev()).contiguous()
    outs = [ops.polar_gather(d(rays), d(lidar), d(proj), d(undo), d(camc), V, in_hw, pc, r0, r_cnt) for _ in range(2)]
    assert same_bits(outs[0], outs[1])
    return outs[0]


@gpu
@pytest.mark.parametrize('case', list(GATHER_CASES))
def test_polar_gather_matches_float64_dyadic(case):
    B, names, Y, X = GATHER_CASES[case]
    V = len(names)
    proj, undo, camc = _dyadic(names, B)
    g = torch.Generator().manual_seed(sum(map(ord, case)))
    rays = torch.randn(B * V, R_D, W_D, 128, generator=g)
    lidar = torch.randn(B, Y, X, 128, generator=g)
    want, allowed, count = _gather_ref(rays.double().to(dev()), lidar.double().to(dev()), proj.double().to(dev()),
                                       undo.double().to(dev()), camc.double().to(dev()), V, IN_D, PC_D, R0_D, float(R_D))
    got = _run_gather(rays, lidar, proj, undo, camc, V, IN_D, PC_D, R0_D, float(R_D))

    # the cases are built on purpose: check that the data holds them
    hom = _cell_points(Y, X, PC_D, 'cpu')
    on_border, clamped = 0, set()
    for b in range(B):
        for v, n in enumerate(names):
            xyz, cz, nx, ny, ok = _project(hom, proj[b, v].double(), IN_D)
            pix = torch.stack([xyz[..., 0] / cz.clamp_min(EPS32), xyz[..., 1] / cz.clamp_min(EPS32)], -1)
            hit = ((pix[..., 0] == 0) | (pix[..., 0] == IN_D[1]) | (pix[..., 1] == 0) | (pix[..., 1] == IN_D[0])) & (cz > EPS32)
            on_border += int((hit & ~ok.any(-1, keepdim=True)).sum())
            if n == 'Z':
                assert bool((cz[..., 2] == EPS32).all() and (cz[..., :2] < EPS32).all() and (cz[..., 3:] > EPS32).all())
    cnt = count.cpu()
    hist = {k: int((cnt == k).sum()) for k in range(V + 1)}
    print(f'polar_gather {case}: cells seen by k cameras {hist}; samples on a border {on_border}')
    if 'A' in names and Y == X:
        assert on_border > 0
    if 'Z' not in names:
        assert hist[0] > 0 and hist[1] > 0
    if V >= 2 and 'S' not in names:
        assert hist[2] > 0 and hist[V] > 0
    unseen = cnt == 0
    assert same_bits(got.cpu()[unseen], lidar[unseen]), 'a cell no camera sees must return lidar unchanged'
    e = row_err(got, want, allowed / TOL)
    print(f'polar_gather {case}: row {e:.2e}')
    assert e < TOL


def _radius_clamped(B, names, Y, X):
    """Cells whose every height sample lies below r0 or beyond r0 + R of a camera that sees them (clamped radius)."""
    proj, undo, camc = _dyadic(names, B)
    hom = _cell_points(Y, X, PC_D, 'cpu')
    below = above = 0
    for b in range(B):
        rxy = hom @ undo[b].double().view(3, 4)[:2].T
        for v in range(len(names)):
            _, _, _, _, ok = _project(hom, proj[b, v].double(), IN_D)
            r = (rxy - camc[b * len(names) + v].double()).norm(dim=-1)[..., 0]
            seen = ok.any(-1)
            below += int((seen & (r < R0_D)).sum())
            above += int((seen & (r > R0_D + R_D)).sum())
    return below, above


def test_dyadic_gather_cases_clamp_the_radius_both_ways():
    """The dyadic cameras see cells nearer than r0 and farther than r0 + R (the clamp to the border rows)."""
    for case in ('b1_v1', 'b2_v6'):
        B, names, Y, X = GATHER_CASES[case]
        below, above = _radius_clamped(B, names, Y, X)
        assert below > 0 and above > 0, (case, below, above)


@gpu
def test_polar_gather_config4_rig():
    """B = 2, V = 6, R = 60, W = 200, 180 x 180 on the synthetic rig, un-augmented: its 3.9M height samples keep clear
    of every strict border (an augmented rig of this size always has a few within 1e-5; the dyadic cases and the block
    test cover the augmentation).  The projected positions are rounded, which the allowed error holds."""
    from deepinteraction_b200 import geom, polar
    B, V, R, W, Y, X = 2, 6, 60, 200, 180, 180
    metas = _metas(B, V, (448, 800), False)
    proj, _ = geom.camera_rows_host(metas)
    _, undo, camc = polar.polar_consts_host(metas)
    in_hw = geom.input_hw(metas)
    assert _well_posed(proj.to(dev()), in_hw, PC, Y, X)
    g = torch.Generator().manual_seed(404)
    rays = torch.randn(B * V, R, W, 128, generator=g)
    lidar = torch.randn(B, Y, X, 128, generator=g)
    want, allowed, count = _gather_ref(rays.double().to(dev()), lidar.double().to(dev()), proj.double().to(dev()),
                                       undo.double().to(dev()), camc.double().to(dev()), V, in_hw, PC, 1.0, float(R))
    got = _run_gather(rays, lidar, proj, undo, camc, V, in_hw, PC, 1.0, float(R))
    hist = {k: int((count == k).sum()) for k in range(V + 1)}
    e = row_err(got, want, allowed / TOL)
    print(f'polar_gather config4: cells seen by k cameras {hist}; row {e:.2e}')
    assert hist[0] > 0 and hist[1] > 0 and hist[2] > 0
    unseen = (count == 0).cpu()
    assert same_bits(got.cpu()[unseen], lidar[unseen])
    assert e < TOL


# ---------------------------------------------------------------------------------------------------------------------
# 4. the block composed
# ---------------------------------------------------------------------------------------------------------------------
_INV = torch.linalg.inv


def _inv32(a):
    return _INV(a.float()).to(a.dtype)


@gpu
@pytest.mark.parametrize('aug', [False, True], ids=['plain', 'augmented'])
def test_polar_block_matches_float64_oracle(aug):
    """polar.polar_forward with the packed weights of a randomised oracle MMRI_I2P_Polar (B = 2, V = 3) against that
    module in float64."""
    import oracle.mmri_pp as opp
    from deepinteraction_b200 import geom, polar
    sys.path.insert(0, os.path.join(ROOT, 'tools'))
    import make_goldens_pp as mgp
    torch.set_grad_enabled(False)
    seed = 2300 + int(aug)
    img_l, pts_l = mgp.pp_layers(True)
    torch.manual_seed(seed)
    o = opp.FusionTransformerv4(2, 2, 16, 24, 128, img_transformerlayers=img_l, pts_transformerlayers=pts_l).eval()
    mgp.randomize_pp(o, seed)
    blk = o.pts_fusion_blocks[0].attentions[1]
    assert isinstance(blk, opp.MMRI_I2P_Polar)
    fr = mgp.pp_frame(seed, aug, views=3, batch=2)
    metas = fr['img_metas']
    B, V, C, Y, X = 2, 3, 128, 36, 36
    h, w = fr['img_levels'][0].shape[-2:]
    g = torch.Generator().manual_seed(seed)
    lidar = torch.randn(B, C, Y, X, generator=g)
    img = torch.randn(B * V, C, h, w, generator=g)
    proj, _ = geom.camera_rows_host(metas)
    in_hw = geom.input_hw(metas)
    assert _well_posed(proj, in_hw, blk.pc_range, Y, X)

    ctx = dict(g=SimpleNamespace(proj=proj.to(dev()), in_hw=in_hw), img_metas=metas)
    ap = polar.pack_polar(blk, dev())
    got = polar.polar_forward(ap, lidar.permute(0, 2, 3, 1).contiguous().to(dev()),
                              img.permute(0, 2, 3, 1).contiguous().to(dev()), ctx).cpu().double()

    o64 = copy.deepcopy(blk).double()
    prev, inv = torch.get_default_dtype(), torch.linalg.inv
    torch.set_default_dtype(torch.float64)
    torch.linalg.inv = _inv32                   # the reference's fp32 inverse of lidar2img (:555)
    try:
        want = o64(lidar.double(), img.double(), metas, None).permute(0, 2, 3, 1)
    finally:
        torch.linalg.inv = inv
        torch.set_default_dtype(prev)
    e, e_dec = rel_err(got, want), rel_err(got - lidar.permute(0, 2, 3, 1).double(), want - lidar.permute(0, 2, 3, 1).double())
    print(f'polar block aug={aug}: rel_err {e:.2e} (decorated part alone {e_dec:.2e}); bar {BLOCK_TOL:.0e}')
    assert e < BLOCK_TOL
