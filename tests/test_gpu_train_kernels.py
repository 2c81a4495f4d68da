"""Kernel-level tests of the training-side kernels against float64: the window-attention backward and its row kernels
(csrc/lcab_bwd.cu: win_dot, win_gather, win_scatter, win_softmax, win_softmax_bwd, relu_bwd, col_sum, ln_bwd) and
train-mode BatchNorm (csrc/bn_train.cu: bn_stats, bn_apply, bn_bwd).  Each float64 reference is written from the
operation's definition; the window scatter's reference is an explicit transpose of the gather (index_add over every
(pixel, tap) pair), so the two references do not share a mistake.  Outputs go into SENT-filled canvases wider and taller
than the output, and every word outside the output must keep its bits.  U = 2^-24 is the fp32 unit roundoff.

Exact cases.  Window inputs are integers of at most 3 bits times a per-pixel power of two in 2^-2 .. 2^2: every
product and every partial sum then sits on a grid of 2^-4 below 2^24 grid units (at most 121 taps of 784 x 16 units, or
512 channels of 49 x 16), so a correct kernel equals float64 bit for bit in any order and a wrong tap, mask, tail,
channel slice or image boundary fails with no tolerance.  Padding columns of strided inputs hold NaN.  col_sum takes
7-bit integers (70001 x 127 < 2^24).  bn_stats takes 3-bit integers at M = 528 * 2^k, k <= 5, so each block holds 2^k
rows: the block mean has k fractional bits, and every deviation from it, every square and every sum is exact (2^k squares
of at most 14 * 2^k grid units stay below 2^24).  The kernel's mean and var must then be the float64 values rounded to
fp32, within 1 ulp (and 2^-40 of the column's magnitude, for a mean that is exactly 0) -- any error of the Chan merge or
its butterfly shows at once.

Bars derived from the kernels' summation order (first-order bound gamma_d = d U on the magnitude of the summed terms):
  win_dot      each lane chains 4 VEC products, then 5 shuffle adds: d = 4 VEC + 5 (9 at C <= 128, 21 at C = 512),
               row_err scale sum_c |a| |b|.
  win_gather / win_scatter   one FMA chain over the KK taps per channel: d = KK (81 at ks = 9), scale sum_j |w| |b|.
  win_softmax  the scaled logit z (|z| <= zmax of its row) is rounded, its max subtracted and rounded (|z - m| <= 2 zmax):
               4 zmax U on the exponent; expf 2 ulp, the sum <= 9 U, the reciprocal and the product 1 U each: a row's
               error relative to its largest weight is at most (4 zmax + 16) U.
  win_softmax_bwd  the sum of A dA chains <= 4 products per lane and 5 shuffle adds, then a difference and two
               products: 16 U with the scale scale * A (|dA| + sum_j A |dA|).
  col_sum      each block sums ceil(M / min(M, 256)) rows in fp32, the blocks are summed in double: d = rows + 1 on
               sum_m |x|.
  ln_bwd       dbeta is a column sum (as col_sum).  dz and dgamma go through xhat = (z - mean) rstd, whose rounding is
               relative to xs = |xhat| + rstd mean|z| (the row mean sums |z|; on rows whose mean is 500x their spread this
               term dominates).  Mean and variance each chain <= 16 values per lane and 5 shuffle adds (21 U), so
               xhat is within about 36 U of xs, and the sums of dz add as much again: the bar 1e-5 (168 U) on dz with
               the scale rstd (|g dy| + mean|g dy| + xs mean(|g dy| xs)) and on dgamma with sum_m |dy| xs leaves margin
               for the second-order terms.
  BatchNorm    mean, var, z, running mean / var, dy, dgamma and dbeta against float64 F.batch_norm(training=True) and its
               autograd; the bar of each is max(floor, 5 x the error fp32 torch makes on the same input and GPU), the rule of
               test_gpu_backward.py::test_lcab_train_mode_matches_oracle_autograd.  The floors (BN_FLOORS) cover the
               cases where torch is nearly exact.  Every case prints its errors next to torch's.

Kernels that only select (relu_bwd) or move data are held to bit equality; every kernel gives the same bits when repeated,
and the documented in-place calls give the same bits as out-of-place ones.  Null and misaligned pointers are rejected too,
but are not passed here: a missing check would then fault the device instead of failing a test.
"""
import math
import zlib

import pytest
import torch
import torch.nn.functional as F

from kernel_check import SENT, _capi, _status, canvas, outside_intact, record_calls, row_err, same_bits

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
DI_ERR_ARG = -1
EPS = 1e-5


def dev():
    return torch.device('cuda:0')


def _ops():
    from deepinteraction_b200 import ops
    return ops


def _p(t):
    return _ops()._ptr(t)


def _gen(seed):
    return torch.Generator(device='cuda').manual_seed(seed)


def _normal(shape, g):
    return torch.randn(shape, generator=g, device=dev())


def _ints(shape, bits, g):
    m = (1 << bits) - 1
    return torch.randint(-m, m + 1, shape, generator=g, device=dev()).float()


def _pow2(shape, lo, hi, g):
    return torch.exp2(torch.randint(lo, hi + 1, shape, generator=g, device=dev()).float())


def _strided(x, ld):
    """x [P, C] in the first C columns of a NaN-filled [P, ld] buffer -> the view."""
    if ld == x.shape[1]:
        return x.contiguous()
    buf = torch.full((x.shape[0], ld), float('nan'), device=dev())
    buf[:, :x.shape[1]] = x
    return buf[:, :x.shape[1]]


def flat_canvas(n, pad=16):
    """(buffer, view): n words at offset `pad` (16-byte aligned) of a SENT-filled buffer of n + 2 pad words."""
    buf = torch.full((n + 2 * pad,), SENT, dtype=torch.int32, device=dev()).view(torch.float32)
    return buf, buf[pad:pad + n]


def flat_intact(buf, n, pad=16):
    b = buf.view(torch.int32)
    return bool((b[:pad] == SENT).all()) and bool((b[pad + n:] == SENT).all())


def exact(got, want):
    """Bit equality with the float64 result rounded to fp32 (exact here); +0 and -0 count as equal."""
    return same_bits(got.float() + 0.0, want.float() + 0.0)


# ---------------------------------------------------------------------------------------------------------------------
# float64 references of the window ops over pixel-major [N*H*W, C] maps; tap j = (dy + r) * ks + (dx + r)
# ---------------------------------------------------------------------------------------------------------------------
def _taps(ks):
    r = ks // 2
    return [(dy, dx) for dy in range(-r, r + 1) for dx in range(-r, r + 1)]


def _neighbours(pix, N, H, W, ks):
    """[S, KK] flat index of tap j of pixel pix[s] (its own image), and whether it lies inside the map."""
    n, y, x = pix // (H * W), (pix // W) % H, pix % W
    t = torch.tensor(_taps(ks), device=dev())
    yy, xx = y[:, None] + t[:, 0], x[:, None] + t[:, 1]
    ok = (yy >= 0) & (yy < H) & (xx >= 0) & (xx < W)
    return torch.where(ok, (n[:, None] * H + yy) * W + xx, 0), ok


def ref_dot(a, b, N, H, W, ks, pix=None):
    """out[p, j] = a[p] . b[nbr(p, j)], 0 for an out-of-map tap -> (values, term scale sum_c |a||b|, in-map mask)."""
    pix = torch.arange(a.shape[0], device=dev()) if pix is None else pix
    idx, ok = _neighbours(pix, N, H, W, ks)
    A, B = a[pix].double(), b.double()[idx] * ok[..., None]              # [S, C], [S, KK, C]
    return torch.einsum('sc,skc->sk', A, B), torch.einsum('sc,skc->sk', A.abs(), B.abs()), ok


def ref_gather(w, b, N, H, W, ks, pix=None):
    """out[p] = sum over in-map taps j of w[p, j] b[nbr(p, j)] -> (values, term scale)."""
    pix = torch.arange(b.shape[0], device=dev()) if pix is None else pix
    idx, ok = _neighbours(pix, N, H, W, ks)
    Wt, B = w[pix].double() * ok, b.double()[idx]
    return torch.einsum('sk,skc->sc', Wt, B), torch.einsum('sk,skc->sc', Wt.abs(), B.abs())


def ref_scatter(w, b, N, H, W, ks):
    """The transpose of the gather: out[p'] = sum over (p, j) with nbr(p, j) = p' of w[p, j] b[p], accumulated pair by pair
    -> (values, term scale)."""
    P, C = b.shape
    out, scale = torch.zeros(P, C, dtype=torch.float64, device=dev()), torch.zeros(P, C, dtype=torch.float64, device=dev())
    idx, ok = _neighbours(torch.arange(P, device=dev()), N, H, W, ks)
    wd, bd = w.double(), b.double()
    for j in range(ks * ks):
        m = ok[:, j]
        out.index_add_(0, idx[m, j], wd[m, j, None] * bd[m])
        scale.index_add_(0, idx[m, j], (wd[m, j, None] * bd[m]).abs())
    return out, scale


def ref_scatter_at(w, b, N, H, W, ks, pix):
    """The scatter at output pixels pix only: the sources p = p' - off_j that lie in the map."""
    n, y, x = pix // (H * W), (pix // W) % H, pix % W
    t = torch.tensor(_taps(ks), device=dev())
    yy, xx = y[:, None] - t[:, 0], x[:, None] - t[:, 1]
    ok = (yy >= 0) & (yy < H) & (xx >= 0) & (xx < W)
    src = torch.where(ok, (n[:, None] * H + yy) * W + xx, 0)
    j = torch.arange(ks * ks, device=dev()).expand_as(src)
    Wt, B = w.double()[src, j] * ok, b.double()[src]
    return torch.einsum('sk,skc->sc', Wt, B), torch.einsum('sk,skc->sc', Wt.abs(), B.abs())


def _vec(C):
    return 1 if C <= 128 else 2 if C <= 256 else 4


def dot_bar(C):
    return (4 * _vec(C) + 5) * U


def apply_bar(ks):
    return ks * ks * U


def win_dot_c(a, b, out, N, H, W, ks):
    return _capi('di_win_dot_f32', _p(a), a.stride(0), _p(b), b.stride(0), _p(out), N, H, W, a.shape[1], ks)


def win_apply_c(name, w, b, out, N, H, W, ks):
    return _capi(name, _p(w), _p(b), b.stride(0), _p(out), out.stride(0), N, H, W, b.shape[1], ks)


# ---------------------------------------------------------------------------------------------------------------------
# 1. win_dot, win_gather, win_scatter
# ---------------------------------------------------------------------------------------------------------------------
WIN_C = (4, 32, 124, 128, 132, 256, 260, 384, 512)     # VEC 1 / 2 / 4 and partly filled channel slices
WIN_KS = (1, 3, 5, 7, 9, 11)                            # ks = 11: KK = 121, the largest accepted
WIN_W = (1, 2, 3, 4, 5, 6, 7, 8, 13, 200)               # x tails of 0..3 pixels per 4-pixel warp, maps narrower than r
WIN_H = (1, 2, 3, 9)


def _window_cases():
    """(N, H, W, C, ks, pad): every C with every W; ks, H, N and the leading-dimension pad cycle through their values.
    pad = lda - C = ldb - C = ldo - C.  The last cases put maps shorter than r next to each other (N = 3, H < r)."""
    cases = []
    for i, C in enumerate(WIN_C):
        for j, W in enumerate(WIN_W):
            ks, H, N, pad = WIN_KS[(i + j) % 6], WIN_H[(i + 2 * j) % 4], (1, 3)[(i + j) % 2], (0, 4, 12)[(i + j) % 3]
            if W == 200:
                N, H = 1, min(H, 3)
            cases.append((N, H, W, C, ks, pad))
    cases += [(3, 1, 5, 32, 11, 4), (3, 2, 13, 128, 9, 0), (3, 3, 7, 256, 11, 0), (3, 2, 3, 512, 7, 4),
              (3, 4, 6, 384, 11, 8), (2, 9, 200, 132, 9, 4)]
    return cases


WINDOW_CASES = _window_cases()


def _exact_window_inputs(P, C, ks, g):
    a = _ints((P, C), 3, g) * _pow2((P, 1), -2, 2, g)
    b = _ints((P, C), 3, g) * _pow2((P, 1), -2, 2, g)
    w = _ints((P, ks * ks), 3, g) * _pow2((P, 1), -2, 2, g)
    return a, b, w


@pytest.mark.parametrize('N,H,W,C,ks,pad', WINDOW_CASES, ids=lambda v: str(v))
def test_window_kernels_exact(N, H, W, C, ks, pad):
    """win_dot, win_gather and win_scatter equal float64 bit for bit; win_dot's out-of-map taps are +0.0; nothing is
    written outside the outputs; NaN in the padding columns of strided inputs does not leak."""
    P, KK = N * H * W, ks * ks
    g = _gen(zlib.crc32(repr((N, H, W, C, ks, pad)).encode()))
    a, b, w = _exact_window_inputs(P, C, ks, g)
    av, bv = _strided(a, C + pad), _strided(b, C + pad)

    buf, out = flat_canvas(P * KK)
    assert win_dot_c(av, bv, out.view(P, KK), N, H, W, ks) == 0
    want, _, ok = ref_dot(a, b, N, H, W, ks)
    assert flat_intact(buf, P * KK)
    assert exact(out.view(P, KK), want), float((out.view(P, KK).double() - want).abs().max())
    assert bool((out.view(P, KK)[~ok].view(torch.int32) == 0).all()), 'out-of-map taps must be +0.0'

    for name, ref in (('di_win_gather_f32', ref_gather), ('di_win_scatter_f32', ref_scatter)):
        cbuf, o = canvas(P, C, pad_cols=pad)
        assert win_apply_c(name, w, bv, o, N, H, W, ks) == 0
        want, _ = ref(w, b, N, H, W, ks)
        assert outside_intact(cbuf, P, C), name
        assert exact(o, want), (name, float((o.double() - want).abs().max()))


@pytest.mark.parametrize('C', [128, 512])
def test_window_kernels_precision_and_determinism(C):
    """Normal inputs at ks = 9 on maps with x tails of 1..3 pixels: row_err against the term scale within the summation
    bound of each kernel (module docstring); a repeated call gives the same bits."""
    ks = 9
    for N, H, W in ((2, 11, 14), (1, 9, 37), (3, 5, 7)):
        g = _gen(C * 1000 + W)
        P = N * H * W
        a, b = _normal((P, C), g), _normal((P, C), g)
        w = torch.softmax(_normal((P, ks * ks), g) * 2, 1)
        d1 = _ops().win_dot(a, b, N, H, W, ks)
        want, scale, _ = ref_dot(a, b, N, H, W, ks)
        e = row_err(d1, want, scale)
        print(f'win_dot C={C} {N}x{H}x{W}: row err {e:.2e} (bar {dot_bar(C):.2e})')
        assert e < dot_bar(C)
        assert same_bits(d1, _ops().win_dot(a, b, N, H, W, ks))
        for fn, ref in ((_ops().win_gather, ref_gather), (_ops().win_scatter, ref_scatter)):
            o1 = fn(w, b, N, H, W, ks)
            want, scale = ref(w, b, N, H, W, ks)
            e = row_err(o1, want, scale)
            print(f'{fn.__name__} C={C} {N}x{H}x{W}: row err {e:.2e} (bar {apply_bar(ks):.2e})')
            assert e < apply_bar(ks)
            assert same_bits(o1, fn(w, b, N, H, W, ks))


# ---------------------------------------------------------------------------------------------------------------------
# 2. win_softmax, win_softmax_bwd
# ---------------------------------------------------------------------------------------------------------------------
SOFTMAX_KK = (1, 9, 25, 31, 32, 33, 81, 96, 97, 121, 128)   # 1..4 lane slots, full and partly filled
SOFTMAX_P = (1, 7, 9, 134400)                               # 8 rows per block: idle warps in the last block
SM_SCALE = 1.0 / math.sqrt(128.0)


def _logits(P, KK, g):
    """Scaled logits z [P, KK] by row kind: a spread of up to +-80; all equal (at -120 .. 120); one dominant by 80;
    unit normal."""
    kind = torch.arange(P, device=dev()) % 4
    spread = torch.exp(torch.rand((P, 1), generator=g, device=dev()) * math.log(800.0)) / 10.0     # 0.1 .. 80
    z = (torch.rand((P, KK), generator=g, device=dev()) * 2 - 1) * spread
    level = torch.tensor([-120.0, 0.0, 37.5, 120.0], device=dev())[torch.randint(0, 4, (P,), generator=g, device=dev())]
    z = torch.where((kind == 1)[:, None], level[:, None].expand(P, KK), z)
    dom = _normal((P, KK), g)
    dom[torch.arange(P, device=dev()), torch.randint(0, KK, (P,), generator=g, device=dev())] += 80.0
    z = torch.where((kind == 2)[:, None], dom, z)
    return torch.where((kind == 3)[:, None], _normal((P, KK), g), z)


def _sm_scale32():
    return float(torch.tensor(SM_SCALE, dtype=torch.float32))


@pytest.mark.parametrize('P', SOFTMAX_P)
@pytest.mark.parametrize('KK', SOFTMAX_KK)
def test_window_softmax_forward_and_backward(KK, P):
    """Forward: each row within (4 zmax + 16) U of its largest weight; backward: row_err 16 U on the scale
    scale * A (|dA| + sum A |dA|); in-place calls (A == S, dS == dA) give the same bits; nothing outside the output is
    written."""
    g = _gen(KK * 7 + P)
    s32 = _sm_scale32()
    S = (_logits(P, KK, g) / s32).float()
    z = S.double() * s32
    want = torch.softmax(z, 1)
    buf, A = flat_canvas(P * KK)
    A = A.view(P, KK)
    assert _capi('di_win_softmax_f32', _p(S), _p(A), P, KK, SM_SCALE) == 0
    assert flat_intact(buf, P * KK)
    zmax = z.abs().amax(1, keepdim=True)
    err = ((A.double() - want).abs().amax(1, keepdim=True) / want.amax(1, keepdim=True)) / ((4 * zmax + 16) * U)
    e = float(err.max())
    print(f'win_softmax KK={KK} P={P}: worst row error / its bar {e:.2f}')
    assert e < 1.0
    S2 = S.clone()
    assert _capi('di_win_softmax_f32', _p(S2), _p(S2), P, KK, SM_SCALE) == 0
    assert same_bits(S2, A)

    Ain = want.float()
    dA = _normal((P, KK), g) * _pow2((P, 1), -6, 6, g)
    Ad, dAd = Ain.double(), dA.double()
    want_dS = Ad * (dAd - (Ad * dAd).sum(1, keepdim=True)) * s32
    scale = Ad * (dAd.abs() + (Ad * dAd.abs()).sum(1, keepdim=True)) * s32
    buf, dS = flat_canvas(P * KK)
    dS = dS.view(P, KK)
    assert _capi('di_win_softmax_bwd_f32', _p(Ain), _p(dA), _p(dS), P, KK, SM_SCALE) == 0
    assert flat_intact(buf, P * KK)
    e = row_err(dS, want_dS, scale)
    print(f'win_softmax_bwd KK={KK} P={P}: row err {e:.2e} (bar {16 * U:.2e})')
    assert e < 16 * U
    dA2 = dA.clone()
    assert _capi('di_win_softmax_bwd_f32', _p(Ain), _p(dA2), _p(dA2), P, KK, SM_SCALE) == 0
    assert same_bits(dA2, dS)
    dS3 = torch.empty_like(dS)
    assert _capi('di_win_softmax_bwd_f32', _p(Ain), _p(dA), _p(dS3), P, KK, SM_SCALE) == 0
    assert same_bits(dS3, dS)


# ---------------------------------------------------------------------------------------------------------------------
# 3. relu_bwd, col_sum, ln_bwd
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('n', [1, 2, 3, 4, 5, 1023, 4097])
def test_relu_bwd_bits(n):
    """dx = dy where the saved output y > 0, +0.0 elsewhere (y = +0.0, -0.0, negative, NaN-free), bit for bit as torch's
    threshold_backward, out of place and in place (dx == dy), with the words around the output untouched."""
    g = _gen(n)
    y = _normal((n,), g)
    kind = torch.randint(0, 4, (n,), generator=g, device=dev())
    y = torch.where(kind == 0, torch.zeros_like(y), torch.where(kind == 1, -torch.zeros_like(y), y))
    y[:4] = torch.tensor([0.0, -0.0, 1e-45, -1e-45], device=dev())[:min(4, n)]
    dy = _normal((n,), g)
    dy[1::5] = -0.0
    want = torch.ops.aten.threshold_backward(dy, y, 0.0)
    buf, dx = flat_canvas(n, pad=4)
    assert _capi('di_relu_bwd_f32', _p(dy), _p(y), _p(dx), n) == 0
    assert flat_intact(buf, n, pad=4)
    assert same_bits(dx, want)
    assert bool((dx[y <= 0].view(torch.int32) == 0).all()), 'the gradient must be +0.0 where y <= 0'
    d2 = dy.clone()
    assert _capi('di_relu_bwd_f32', _p(d2), _p(y), _p(d2), n) == 0
    assert same_bits(d2, want)


COLSUM_M = (1, 2, 255, 256, 257, 70001)       # M < 256: one row per block; 257: empty trailing blocks
COLSUM_C = (1, 4, 255, 256, 257, 512)         # C > 256: several blockIdx.y


def colsum_bar(M):
    return (-(-M // min(M, 256)) + 1) * U


@pytest.mark.parametrize('C', COLSUM_C)
@pytest.mark.parametrize('M', COLSUM_M)
def test_col_sum(M, C):
    """Integer rows sum exactly; normal rows within (rows per block + 1) U of sum |x|; a strided view (ld > C, NaN in the
    padding) reads only its C columns; repeated calls give the same bits; the words around the output are untouched."""
    g = _gen(M * 600 + C)
    ld = C + (0, 3, 8)[(M + C) % 3]
    work = torch.empty(256 * C, device=dev())
    for kind in ('ints', 'normal'):
        x = _ints((M, C), 7, g) if kind == 'ints' else _normal((M, C), g) * _pow2((1, C), -8, 8, g)
        xv = _strided(x, ld)
        buf, out = flat_canvas(C, pad=4)
        assert _capi('di_col_sum_f32', _p(xv), ld, M, C, _p(work), _p(out)) == 0
        assert flat_intact(buf, C, pad=4)
        want = x.double().sum(0)
        if kind == 'ints':
            assert exact(out, want)
        else:
            e = row_err(out, want, x.double().abs().sum(0), width=1)
            assert e < colsum_bar(M), (e, colsum_bar(M))
        out2 = torch.empty(C, device=dev())
        assert _capi('di_col_sum_f32', _p(xv), ld, M, C, _p(work), _p(out2)) == 0
        assert same_bits(out, out2)


LN_BAR = 1e-5
LN_C = (4, 32, 100, 128, 256, 500, 512)
LN_M = (1, 7, 200, 513)


@pytest.mark.parametrize('M', LN_M)
@pytest.mark.parametrize('C', LN_C)
def test_ln_bwd(C, M):
    """dz, dgamma and dbeta against float64 autograd of F.layer_norm (scales in the module docstring), with strided dy
    and z (NaN in their padding) and a strided dz canvas; rows of mean >> spread."""
    g = _gen(C * 1000 + M)
    z = _normal((M, C), g) * 2
    z[::3] = 500.0 + _normal(((M + 2) // 3, C), g)
    gamma, beta = torch.rand(C, generator=g, device=dev()) + 0.5, _normal((C,), g)
    dy = _normal((M, C), g)
    dyv, zv = _strided(dy, C + 4), _strided(z, C + 8)
    zz, gg, bb = (t.double().requires_grad_(True) for t in (z, gamma, beta))
    with torch.enable_grad():
        F.layer_norm(zz, (C,), gg, bb, EPS).mul(dy.double()).sum().backward()
    cbuf, dz = canvas(M, C, pad_cols=12)
    obuf, dgb = flat_canvas(2 * C, pad=4)
    dg, db = dgb[:C], dgb[C:]
    work = torch.empty(M * C + 256 * C, device=dev())
    assert _capi('di_ln_bwd_f32', _p(dyv), C + 4, _p(zv), C + 8, _p(gamma), _p(dz), C + 12, _p(dg), _p(db), _p(work), M, C,
                 EPS) == 0
    assert outside_intact(cbuf, M, C) and flat_intact(obuf, 2 * C, pad=4)
    zd = z.double()
    mu, var = zd.mean(1, keepdim=True), zd.var(1, unbiased=False, keepdim=True)
    rstd = (var + EPS).rsqrt()
    xh = (zd - mu) * rstd
    gdy = gamma.double() * dy.double()
    xs = xh.abs() + rstd * zd.abs().mean(1, keepdim=True)
    scale = rstd * (gdy.abs() + gdy.abs().mean(1, keepdim=True) + xs * (gdy.abs() * xs).mean(1, keepdim=True))
    e_dz = row_err(dz, zz.grad, scale)
    e_dg = row_err(dg, gg.grad, (dy.double().abs() * xs).sum(0), width=1)
    e_db = row_err(db, bb.grad, dy.double().abs().sum(0), width=1)
    print(f'ln_bwd C={C} M={M}: dz {e_dz:.2e} dgamma {e_dg:.2e} dbeta {e_db:.2e}')
    assert e_dz < LN_BAR and e_dg < LN_BAR and e_db < colsum_bar(M)
    dz2 = torch.empty(M, C, device=dev())
    dgb2 = torch.empty(2 * C, device=dev())
    assert _capi('di_ln_bwd_f32', _p(dyv), C + 4, _p(zv), C + 8, _p(gamma), _p(dz2), C, _p(dgb2), _p(dgb2[C:]), _p(work),
                 M, C, EPS) == 0
    assert same_bits(dz2, dz) and same_bits(dgb2, dgb)


# ---------------------------------------------------------------------------------------------------------------------
# 4. bn_stats, bn_apply, bn_bwd
# ---------------------------------------------------------------------------------------------------------------------
# Floors of the BatchNorm bars (the bar is max(floor, 5 x fp32 torch's error)); metrics: mean |d| / (|mean| + std) and
# var |d| / var per channel; z and dy max |d| per column over that column's max |ref|; running statistics |d| over the
# magnitude of their update, 0.9 |old| + 0.1 (|mean| + std) and 0.9 old + 0.1 var; dgamma and dbeta max |d| / max |ref|.
BN_FLOORS = dict(mean=1e-6, var=4e-6, z=1e-5, run_mean=1e-6, run_var=2e-6, dy=4e-5, dgamma=2e-5, dbeta=2e-5)
BN_BLOCKS = 528


def col_err(got, want, scale=None):
    """max over columns of max|got - want| / max(scale) in that column (scale defaults to |want|; [C] vectors: per
    element).  A column whose scale is zero must match exactly."""
    g, w = got.double().reshape(-1, got.shape[-1]), want.double().reshape(-1, want.shape[-1])
    s = w.abs() if scale is None else torch.broadcast_to(scale.double().abs().reshape(-1, w.shape[-1]), w.shape)
    den, err = s.amax(0), (g - w).abs().amax(0)
    return float(torch.where(den > 0, err / den.clamp_min(1e-300), err * 1e30).max())


def _bn_reference(y, dz, gamma, beta, relu, rm, rv, dtype):
    """torch in `dtype`: mean, var (biased), z, running mean / var after the step, dy, dgamma, dbeta."""
    yr = y.to(dtype).requires_grad_(True)
    gr = None if gamma is None else gamma.to(dtype).requires_grad_(True)
    br = None if beta is None else beta.to(dtype).requires_grad_(True)
    rmr, rvr = rm.to(dtype).clone(), rv.to(dtype).clone()
    with torch.enable_grad():
        z = F.batch_norm(yr, rmr, rvr, gr, br, True, 0.1, EPS)
        if relu:
            z = F.relu(z)
        (z * dz.to(dtype)).sum().backward()
    var, mean = torch.var_mean(y.to(dtype), 0, correction=0)
    return dict(mean=mean, var=var, z=z.detach(), run_mean=rmr, run_var=rvr, dy=yr.grad, rm_old=rm.to(dtype),
                rv_old=rv.to(dtype),
                dgamma=None if gr is None else gr.grad, dbeta=None if br is None else br.grad)


def _bn_kernels(y, dz, gamma, beta, relu, rm, rv):
    ops = _ops()
    rmd, rvd = rm.clone(), rv.clone()
    mean, var = ops.bn_stats(y, rmd, rvd, 0.1)
    z = ops.bn_apply(y, mean, var, gamma, beta, EPS, relu)
    dy, dg, db = ops.bn_bwd(dz, z if relu else None, y, mean, var, gamma, EPS)
    return dict(mean=mean, var=var, z=z, run_mean=rmd, run_var=rvd, dy=dy, dgamma=dg, dbeta=db)


def _bn_errors(got, ref, cols=slice(None)):
    """The metric of each BatchNorm output (BN_FLOORS) over the channels `cols`."""
    std = ref['var'][cols].clamp_min(0).sqrt()
    e = dict(mean=col_err(got['mean'][cols], ref['mean'][cols], ref['mean'][cols].abs() + std),
             var=col_err(got['var'][cols], ref['var'][cols]), z=col_err(got['z'][:, cols], ref['z'][:, cols]),
             run_mean=col_err(got['run_mean'][cols], ref['run_mean'][cols],
                              0.9 * ref['rm_old'][cols].abs() + 0.1 * (ref['mean'][cols].abs() + std)),
             run_var=col_err(got['run_var'][cols], ref['run_var'][cols], 0.9 * ref['rv_old'][cols] + 0.1 * ref['var'][cols]),
             dy=col_err(got['dy'][:, cols], ref['dy'][:, cols]))
    if ref['dgamma'] is not None:
        for k in ('dgamma', 'dbeta'):
            r = ref[k][cols].double()
            e[k] = float((got[k][cols].double() - r).abs().max() / r.abs().max().clamp_min(1e-300))
    return e


def _bn_check(label, y, dz, gamma, beta, relu, rm, rv, groups=None):
    """Kernels vs float64 and fp32 torch vs float64; every output within max(floor, 5 x torch's error), per column group."""
    r64 = _bn_reference(y, dz, gamma, beta, relu, rm, rv, torch.float64)
    r32 = _bn_reference(y, dz, gamma, beta, relu, rm, rv, torch.float32)
    got = _bn_kernels(y, dz, gamma, beta, relu, rm, rv)
    bad = []
    for gname, cols in (groups or {'all': slice(None)}).items():
        e, e32 = _bn_errors(got, r64, cols), _bn_errors(r32, r64, cols)
        print(f'{label} {gname}: ' + ', '.join(f'{k} {e[k]:.1e} (torch {e32[k]:.1e})' for k in e))
        bad += [(gname, k, e[k], e32[k]) for k in e if not e[k] <= max(BN_FLOORS[k], 5 * e32[k])]
    assert not bad, (label, bad)
    return got


def _bn_inputs(M, C, affine, g):
    y = _normal((M, C), g) * (torch.rand(C, generator=g, device=dev()) + 0.2) + _normal((C,), g) * 3
    gamma = (torch.rand(C, generator=g, device=dev()) + 0.5) if affine else None
    beta = _normal((C,), g) * 0.1 if affine else None
    rm, rv = _normal((C,), g) * 0.1, torch.rand(C, generator=g, device=dev()) + 0.5
    return y, gamma, beta, rm, rv, _normal((M, C), g)


def _ulp(x):
    return (torch.nextafter(x, torch.full_like(x, math.inf)) - x).abs()


@pytest.mark.parametrize('k', [0, 1, 3, 5])
@pytest.mark.parametrize('C', [4, 128, 132, 384])
def test_bn_stats_exact_moments(k, C):
    """M = 528 * 2^k: every block holds 2^k rows of 3-bit integers (plus a per-column offset of up to 2^10), so each block's
    sums, mean and M2 are exact and the merged mean and var must be float64's rounded to fp32 within 1 ulp."""
    g = _gen(k * 1000 + C)
    M = BN_BLOCKS << k
    y = _ints((M, C), 3, g) + torch.randint(-1024, 1025, (C,), generator=g, device=dev()).float()
    y[:, :C // 4] = _ints((M, C // 4), 3, g)              # and columns around zero
    mean, var = _ops().bn_stats(y)
    var64, mean64 = torch.var_mean(y.double(), 0, correction=0)
    m32, v32 = mean64.float(), var64.float()
    tol = _ulp(m32) + 2.0 ** -40 * y.abs().amax(0)
    assert bool(((mean - m32).abs() <= tol).all()), float(((mean - m32).abs() / tol).max())
    assert bool(((var - v32).abs() <= _ulp(v32)).all()), float(((var.double() - var64).abs() / var64).max())


BN_M = (2, 7, 527, 528, 529, 1057, 134400, 32400)   # one row per block, exactly one block each, empty trailing blocks
BN_C = (4, 124, 128, 132, 256, 384)                 # 128-channel tiles, partly filled


@pytest.mark.parametrize('C', BN_C)
@pytest.mark.parametrize('M', BN_M)
def test_bn_train_kernels(M, C):
    """bn_stats -> bn_apply -> bn_bwd at every row-block and channel-tile edge, with and without ReLU and affine."""
    relu, affine = [(True, True), (False, True), (True, False), (False, False)][(BN_M.index(M) + BN_C.index(C)) % 4]
    g = _gen(M * 1000 + C)
    y, gamma, beta, rm, rv, dz = _bn_inputs(M, C, affine, g)
    y[:, 0] += 100.0
    _bn_check(f'bn M={M} C={C} relu={relu} affine={affine}', y, dz, gamma, beta, relu, rm, rv)


def _moment_edges(M, g):
    """[M, 128] columns in groups of 16: the edges of the one-pass block moments (pivot = a block's first row)."""
    C, rows = 128, -(-M // BN_BLOCKS)
    y = _normal((M, C), g)
    pivots = torch.arange(0, M, rows, device=dev())
    groups = {'normal': slice(0, 16)}
    y[:, 16:32] = 1e4 + _normal((M, 16), g) * 1e-2
    groups['mean 1e4, std 1e-2'] = slice(16, 32)
    y[pivots, 32:48] = 1000.0
    groups['pivots 1000 sigma'] = slice(32, 48)
    sparse = torch.rand((M, 16), generator=g, device=dev()) < 0.02
    y[:, 48:64] = torch.where(sparse, 30.0 + _normal((M, 16), g), torch.zeros(M, 16, device=dev()))
    y[pivots, 48:64] = 30.0 + _normal((len(pivots), 16), g)
    groups['sparse, pivots on the few'] = slice(48, 64)
    sparse = torch.rand((M, 16), generator=g, device=dev()) < 0.02
    y[:, 64:80] = torch.where(sparse, 30.0 + _normal((M, 16), g), torch.zeros(M, 16, device=dev()))
    groups['sparse, pivots on zeros'] = slice(64, 80)
    y[:, 80:96] = 3.75
    groups['constant'] = slice(80, 96)
    y[:, 96:] = _normal((M, 32), g) * 5 + 40
    groups['offset normal'] = slice(96, 128)
    return y, groups


@pytest.mark.parametrize('M', [134400, 32400])
def test_bn_moment_edges(M):
    """The edges of the one-pass block moments at the production row counts, against float64 and fp32 torch: a column of
    mean 1e4 and std 1e-2, block pivots that are 1000 sigma outliers, sparse columns of exact zeros with a few large
    rows (pivots on them, or not), and a constant column whose var must be exactly 0 with every output finite."""
    g = _gen(M)
    y, groups = _moment_edges(M, g)
    C = y.shape[1]
    gamma, beta = torch.rand(C, generator=g, device=dev()) + 0.5, _normal((C,), g) * 0.1
    rm, rv = _normal((C,), g) * 0.1, torch.rand(C, generator=g, device=dev()) + 0.5
    dz = _normal((M, C), g)
    got = _bn_check(f'bn edges M={M}', y, dz, gamma, beta, True, rm, rv, groups)
    const = groups['constant']
    assert bool((got['var'][const] == 0).all())
    for k in ('z', 'dy'):
        assert bool(torch.isfinite(got[k]).all()), k


def test_bn_aliasing_and_determinism():
    """bn_apply with z == y and bn_bwd with dy == dz give the bits of separate buffers; repeated calls give the same
    bits."""
    M, C = 4321, 132
    g = _gen(77)
    y, gamma, beta, rm, rv, dz = _bn_inputs(M, C, True, g)
    ops = _ops()
    mean, var = ops.bn_stats(y)
    m2, v2 = ops.bn_stats(y)
    assert same_bits(mean, m2) and same_bits(var, v2)
    z = ops.bn_apply(y, mean, var, gamma, beta, EPS, 1)
    assert same_bits(z, ops.bn_apply(y, mean, var, gamma, beta, EPS, 1))
    yz = y.clone()
    assert _capi('di_bn_apply_f32', _p(yz), M, C, _p(mean), _p(var), _p(gamma), _p(beta), EPS, 1, _p(yz)) == 0
    assert same_bits(yz, z)
    dy, dg, db = ops.bn_bwd(dz, z, y, mean, var, gamma, EPS)
    dy2, dg2, db2 = ops.bn_bwd(dz, z, y, mean, var, gamma, EPS)
    assert same_bits(dy, dy2) and same_bits(dg, dg2) and same_bits(db, db2)
    work = torch.empty(592 * C * 2, device=dev())
    d = dz.clone()
    dg3, db3 = torch.empty(C, device=dev()), torch.empty(C, device=dev())
    assert _capi('di_bn_bwd_f32', _p(d), _p(z), _p(y), M, C, _p(mean), _p(var), _p(gamma), EPS, _p(work), _p(d), _p(dg3),
                 _p(db3)) == 0
    assert same_bits(d, dy) and same_bits(dg3, dg) and same_bits(db3, db)


# ---------------------------------------------------------------------------------------------------------------------
# 5. documented rejections: -1 and the output untouched; every buffer is sized for the rejected shape
# ---------------------------------------------------------------------------------------------------------------------
def _rejection_cases():
    """name -> builder(out canvas, keep) -> (entry point, args); the builder appends its buffers to `keep`.  Window
    shapes are (N, H, W, C, ks, ld)."""
    def zeros(keep, *shape):
        keep.append(torch.zeros(*shape, device=dev()))
        return _p(keep[-1])

    def win(name, N, H, W, C, ks, ld=None):
        ld = ld or C

        def build(out, keep):
            P = max(N, 1) * max(H, 1) * max(W, 1)
            a = zeros(keep, P, ld)
            if name == 'di_win_dot_f32':
                return name, [a, ld, a, ld, _p(out), N, H, W, C, ks]
            return name, [zeros(keep, P, ks * ks), a, ld, _p(out), ld, N, H, W, C, ks]
        return build

    def softmax(name, P, KK):
        def build(out, keep):
            s = zeros(keep, max(P, 1) * max(KK, 1))
            if name == 'di_win_softmax_f32':
                return name, [s, _p(out), P, KK, 1.0]
            return name, [s, s, _p(out), P, KK, 1.0]
        return build

    def col_sum(M):
        def build(out, keep):
            return 'di_col_sum_f32', [zeros(keep, max(M, 1), 64), 64, M, 64, zeros(keep, 256 * 64), _p(out)]
        return build

    def ln_bwd(M, C):
        def build(out, keep):
            Mx = max(M, 1)
            x = zeros(keep, Mx, C)
            return 'di_ln_bwd_f32', [x, C, x, C, zeros(keep, C), _p(out), C, _p(out[Mx * C:]), _p(out[Mx * C + C:]),
                                     zeros(keep, Mx * C + 256 * C), M, C, EPS]
        return build

    def bn_stats(M, C, run_mean, run_var):
        # C = 6 on one row: the float4 loads of a missing check would stay aligned and inside the 8-word row buffer
        def build(out, keep):
            r = zeros(keep, C + 4)
            return 'di_bn_stats_f32', [zeros(keep, M, -(-C // 4) * 4), M, C, zeros(keep, 592 * C * 3), _p(out),
                                       _p(out[C + 4:]), r if run_mean else None, r if run_var else None, 0.1]
        return build

    cases = {}
    for name in ('di_win_dot_f32', 'di_win_gather_f32', 'di_win_scatter_f32'):
        s = name[7:-4]
        cases.update({
            f'{s}_C_6': win(name, 1, 4, 5, 6, 3, ld=8),
            f'{s}_C_516': win(name, 1, 4, 5, 516, 3),
            f'{s}_ks_2': win(name, 1, 4, 5, 32, 2),
            f'{s}_ks_13': win(name, 1, 4, 5, 32, 13),
            f'{s}_N_0': win(name, 0, 4, 5, 32, 3),
            f'{s}_H_0': win(name, 1, 0, 5, 32, 3),
            f'{s}_W_0': win(name, 1, 4, 0, 32, 3),
        })
    for name in ('di_win_softmax_f32', 'di_win_softmax_bwd_f32'):
        s = name[3:-4]
        cases.update({f'{s}_KK_0': softmax(name, 5, 0), f'{s}_KK_129': softmax(name, 5, 129), f'{s}_P_0': softmax(name, 0, 9)})
    cases.update({
        'col_sum_M_0': col_sum(0),
        'ln_bwd_M_0': ln_bwd(0, 64),
        'ln_bwd_C_513': ln_bwd(3, 513),
        'bn_stats_C_6': bn_stats(1, 6, True, True),
        'bn_stats_run_mean_without_run_var': bn_stats(64, 64, True, False),
    })
    return cases


REJECTIONS = _rejection_cases()


@pytest.mark.parametrize('case', list(REJECTIONS))
def test_documented_rejections(case):
    buf, out = flat_canvas(1 << 16)
    keep = []
    name, args = REJECTIONS[case](out, keep)
    assert _status(name, *args) == DI_ERR_ARG
    assert bool((buf.view(torch.int32) == SENT).all())


# ---------------------------------------------------------------------------------------------------------------------
# 6. the production calls of the base model
# ---------------------------------------------------------------------------------------------------------------------
TRAIN = ('di_win_dot_f32', 'di_win_gather_f32', 'di_win_scatter_f32', 'di_win_softmax_f32', 'di_win_softmax_bwd_f32',
         'di_relu_bwd_f32', 'di_col_sum_f32', 'di_ln_bwd_f32', 'di_bn_stats_f32', 'di_bn_apply_f32', 'di_bn_bwd_f32')
PILLARS = 'pillars'   # a row count equal to the frame's number of pillars (MMRI_I2P backward); tested at 24000
PILLARS_TESTED = 24000


def call_key(name, a):
    """The shape signature of a call: window (N, H, W, C, ks, lda / ldb or ldb / ldo), softmax (P, KK), relu (n),
    col_sum (M, C, ld), ln_bwd (M, C, ldy, ldz, lddz), bn_stats (M, C, running statistics), bn_apply (M, C, affine, ReLU),
    bn_bwd (M, C, ReLU, affine)."""
    if name == 'di_win_dot_f32':
        return (name,) + tuple(a[5:10]) + (a[1], a[3])
    if name in ('di_win_gather_f32', 'di_win_scatter_f32'):
        return (name,) + tuple(a[5:10]) + (a[2], a[4])
    if name == 'di_win_softmax_f32':
        return (name, a[2], a[3])
    if name == 'di_win_softmax_bwd_f32':
        return (name, a[3], a[4])
    if name == 'di_relu_bwd_f32':
        return (name, a[3])
    if name == 'di_col_sum_f32':
        return (name, a[2], a[3], a[1])
    if name == 'di_ln_bwd_f32':
        return (name, a[10], a[11], a[1], a[3], a[6])
    if name == 'di_bn_stats_f32':
        return (name, a[1], a[2], a[6] is not None)
    if name == 'di_bn_apply_f32':
        return (name, a[1], a[2], a[5] is not None, a[8])
    return (name, a[3], a[4], a[1] is not None, a[7] is not None)


IMG, BEV = (6, 112, 200), (1, 180, 180)
M_IMG, M_BEV = 6 * 112 * 200, 180 * 180

# Every call of these entry points in the base model (projects/configs/nuscenes/di_b200_base_hotpath.py: 6 views of
# 112 x 200 image rows, a 180 x 180 BEV map, hidden width 128, 9 x 9 windows, 200 proposals) made by
# train.encoder_train_step and by backward.encoder_backward, decoder_layer_backward and point_rcnn_backward.
TABLE = {}
for _dims, _M, _where in ((IMG, M_IMG, 'image'), (BEV, M_BEV, 'BEV')):
    TABLE.update({
        ('di_win_dot_f32',) + _dims + (128, 9, 128, 128): f'{_where} LCAB logits q.k and dA = dO.v',
        ('di_win_gather_f32',) + _dims + (128, 9, 128, 128): f'{_where} LCAB out = A v, dq = dS k',
        ('di_win_scatter_f32',) + _dims + (128, 9, 128, 128): f'{_where} LCAB dv = A^T dO, dk = dS^T q',
        ('di_win_softmax_f32', _M, 81): f'{_where} LCAB window softmax',
        ('di_win_softmax_bwd_f32', _M, 81): f'{_where} LCAB softmax backward',
        ('di_bn_stats_f32', _M, 128, True): f'{_where} ConvBN batch statistics (training step)',
        ('di_bn_apply_f32', _M, 128, True, 1): f'{_where} LCAB ConvBNReLU normalise',
        ('di_bn_apply_f32', _M, 128, True, 0): f'{_where} fuse ConvBN normalise',
        ('di_bn_bwd_f32', _M, 128, True, True): f'{_where} LCAB ConvBNReLU backward',
        ('di_bn_bwd_f32', _M, 128, False, True): f'{_where} fuse ConvBN backward',
        ('di_col_sum_f32', _M, 128, 128): f'{_where} shared conv / LCAB / fuse bias gradients',
        ('di_relu_bwd_f32', _M * 128): f'{_where} LCAB ReLU masks (eval-mode backward)' +
                                         (', decoder key pos-MLP hidden' if _M == M_BEV else ''),
    })
TABLE.update({
    ('di_col_sum_f32', PILLARS, 128, 128): 'I2P bias gradients over the pillars',
    ('di_col_sum_f32', M_BEV, 256, 256): 'decoder layer cross-attention K | V bias gradient over the BEV rows',
    ('di_col_sum_f32', 200, 128, 128): 'query-row bias gradients of the 128-wide decoder layers',
    ('di_col_sum_f32', 200, 256, 256): 'decoder layer FFN linear1 and query pos-MLP bias gradients',
    ('di_col_sum_f32', 200, 384, 384): 'self-attention in_proj bias gradient',
    ('di_col_sum_f32', 200, 512, 512): 'PointRCNN FFN linear1 bias and DynamicConv norm gradients',
    ('di_col_sum_f32', 200, 32768, 32768): 'PointRCNN DynamicConv parameter generator bias gradient',
    ('di_ln_bwd_f32', 200, 128, 128, 128, 128): 'decoder layer and PointRCNN LayerNorm backward',
    ('di_relu_bwd_f32', 200 * 128): 'query-row ReLU masks (pos-MLP hidden, PointRCNN DynamicConv)',
    ('di_relu_bwd_f32', 200 * 256): 'decoder layer FFN ReLU mask',
})


def _sample_pixels(dims, ks, g):
    """Flat pixels of an (N, H, W) map: the first and last pixel of every image, pixels within r of every border, and
    random ones."""
    N, H, W = dims
    r = ks // 2
    edge_y = torch.tensor(list(range(r + 1)) + list(range(H - r - 1, H)), device=dev())
    edge_x = torch.tensor(list(range(r + 1)) + list(range(W - r - 1, W)), device=dev())
    pix = []
    for n in range(N):
        base = n * H * W
        pix += [torch.tensor([base, base + H * W - 1], device=dev())]
        pix.append(base + edge_y * W + torch.randint(0, W, edge_y.shape, generator=g, device=dev()))
        pix.append(base + torch.randint(0, H, edge_x.shape, generator=g, device=dev()) * W + edge_x)
    pix.append(torch.randint(0, N * H * W, (300,), generator=g, device=dev()))
    return torch.unique(torch.cat(pix))


def _run_window_entry(key, g):
    name, N, H, W, C, ks, ld1, ld2 = key
    ops = _ops()
    P, dims = N * H * W, (N, H, W)
    b = _strided(_normal((P, C), g), ld1 if name != 'di_win_dot_f32' else ld2)
    pix = _sample_pixels(dims, ks, g)
    with record_calls() as calls:
        if name == 'di_win_dot_f32':
            a = _strided(_normal((P, C), g), ld1)
            out = ops.win_dot(a, b, N, H, W, ks)
        else:
            w = _normal((P, ks * ks), g)
            out = (ops.win_gather if 'gather' in name else ops.win_scatter)(w, b, N, H, W, ks)
    if name == 'di_win_dot_f32':
        want, scale, _ = ref_dot(a, b, N, H, W, ks, pix)
        bar = dot_bar(C)
    elif 'gather' in name:
        want, scale = ref_gather(w, b, N, H, W, ks, pix)
        bar = apply_bar(ks)
    else:
        want, scale = ref_scatter_at(w, b, N, H, W, ks, pix)
        bar = apply_bar(ks)
    return calls, row_err(out[pix], want, scale), bar


def _run_row_entry(key, g):
    name = key[0]
    ops = _ops()
    s32 = _sm_scale32()
    with record_calls() as calls:
        if name == 'di_win_softmax_f32':
            S = (_logits(key[1], key[2], g) / s32).float()
            out = ops.win_softmax(S, SM_SCALE)
        elif name == 'di_win_softmax_bwd_f32':
            A = torch.softmax(_normal((key[1], key[2]), g) * 3, 1)
            dA = _normal((key[1], key[2]), g)
            out = ops.win_softmax_bwd(A, dA, SM_SCALE)
        elif name == 'di_relu_bwd_f32':
            y, dy = _normal((key[1],), g), _normal((key[1],), g)
            y[::7] = 0.0
            out = ops.relu_bwd(dy, y)
        elif name == 'di_col_sum_f32':
            M = PILLARS_TESTED if key[1] == PILLARS else key[1]
            x = _strided(_normal((M, key[2]), g), key[3])
            out = ops.col_sum(x)
        else:                                                      # ln_bwd
            _, M, C, ldy, ldz, lddz = key
            z = _normal((M, C), g) * 2 + 3
            gamma = torch.rand(C, generator=g, device=dev()) + 0.5
            dy = _normal((M, C), g)
            out = ops.ln_bwd(_strided(dy, ldy), _strided(z, ldz), gamma)
    if name == 'di_win_softmax_f32':
        z = S.double() * s32
        want = torch.softmax(z, 1)
        bars = (4 * z.abs().amax(1, keepdim=True) + 16) * U
        e = float((((out.double() - want).abs().amax(1, keepdim=True) / want.amax(1, keepdim=True)) / bars).max())
        return calls, e, 1.0
    if name == 'di_win_softmax_bwd_f32':
        Ad, dAd = A.double(), dA.double()
        want = Ad * (dAd - (Ad * dAd).sum(1, keepdim=True)) * s32
        return calls, row_err(out, want, Ad * (dAd.abs() + (Ad * dAd.abs()).sum(1, keepdim=True)) * s32), 16 * U
    if name == 'di_relu_bwd_f32':
        return calls, 0.0 if same_bits(out, torch.ops.aten.threshold_backward(dy, y, 0.0)) else math.inf, 0.5
    if name == 'di_col_sum_f32':
        return calls, row_err(out, x.double().sum(0), x.double().abs().sum(0), width=1), colsum_bar(x.shape[0])
    zz = z.double().requires_grad_(True)
    with torch.enable_grad():
        F.layer_norm(zz, (C,), gamma.double(), None, EPS).mul(dy.double()).sum().backward()
    return calls, float((out[0].double() - zz.grad).abs().max() / zz.grad.abs().max()), LN_BAR


def _run_bn_entry(key, g):
    name, M, C = key[:3]
    relu = key[4] if name == 'di_bn_apply_f32' else key[3] if name == 'di_bn_bwd_f32' else True
    y, gamma, beta, rm, rv, dz = _bn_inputs(M, C, True, g)
    with record_calls() as calls:
        _bn_check(f'production {TABLE[key]}', y, dz, gamma, beta, relu, rm, rv)
    return [c for c in calls if c[0] == name], 0.0, 1.0


@pytest.mark.parametrize('key', list(TABLE), ids=lambda k: '-'.join(map(str, k)))
def test_production_calls(key):
    """Every table entry at its real size through ops (the entry point and shape it takes are asserted), against float64
    on sampled pixels (window ops) or in full."""
    g = _gen(zlib.crc32(repr(key).encode()))
    run = _run_window_entry if key[0].startswith('di_win_') and 'softmax' not in key[0] else \
        _run_bn_entry if key[0].startswith('di_bn_') else _run_row_entry
    calls, e, bar = run(key, g)
    keys = [call_key(n, a) for n, a in calls if n in TRAIN]
    if key[0] == 'di_col_sum_f32' and key[1] == PILLARS:
        keys = [(k[0], PILLARS) + k[2:] for k in keys]
    assert key in keys, keys
    print(f'production {TABLE[key]}: error {e:.2e} (bar {bar:.2e})')
    assert e < bar


def _pillar_key(k, n_pillars):
    return (k[0], PILLARS) + k[2:] if k[0] == 'di_col_sum_f32' and k[1] == n_pillars else k


def test_production_table_covers_base_training():
    """One base-shape training step of the encoder and one run of backward.encoder_backward, decoder_layer_backward and
    point_rcnn_backward (both PointRCNN blocks): every call of these entry points they issue is in the table."""
    import bench
    from deepinteraction_b200 import backward, synth, train
    from test_gpu_decoder_layer_backward import _decoder as layer_decoder, _layer_inputs
    from test_gpu_rcnn_backward import _decoder as rcnn_decoder, _block_inputs, BLOCK_SEEDS
    d = dev()
    neck, _ = bench.build_models(d)
    fr = synth.to_device(synth.make_frame_batch(bench.SEED + 5, batch=1, cloud='lidar'), d)
    pm = fr['pts_metas']
    n_pillars = int(pm['pillars'].shape[0])
    BV, _, h, w = fr['img_feats'].shape
    B, _, Y, X = fr['pts_feats'].shape
    g = _gen(5)
    with record_calls() as calls:
        train.encoder_train_step(neck.train(), fr['img_feats'], fr['pts_feats'], fr['img_metas'], pm,
                                 lambda a, b, c: tuple(torch.randn_like(t) for t in (a, b, c)))
        neck.eval()
        backward.encoder_backward(neck, fr['img_feats'], fr['pts_feats'], fr['img_metas'], pm, _normal((BV, h, w, 128), g),
                                  _normal((B, Y, X, 128), g), _normal((B, Y, X, 128), g))
        m = layer_decoder(True, False)
        backward.decoder_layer_backward(m, *(t.to(d) for t in _layer_inputs(m, 1, 91)))
        m = rcnn_decoder(True)
        for li in (1, 3):
            backward.point_rcnn_backward(m, li, *(t.to(d) for t in _block_inputs(m, 1, BLOCK_SEEDS[(True, li)])))
    torch.cuda.synchronize()
    keys = {_pillar_key(call_key(n, a), n_pillars) for n, a in calls if n in TRAIN}
    print('base training calls:', sorted(keys, key=str))
    missing = sorted(keys - set(TABLE), key=str)
    assert not missing, missing
