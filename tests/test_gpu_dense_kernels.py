"""Kernel-level tests of the dense layers against float64: the wgmma split-product GEMM and 3x3 convolution
(csrc/gemm_tc.cu, bf16-split and 3xTF32) and the FFMA SGEMM with its small-M kernel and split-K (csrc/gemm.cu).  The C
entry points are called directly wherever the variant matters, so that the operand precision, the weight placement
(mode 3 = resident when K <= 128, mode 4 = streamed), the SM limit of the persistent grid, the NCHW-direct conv and the
split kinds are chosen by the test, not by ops routing.  Calls that go through ops record the entry point they took.

Exact cases.  Integer operands, scaled by powers of two per row of A and per output column, with every product and
every partial sum below 2^24: any correct kernel, in any summation order, equals the float64 result bit for bit, so a
wrong k chunk, tap, source, tile, halo or padding fails with zero tolerance.  The compensation terms are exercised by
operands wider than the hi part (bf16: 8 significant bits, tf32: 11): A of 10-12 bits against W of 3-4 bits makes
A_mid / A_lo nonzero, and the reverse makes W_mid / W_lo nonzero, so dropping any one of the three products breaks
exactness.

Precision cases.  Random normal operands with per-row magnitudes spread over 2^-20..2^20, bias, residuals and GELU;
row_err (kernel_check.py) against the per-element scale |A| |W|^T + |bias| + |res|, the magnitude of the terms summed.
Each mode has its own bar, set from the H100 measurement (see BARS).

Bounds.  Outputs are views of a larger buffer filled with a NaN sentinel (extra rows past M, ldc > N): every word
outside the [M, N] window keeps its bits; so do the output and the unused partials of every rejected call.
"""
import contextlib
import ctypes
import os
import zlib

import pytest
import torch
import torch.nn.functional as F

from kernel_check import SENT, _capi, _status, canvas, outside_intact, record_calls, row_err, same_bits

pytestmark = pytest.mark.gpu

DI_ERR_ARG, DI_ERR_UNSUPPORTED = -1, -3
SM_LIMITS = (0, 1, 7, 131)        # 0 = one CTA per SM; 1 and 7 are below / not multiples of n_tiles = 3, 5

# Bars of row_err per mode: the maxima over every precision and production case of this file measured on an H100 80GB
# HBM3 (132 SMs, 700 W power limit), times a margin:
#   bf16 split  3.5e-6 at every K (64 .. 4608)        bar 1.5e-5  (margin 4.3x)
#   3xTF32      4.3e-7 for K <= 384                   bar 1e-6    (margin 2.3x)
#               1.04e-6 up to K = 4608                bar 4e-6    (margin 3.8x)
#   FFMA        2.5e-7                                bar 1e-6    (margin 4x)
# The 3xTF32 error grows with K (the tensor core truncates its accumulator at every step); the bf16-split error is set
# by the 16 operand bits and does not.  At K <= 384 the two modes are 3.5x - 20x apart and the test asserts that every
# bf16-split result there exceeds the 3xTF32 bar: the smallest bf16-split error is 1.5e-6, 1.5x over that bar, which is
# the slack a rebuild of either mode has before the separation assertion fails.  At K = 1152 and 4608 they are only
# 1.5x apart and no bar separates them.
BARS = dict(bf16=1.5e-5, tf32=4e-6, ffma=1e-6)
TF32_BAR_SHORT_K = 1e-6          # 3xTF32 with K <= 384


def bar(mode, K):
    return TF32_BAR_SHORT_K if mode == 'tf32' and K <= 384 else BARS[mode]


def dev():
    return torch.device('cuda:0')


def _ops():
    from deepinteraction_b200 import ops
    return ops


def _fold():
    from deepinteraction_b200 import fold
    return fold


def _lib():
    from deepinteraction_b200 import _lib
    return _lib.lib()


def _p(t):
    return _ops()._ptr(t)


def _gen(seed):
    return torch.Generator(device='cuda').manual_seed(seed)


def _ints(shape, bits, g):
    """Integers of up to `bits` magnitude bits (|x| < 2^bits), as fp32 on the device."""
    m = (1 << bits) - 1
    return torch.randint(-m, m + 1, shape, generator=g, device=dev()).float()


def _pow2(n, lo, hi, g):
    return torch.exp2(torch.randint(lo, hi + 1, (n,), generator=g, device=dev()).float())


@contextlib.contextmanager
def tc_state(mode=3, sm_limit=0):
    """Weight placement and SM limit of the tensor-core launches; restores the defaults."""
    L = _lib()
    assert L.di_tc_set_mode(mode) == 0 and L.di_tc_set_sm_limit(sm_limit) == 0
    try:
        yield
    finally:
        L.di_tc_set_mode(3)
        L.di_tc_set_sm_limit(int(os.environ.get('DI_B200_TC_SMS', '0')))


def exact(got, want):
    """Bit equality with the float64 result rounded to fp32 (exact here); +0 and -0 count as equal."""
    return same_bits(got.float() + 0.0, want.float() + 0.0)


def _src_views(Ks, M, pad, g, make):
    """Sources [M, K_s], each a view with lda = K_s + pad of its own buffer (pad % 4 == 0 keeps 16-byte rows)."""
    out = []
    for k in Ks:
        buf = make((M, k + pad), g)
        out.append(buf[:, :k] if pad else buf)
    return out


def _srcs_args(srcs):
    a = []
    for s in srcs:
        assert s.stride(1) == 1
        a += [_p(s), s.stride(0), s.shape[1]]
    while len(a) < 9:
        a += [None, 0, 0]
    return a


def _wsplit(w, bf):
    fold = _fold()
    hi, lo = (fold.split_bf16 if bf else fold.split_tf32)(w.float())
    return hi.to(dev()), lo.to(dev())


def tc_linear(bf, srcs, w, out, bias=None, res=None, res_mod=0, act=0, split=None, ws=None):
    hi, lo = ws if ws is not None else _wsplit(w, bf)
    M, N = srcs[0].shape[0], w.shape[0]
    args = _srcs_args(srcs) + [_p(hi), _p(lo), _p(bias), _p(res), 0 if res is None else res.stride(0), res_mod, _p(out),
                               out.stride(0), M, N, act]
    if split is not None:
        return _capi('di_linear_tcb_split_f32', *args, *split)
    return _capi('di_linear_tcb_f32' if bf else 'di_linear_tc_f32', *args)


def ffma_linear(srcs, w, out, bias=None, res=None, res_mod=0, act=0, splits=1, split_stride=0):
    M, N = srcs[0].shape[0], w.shape[0]
    return _capi('di_linear_f32', *_srcs_args(srcs), _p(w), _p(bias), _p(res), 0 if res is None else res.stride(0),
                 res_mod, _p(out), out.stride(0), M, N, act, splits, split_stride)


def _act(y, act):
    return {0: lambda x: x, 1: F.relu, 2: F.gelu}[act](y)


def ref_linear(srcs, w, bias=None, res=None, res_mod=0, act=0):
    A = torch.cat([s.double() for s in srcs], 1)
    y = A @ w.double().t()
    if bias is not None:
        y = y + bias.double()
    if res is not None:
        M = A.shape[0]
        y = y + res.double()[torch.arange(M, device=y.device) % (res_mod or M)]
    return _act(y, act)


def scale_linear(srcs, w, bias=None, res=None, res_mod=0):
    """|A| |W|^T + |bias| + |res|: the magnitude of the terms summed into each output."""
    A = torch.cat([s.double().abs() for s in srcs], 1)
    s = A @ w.double().abs().t()
    if bias is not None:
        s = s + bias.double().abs()
    if res is not None:
        M = A.shape[0]
        s = s + res.double().abs()[torch.arange(M, device=s.device) % (res_mod or M)]
    return s


def _res(M, N, res_mod, g, make):
    if res_mod is None:
        return None
    return make((res_mod or M, N), g)


# ---------------------------------------------------------------------------------------------------------------------
# 1. tensor-core linear: exact cases
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('bf', [True, False], ids=['bf16split', '3xtf32'])
@pytest.mark.parametrize('wide', ['A', 'W'])
@pytest.mark.parametrize('mode', [3, 4])
def test_tc_linear_exact_compensation(bf, wide, mode):
    """A (or W) wider than the hi part: the A_mid / A_lo (W_mid / W_lo) products carry the low bits.  K = 64 keeps
    every sum below 2^24 (64 * 2^12 * 15 for bf16, 64 * 2^14 * 15 for 3xTF32)."""
    g = _gen(11 + bf + 2 * (wide == 'W'))
    M, N, K = 300, 132, 64
    wb = 12 if bf else 14
    A = _ints((M, K), wb if wide == 'A' else 4, g)
    W = _ints((N, K), 4 if wide == 'A' else wb, g)
    bias = _ints((N,), 10, g)
    hi, lo = _wsplit(W, bf)
    assert bool((lo != 0).any()) == (wide == 'W')
    buf, out = canvas(M, N)
    with tc_state(mode):
        tc_linear(bf, [A], W, out, bias=bias, act=1, ws=(hi, lo))
    assert exact(out, ref_linear([A], W, bias, act=1))
    assert outside_intact(buf, M, N)


# (M, N, K per source, extra lda, res_mod (None: no residual, 0: one row per output row), act, bias)
TC_SHAPES = [
    (1, 4, [64], 0, None, 0, True),
    (127, 20, [64, 64], 36, 0, 1, True),
    (128, 132, [128], 0, 1, 0, False),
    (129, 640, [64, 64], 0, None, 1, True),             # resident W, n_tiles = 5, tiles < SMs
    (17019, 128, [128], 0, None, 0, False),             # resident W, n_tiles = 1, tiles = 133 >= SMs
    (6000, 384, [64, 64], 4, 97, 1, True),              # resident W, n_tiles = 3, tiles = 141 >= SMs
    (3500, 640, [128], 0, None, 0, False),              # resident W, n_tiles = 5, tiles = 140 >= SMs
    (100, 2112, [64], 0, None, 1, True),                # N > 2048 with M < 128
    (1000, 256, [64, 128, 64], 8, 97, 0, True),         # three sources, streamed W
    (33000, 132, [128, 128, 128], 0, None, 1, False),   # large M with M % 128 != 0, N tail
    (700, 36, [32, 64, 32], 4, 0, 0, True),             # 3xTF32 only: source boundaries at multiples of 32
    (300, 384, [32, 96], 0, None, 1, False),            # 3xTF32 only, resident W (K = 128)
]


def _exact_linear_case(M, N, Ks, pad, res_mod, act, has_bias, seed):
    """Integer operands of 4 bits: per-output-column powers of two, and per-row ones when nothing is added per column
    (bias / residual values are not scaled by the row)."""
    g = _gen(seed)
    rs = _pow2(M, -6, 6, g)[:, None] if not has_bias and res_mod is None else 1.0
    srcs = _src_views(Ks, M, pad, g, lambda shape, g: _ints(shape, 4, g) * rs)
    cs = _pow2(N, -6, 6, g)
    W = _ints((N, sum(Ks)), 4, g) * cs[:, None]
    bias = _ints((N,), 10, g) * cs if has_bias else None
    res = _res(M, N, res_mod, g, lambda shape, g: _ints(shape, 8, g) * cs)
    return srcs, W, bias, res


@pytest.mark.parametrize('M,N,Ks,pad,res_mod,act,has_bias', TC_SHAPES,
                         ids=['x'.join(map(str, (c[0], c[1], '+'.join(map(str, c[2]))))) for c in TC_SHAPES])
def test_tc_linear_exact_shapes(M, N, Ks, pad, res_mod, act, has_bias):
    """Every placement and SM limit on the same exact inputs: each result equals float64 bit for bit."""
    srcs, W, bias, res = _exact_linear_case(M, N, Ks, pad, res_mod, act, has_bias, M + N)
    want = ref_linear(srcs, W, bias, res, res_mod or 0, act)
    for bf in (True, False):
        if bf and any(k % 64 for k in Ks):
            continue
        ws = _wsplit(W, bf)
        for mode in (3, 4):
            for lim in SM_LIMITS:
                buf, out = canvas(M, N)
                with tc_state(mode, lim):
                    tc_linear(bf, srcs, W, out, bias, res, res_mod or 0, act, ws=ws)
                assert exact(out, want), (bf, mode, lim)
                assert outside_intact(buf, M, N), (bf, mode, lim)


# ---------------------------------------------------------------------------------------------------------------------
# 2. tensor-core linear: precision, mode separation, invariants
# ---------------------------------------------------------------------------------------------------------------------
def _normal(shape, g):
    return torch.randn(shape, generator=g, device=dev())


def _precision_case(M, N, Ks, res_mod, has_bias, seed):
    g = _gen(seed)
    rs = _pow2(M, -20, 20, g)
    srcs = [_normal((M, k), g) * rs[:, None] for k in Ks]
    W = _normal((N, sum(Ks)), g) / sum(Ks) ** 0.5
    bias = _normal((N,), g) if has_bias else None
    res = _res(M, N, res_mod, g, _normal)
    return srcs, W, bias, res


# (M, N, K per source, res_mod, act, bias)
PREC_SHAPES = [
    (3000, 128, [128], 97, 2, True),
    (1500, 384, [128, 128, 128], None, 0, True),
    (700, 256, [64], 0, 2, False),
    (400, 128, [1152], None, 1, True),
    (300, 128, [4608], None, 0, False),
]


@pytest.mark.parametrize('M,N,Ks,res_mod,act,has_bias', PREC_SHAPES,
                         ids=['x'.join(map(str, (c[0], c[1], '+'.join(map(str, c[2]))))) for c in PREC_SHAPES])
def test_tc_linear_precision(M, N, Ks, res_mod, act, has_bias):
    """Per-row error of each mode within its bar, and for K <= 384 the 3xTF32 bar rejects the bf16-split result of the
    same inputs (the backward's precision rests on that gap)."""
    srcs, W, bias, res = _precision_case(M, N, Ks, res_mod, has_bias, M + 3 * N)
    want = ref_linear(srcs, W, bias, res, res_mod or 0, act)
    scale = scale_linear(srcs, W, bias, res, res_mod or 0)
    errs = {}
    for bf, mode in ((True, 'bf16'), (False, 'tf32')):
        out = torch.empty(M, N, device=dev())
        tc_linear(bf, srcs, W, out, bias, res, res_mod or 0, act)
        errs[mode] = row_err(out, want, scale)
    out = torch.empty(M, N, device=dev())
    ffma_linear(srcs, W.contiguous(), out, bias, res, res_mod or 0, act)
    errs['ffma'] = row_err(out, want, scale)
    print(f'precision M={M} N={N} K={Ks}: ' + ' '.join(f'{k} {v:.2e}' for k, v in errs.items()) +
          f'  gap bf16/tf32 {errs["bf16"] / max(errs["tf32"], 1e-30):.1f}')
    K = sum(Ks)
    for mode, e in errs.items():
        assert e < bar(mode, K), (mode, e)
    if K <= 384:
        assert errs['bf16'] > bar('tf32', K), errs


@pytest.mark.parametrize('M,N,Ks', [(17019, 128, [128]), (6000, 384, [64, 64]), (3500, 640, [128]), (129, 640, [64]),
                                    (2000, 256, [128, 64, 64])])
@pytest.mark.parametrize('bf', [True, False], ids=['bf16split', '3xtf32'])
def test_tc_linear_same_bits_for_every_sm_limit_and_placement(M, N, Ks, bf):
    """Each tile is computed by one CTA with one instruction sequence: the grid size and the weight placement do not
    change a bit, and a second launch reproduces the first."""
    srcs, W, bias, res = _precision_case(M, N, Ks, 97, True, 7 * M + N)
    ws = _wsplit(W, bf)
    base = torch.empty(M, N, device=dev())
    tc_linear(bf, srcs, W, base, bias, res, 97, 2, ws=ws)
    for mode in (3, 4):
        for lim in SM_LIMITS:
            out = torch.empty(M, N, device=dev())
            with tc_state(mode, lim):
                tc_linear(bf, srcs, W, out, bias, res, 97, 2, ws=ws)
            assert same_bits(out, base), (mode, lim)


# ---------------------------------------------------------------------------------------------------------------------
# 3. pre-split outputs (di_linear_tcb_split_f32)
# ---------------------------------------------------------------------------------------------------------------------
def _bf16_bits(x):
    return x.to(torch.bfloat16).view(torch.int16).to(torch.int64) & 0xFFFF


def _expected_split_words(y, col0, kind):
    """The word format of the gemm_tc.cu epilogue, from the fp32 values y [M, N]: for each channel pair (c, c + 1),
    c even and >= col0, hi = bf16(y) and mid = bf16(y - hi) packed bf16x2 (lower channel in the low half); kind 1:
    words c (hi), c + 1 (mid); kind 2: in the group of 8 at g = c & ~7, words g + (c & 7) / 2 (hi) and that + 4 (mid);
    kind 3: r = c - col0, words col0 + 128 (r // 128) + (r % 128) / 2 (hi) and that + 64 (mid).  Columns below col0
    keep their fp32 bits."""
    y = y.float()
    words = y.view(torch.int32).to(torch.int64) & 0xFFFFFFFF
    z = y[:, col0:]
    hb = _bf16_bits(z)
    mb = _bf16_bits(z - z.to(torch.bfloat16).float())
    hi = hb[:, 0::2] | (hb[:, 1::2] << 16)
    mid = mb[:, 0::2] | (mb[:, 1::2] << 16)
    c = torch.arange(col0, y.shape[1], 2, device=y.device)
    if kind == 1:
        wh, wm = c, c + 1
    elif kind == 2:
        wh = (c & ~7) + (c & 7) // 2
        wm = wh + 4
    else:
        r = c - col0
        wh = col0 + (r // 128) * 128 + (r % 128) // 2
        wm = wh + 64
    words[:, wh] = hi
    words[:, wm] = mid
    return torch.where(words >= 2 ** 31, words - 2 ** 32, words).to(torch.int32)


@pytest.mark.parametrize('kind,M,N,col0', [(1, 200, 96, 32), (1, 129, 160, 0), (2, 131, 160, 64), (2, 1000, 384, 128),
                                           (3, 1000, 384, 128), (3, 127, 256, 0)])
def test_tc_linear_split_words(kind, M, N, col0):
    srcs, W, bias, _ = _precision_case(M, N, [128], None, True, 31 * kind + M)
    ws = _wsplit(W, True)
    plain = torch.empty(M, N, device=dev())
    tc_linear(True, srcs, W, plain, bias, act=1, ws=ws)
    buf, out = canvas(M, N)
    tc_linear(True, srcs, W, out, bias, act=1, split=(col0, kind), ws=ws)
    assert torch.equal(out.contiguous().view(torch.int32), _expected_split_words(plain, col0, kind))
    assert outside_intact(buf, M, N)


# ---------------------------------------------------------------------------------------------------------------------
# 4. tensor-core 3x3 convolution
# ---------------------------------------------------------------------------------------------------------------------
def _conv_ref(x_nchw, w4, bias, act):
    y = F.conv2d(x_nchw.double(), w4.double(), None if bias is None else bias.double(), padding=1)
    return _act(y, act).permute(0, 2, 3, 1)


def tc_conv(bf, nchw, x, w4, bias, act, ws=None):
    """x: NCHW [N, Cin, H, W] on the device; the input is passed NCHW (direct kernel) or transposed to NHWC."""
    N, Cin, H, W = x.shape
    Cout = w4.shape[0]
    hi, lo = ws if ws is not None else _wsplit(_fold().pack_conv3x3(w4), bf)
    xin = x.contiguous() if nchw else x.permute(0, 2, 3, 1).contiguous()
    buf = torch.full((N * H * W + 5, Cout), SENT, dtype=torch.int32, device=dev()).view(torch.float32)
    name = 'di_conv3x3_tc%s%s_f32' % ('b' if bf else '', '_nchw' if nchw else '')
    _capi(name, _p(xin), _p(hi), _p(lo), _p(bias), _p(buf), N, Cin, H, W, Cout, act)
    assert bool((buf[N * H * W:].view(torch.int32) == SENT).all())
    return buf[:N * H * W].view(N, H, W, Cout)


# (images, Cin, H, W, Cout, act): H % 8 and W % 16 != 0, H or W in {1, 2}, several images
CONV_SHAPES = [(2, 64, 13, 21, 12, 1), (3, 64, 1, 37, 20, 0), (1, 128, 9, 2, 128, 1), (2, 64, 17, 36, 256, 0),
               (1, 64, 10, 20, 512, 1), (2, 64, 2, 44, 128, 0), (5, 128, 7, 8, 20, 0)]


@pytest.mark.parametrize('n,cin,H,W,cout,act', CONV_SHAPES, ids=['x'.join(map(str, c[:5])) for c in CONV_SHAPES])
def test_conv3x3_tc_exact(n, cin, H, W, cout, act):
    """Both precisions, NHWC input and (W % 4 == 0) the NCHW-direct kernel: equal to float64 bit for bit."""
    g = _gen(n * 1000 + W)
    x = _ints((n, cin, H, W), 4, g)
    cs = _pow2(cout, -6, 6, g)
    w4 = _ints((cout, cin, 3, 3), 4, g) * cs[:, None, None, None]
    bias = _ints((cout,), 10, g) * cs
    want = _conv_ref(x, w4, bias, act)
    for bf in (True, False):
        ws = _wsplit(_fold().pack_conv3x3(w4), bf)
        for nchw in ((False, True) if W % 4 == 0 else (False,)):
            assert exact(tc_conv(bf, nchw, x, w4, bias, act, ws), want), (bf, nchw)


@pytest.mark.parametrize('bf', [True, False], ids=['bf16split', '3xtf32'])
@pytest.mark.parametrize('wide', ['x', 'w'])
def test_conv3x3_tc_exact_compensation(bf, wide):
    """Wide inputs or wide weights through every tap: K = 9 * 64 with 10 x 4 bits (bf16), 9 * 32 with 12 x 3 bits
    (3xTF32), all sums below 2^24."""
    cin = 64 if bf else 32
    xb, wb = (10, 4) if bf else (12, 3)
    if wide == 'w':
        xb, wb = wb, xb
    g = _gen(5 + bf + 2 * (wide == 'w'))
    x = _ints((2, cin, 11, 20), xb, g)
    w4 = _ints((20, cin, 3, 3), wb, g)
    want = _conv_ref(x, w4, None, 0)
    for nchw in (False, True):
        assert exact(tc_conv(bf, nchw, x, w4, None, 0), want), nchw


def test_shared_conv_backward_dx_exact():
    """The dx convolution of the backward: the forward's packed weight flipped and transposed on the device, run on the
    3xTF32 path (_precise), equals the float64 input gradient bit for bit."""
    from deepinteraction_b200 import backward, fold
    g = _gen(77)
    n, cin, cout, H, W = 2, 256, 128, 9, 21
    x = _ints((n, cin, H, W), 3, g)
    w4 = _ints((cout, cin, 3, 3), 4, g)
    gy = _ints((n, cout, H, W), 4, g)
    wk = fold.Weight(fold.pack_conv3x3(w4), dev())
    with record_calls() as calls, backward._precise():
        dx, _ = backward._shared_conv_backward(gy.permute(0, 2, 3, 1).reshape(-1, cout).contiguous(), wk, x)
    assert [c[0] for c in calls if 'conv3x3' in c[0]] == ['di_conv3x3_tc_f32']
    want = torch.nn.grad.conv2d_input(x.shape, w4.double(), gy.double(), padding=1).permute(0, 2, 3, 1)
    assert exact(dx, want)


# ---------------------------------------------------------------------------------------------------------------------
# 5. FFMA linear (gemm.cu): small-M kernel / SGEMM boundary, loaders, stores, split-K
# ---------------------------------------------------------------------------------------------------------------------
# (M, N, K per source, column offset of the sources (misaligned pointer when % 4 != 0), res_mod, act, bias)
FFMA_SHAPES = [
    (640, 2048, [64], 0, None, 1, True),          # small-M kernel (M <= 640, N <= 2048)
    (641, 2048, [64], 0, None, 0, True),          # SGEMM
    (640, 2049, [64], 0, 97, 1, True),            # SGEMM, N > 2048: vector store with a scalar tail
    (641, 130, [64], 0, None, 0, True),           # SGEMM, ldc % 4 != 0: scalar store
    (1000, 132, [3, 10, 7], 0, None, 0, True),    # source boundaries inside a BK = 8 tile, K % 4 != 0: scalar loader
    (200, 64, [3, 10, 7], 0, 0, 1, True),         # the same on the small-M kernel
    (900, 128, [68], 1, None, 0, False),          # misaligned source pointer: scalar loader
    (5000, 36, [128, 64], 0, 97, 1, True),        # two sources, vector loader and store
]


@pytest.mark.parametrize('M,N,Ks,off,res_mod,act,has_bias', FFMA_SHAPES,
                         ids=['x'.join(map(str, (c[0], c[1], '+'.join(map(str, c[2]))))) + f'o{c[3]}' for c in FFMA_SHAPES])
def test_ffma_linear_exact(M, N, Ks, off, res_mod, act, has_bias):
    g = _gen(M * 3 + N)
    srcs = [_ints((M, k + off + 4), 4, g)[:, off:off + k] for k in Ks]
    cs = _pow2(N, -6, 6, g)
    W = _ints((N, sum(Ks)), 4, g) * cs[:, None]
    bias = _ints((N,), 10, g) * cs if has_bias else None
    res = _res(M, N, res_mod, g, lambda shape, g: _ints(shape, 8, g) * cs)
    buf, out = canvas(M, N, pad_cols=8 if N % 4 == 0 else 7)     # ldc % 4 != 0 with N: the scalar store
    assert ffma_linear(srcs, W, out, bias, res, res_mod or 0, act) == 1
    assert exact(out, ref_linear(srcs, W, bias, res, res_mod or 0, act))
    assert outside_intact(buf, M, N)


@pytest.mark.parametrize('M,N,K', [(641, 128, 256), (300, 2112, 128), (400, 128, 256)])
def test_ffma_linear_gelu_precision(M, N, K):
    """GELU in the SGEMM epilogue (M > 640 or N > 2048) and in the small-M kernel."""
    srcs, W, bias, res = _precision_case(M, N, [K], 97, True, M + N + K)
    out = torch.empty(M, N, device=dev())
    ffma_linear(srcs, W, out, bias, res, 97, 2)
    e = row_err(out, ref_linear(srcs, W, bias, res, 97, 2), scale_linear(srcs, W, bias, res, 97))
    print(f'ffma GELU M={M} N={N} K={K}: row err {e:.2e}')
    assert e < BARS['ffma'], e


@pytest.mark.parametrize('K,splits,n_expected', [(100, 6, 5), (100, 20, 13), (100, 4, 4), (100, 1, 1), (1000, 256, 125),
                                                 (1003, 7, 7)])
def test_ffma_split_k(K, splits, n_expected):
    """The returned partial count (splits capped at the k-tiles, and fewer when splits does not divide them), the unused
    partials untouched, the exact sum of the partials and its fixed-order reduction, and determinism."""
    M, N = 300, 132
    g = _gen(K + splits)
    A = _ints((M, K), 4, g)
    W = _ints((N, K), 4, g)
    want = ref_linear([A], W)
    buf = torch.full((splits + 1, M, N), SENT, dtype=torch.int32, device=dev()).view(torch.float32)
    n = ffma_linear([A], W, buf[0], splits=splits, split_stride=M * N)
    assert n == n_expected
    assert bool((buf[n:].view(torch.int32) == SENT).all())
    assert exact(buf[:n].double().sum(0), want)
    assert exact(_ops().rows_finish(buf[:n]) if n > 1 else buf[0], want)
    again = torch.empty_like(buf)
    assert ffma_linear([A], W, again[0], splits=splits, split_stride=M * N) == n
    assert same_bits(again[:n], buf[:n])


# ---------------------------------------------------------------------------------------------------------------------
# 6. FFMA 3x3 convolution
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('x_nhwc,y_nchw,n,cin,H,W,cout', [(False, False, 2, 3, 9, 21, 20), (False, True, 1, 5, 8, 17, 12),
                                                          (True, False, 3, 8, 5, 7, 12), (True, True, 2, 4, 1, 9, 6)])
def test_ffma_conv3x3_exact(x_nhwc, y_nchw, n, cin, H, W, cout):
    g = _gen(n + cin + H)
    x = _ints((n, cin, H, W), 4, g)
    w4 = _ints((cout, cin, 3, 3), 4, g)
    bias = _ints((cout,), 8, g)
    want = _conv_ref(x, w4, bias, 1)
    xin = x.permute(0, 2, 3, 1).contiguous() if x_nhwc else x
    y = torch.full((n * H * W * cout + 8,), SENT, dtype=torch.int32, device=dev()).view(torch.float32)
    _capi('di_conv3x3_f32', _p(xin), int(x_nhwc), _p(_fold().pack_conv3x3(w4).contiguous()), _p(bias), _p(y), int(y_nchw),
          n, cin, H, W, cout, 1)
    got = y[:-8].view(n, cout, H, W).permute(0, 2, 3, 1) if y_nchw else y[:-8].view(n, H, W, cout)
    assert exact(got, want)
    assert bool((y[-8:].view(torch.int32) == SENT).all())


# ---------------------------------------------------------------------------------------------------------------------
# 7. documented rejections: the error code, and the output untouched (no launch)
# ---------------------------------------------------------------------------------------------------------------------
def _rejection_cases():
    """name -> (entry point, args builder(A, W, out, hi/lo bf16, hi/lo tf32), expected status)."""
    def lin(bf, Ks=(64,), N=128, A_off=0, lda=None, split=None, res=False):
        def build(A, Wb, Wt, out, resb):
            hi, lo = Wb if bf else Wt
            ptr = ctypes.c_void_p(A.data_ptr() + 4 * A_off)
            a = []
            for k in Ks:
                a += [ptr if k else None, lda or A.stride(0), k]
            a += [None, 0, 0] * (3 - len(Ks))
            args = a + [_p(hi), _p(lo), None, _p(resb) if res else None, resb.stride(0) if res else 0, 0, _p(out),
                        out.stride(0), 256, N, 0]
            if split is not None:
                return ('di_linear_tcb_split_f32', args + list(split))
            return ('di_linear_tcb_f32' if bf else 'di_linear_tc_f32', args)
        return build

    def ffma(Ks=(64,), splits=1, res=False):
        def build(A, Wb, Wt, out, resb):
            a = []
            for k in Ks:
                a += [_p(A) if k else None, A.stride(0), k]
            a += [None, 0, 0] * (3 - len(Ks))
            return ('di_linear_f32', a + [_p(Wt[0]), None, _p(resb) if res else None, resb.stride(0) if res else 0, 0,
                                          _p(out), out.stride(0), 256, 128, 0, splits, 256 * 128])
        return build

    def conv(name, cin, W=16, x_nhwc=1):
        def build(A, Wb, Wt, out, resb):
            if name == 'di_conv3x3_f32':
                return (name, [_p(A), x_nhwc, _p(Wt[0]), None, _p(out), 0, 1, cin, 4, W, 128, 0])
            hi, lo = Wb if 'tcb' in name else Wt
            return (name, [_p(A), _p(hi), _p(lo), None, _p(out), 1, cin, 4, W, 128, 0])
        return build

    return {
        'tcb_K_not_multiple_of_64': (lin(True, Ks=(32,)), DI_ERR_UNSUPPORTED),
        'tc_K_not_multiple_of_32': (lin(False, Ks=(48,)), DI_ERR_UNSUPPORTED),
        'tcb_second_source_K_not_multiple_of_64': (lin(True, Ks=(64, 96)), DI_ERR_UNSUPPORTED),
        'tcb_N_not_multiple_of_4': (lin(True, N=126), DI_ERR_UNSUPPORTED),
        'tc_N_not_multiple_of_4': (lin(False, N=130), DI_ERR_UNSUPPORTED),
        'tcb_misaligned_A': (lin(True, A_off=1), DI_ERR_UNSUPPORTED),
        'tc_misaligned_A': (lin(False, A_off=2), DI_ERR_UNSUPPORTED),
        'tcb_lda_not_multiple_of_4': (lin(True, lda=130), DI_ERR_UNSUPPORTED),
        'tcb_K2_without_K1': (lin(True, Ks=(64, 0, 64)), DI_ERR_UNSUPPORTED),
        'split_kind_4': (lin(True, split=(0, 4)), DI_ERR_ARG),
        'split_kind_1_col0_16': (lin(True, split=(16, 1)), DI_ERR_ARG),
        'split_kind_2_negative_col0': (lin(True, split=(-32, 2)), DI_ERR_ARG),
        'split_kind_3_col0_64': (lin(True, split=(64, 3)), DI_ERR_ARG),
        'split_kind_3_N_96': (lin(True, N=96, split=(0, 3)), DI_ERR_ARG),
        'split_kind_1_N_100': (lin(True, N=100, split=(0, 1)), DI_ERR_ARG),
        'ffma_res_with_split_k': (ffma(splits=2, res=True), DI_ERR_ARG),
        'ffma_K2_without_K1': (ffma(Ks=(64, 0, 64)), DI_ERR_ARG),
        'ffma_conv_nhwc_cin_6': (conv('di_conv3x3_f32', 6), DI_ERR_ARG),
        'tcb_conv_cin_32': (conv('di_conv3x3_tcb_f32', 32), DI_ERR_UNSUPPORTED),
        'tc_conv_cin_48': (conv('di_conv3x3_tc_f32', 48), DI_ERR_UNSUPPORTED),
        'tcb_conv_nchw_W_10': (conv('di_conv3x3_tcb_nchw_f32', 64, W=10), DI_ERR_UNSUPPORTED),
        'tc_conv_cout_not_multiple_of_4': (None, DI_ERR_UNSUPPORTED),
    }


REJECTIONS = _rejection_cases()


@pytest.mark.parametrize('case', list(REJECTIONS))
def test_documented_rejections(case):
    build, want = REJECTIONS[case]
    g = _gen(3)
    A = _normal((256, 1024), g)
    W = _normal((128, 4608), g)
    Wb, Wt = _wsplit(W, True), _wsplit(W, False)
    resb = _normal((256, 128), g)
    buf = torch.full((2, 256 * 256 * 2), SENT, dtype=torch.int32, device=dev()).view(torch.float32)
    out = buf[0].view(512, 256)[:256, :128]
    if build is None:                          # Cout = 126 on the tensor-core conv
        Wt126 = _wsplit(W[:126], False)
        name, args = 'di_conv3x3_tc_f32', [_p(A), _p(Wt126[0]), _p(Wt126[1]), None, _p(out), 1, 32, 4, 16, 126, 0]
    else:
        name, args = build(A, Wb, Wt, out, resb)
    assert _status(name, *args) == want
    assert bool((buf.view(torch.int32) == SENT).all())


# ---------------------------------------------------------------------------------------------------------------------
# 8. routing and the production calls of the base model
# ---------------------------------------------------------------------------------------------------------------------
DENSE = ('di_linear_f32', 'di_linear_tc_f32', 'di_linear_tcb_f32', 'di_linear_tcb_split_f32', 'di_conv3x3_f32',
         'di_conv3x3_tc_f32', 'di_conv3x3_tcb_f32', 'di_conv3x3_tc_nchw_f32', 'di_conv3x3_tcb_nchw_f32')
PILLARS = 'pillars'   # a row count or K equal to the frame's number of pillars (MMRI_I2P backward); tested at 24000
PILLARS_TESTED = 24000


def call_key(name, args):
    """The shape signature of a dense C call: ('linear', entry, M, N, K per source, act, residual, splits) or
    ('conv', entry, images, Cin, H, W, Cout, act)."""
    if 'conv3x3' in name:
        if name == 'di_conv3x3_f32':
            return ('conv', name) + tuple(args[6:12])
        return ('conv', name) + tuple(args[5:11])
    Ks = tuple(k for k in (args[2], args[5], args[8]) if k)
    if name == 'di_linear_f32':
        return ('linear', name, args[16], args[17], Ks, args[18], args[11] is not None, args[19])
    return ('linear', name, args[17], args[18], Ks, args[19], args[12] is not None, 1)


# Every dense call of the base model (projects/configs/nuscenes/di_b200_base_hotpath.py: 6 views of 112 x 200 image
# features with 256 channels, a 180 x 180 BEV map with 512 channels, hidden width 128, 200 proposals, 10 classes).
# FWD_TABLE: the forward of mmri.py (encoder, bf16 split) and mmpi.py (decoder, 3xTF32).  The LCAB projections of the
# base width run in the fused di_lcab_forward_f32 and the query-row layers of the decoder in di_rows_mlp_f32: neither
# is a dense call.  BWD_TABLE: the calls of backward.py's encoder_backward, decoder_layer_backward and
# point_rcnn_backward (both PointRCNN blocks) that the forward does not already make; everything there runs under
# _precise (3xTF32), the weight gradients dy^T x on the FFMA kernel with split-K over the rows (_wgrad), and the forward
# intermediates are recomputed.  Key: ('linear', entry, M, N, K per source, act, residual, splits) or
# ('conv', entry, images, Cin, H, W, Cout, act).  One guard test per table keeps it complete.
FWD_TABLE = {
    ('conv', 'di_conv3x3_tcb_f32', 6, 256, 112, 200, 128, 0): 'encoder shared_conv_img (NCHW input transposed)',
    ('conv', 'di_conv3x3_tcb_f32', 1, 512, 180, 180, 128, 0): 'encoder shared_conv_pts (NCHW input transposed)',
    ('linear', 'di_linear_tcb_f32', 32400, 128, (128,), 0, False, 1):
        'encoder MMRI_I2P qk = M1 rows + c1 and out = M2 s + c2, over the pillar rows staged at the capacity B * Y * X',
    ('linear', 'di_linear_tcb_f32', 32400, 128, (128, 128, 128), 0, False, 1): 'encoder P_out_proj + P_integration',
    ('linear', 'di_linear_tcb_f32', 134400, 128, (128, 128, 128), 0, False, 1): 'encoder I_out_proj + I_integration',
    ('conv', 'di_conv3x3_tc_f32', 1, 128, 180, 180, 128, 1): 'decoder heatmap_head[_img] conv 0 (ReLU)',
    ('conv', 'di_conv3x3_tc_f32', 1, 128, 180, 180, 12, 0): 'decoder heatmap_head[_img] conv 1 (10 classes, padded to 12)',
    ('linear', 'di_linear_tc_f32', 32400, 256, (128,), 0, True, 1): 'decoder cross-attention K | V of the BEV map (+ pos)',
    ('linear', 'di_linear_tc_f32', 200, 32768, (128,), 0, False, 1): 'decoder DynamicConv parameter generator',
    ('linear', 'di_linear_f32', 200, 128, (6272,), 0, False, 49): 'decoder DynamicConv output layer (split-K 49)',
}
BWD_TABLE = {
    ('conv', 'di_conv3x3_tc_f32', 6, 256, 112, 200, 128, 0):
        'encoder recompute: shared_conv_img',
    ('conv', 'di_conv3x3_tc_f32', 1, 512, 180, 180, 128, 0):
        'encoder recompute: shared_conv_pts',
    ('conv', 'di_conv3x3_tc_f32', 6, 128, 112, 200, 256, 0):
        'shared_conv_img dx (flipped, transposed weight)',
    ('conv', 'di_conv3x3_tc_f32', 1, 128, 180, 180, 512, 0):
        'shared_conv_pts dx (flipped, transposed weight)',
    ('linear', 'di_linear_tc_f32', 32400, 128, (128, 128, 128), 0, False, 1):
        'encoder recompute P fuse; BEV LCAB dX [dq1 | dk1 | dv] self1^T',
    ('linear', 'di_linear_tc_f32', 134400, 384, (128,), 1, False, 1):
        'image LCAB recompute q1 | k1 | v (self attention)',
    ('linear', 'di_linear_tc_f32', 32400, 384, (128,), 1, False, 1):
        'BEV LCAB recompute q1 | k1 | v (self attention)',
    ('linear', 'di_linear_tc_f32', 134400, 256, (128,), 1, False, 1):
        'P2I LCAB recompute k1 | v of the warped BEV rows',
    ('linear', 'di_linear_tc_f32', 134400, 128, (128,), 1, False, 1):
        'image LCAB recompute q1 (P2I), q2, k2',
    ('linear', 'di_linear_tc_f32', 32400, 128, (128,), 1, False, 1):
        'BEV LCAB recompute q2, k2',
    ('linear', 'di_linear_tc_f32', PILLARS, 128, (128,), 0, False, 1):
        'I2P recompute qk = M1 rows; dX ds = do M2^T, drows = dqk M1^T',
    ('linear', 'di_linear_tc_f32', 134400, 384, (128,), 0, False, 1):
        'I fuse dX: d [p2i | i2i | img] = d new_img Wf',
    ('linear', 'di_linear_tc_f32', 32400, 384, (128,), 0, False, 1):
        'P fuse dX: d [i2p | p2p | pts] = d new_pts Wf',
    ('linear', 'di_linear_tc_f32', 134400, 128, (128, 128, 128), 0, False, 1):
        'image LCAB dX [dq1 | dk1 | dv] self1^T',
    ('linear', 'di_linear_tc_f32', 134400, 128, (128, 128), 0, False, 1):
        'P2I LCAB dX [dk1 | dv] kv1^T',
    ('linear', 'di_linear_tc_f32', 134400, 128, (128,), 0, False, 1):
        'image LCAB dX dq q2^T, dk k2^T, dq1 q1^T',
    ('linear', 'di_linear_tc_f32', 32400, 128, (128,), 0, False, 1):
        'BEV LCAB dX dq q2^T, dk k2^T; decoder layer key pos-MLP dX cpe2^T',
    ('linear', 'di_linear_tc_f32', 32400, 128, (256,), 0, False, 1):
        'decoder layer d bev = d kv W_kv',
    ('linear', 'di_linear_tc_f32', 200, 128, (128,), 0, False, 1):
        'query-row dX: cross_out^T, cross_q^T, self_out^T, spe2^T, attn_out^T',
    ('linear', 'di_linear_tc_f32', 200, 256, (128,), 0, False, 1):
        'decoder layer FFN dX dz ffn2^T',
    ('linear', 'di_linear_tc_f32', 200, 128, (256,), 0, True, 1):
        'decoder layer FFN dX dh ffn1^T + dz',
    ('linear', 'di_linear_tc_f32', 200, 128, (384,), 0, False, 1):
        'decoder layer self-attention dX dqkv self_in^T',
    ('linear', 'di_linear_tc_f32', 200, 512, (128,), 0, False, 1):
        'PointRCNN FFN dX dz ffn2^T',
    ('linear', 'di_linear_tc_f32', 200, 128, (512,), 0, True, 1):
        'PointRCNN FFN dX dh ffn1^T + dz',
    ('linear', 'di_linear_tc_f32', 200, 6272, (128,), 0, False, 1):
        'PointRCNN DynamicConv out_layer dX dzd3 dout^T',
    ('linear', 'di_linear_tc_f32', 200, 128, (384,), 0, True, 1):
        'PointRCNN self-attention dX dqkv attn_in^T + dz1',
    ('linear', 'di_linear_f32', 200, 128, (32768,), 0, False, 64):
        'PointRCNN DynamicConv generator dX d params W_dyn (split-K 64)',
    ('linear', 'di_linear_f32', 128, 128, (134400,), 0, False, 256):
        'weight gradients over the image pixels (LCAB, I fuse)',
    ('linear', 'di_linear_f32', 128, 128, (32400,), 0, False, 63):
        'weight gradients over the BEV pixels (LCAB, P fuse)',
    ('linear', 'di_linear_f32', 128, 256, (134400,), 0, False, 256):
        'shared_conv_img dW per tap over the shifted input',
    ('linear', 'di_linear_f32', 128, 512, (32400,), 0, False, 63):
        'shared_conv_pts dW per tap over the shifted input',
    ('linear', 'di_linear_f32', 128, 128, (PILLARS,), 0, False, PILLARS):
        'I2P dM1, dM2 over the pillars',
    ('linear', 'di_linear_f32', 256, 128, (32400,), 0, False, 63):
        'decoder layer cross_kv dW over the BEV rows',
    ('linear', 'di_linear_f32', 128, 2, (32400,), 0, False, 63):
        'decoder layer key pos-MLP conv 0 dW over the grid positions',
    ('linear', 'di_linear_f32', 128, 2, (200,), 0, False, 1):
        'decoder layer query pos-MLP conv 0 dW',
    ('linear', 'di_linear_f32', 128, 128, (200,), 0, False, 1):
        'query-row weight gradients: out_proj, cross_q, pos-MLP conv 1',
    ('linear', 'di_linear_f32', 128, 256, (200,), 0, False, 1):
        'decoder layer FFN linear2 dW; cross_q dW over [q1 | qpe]',
    ('linear', 'di_linear_f32', 256, 128, (200,), 0, False, 1):
        'decoder layer FFN linear1 dW',
    ('linear', 'di_linear_f32', 384, 256, (200,), 0, False, 1):
        'decoder layer self_in dW over [query | qpe]',
    ('linear', 'di_linear_f32', 384, 128, (200,), 0, False, 1):
        'PointRCNN attention in_proj dW',
    ('linear', 'di_linear_f32', 128, 512, (200,), 0, False, 1):
        'PointRCNN FFN linear2 dW',
    ('linear', 'di_linear_f32', 512, 128, (200,), 0, False, 1):
        'PointRCNN FFN linear1 dW',
    ('linear', 'di_linear_f32', 128, 6272, (200,), 0, False, 1):
        'PointRCNN DynamicConv out_layer dW',
    ('linear', 'di_linear_f32', 32768, 128, (200,), 0, False, 1):
        'PointRCNN DynamicConv generator dW',
}


def _sample_rows(M, g, images=None, hw=None):
    rows = {0, 127, 128, M - 1}
    if images:
        for i in range(images):
            rows |= {i * hw, (i + 1) * hw - 1}
    rows |= set(torch.randint(0, M, (600,), generator=g, device=dev()).tolist())
    return torch.tensor(sorted(r for r in rows if r < M), device=dev())


def _mode_of(name):
    return 'ffma' if name in ('di_linear_f32', 'di_conv3x3_f32') else 'bf16' if 'tcb' in name else 'tf32'


@contextlib.contextmanager
def _bf16(on):
    ops = _ops()
    saved, ops.TC_BF16[0] = ops.TC_BF16[0], on
    try:
        yield
    finally:
        ops.TC_BF16[0] = saved


def _run_linear_entry(key, g):
    _, name, M, N, Ks, act, has_res, splits = key
    ops, fold = _ops(), _fold()
    M = PILLARS_TESTED if M == PILLARS else M
    if Ks == (PILLARS,):                          # weight gradient over the pillars: _wgrad's split count
        Ks, splits = (PILLARS_TESTED,), max(1, min(256, PILLARS_TESTED // 512))
    srcs = [_normal((M, k), g) for k in Ks]
    Wf = _normal((N, sum(Ks)), g) / sum(Ks) ** 0.5
    bias = _normal((N,), g) if splits == 1 else None
    res = _normal((M, N), g) if has_res else None
    with record_calls() as calls, _bf16('tcb' in name):
        if splits > 1:
            part = ops.linear(srcs, Wf, splits=splits)
            out = ops.rows_finish(part) if part.shape[0] > 1 else part[0]
        else:                                     # the FFMA entries of the table take a plain weight tensor
            w = Wf if name == 'di_linear_f32' else fold.Weight(Wf, dev())
            out = ops.linear(srcs, w, bias, act, res=res, res_mod=M if has_res else 0)
    assert call_key(*calls[0]) == ('linear', name, M, N, Ks, act, has_res, splits), call_key(*calls[0])
    rows = _sample_rows(M, g)
    sub = [s[rows] for s in srcs]
    rsub = None if res is None else res[rows]
    return (row_err(out[rows], ref_linear(sub, Wf, bias, rsub, 0, act), scale_linear(sub, Wf, bias, rsub, 0)),
            calls[0][0])


def _conv_at(x, w4, bias, pix, act):
    """float64 3x3 convolution of NCHW x at the flat output pixels pix -> ([P, Cout] values, [P, Cout] term scale)."""
    n, cin, H, W = x.shape
    xp = F.pad(x.double(), (1, 1, 1, 1))
    img, yx = pix // (H * W), pix % (H * W)
    yy, xx = yx // W, yx % W
    cols = torch.stack([xp[img, :, yy + ky, xx + kx] for ky in range(3) for kx in range(3)], 2)   # [P, cin, 9]
    wm = w4.double().reshape(w4.shape[0], cin * 9)
    cols = cols.reshape(len(pix), cin * 9)
    y = cols @ wm.t() + bias.double()
    return _act(y, act), cols.abs() @ wm.abs().t() + bias.double().abs()


def _run_conv_entry(key, g):
    _, name, n, cin, H, W, cout, act = key
    ops, fold = _ops(), _fold()
    x = _normal((n, cin, H, W), g)
    w4 = _normal((cout, cin, 3, 3), g) / (9 * cin) ** 0.5
    bias = _normal((cout,), g)
    with record_calls() as calls, _bf16('tcb' in name):
        y = ops.conv3x3(x if 'nchw' in name or 'tcb' in name else x.permute(0, 2, 3, 1).contiguous(),
                        fold.Weight(fold.pack_conv3x3(w4), dev()), bias, cout, 'tcb' not in name, False, act)
    assert call_key(*[c for c in calls if c[0] in DENSE][0]) == key
    pix = _sample_rows(n * H * W, g, n, H * W)
    want, scale = _conv_at(x, w4, bias, pix, act)
    return row_err(y.reshape(-1, cout)[pix], want, scale), name


@pytest.mark.parametrize('key', list(FWD_TABLE) + list(BWD_TABLE), ids=lambda k: '-'.join(map(str, k[1:])))
def test_production_dense_calls(key):
    """Every table entry at its real size through ops (the entry point it takes is asserted), against float64 on a
    sample of rows that includes 0, 127, 128, M - 1 and the first and last pixel of every image."""
    g = _gen(zlib.crc32(repr(key).encode()))
    e, name = (_run_conv_entry if key[0] == 'conv' else _run_linear_entry)(key, g)
    mode = _mode_of(name)
    K = 9 * key[3] if key[0] == 'conv' else PILLARS_TESTED if key[4] == (PILLARS,) else sum(key[4])
    print(f'production {FWD_TABLE.get(key) or BWD_TABLE.get(key)}: {mode} row err {e:.2e}')
    assert e < bar(mode, K), e


def test_production_table_covers_base_forward():
    """One base-shape forward of encoder and decoder: every dense call it issues is in the table."""
    import bench
    from deepinteraction_b200 import synth
    neck, head = bench.build_models(dev())
    fr = synth.to_device(synth.make_frame_batch(bench.SEED + 5, batch=1, cloud='lidar'), dev())
    with torch.no_grad(), record_calls() as calls:
        img, pts = neck(fr['img_feats'], fr['pts_feats'], fr['img_metas'], fr['pts_metas'])
        head(pts, img, fr['img_metas'])
    torch.cuda.synchronize()
    keys = {call_key(n, a) for n, a in calls if n in DENSE}
    print('base forward dense calls:', sorted(keys, key=str))
    missing = sorted(keys - set(FWD_TABLE), key=str)
    assert not missing, missing


def _pillar_key(k, n_pillars):
    """A linear call key with the frame's pillar count (as M, or as the K of a weight gradient with its split count)
    replaced by PILLARS."""
    if k[0] != 'linear':
        return k
    if k[2] == n_pillars:
        k = k[:2] + (PILLARS,) + k[3:]
    if k[4] == (n_pillars,):
        k = k[:4] + ((PILLARS,), k[5], k[6], PILLARS)
    return k


def test_production_table_covers_base_backward():
    """One base-shape run of backward.encoder_backward, decoder_layer_backward and point_rcnn_backward (both PointRCNN
    blocks): every dense call they issue is in the table."""
    import bench
    from deepinteraction_b200 import backward, synth
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
        backward.encoder_backward(neck, fr['img_feats'], fr['pts_feats'], fr['img_metas'], pm, _normal((BV, h, w, 128), g),
                                  _normal((B, Y, X, 128), g), _normal((B, Y, X, 128), g))
        m = layer_decoder(True, False)
        backward.decoder_layer_backward(m, *(t.to(d) for t in _layer_inputs(m, 1, 91)))
        m = rcnn_decoder(True)
        for li in (1, 3):
            backward.point_rcnn_backward(m, li, *(t.to(d) for t in _block_inputs(m, 1, BLOCK_SEEDS[(True, li)])))
    torch.cuda.synchronize()
    keys = {_pillar_key(call_key(n, a), n_pillars) for n, a in calls if n in DENSE}
    print('base backward dense calls:', sorted(keys, key=str))
    missing = sorted(keys - set(FWD_TABLE) - set(BWD_TABLE), key=str)
    assert not missing, missing


def test_conv3x3_routing_of_nchw_direct():
    """ops.conv3x3 takes the NCHW-direct kernel exactly when it is enabled and W % 4 == 0."""
    ops, fold = _ops(), _fold()
    g = _gen(9)
    w = fold.Weight(fold.pack_conv3x3(_normal((128, 64, 3, 3), g)), dev())
    saved = ops.NCHW_DIRECT[0]
    try:
        for direct in (False, True):
            ops.NCHW_DIRECT[0] = direct
            for W, want in ((50, 'di_conv3x3_tcb_f32'), (44, 'di_conv3x3_tcb_nchw_f32' if direct else 'di_conv3x3_tcb_f32')):
                with record_calls() as calls:
                    ops.conv3x3(_normal((1, 64, 8, W), g), w, None, 128, False)
                assert [c[0] for c in calls if c[0] in DENSE] == [want], (direct, W)
    finally:
        ops.NCHW_DIRECT[0] = saved
