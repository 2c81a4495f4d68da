"""Tests of the NHWC tensor-core 3x3 convolution (csrc/conv_tc.cu) where test_gpu_dense_kernels.py does not reach: the
16-column tile that serves Cout <= 16, several channel chunks through the double-buffered halo ring (3xTF32) and the
tap-major steps (bf16 split), and the persistent grid's tile striding under every SM limit.

Exact cases use integer operands scaled by powers of two per output column, with every partial sum below 2^24, so any
correct kernel equals the float64 result bit for bit; the output canvas has sentinel rows past the last pixel that
must keep their bits."""
import os

import pytest
import torch
import torch.nn.functional as F

from kernel_check import _capi, same_bits

pytestmark = pytest.mark.gpu

SENT = 0x7FA5A5A5
SM_LIMITS = (0, 1, 7, 131)


def dev():
    return torch.device('cuda:0')


def _gen(seed):
    return torch.Generator(device='cuda').manual_seed(seed)


def _ints(shape, bits, g):
    m = (1 << bits) - 1
    return torch.randint(-m, m + 1, shape, generator=g, device=dev()).float()


def _split(w4, bf):
    from deepinteraction_b200 import fold
    wk = fold.Weight(fold.pack_conv3x3(w4), dev())
    return (wk.bh, wk.bm) if bf else (wk.hi, wk.lo)


def conv(bf, x, w4, bias, act, ws=None):
    """x: NCHW on the device, passed to di_conv3x3_tc[b]_f32 as NHWC; returns NHWC."""
    from deepinteraction_b200 import ops
    N, Cin, H, W = x.shape
    Cout = w4.shape[0]
    hi, lo = ws if ws is not None else _split(w4, bf)
    buf = torch.full((N * H * W + 5, Cout), SENT, dtype=torch.int32, device=dev()).view(torch.float32)
    _capi('di_conv3x3_tc%s_f32' % ('b' if bf else ''), ops._ptr(x.permute(0, 2, 3, 1).contiguous()), ops._ptr(hi),
          ops._ptr(lo), ops._ptr(bias), ops._ptr(buf), N, Cin, H, W, Cout, act)
    assert bool((buf[N * H * W:].view(torch.int32) == SENT).all())
    return buf[:N * H * W].view(N, H, W, Cout)


def want(x, w4, bias, act):
    y = F.conv2d(x.double(), w4.double(), None if bias is None else bias.double(), padding=1)
    return (y.clamp_min(0) if act else y).permute(0, 2, 3, 1)


def exact(got, ref):
    return same_bits(got.float() + 0.0, ref.float() + 0.0)


# (images, Cin, H, W, Cout, act): partial tiles in y and x; Cout <= 16 takes the 16-column tile; Cin = 256 runs
# four (bf16) or eight (3xTF32) channel chunks; the production frame sizes take other tile shapes than 8 x 16 on a
# 132-SM H100 (7 x 18 at 180 x 180, 16 x 8 for six 112 x 200 maps)
EXACT = [(2, 64, 13, 21, 4, 1), (1, 64, 9, 17, 12, 0), (3, 128, 8, 16, 16, 1), (1, 256, 20, 33, 16, 0),
         (1, 256, 11, 35, 128, 1), (2, 128, 5, 50, 24, 0), (1, 64, 180, 180, 16, 1), (1, 64, 180, 180, 128, 0),
         (6, 64, 112, 200, 128, 1)]


@pytest.mark.parametrize('n,cin,H,W,cout,act', EXACT, ids=['x'.join(map(str, c[:5])) for c in EXACT])
@pytest.mark.parametrize('bf', [True, False], ids=['bf16split', '3xtf32'])
def test_conv3x3_nhwc_exact(bf, n, cin, H, W, cout, act):
    g = _gen(n * 7919 + cin * 31 + W * 7 + cout)
    x = _ints((n, cin, H, W), 4, g)
    cs = torch.exp2(torch.randint(-6, 7, (cout,), generator=g, device=dev()).float())
    w4 = _ints((cout, cin, 3, 3), 4, g) * cs[:, None, None, None]
    bias = _ints((cout,), 10, g) * cs
    assert exact(conv(bf, x, w4, bias, act), want(x, w4, bias, act))


@pytest.mark.parametrize('cout', [12, 256])
@pytest.mark.parametrize('bf', [True, False], ids=['bf16split', '3xtf32'])
def test_conv3x3_nhwc_same_bits_for_every_sm_limit(bf, cout):
    """The grid and the tile shape picked for it change with the SM limit (limit 1 takes 7 x 17 tiles here), the steps of
    a pixel's sum do not: every SM limit gives the same bits."""
    from deepinteraction_b200 import _lib
    L = _lib.lib()
    g = _gen(11 + cout + bf)
    x = torch.randn((2, 128, 37, 50), generator=g, device=dev())
    w4 = torch.randn((cout, 128, 3, 3), generator=g, device=dev()) / 34
    bias = torch.randn((cout,), generator=g, device=dev())
    ws = _split(w4, bf)
    outs = []
    try:
        for lim in SM_LIMITS:
            assert L.di_tc_set_sm_limit(lim) == 0
            outs.append(conv(bf, x, w4, bias, 1, ws))
    finally:
        L.di_tc_set_sm_limit(int(os.environ.get('DI_B200_TC_SMS', '0')))
    for lim, o in zip(SM_LIMITS[1:], outs[1:]):
        assert same_bits(o, outs[0]), lim
    ref = want(x, w4, bias, 1)
    err = float(((outs[0].double() - ref).abs().max() / ref.abs().max()).item())
    assert err < (1e-4 if bf else 1e-5), err
