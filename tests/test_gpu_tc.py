"""GPU parity of the wgmma (split-product, TMA-staged) dense kernels vs float64 references, and FFMA/TC agreement.
Both operand precisions (bf16 split = the default where K % 64 == 0, and 3xTF32) and both weight placements."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from conftest import rel_err
from kernel_check import record_calls

pytestmark = pytest.mark.gpu
TIGHT = 5e-5


def dev():
    return torch.device('cuda:0')


@pytest.fixture(params=[(3, True), (4, True), (3, False), (4, False)],
                ids=['bf16split+W-resident', 'bf16split+W-streamed', '3xtf32+W-resident', '3xtf32+W-streamed'])
def tc_mode(request):
    from deepinteraction_b200 import _lib, ops
    mode, bf = request.param
    _lib.check(_lib.lib().di_tc_set_mode(mode))
    old = ops.TC_BF16[0]
    ops.TC_BF16[0] = bf
    yield request.param
    ops.TC_BF16[0] = old
    _lib.lib().di_tc_set_mode(3)


@pytest.mark.parametrize('M,N,Ks,act,use_res', [
    (128, 128, [128], 1, False), (1000, 128, [128], 0, False), (32400, 128, [128, 128, 128], 0, False),
    (777, 384, [128], 1, False), (4096, 256, [64, 32], 2, True), (4096, 256, [64, 128], 2, True),
    (200, 32768, [128], 0, False),
    (300, 20, [384], 0, False), (50001, 128, [256], 1, True)])
def test_linear_tc_matches_float64(M, N, Ks, act, use_res, tc_mode):
    from deepinteraction_b200 import ops, fold
    g = torch.Generator().manual_seed(M + N)
    srcs = [torch.randn(M, k, generator=g) * (1 + i) for i, k in enumerate(Ks)]
    W = torch.randn(N, sum(Ks), generator=g) / np.sqrt(sum(Ks))
    b = torch.randn(N, generator=g)
    res = torch.randn(97, N, generator=g) if use_res else None
    ref = torch.cat(srcs, 1).double() @ W.double().t() + b.double()
    if use_res:
        ref = ref + res.double()[torch.arange(M) % 97]
    ref = {0: lambda x: x, 1: F.relu, 2: F.gelu}[act](ref).float()
    Wt = fold.Weight(W, dev())
    n0 = ops.LAUNCHES[0]
    out = ops.linear([s.to(dev()) for s in srcs], Wt, b.to(dev()), act, res=None if res is None else res.to(dev()),
                     res_mod=97 if use_res else 0)
    e = rel_err(out.cpu(), ref)
    print(f'linear_tc M={M} N={N} K={Ks}: rel err {e:.2e}')
    assert e < TIGHT


def test_linear_tc_strided_sources_and_ffma_agreement():
    from deepinteraction_b200 import ops, fold
    g = torch.Generator().manual_seed(5)
    big = torch.randn(5000, 384, generator=g).to(dev())
    W = torch.randn(128, 128, generator=g) / 11
    Wt = fold.Weight(W, dev())
    a = ops.linear([big[:, 128:256]], Wt, act=ops.ACT_RELU)
    ops.USE_TC[0] = False
    try:
        b = ops.linear([big[:, 128:256]], Wt, act=ops.ACT_RELU)
    finally:
        ops.USE_TC[0] = True
    ref = F.relu(big[:, 128:256].cpu().double() @ W.double().t()).float()
    assert rel_err(a.cpu(), ref) < TIGHT and rel_err(b.cpu(), ref) < TIGHT
    # the compensated products must be far better than a single TF32 / BF16 pass (~5e-4 / 4e-3)
    assert rel_err(a.cpu(), ref) < 1e-5
    ops.TC_BF16[0] = False
    try:
        c = ops.linear([big[:, 128:256]], Wt, act=ops.ACT_RELU)
    finally:
        ops.TC_BF16[0] = True
    assert rel_err(c.cpu(), ref) < 2e-6


@pytest.mark.parametrize('N,Cin,H,W,Cout,nhwc_in,act', [(1, 32, 8, 16, 128, True, 0), (2, 128, 37, 45, 128, True, 1),
                                                          (6, 256, 28, 50, 128, False, 0), (1, 64, 180, 180, 128, False, 0),
                                                          (1, 128, 5, 7, 256, True, 1), (2, 128, 37, 44, 128, False, 1),
                                                          (1, 64, 9, 200, 20, False, 0)])
def test_conv3x3_tc_matches_float64(N, Cin, H, W, Cout, nhwc_in, act, tc_mode):
    from deepinteraction_b200 import ops, fold
    g = torch.Generator().manual_seed(N * 100 + Cin)
    x = torch.randn(N, Cin, H, W, generator=g)
    w = torch.randn(Cout, Cin, 3, 3, generator=g) / np.sqrt(9 * Cin)
    b = torch.randn(Cout, generator=g)
    ref = F.conv2d(x.double(), w.double(), b.double(), padding=1)
    if act:
        ref = F.relu(ref)
    xin = x.permute(0, 2, 3, 1).contiguous() if nhwc_in else x
    Wt = fold.Weight(fold.pack_conv3x3(w), dev())
    # NCHW inputs: via transposition, and read in place where the direct kernel applies (W % 4 == 0)
    for direct in ((False,) if nhwc_in or W % 4 else (False, True)):
        old = ops.NCHW_DIRECT[0]
        ops.NCHW_DIRECT[0] = direct
        try:
            with record_calls() as calls:
                y = ops.conv3x3(xin.to(dev()), Wt, b.to(dev()), Cout, nhwc_in, False, act).cpu().permute(0, 3, 1, 2)
        finally:
            ops.NCHW_DIRECT[0] = old
        bf = ops.TC_BF16[0] and Cin % 64 == 0
        assert [c[0] for c in calls if 'conv3x3' in c[0]] == ['di_conv3x3_tc%s%s_f32' % ('b' if bf else '',
                                                                                        '_nchw' if direct else '')]
        e = rel_err(y, ref.float())
        print(f'conv_tc N={N} Cin={Cin} {H}x{W} direct={direct}: rel err {e:.2e}')
        assert e < TIGHT


def test_bf16_split_keeps_16_bits():
    from deepinteraction_b200 import fold
    w = torch.randn(4096) * torch.logspace(-6, 6, 4096)
    hi, mid = fold.split_bf16(w)
    assert hi.dtype == torch.bfloat16 and mid.dtype == torch.bfloat16
    err = (hi.float() + mid.float() - w).abs() / w.abs()
    assert float(err.max()) <= 2.0 ** -17


def test_tf32_split_is_exact():
    from deepinteraction_b200 import fold
    w = torch.randn(4096) * torch.logspace(-6, 6, 4096)
    hi, lo = fold.split_tf32(w)
    assert int((hi.view(torch.int32) & 0x1FFF).abs().max()) == 0
    assert torch.equal(hi + lo, w)
    assert float((lo.abs() / w.abs()).max()) <= 2.0 ** -11
