"""GPU: the fused LCAB projection kernel (di_lcab_proj_f32, mode 1) equals the five-launch chain (mode 0) bit for bit:
every row count around the 64-row work items, self and cross attention, strided input views, small grids (the
Q / K / V role partition must cover every work item) and two streams running it at once."""
import os

import pytest
import torch

pytestmark = pytest.mark.gpu
C = 128


def dev():
    return torch.device('cuda:0')


def weights(g):
    from deepinteraction_b200 import fold
    w1 = fold.Weight(torch.randn(3 * C, C, generator=g) / 11, dev())
    w2 = fold.Weight(torch.randn(2 * C, C, generator=g) / 11, dev())
    b1, b2 = torch.randn(3 * C, generator=g).to(dev()), torch.randn(2 * C, generator=g).to(dev())
    return w1, b1, w2, b2


def proj(fused, xt, xs, w):
    from deepinteraction_b200 import ops
    ops.set_lcab_fused(fused)
    try:
        return [t.contiguous().view(torch.int32).clone() for t in ops.lcab_proj(xt, xs, *w)]
    finally:
        ops.set_lcab_fused(True)


def assert_equal(got, want):
    for name, a, b in zip('qkv', got, want):
        assert torch.equal(a, b), f'{name}: {int((a != b).sum())} words differ'


@pytest.mark.parametrize('self_attn', [True, False])
@pytest.mark.parametrize('M', [1, 127, 128, 129, 1000, 32400, 134400])
def test_fused_equals_chain(M, self_attn):
    g = torch.Generator().manual_seed(M + 7 * self_attn)
    w = weights(g)
    xt = torch.randn(M, C, generator=g).to(dev())
    xs = xt if self_attn else torch.randn(M, C, generator=g).to(dev())
    assert_equal(proj(True, xt, xs, w), proj(False, xt, xs, w))


@pytest.mark.parametrize('self_attn', [True, False])
def test_fused_strided_views(self_attn):
    """x_t / x_s as column views of wider row-major tensors (ld > 128)."""
    g = torch.Generator().manual_seed(31)
    M = 3001
    w = weights(g)
    wide_t = torch.randn(M, 3 * C, generator=g).to(dev())
    xt = wide_t[:, C:2 * C]
    xs = xt if self_attn else torch.randn(M, 2 * C + 32, generator=g).to(dev())[:, 32:32 + C]
    got = proj(True, xt, xs, w)
    assert_equal(got, proj(False, xt, xs, w))
    assert_equal(got, proj(True, xt.contiguous(), xt.contiguous() if self_attn else xs.contiguous(), w))


@pytest.mark.parametrize('sms', [3, 5, 7])
def test_fused_small_grids(sms):
    """With at most 3 / 5 / 7 CTAs (one or two per role) every work item is still computed."""
    from deepinteraction_b200 import _lib
    L = _lib.lib()
    g = torch.Generator().manual_seed(sms)
    M = 20000 + 37
    w = weights(g)
    xt = torch.randn(M, C, generator=g).to(dev())
    xs = torch.randn(M, C, generator=g).to(dev())
    want = proj(False, xt, xs, w)
    _lib.check(L.di_tc_set_sm_limit(sms), 'di_tc_set_sm_limit')
    try:
        got = proj(True, xt, xs, w)
    finally:
        # the limit has no getter: back to the process default (ops.py reads DI_B200_TC_SMS once at import)
        _lib.check(L.di_tc_set_sm_limit(int(os.environ.get('DI_B200_TC_SMS', '0'))), 'di_tc_set_sm_limit')
    assert_equal(got, want)


def test_fused_two_streams():
    """Two streams running the fused kernel on different inputs at the same time == sequential runs."""
    from deepinteraction_b200 import ops
    g = torch.Generator().manual_seed(41)
    M = 134400
    ins = []
    for _ in range(2):
        w = weights(g)
        xt = torch.randn(M, C, generator=g).to(dev())
        ins.append((xt, torch.randn(M, C, generator=g).to(dev()), w))
    want = [proj(True, xt, xs, w) for xt, xs, w in ins]
    streams = [torch.cuda.Stream() for _ in ins]
    torch.cuda.synchronize()
    outs = [None, None]
    for rep in range(3):
        for i, ((xt, xs, w), s) in enumerate(zip(ins, streams)):
            with torch.cuda.stream(s):
                outs[i] = ops.lcab_proj(xt, xs, *w)
        torch.cuda.synchronize()
        for got, ref in zip(outs, want):
            assert_equal([t.contiguous().view(torch.int32) for t in got], ref)
