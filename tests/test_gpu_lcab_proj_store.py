"""GPU: the fused LCAB projection kernel stores q / k / v by TMA, which must not write past row M: with the outputs as
views into larger buffers, the guard rows after row M come back untouched and rows < M equal the five-launch chain bit
for bit.  Also the fused kernel at more grid sizes than the 3 / 5 / 7 CTAs of test_gpu_lcab_proj_fused.py, so that the
Q / K / V partition of other SM budgets covers every work item, and with one or two items per CTA (one consumer
warpgroup idle, or the two taking one turn each)."""
import os

import pytest
import torch

pytestmark = pytest.mark.gpu
C = 128
GUARD = 0x7FC0DEAD                                   # a NaN pattern the kernel never writes


def dev():
    return torch.device('cuda:0')


def weights(g):
    from deepinteraction_b200 import fold
    w1 = fold.Weight(torch.randn(3 * C, C, generator=g) / 11, dev())
    w2 = fold.Weight(torch.randn(2 * C, C, generator=g) / 11, dev())
    b1, b2 = torch.randn(3 * C, generator=g).to(dev()), torch.randn(2 * C, generator=g).to(dev())
    return w1, b1, w2, b2


def chain(xt, xs, w):
    from deepinteraction_b200 import ops
    ops.set_lcab_fused(False)
    try:
        return [t.contiguous().view(torch.int32).clone() for t in ops.lcab_proj(xt, xs, *w)]
    finally:
        ops.set_lcab_fused(True)


def fused_into(xt, xs, w, bufs):
    """di_lcab_proj_f32 (fused) writing q, k, v into the first M rows of each buffer in bufs."""
    from deepinteraction_b200 import ops
    w1, b1, w2, b2 = w
    M = xt.shape[0]
    (pt, lt), (ps, ls) = ops._rows(xt), ops._rows(xs)
    ops._call('di_lcab_proj_f32', pt, lt, ps, ls, ops._ptr(w1.bh), ops._ptr(w1.bm), ops._ptr(b1), ops._ptr(w2.bh),
              ops._ptr(w2.bm), ops._ptr(b2), ops._ptr(bufs[0]), ops._ptr(bufs[1]), ops._ptr(bufs[2]), M, ops._stream())


@pytest.mark.parametrize('self_attn', [True, False])
@pytest.mark.parametrize('M', [1, 63, 65, 3001, 32400])
def test_fused_store_leaves_guard_rows(M, self_attn):
    g = torch.Generator().manual_seed(1000 + M + self_attn)
    w = weights(g)
    xt = torch.randn(M, C, generator=g).to(dev())
    xs = xt if self_attn else torch.randn(M, C, generator=g).to(dev())
    guard_rows = 200                                  # more than one 64-row box past the last item
    bufs = [torch.full((M + guard_rows, C), GUARD, dtype=torch.int32, device=dev()) for _ in range(3)]
    fused_into(xt, xs, w, bufs)
    torch.cuda.synchronize()
    want = chain(xt, xs, w)
    for name, buf, ref in zip('qkv', bufs, want):
        assert torch.equal(buf[:M], ref), f'{name}: {int((buf[:M] != ref).sum())} words differ'
        assert bool((buf[M:] == GUARD).all()), f'{name}: {int((buf[M:] != GUARD).sum())} guard words overwritten'


@pytest.mark.parametrize('sms', [4, 6, 11, 40])
@pytest.mark.parametrize('M', [64 * 9 + 5, 20000 + 37])
def test_fused_more_grids(sms, M):
    """SM budgets other than 3 / 5 / 7, at a row count with about one item per CTA and at one with many."""
    from deepinteraction_b200 import _lib, ops
    L = _lib.lib()
    g = torch.Generator().manual_seed(sms * 7 + M)
    w = weights(g)
    xt = torch.randn(M, C, generator=g).to(dev())
    xs = torch.randn(M, C, generator=g).to(dev())
    want = chain(xt, xs, w)
    _lib.check(L.di_tc_set_sm_limit(sms), 'di_tc_set_sm_limit')
    try:
        got = [t.contiguous().view(torch.int32).clone() for t in ops.lcab_proj(xt, xs, *w)]
    finally:
        # the limit has no getter: back to the process default (ops.py reads DI_B200_TC_SMS once at import)
        _lib.check(L.di_tc_set_sm_limit(int(os.environ.get('DI_B200_TC_SMS', '0'))), 'di_tc_set_sm_limit')
    for name, a, b in zip('qkv', got, want):
        assert torch.equal(a, b), f'{name}: {int((a != b).sum())} words differ'
