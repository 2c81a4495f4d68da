"""GPU: the fused LCAB projection kernel (di_lcab_proj_f32) equals the five-launch chain of tests/lcab_chain.py bit for
bit: every row count around the 64-row work items, self and cross attention, outputs as fresh tensors and as views into
larger buffers (the TMA stores must leave the guard rows after row M untouched), strided input views, SM budgets from
one or two CTAs per role up (the Q / K / V role partition must cover every work item, with one or two items per CTA or
many) and two streams running it at once."""
import pytest
import torch

from deepinteraction_b200 import ops
from lcab_chain import C, chain, dev, sm_limit, weights

pytestmark = pytest.mark.gpu
GUARD = 0x7FC0DEAD                                   # a NaN pattern the kernel never writes


def fused(xt, xs, w):
    return [t.view(torch.int32) for t in ops.lcab_proj(xt, xs, *w)]


def fused_into(xt, xs, w, bufs):
    """di_lcab_proj_f32 writing q, k, v into the first M rows of each buffer in bufs."""
    w1, b1, w2, b2 = w
    (pt, lt), (ps, ls) = ops._rows(xt), ops._rows(xs)
    ops._call('di_lcab_proj_f32', pt, lt, ps, ls, ops._ptr(w1.bh), ops._ptr(w1.bm), ops._ptr(b1), ops._ptr(w2.bh),
              ops._ptr(w2.bm), ops._ptr(b2), ops._ptr(bufs[0]), ops._ptr(bufs[1]), ops._ptr(bufs[2]), xt.shape[0],
              ops._stream())


def assert_equal(got, want):
    for name, a, b in zip('qkv', got, want):
        assert torch.equal(a, b), f'{name}: {int((a != b).sum())} words differ'


@pytest.mark.parametrize('out', ['fresh', 'guarded'])
@pytest.mark.parametrize('self_attn', [True, False])
@pytest.mark.parametrize('M', [1, 63, 65, 127, 128, 129, 1000, 3001, 32400, 134400])
def test_fused_equals_chain(M, self_attn, out):
    g = torch.Generator().manual_seed(M + 7 * self_attn)
    w = weights(g)
    xt = torch.randn(M, C, generator=g).to(dev())
    xs = xt if self_attn else torch.randn(M, C, generator=g).to(dev())
    want = chain(xt, xs, *w)
    if out == 'fresh':
        assert_equal(fused(xt, xs, w), want)
        return
    guard_rows = 200                                  # more than one 64-row box past the last item
    bufs = [torch.full((M + guard_rows, C), GUARD, dtype=torch.int32, device=dev()) for _ in range(3)]
    fused_into(xt, xs, w, bufs)
    assert_equal([b[:M] for b in bufs], want)
    for name, buf in zip('qkv', bufs):
        assert bool((buf[M:] == GUARD).all()), f'{name}: {int((buf[M:] != GUARD).sum())} guard words overwritten'


@pytest.mark.parametrize('self_attn', [True, False])
def test_fused_strided_views(self_attn):
    """x_t / x_s as column views of wider row-major tensors (ld > 128)."""
    g = torch.Generator().manual_seed(31)
    M = 3001
    w = weights(g)
    wide_t = torch.randn(M, 3 * C, generator=g).to(dev())
    xt = wide_t[:, C:2 * C]
    xs = xt if self_attn else torch.randn(M, 2 * C + 32, generator=g).to(dev())[:, 32:32 + C]
    got = fused(xt, xs, w)
    assert_equal(got, chain(xt, xs, *w))
    assert_equal(got, fused(xt.contiguous(), xt.contiguous() if self_attn else xs.contiguous(), w))


@pytest.mark.parametrize('sms', [3, 4, 5, 6, 7, 11, 40])
@pytest.mark.parametrize('M', [64 * 9 + 5, 20000 + 37])
def test_fused_sm_limits(M, sms):
    """At most 3 .. 40 CTAs, at a row count with about one item per CTA and at one with many: every work item is
    computed."""
    g = torch.Generator().manual_seed(sms * 7 + M)
    w = weights(g)
    xt = torch.randn(M, C, generator=g).to(dev())
    xs = torch.randn(M, C, generator=g).to(dev())
    want = chain(xt, xs, *w)
    with sm_limit(sms):
        got = fused(xt, xs, w)
    assert_equal(got, want)


def test_fused_two_streams():
    """Two streams running the fused kernel on different inputs at the same time == sequential runs."""
    g = torch.Generator().manual_seed(41)
    M = 134400
    ins = []
    for _ in range(2):
        w = weights(g)
        xt = torch.randn(M, C, generator=g).to(dev())
        ins.append((xt, torch.randn(M, C, generator=g).to(dev()), w))
    want = [[t.clone() for t in fused(xt, xs, w)] for xt, xs, w in ins]
    streams = [torch.cuda.Stream() for _ in ins]
    torch.cuda.synchronize()
    outs = [None, None]
    for rep in range(3):
        for i, ((xt, xs, w), s) in enumerate(zip(ins, streams)):
            with torch.cuda.stream(s):
                outs[i] = fused(xt, xs, w)
        torch.cuda.synchronize()
        for got, ref in zip(outs, want):
            assert_equal(got, ref)


@pytest.mark.parametrize('self_attn', [True, False])
@pytest.mark.parametrize('offset', [0, 1], ids=['aligned', 'misaligned'])
def test_lcab_forward_row_views(offset, self_attn):
    """mmri.lcab_forward at C = 128 on column views of wider tensors: aligned rows go in through their leading dimension,
    rows that are not 16-byte aligned as a contiguous copy; both equal the run on contiguous rows bit for bit."""
    from deepinteraction_b200 import mmri, synth
    N, H, W = 2, 37, 21
    torch.manual_seed(3)
    holder = mmri.LocalContextAttentionBlock(C, C, 9)
    synth.randomize_norm_stats(holder, 3)
    pk = mmri._pack_lcab(holder.eval(), dev())
    g = torch.Generator().manual_seed(5 + offset)
    wide = torch.randn(N * H * W, 3 * C, generator=g).to(dev())
    xt = wide[:, C + offset:2 * C + offset]
    xs = xt if self_attn else wide[:, 2 * C - 4 * offset:3 * C - 4 * offset]
    ct = xt.contiguous()
    want = mmri.lcab_forward(pk, ct, ct if self_attn else xs.contiguous(), N, H, W)
    got = mmri.lcab_forward(pk, xt, xs, N, H, W)
    assert torch.equal(got.view(torch.int32), want.view(torch.int32))
