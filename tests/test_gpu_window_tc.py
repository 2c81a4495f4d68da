"""GPU: the planar 9x9 window kernel (di_lcab_window_tc_f32, C = 128) and the fp32-operand kernel
(di_lcab_window_f32, any C % 32 == 0) against the interleaved pre-split kernel (di_lcab_window_pre_f32, q / k kind 1,
v kind 2), bit for bit.

All three kernels feed the same bf16 hi / mid words into the same fragment algebra (2 x 8 query patch per warp, the same
k16 steps, split products, softmax and P V key grouping), so only the operand layout and the way the operands reach
shared memory differ; the fp32-operand kernel splits in shared memory exactly as the dense layers' epilogue does.  The cases cover one tile, tiles cut by the image border, several images, non-contiguous row
strides, persistent grids of 1, 3 and 7 CTAs (also with fewer tiles than CTAs), concurrent streams and CUDA-graph
replays on two streams."""
import os

import pytest
import torch

from deepinteraction_b200 import _lib, fold, ops

pytestmark = pytest.mark.gpu
C = 128
SHAPES = [(1, 8, 16), (1, 3, 5), (2, 16, 8), (1, 9, 50), (3, 37, 21), (1, 180, 180), (6, 112, 200)]


def dev():
    return torch.device('cuda:0')


def i32(t):
    return t.contiguous().view(torch.int32)


def strided(x, pad):
    """x [M, 128] as a row view with leading dimension 128 + 2 * pad (starting `pad` words into each row)."""
    buf = torch.full((x.shape[0], C + 2 * pad), float('nan'), device=x.device)
    view = buf[:, pad:pad + C]
    view.copy_(x)
    return view


def inputs(N, H, W, seed, c=C):
    g = torch.Generator().manual_seed(seed)
    M = N * H * W
    q, k, v = (torch.randn(M, c, generator=g).to(dev()) for _ in range(3))
    return q * 1.7, k, v                               # logits spread over a few units after the 1/sqrt(C) scale


def planar(q, k, v, pad=0):
    return [strided(fold.split_rows(x, 3), pad) if pad else fold.split_rows(x, 3) for x in (q, k, v)]


def interleaved(q, k, v, N, H, W):
    return ops.lcab_window_pre(fold.split_rows(q, 1), fold.split_rows(k, 1), fold.split_rows(v, 2), N, H, W, q.shape[1])


def window_tc(ops_in, N, H, W, out=None):
    return ops.lcab_window_tc(*ops_in, N, H, W, C, out=out)


@pytest.mark.parametrize('N,H,W', SHAPES)
@pytest.mark.parametrize('pad', [0, 4], ids=['contiguous', 'strided'])
def test_planar_equals_interleaved(N, H, W, pad):
    q, k, v = inputs(N, H, W, 100 + H + W)
    want = interleaved(q, k, v, N, H, W)
    out = strided(torch.zeros(N * H * W, C, device=dev()), 8) if pad else None
    got = window_tc(planar(q, k, v, pad), N, H, W, out=out)
    assert torch.equal(i32(got), i32(want))
    if pad:                                            # the words around the written rows stay untouched
        base = got.as_strided((got.shape[0], C + 16), (C + 16, 1), got.storage_offset() - 8)
        assert torch.isnan(base[:, :8]).all() and torch.isnan(base[:, C + 8:]).all()


@pytest.mark.parametrize('c', [32, 64, 128, 256])
@pytest.mark.parametrize('N,H,W', SHAPES)
def test_fp32_operands_equal_interleaved(N, H, W, c):
    """The fp32-operand kernel (default for a 9x9 window and C % 32 == 0) == the interleaved kernel on split_rows of the
    same rows."""
    q, k, v = inputs(N, H, W, 300 + H + W + c, c)
    assert torch.equal(i32(ops.lcab_window(q, k, v, N, H, W, c)), i32(interleaved(q, k, v, N, H, W)))


@pytest.mark.parametrize('sms', [1, 3, 7, 0], ids=['sm1', 'sm3', 'sm7', 'nolimit'])
@pytest.mark.parametrize('N,H,W', [(1, 8, 16), (1, 3, 5), (2, 16, 8), (3, 37, 21), (2, 112, 200)])
def test_persistent_grid_sizes(N, H, W, sms):
    """Every tile is computed whatever the number of CTAs: 1 (all tiles in one ring), 3 and 7 (also more CTAs than
    tiles), and the whole GPU."""
    q, k, v = inputs(N, H, W, 7 * sms + H)
    want = interleaved(q, k, v, N, H, W)
    L = _lib.lib()
    _lib.check(L.di_tc_set_sm_limit(sms), 'di_tc_set_sm_limit')
    try:
        got = window_tc(planar(q, k, v), N, H, W)
    finally:
        # the limit has no getter: back to the process default (ops.py reads DI_B200_TC_SMS once at import)
        _lib.check(L.di_tc_set_sm_limit(int(os.environ.get('DI_B200_TC_SMS', '0'))), 'di_tc_set_sm_limit')
    assert torch.equal(i32(got), i32(want))


def test_two_streams():
    """Two streams running the kernel on different inputs at the same time == sequential launches."""
    shapes = [(6, 112, 200), (1, 180, 180)]
    ins = [planar(*inputs(*s, 61 + i)) for i, s in enumerate(shapes)]
    want = [window_tc(x, *s) for x, s in zip(ins, shapes)]
    streams = [torch.cuda.Stream() for _ in shapes]
    torch.cuda.synchronize()
    for _ in range(3):
        outs = []
        for x, s, st in zip(ins, shapes, streams):
            with torch.cuda.stream(st):
                outs.append(window_tc(x, *s))
        torch.cuda.synchronize()
        for got, ref in zip(outs, want):
            assert torch.equal(i32(got), i32(ref))


def test_graph_replay_two_streams():
    """Graphs captured on two streams and replayed concurrently read the captured buffers in place: refilled inputs give
    exactly what sequential launches give on the new data."""
    shapes = [(6, 112, 200), (1, 180, 180)]
    static = [planar(*inputs(*s, 71 + i)) for i, s in enumerate(shapes)]
    outs = [torch.empty(N * H * W, C, device=dev()) for N, H, W in shapes]
    window_tc(static[0], *shapes[0], out=outs[0])       # load the module and reserve shared memory before capture
    streams = [torch.cuda.Stream() for _ in shapes]
    graphs = []
    torch.cuda.synchronize()
    for x, s, o, st in zip(static, shapes, outs, streams):
        gr = torch.cuda.CUDAGraph()
        with torch.cuda.graph(gr, stream=st):
            window_tc(x, *s, out=o)
        graphs.append(gr)
    for rep in range(2):
        fresh = [planar(*inputs(*s, 81 + 2 * rep + i)) for i, s in enumerate(shapes)]
        want = [window_tc(x, *s) for x, s in zip(fresh, shapes)]
        for dst, src in zip(static, fresh):
            for d, f in zip(dst, src):
                d.copy_(f)
        torch.cuda.synchronize()
        for gr, st in zip(graphs, streams):
            with torch.cuda.stream(st):
                gr.replay()
        torch.cuda.synchronize()
        for got, ref in zip(outs, want):
            assert torch.equal(i32(got), i32(ref))
