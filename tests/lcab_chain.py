"""Reference for the fused LCAB projections (di_lcab_proj_f32): the five 1x1 layers as five launches of the bf16-split
tensor-core GEMM (di_linear_tcb_split_f32), one per layer -- q1 / k1 as plain fp32 rows, q / k / v in the planar split
format (kind 3) of the window kernel.  The GEMM is called directly whatever M is: ops.linear sends fewer than 128 rows to
the FFMA kernels, whose sums differ from the tensor-core ones in the last bits."""
import contextlib
import os

import torch

from deepinteraction_b200 import _lib, fold, ops

C = 128


def dev():
    return torch.device('cuda:0')


def weights(g):
    """w1 = [q1 | k1 | v] (384 x 128), b1, w2 = [q2 | k2] (256 x 128), b2 from the CPU generator g."""
    w1 = fold.Weight(torch.randn(3 * C, C, generator=g) / 11, dev())
    w2 = fold.Weight(torch.randn(2 * C, C, generator=g) / 11, dev())
    b1, b2 = torch.randn(3 * C, generator=g).to(dev()), torch.randn(2 * C, generator=g).to(dev())
    return w1, b1, w2, b2


def _layer(x, w, i, b, kind):
    """relu(x @ W[i*128 : (i+1)*128].T + b) as a new [M, 128] tensor, split kind 0 (fp32) or 3 (planar)."""
    M = x.shape[0]
    out = torch.empty(M, C, device=x.device, dtype=torch.float32)
    p, ld = ops._rows(x)
    rows = slice(i * C, (i + 1) * C)
    _lib.check(_lib.lib().di_linear_tcb_split_f32(p, ld, C, None, 0, 0, None, 0, 0, ops._ptr(w.bh[rows]),
                                                  ops._ptr(w.bm[rows]), ops._ptr(b), None, 0, 0, ops._ptr(out), C, M, C,
                                                  ops.ACT_RELU, 0, kind, ops._stream()), 'di_linear_tcb_split_f32')
    return out


def chain(x_t, x_s, w1, b1, w2, b2):
    """q, k, v of the five-launch chain as int32 words [M, 128] each."""
    q = _layer(_layer(x_t, w1, 0, b1[:C], 0), w2, 0, b2[:C], 3)
    k = _layer(_layer(x_s, w1, 1, b1[C:2 * C], 0), w2, 1, b2[C:], 3)
    v = _layer(x_s, w1, 2, b1[2 * C:], 3)
    return [t.view(torch.int32) for t in (q, k, v)]


@contextlib.contextmanager
def sm_limit(n):
    """Persistent tensor-core grids capped at n CTAs inside the block."""
    L = _lib.lib()
    _lib.check(L.di_tc_set_sm_limit(n), 'di_tc_set_sm_limit')
    try:
        yield
    finally:
        # the limit has no getter: back to the process default (ops.py reads DI_B200_TC_SMS once at import)
        _lib.check(L.di_tc_set_sm_limit(int(os.environ.get('DI_B200_TC_SMS', '0'))), 'di_tc_set_sm_limit')
