"""Inputs of the comparisons with the reference's own CUDA extension `localattention`, and the stored form of its
outputs (tests/golden/locatt_ref.pt, written by tools/make_goldens_locatt.py from the extension compiled unmodified by
oracle/build_ref.py).  Every case's inputs come from a seeded CPU generator, so the test and the generator build the
same tensors.  An output larger than SAMPLE elements is stored as the values at SAMPLE flat positions drawn with a
fixed seed; the test compares its own output at the same positions."""
import numpy as np
import torch

GOLDEN = 'locatt_ref.pt'
SAMPLE = 8000


def take(t):
    """The stored form of an output: all elements, or a fixed seeded sample of them (flattened, float32, CPU)."""
    flat = t.detach().reshape(-1).float().cpu()
    if flat.numel() <= SAMPLE:
        return flat.clone()
    idx = np.sort(np.random.default_rng(0).choice(flat.numel(), SAMPLE, replace=False))
    return flat[torch.from_numpy(idx)].clone()


DROP_IN = [(2, 16, 9, 13, 9, 9), (1, 128, 20, 17, 9, 9), (2, 8, 7, 11, 3, 5), (1, 32, 5, 6, 5, 3)]


def drop_in_inputs(N, C, H, W, kH, kW):
    g = torch.Generator().manual_seed(100 + C)
    x_ori = torch.randn(N, C, H, W, generator=g)
    x_loc = torch.randn(N, C, H, W, generator=g)
    wgt = torch.randn(N, H, W, kH * kW, generator=g)
    grad_c = torch.randn(N, C, H, W, generator=g)
    return x_ori, x_loc, wgt, grad_c


def drop_in_calls(m, x_ori, x_loc, wgt, grad_c, kH, kW):
    """name -> output of the six entry points of module m (the reference extension or the drop-in replacement)."""
    return {
        'similar_forward': m.similar_forward(x_ori, x_loc, kH, kW),
        'similar_backward(is_ori)': m.similar_backward(x_loc, wgt, kH, kW, True),
        'similar_backward(is_loc)': m.similar_backward(x_ori, wgt, kH, kW, False),
        'weighting_forward': m.weighting_forward(x_ori, wgt, kH, kW),
        'weighting_backward_ori': m.weighting_backward_ori(wgt, grad_c, kH, kW),
        'weighting_backward_weight': m.weighting_backward_weight(x_ori, grad_c, kH, kW),
    }


FUSED = [(2, 40, 33), (1, 17, 50)]


def fused_inputs(N, H, W, C=128):
    g = torch.Generator().manual_seed(31 + H)
    return tuple(torch.randn(N, C, H, W, generator=g) for _ in range(3))


def oracle_inputs():
    g = torch.Generator().manual_seed(5)
    N, C, H, W, k = 2, 64, 11, 14, 9
    return tuple(torch.randn(N, C, H, W, generator=g) for _ in range(3)) + (k,)


BACKWARD = [(2, 128, 11, 14, 9), (1, 32, 7, 9, 9), (1, 256, 6, 5, 5)]


def backward_inputs(N, C, H, W, ks):
    g = torch.Generator().manual_seed(7 + C)
    a = torch.randn(N, C, H, W, generator=g)
    b = torch.randn(N, C, H, W, generator=g)
    w = torch.randn(N, H, W, ks * ks, generator=g)
    return a, b, w


def key(*parts):
    return '/'.join(str(p) for p in parts)
