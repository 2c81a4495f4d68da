"""Sampled storage of large golden outputs (every file under tests/golden stays below 1 MB).

shrink() replaces each floating-point tensor of more than LIMIT elements by a record holding its shape, max|x| and the
values at SAMPLE flat positions drawn with a fixed seed (the positions depend only on the element count).
golden_err() is conftest.rel_err = max|a - b| / max|b| against such a record: the numerator over the stored positions of
a, the denominator from the full tensor the record was made of."""
import numpy as np
import torch

LIMIT = 30000
SAMPLE = 30000


def _positions(n):
    return torch.from_numpy(np.sort(np.random.default_rng(0).choice(n, SAMPLE, replace=False)))


def is_sampled(g):
    return isinstance(g, dict) and 'sampled' in g


def shrink(obj):
    if isinstance(obj, torch.Tensor):
        if obj.is_floating_point() and obj.numel() > LIMIT:
            flat = obj.detach().reshape(-1).float().cpu()
            return dict(sampled=flat[_positions(flat.numel())].clone(), shape=tuple(obj.shape),
                        absmax=float(flat.abs().max()))
        return obj
    if isinstance(obj, dict):
        return {k: shrink(v) for k, v in obj.items()}
    if isinstance(obj, (list, tuple)):
        return type(obj)(shrink(v) for v in obj)
    return obj


def shape_of(g):
    return tuple(g['shape']) if is_sampled(g) else tuple(g.shape)


def golden_err(a, g):
    """max|a - g| / max|g| for a full tensor a and a golden g (a tensor or a shrink() record)."""
    a = a.detach().float().cpu()
    if not is_sampled(g):
        return float((a - g).abs().max() / g.abs().max().clamp_min(1e-12))
    assert tuple(a.shape) == tuple(g['shape']), (tuple(a.shape), g['shape'])
    s = a.reshape(-1)[_positions(a.numel())]
    return float((s - g['sampled']).abs().max() / max(g['absmax'], 1e-12))
