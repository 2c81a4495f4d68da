"""Helpers of the kernel-level GPU tests: direct calls of the C entry points, the per-row error metric and bit equality.

row_err takes the max over output rows of max|a-b| / scale_row, where scale_row is the magnitude of the terms summed into
that row (>= max|b_row|).  A global max hides a wrong row whose values are small; and fp32 rounding is relative to the
summed terms, not to their sum, which may cancel.  A row whose terms are all zero must be exactly zero."""
import torch

SENT = 0x7FA5A5A5                 # NaN bit pattern of the output canvases


def _ops():
    from deepinteraction_b200 import ops
    return ops


def _capi(name, *args):
    """Call a C entry point directly (the wrappers allocate their outputs; these tests pre-fill them); returns its
    status (a count where the entry point returns one)."""
    ops = _ops()
    rc = ops._call(name, *args, ops._stream())
    torch.cuda.synchronize()
    return rc


def _status(name, *args):
    """The raw status of a C entry point, without raising on an error code (tests of the documented rejections)."""
    from deepinteraction_b200 import _lib
    ops = _ops()
    rc = getattr(_lib.lib(), name)(*args, ops._stream())
    torch.cuda.synchronize()
    return rc


class record_calls:
    """`with record_calls() as calls:` lists (entry point, args) of every C call the ops wrappers issue inside."""

    def __enter__(self):
        ops = _ops()
        self.calls, self.saved = [], ops._call

        def rec(name, *args, **kw):
            self.calls.append((name, args))
            return self.saved(name, *args, **kw)
        ops._call = rec
        return self.calls

    def __exit__(self, *a):
        _ops()._call = self.saved
        return False


def row_err(got, want, scale, width=None):
    """max over rows of max|got - want| / max(scale_row, max|want_row|); rows are the last dimension, or groups of
    `width` values of it."""
    g, w, s = (t.detach().double().cpu() for t in (got, want, scale))
    s = torch.broadcast_to(s, g.shape)
    n = width or g.shape[-1]
    g, w, s = g.reshape(-1, n), w.reshape(-1, n), s.reshape(-1, n)
    den = torch.maximum(w.abs().amax(1), s.abs().amax(1))
    err = (g - w).abs().amax(1)
    return float(torch.where(den > 0, err / den.clamp_min(1e-300), err * 1e30).max())


def same_bits(a, b):
    a, b = a.detach().cpu().contiguous(), b.detach().cpu().contiguous()
    return a.shape == b.shape and torch.equal(a.view(torch.int32), b.view(torch.int32))


def canvas(rows, cols, pad_cols=8, pad_rows=3):
    """(buffer, view): a [rows, cols] output view with ldc = cols + pad_cols inside a SENT-filled buffer."""
    buf = torch.full((rows + pad_rows, cols + pad_cols), SENT, dtype=torch.int32, device='cuda').view(torch.float32)
    return buf, buf[:rows, :cols]


def outside_intact(buf, rows, cols):
    """Every word of a canvas outside its [rows, cols] view still holds SENT."""
    b = buf.view(torch.int32)
    keep = torch.ones_like(b, dtype=torch.bool)
    keep[:rows, :cols] = False
    return bool((b[keep] == SENT).all())
