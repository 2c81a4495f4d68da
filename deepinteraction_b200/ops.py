"""Thin torch-tensor wrappers over the C ABI (include/di_b200.h).

torch is used for device memory and the current CUDA stream only; every computation is a
kernel of libdi_b200.so.  All wrappers require CUDA fp32 contiguous tensors and raise on
anything else -- there is no fallback path.
"""
import ctypes
import os

import torch

from . import _lib
from .fold import Weight

ACT_NONE, ACT_RELU, ACT_GELU = 0, 1, 2

LAUNCHES = [0]   # number of libdi_b200 kernel-launching calls (bench.py reports it)
USE_TC = [os.environ.get('DI_B200_TC', '1') != '0']   # wgmma split-product path for Weight objects (else FFMA)
TC_CONV = [os.environ.get('DI_B200_TC_CONV', '1') != '0']
TC_MIN_M = [int(os.environ.get('DI_B200_TC_MIN_M', '128'))]   # fewer rows: fp32 FFMA kernels of gemm.cu (threshold not re-measured on the H100)
TC_BF16 = [os.environ.get('DI_B200_TC_BF16', '1') != '0']   # bf16-split operands where K % 64 == 0 (else 3xTF32)
_TAG = ['']        # optional shape tag for the next profiled call (bench.py --shapes table)
PROFILE = [None]   # bench.py sets PROFILE[0] = [] to record (name, start_event, end_event, bytes, flops, module) per call
PROFILE_FLUSH = [None]     # optional > L2 scratch tensor zeroed before every profiled launch (bench.py)
_MODULE = [None]  # (name, module-boundary bytes, flops) of the nn.Module whose kernels are being issued (bench.py roofline table)


class module:
    """`with ops.module('lcab_img_self', nbytes, flops):` tags the calls issued inside with the reference nn.Module
    they belong to and that module's ALGORITHMIC bytes (SURVEY.md 8(d): every distinct input map read once, the
    output written once).  Only bench.py's profile pass reads the tags; zero cost otherwise."""

    def __init__(self, name, nbytes=0, flops=0):
        self.tag = (name, int(nbytes), int(flops))

    def __enter__(self):
        self.prev, _MODULE[0] = _MODULE[0], self.tag

    def __exit__(self, *a):
        _MODULE[0] = self.prev
        return False


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _ptr(t):
    if t is None:
        return None
    assert t.is_cuda, 'libdi_b200 needs CUDA tensors'
    return ctypes.c_void_p(t.data_ptr())


def _f32(t, name='tensor'):
    if not (t.is_cuda and t.dtype == torch.float32):
        raise TypeError(f'{name}: expected a CUDA float32 tensor, got {t.dtype} on {t.device}')
    return t


def _call(name, *args, nbytes=0, flops=0, launches=1):
    """nbytes / flops: ALGORITHMIC traffic and work of the call (inputs read once, outputs written once); launches: kernels
    the entry point issues (for bench.py's launch count)."""
    LAUNCHES[0] += launches
    prof = PROFILE[0]
    if prof is None:
        return _lib.check(getattr(_lib.lib(), name)(*args), name)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    if PROFILE_FLUSH[0] is not None:
        # keeps the GPU busy (and evicts L2) while the host enqueues e0 / kernel / e1: the interval then is the kernel's
        # own duration from a cold cache, like an ncu launch list -- not launch latency on an idle stream
        PROFILE_FLUSH[0].zero_()
    e0.record()
    rc = _lib.check(getattr(_lib.lib(), name)(*args), name)
    e1.record()
    prof.append((name + _TAG[0], e0, e1, nbytes, flops, _MODULE[0]))
    _TAG[0] = ''
    return rc


def _rows(t):
    """(pointer, leading dimension) of a 2-D row-major view whose rows are contiguous."""
    assert t.dim() == 2 and t.stride(1) == 1, (t.shape, t.stride())
    return _ptr(t), t.stride(0)


def linear(srcs, W, bias=None, act=ACT_NONE, out=None, res=None, res_mod=0, splits=1):
    """out[M,N] = act(cat(srcs,1) @ W.T + bias + res[m % res_mod]).  srcs: 1..3 2-D row views."""
    srcs = list(srcs)
    M = srcs[0].shape[0]
    N, K = W.shape
    if isinstance(W, Weight):
        if (USE_TC[0] and splits == 1 and (M >= TC_MIN_M[0] or N > 2048) and N % 4 == 0
                and all(s_.shape[1] % 32 == 0 and s_.stride(0) % 4 == 0 and s_.data_ptr() % 16 == 0 for s_ in srcs)):
            return _linear_tc(srcs, W, bias, act, out, res, res_mod, M, N, K)
        W = W.w
    assert sum(s.shape[1] for s in srcs) == K, (K, [s.shape for s in srcs])
    a = []
    for s in srcs:
        _f32(s)
        p, ld = _rows(s)
        a += [p, ld, s.shape[1]]
    while len(a) < 9:
        a += [None, 0, 0]
    assert W.is_contiguous()
    if splits > 1:
        assert res is None and bias is None and act == ACT_NONE
        part = torch.empty(splits, M, N, device=W.device, dtype=torch.float32) if out is None else out
        if PROFILE[0] is not None:
            _TAG[0] = ' M%d N%d K%d s%d' % (M, N, K, splits)
        n = _call('di_linear_f32', *a, _ptr(W), None, None, 0, 0, _ptr(part), N, M, N, ACT_NONE, splits, M * N,
                  _stream(), nbytes=4 * (M * K + N * K + splits * M * N), flops=2 * M * N * K)
        return part[:n]
    if out is None:
        out = torch.empty(M, N, device=W.device, dtype=torch.float32)
    po, ldo = _rows(out)
    pr, ldr = (None, 0) if res is None else _rows(res)
    if PROFILE[0] is not None:
        _TAG[0] = ' M%d N%d K%d' % (M, N, K)
    _call('di_linear_f32', *a, _ptr(W), _ptr(bias), pr, ldr, res_mod, po, ldo, M, N, act, 1, 0, _stream(),
          nbytes=4 * (M * K + N * K + M * N + (0 if res is None else res.numel())), flops=2 * M * N * K)
    return out


def _linear_tc(srcs, W, bias, act, out, res, res_mod, M, N, K):
    a = []
    for s in srcs:
        _f32(s)
        p, ld = _rows(s)
        a += [p, ld, s.shape[1]]
    while len(a) < 9:
        a += [None, 0, 0]
    if out is None:
        out = torch.empty(M, N, device=W.w.device, dtype=torch.float32)
    po, ldo = _rows(out)
    pr, ldr = (None, 0) if res is None else _rows(res)
    bf = TC_BF16[0] and all(s.shape[1] % 64 == 0 for s in srcs)
    if PROFILE[0] is not None:
        _TAG[0] = ' M%d N%d K%s' % (M, N, '+'.join(str(s.shape[1]) for s in srcs))
    _call('di_linear_tcb_f32' if bf else 'di_linear_tc_f32', *a, _ptr(W.bh if bf else W.hi), _ptr(W.bm if bf else W.lo),
          _ptr(bias), pr, ldr, res_mod, po, ldo, M, N, act, _stream(),
          nbytes=4 * (M * K + N * K + M * N + (0 if res is None else res.numel())), flops=2 * M * N * K)
    return out


if os.environ.get('DI_B200_TC_SMS'):
    _lib.check(_lib.lib().di_tc_set_sm_limit(int(os.environ['DI_B200_TC_SMS'])), 'di_tc_set_sm_limit')

# shared convs read the NCHW boundary tensors in place (no transposition pass); off by default (not measured on the
# H100).
NCHW_DIRECT = [os.environ.get('DI_B200_NCHW_DIRECT', '0') != '0']
PRESPLIT = [os.environ.get('DI_B200_PRESPLIT', '1') != '0']   # q/k/v projections emit bf16 (hi, mid) words for the window kernel


def can_presplit(M, C, ksize):
    """True when the k/q/v projections may write the window kernel's operand format directly."""
    return bool(PRESPLIT[0] and USE_TC[0] and TC_BF16[0] and ksize == 9 and C % 64 == 0 and M >= TC_MIN_M[0])


def linear_split(srcs, W, bias, act, split_col0, split_kind):
    """linear() on the bf16-split tensor-core path whose output columns >= split_col0 are pre-split (kind 1: Q/K
    layout, 2: V layout) for lcab_window_pre.  Only valid where can_presplit() holds."""
    M, N = srcs[0].shape[0], W.shape[0]
    assert isinstance(W, Weight) and all(s.shape[1] % 64 == 0 for s in srcs) and N % 32 == 0 and split_col0 % 32 == 0
    assert split_kind != 3 or (N % 128 == 0 and split_col0 % 128 == 0)
    a = []
    for s in srcs:
        _f32(s)
        p, ld = _rows(s)
        a += [p, ld, s.shape[1]]
    while len(a) < 9:
        a += [None, 0, 0]
    out = torch.empty(M, N, device=W.w.device, dtype=torch.float32)
    K = sum(s.shape[1] for s in srcs)
    if PROFILE[0] is not None:
        _TAG[0] = ' M%d N%d K%d split' % (M, N, K)
    _call('di_linear_tcb_split_f32', *a, _ptr(W.bh), _ptr(W.bm), _ptr(bias), None, 0, 0, _ptr(out), N, M, N, act,
          split_col0, split_kind, _stream(), nbytes=4 * (M * K + N * K + M * N), flops=2 * M * N * K)
    return out


def can_window_tc(M, C, ksize):
    """True when LocalContextAttentionBlock runs as lcab_forward_tc (fused projections + planar window kernel)."""
    return bool(can_presplit(M, C, ksize) and C == 128)


def lcab_window_tc(q, k, v, N, H, W, C, out=None):
    """9x9 window attention for planar pre-split q, k, v row views (linear_split kind 3)."""
    if out is None:
        out = torch.empty(N * H * W, C, device=q.device, dtype=torch.float32)
    (pq, lq), (pk, lk), (pv, lv), (po, lo) = _rows(q), _rows(k), _rows(v), _rows(out)
    _call('di_lcab_window_tc_f32', pq, lq, pk, lk, pv, lv, po, lo, N, H, W, C, _stream(),
          nbytes=4 * 4 * N * H * W * C, flops=2 * 2 * 81 * N * H * W * C)
    return out


def lcab_proj(x_t, x_s, w1, b1, w2, b2):
    """q, k, v (planar operands of lcab_window_tc) from the target / source rows in one fused launch: w1 = Weight of
    [q1 | k1 | v] (384 x 128), w2 = Weight of [q2 | k2] (256 x 128), BN folded."""
    M = x_t.shape[0]
    assert x_t.shape[1] == 128 and x_s.shape == x_t.shape and w1.shape == (384, 128) and w2.shape == (256, 128)
    out = torch.empty(3, M, 128, device=x_t.device, dtype=torch.float32)
    (pt, lt), (ps, ls) = _rows(x_t), _rows(x_s)
    _call('di_lcab_proj_f32', pt, lt, ps, ls, _ptr(w1.bh), _ptr(w1.bm), _ptr(b1), _ptr(w2.bh), _ptr(w2.bm), _ptr(b2),
          _ptr(out[0]), _ptr(out[1]), _ptr(out[2]), M, _stream(),
          nbytes=4 * M * 128 * (4 if x_t is x_s else 5), flops=2 * 5 * M * 128 * 128)
    return out[0], out[1], out[2]


def lcab_forward_tc(x_t, x_s, w1, b1, w2, b2, N, H, W):
    """LocalContextAttentionBlock for C = 128 in one C-ABI call (fused projections + planar window kernel).  x_t / x_s:
    row views with 16-byte aligned rows (leading dimension % 4 == 0).  The byte count is the MODULE-boundary one of
    SURVEY.md 8(d): each distinct input map read once, the output written once."""
    M = x_t.shape[0]
    assert M == N * H * W and x_t.shape[1] == 128 and x_s.shape == x_t.shape
    qkv = torch.empty(3, M, 128, device=x_t.device, dtype=torch.float32)
    out = torch.empty(M, 128, device=x_t.device, dtype=torch.float32)
    (pt, lt), (ps, ls) = _rows(x_t), _rows(x_s)
    _call('di_lcab_forward_f32', pt, lt, ps, ls, _ptr(w1.bh), _ptr(w1.bm), _ptr(b1), _ptr(w2.bh), _ptr(w2.bm), _ptr(b2),
          _ptr(qkv), _ptr(out), 128, N, H, W, _stream(),
          nbytes=4 * M * 128 * (2 if x_t is x_s else 3), flops=2 * 5 * M * 128 * 128 + 2 * 2 * 81 * M * 128,
          launches=2)
    return out


def lcab_window_pre(q, k, v, N, H, W, C, out=None):
    """lcab_window for pre-split q, k (kind 1) and v (kind 2) row views."""
    if out is None:
        out = torch.empty(N * H * W, C, device=q.device, dtype=torch.float32)
    (pq, lq), (pk, lk), (pv, lv), (po, lo) = _rows(q), _rows(k), _rows(v), _rows(out)
    _call('di_lcab_window_pre_f32', pq, lq, pk, lk, pv, lv, po, lo, N, H, W, C, _stream(),
          nbytes=4 * 4 * N * H * W * C, flops=2 * 2 * 81 * N * H * W * C)
    return out


def conv3x3(x, w_packed, bias, cout, x_nhwc, y_nchw=False, act=ACT_NONE):
    """x: NCHW (N,Cin,H,W) or NHWC (N,H,W,Cin) contiguous; returns NHWC (N,H,W,cout) or NCHW."""
    _f32(x)
    assert x.is_contiguous()
    if x_nhwc:
        N, H, W, Cin = x.shape
    else:
        N, Cin, H, W = x.shape
    if isinstance(w_packed, Weight):
        if USE_TC[0] and TC_CONV[0] and not y_nchw and cout % 4 == 0 and Cin % 32 == 0:
            bf = TC_BF16[0] and Cin % 64 == 0
            direct = NCHW_DIRECT[0] and not x_nhwc and W % 4 == 0     # NCHW input read in place (channel-major TMA boxes)
            xin = x if (x_nhwc or direct) else nchw_to_nhwc(x)
            y = torch.empty((N, H, W, cout), device=x.device, dtype=torch.float32)
            name = 'di_conv3x3_tc%s%s_f32' % ('b' if bf else '', '_nchw' if direct else '')
            _call(name, _ptr(xin), _ptr(w_packed.bh if bf else w_packed.hi), _ptr(w_packed.bm if bf else w_packed.lo),
                  _ptr(bias), _ptr(y), N, Cin, H, W, cout, act, _stream(),
                  nbytes=4 * (x.numel() + w_packed.w.numel() + y.numel()), flops=2 * N * H * W * cout * 9 * Cin)
            return y
        w_packed = w_packed.w
    y = torch.empty((N, cout, H, W) if y_nchw else (N, H, W, cout), device=x.device, dtype=torch.float32)
    _call('di_conv3x3_f32', _ptr(x), int(x_nhwc), _ptr(w_packed), _ptr(bias), _ptr(y), int(y_nchw), N, Cin, H, W, cout,
          act, _stream(), nbytes=4 * (x.numel() + w_packed.numel() + y.numel()), flops=2 * N * H * W * cout * 9 * Cin)
    return y


def lcab_window(q, k, v, N, H, W, C, ksize=9, out=None):
    """q,k,v: 2-D row views [N*H*W, >=C] (pixel-major); returns [N*H*W, C]."""
    if out is None:
        out = torch.empty(N * H * W, C, device=q.device, dtype=torch.float32)
    (pq, lq), (pk, lk), (pv, lv), (po, lo) = _rows(q), _rows(k), _rows(v), _rows(out)
    _call('di_lcab_window_f32', pq, lq, pk, lk, pv, lv, po, lo, N, H, W, C, ksize, _stream(),
          nbytes=4 * 4 * N * H * W * C, flops=2 * 2 * ksize * ksize * N * H * W * C)
    return out


def gather_rows(map_nhwc, coors, n_dev=None):
    """n_dev (here and in scatter_rows / i2p_attend / depth_scatter): int32 device tensor holding the live count when
    the arrays are allocated at capacity (shape-independent graph replay); None = all rows."""
    B, Y, X, C = map_nhwc.shape
    P = coors.shape[0]
    rows = torch.zeros(P, C, device=map_nhwc.device, dtype=torch.float32) if n_dev is not None else \
        torch.empty(P, C, device=map_nhwc.device, dtype=torch.float32)
    _call('di_gather_rows_f32', _ptr(map_nhwc), _ptr(coors), _ptr(rows), P, Y, X, C, _ptr(n_dev), _stream())
    return rows


def scatter_rows(rows, cnt, coors, map_nhwc, n_dev=None):
    B, Y, X, C = map_nhwc.shape
    _call('di_scatter_rows_f32', _ptr(rows), _ptr(cnt), _ptr(coors), _ptr(map_nhwc), coors.shape[0], Y, X, C,
          _ptr(n_dev), _stream())
    return map_nhwc


def pillarize(pts_list, bev_hw, pc_range, max_pts=20, n_dev=None, cap=None):
    """GPU pillar generation.  pts_list: B device tensors [n_b, >=3] (capacity rows when n_dev [B] int32 holds the live
    counts).  -> pillars [cap, max_pts, pdim], coors [cap, 4] int32, npts [cap] int32, n_pillars [1] int32 (device)."""
    B = len(pts_list)
    Y, X = bev_hw
    dev = pts_list[0].device
    pdim = pts_list[0].shape[1]
    assert all(p.dtype == torch.float32 and p.stride(1) == 1 and p.shape[1] == pdim and p.stride(0) == pts_list[0].stride(0)
               for p in pts_list)
    caps = [int(p.shape[0]) for p in pts_list]
    cap = B * Y * X if cap is None else cap
    work = torch.empty(4 * B * Y * X + 1 + B * max(caps + [1]) + sum(caps) + 1, device=dev, dtype=torch.int32)
    pillars = torch.empty(cap, max_pts, pdim, device=dev, dtype=torch.float32)
    coors = torch.zeros(cap, 4, device=dev, dtype=torch.int32)
    npts = torch.zeros(cap, device=dev, dtype=torch.int32)
    n_out = torch.empty(1, device=dev, dtype=torch.int32)
    ptrs = (ctypes.c_void_p * B)(*[p.data_ptr() if p.shape[0] else None for p in pts_list])
    ncap = (ctypes.c_int * B)(*caps)
    rng = (ctypes.c_float * 6)(*[float(v) for v in pc_range])
    _call('di_pillarize_f32', ptrs, ncap, _ptr(n_dev), B, pts_list[0].stride(0), pdim, Y, X, max_pts, rng, _ptr(work),
          _ptr(pillars), _ptr(coors), _ptr(npts), _ptr(n_out), cap, _stream())
    return pillars, coors, npts, n_out


def scatter_rows_add(rows, cnt, coors, map_nhwc, n_dev=None):
    """map[coors[p]] += rows[p] where cnt[p] > 0 (in place)."""
    B, Y, X, C = map_nhwc.shape
    _call('di_scatter_rows_add_f32', _ptr(rows), _ptr(cnt), _ptr(coors), _ptr(map_nhwc), coors.shape[0], Y, X, C,
          _ptr(n_dev), _stream())
    return map_nhwc


def msdeform(values, raw, B, hq, wq, heads=8, points=4):
    """values: list of 1 or 2 projected value maps [B, H_l, W_l, C]; raw [B*hq*wq, heads*L*P*3] (offsets | logits)
    -> [B*hq*wq, C]."""
    L = len(values)
    C = values[0].shape[-1]
    assert all(v.is_contiguous() and v.shape[0] == B for v in values) and raw.shape[0] == B * hq * wq
    out = torch.empty(B * hq * wq, C, device=raw.device, dtype=torch.float32)
    sh = (ctypes.c_int * (2 * L))(*[d for v in values for d in v.shape[1:3]])
    pr, ldr = _rows(raw)
    _call('di_msdeform_f32', _ptr(values[0]), _ptr(values[1]) if L > 1 else None, pr, ldr, _ptr(out), C, B, hq * wq, hq, wq,
          heads, C // heads, L, points, sh, _stream(),
          nbytes=4 * (sum(v.numel() for v in values) + raw.numel() + out.numel()),
          flops=2 * 4 * heads * L * points * (C // heads) * B * hq * wq)
    return out


def polar_grid(cam, BV, R, W, h_feat, im_scale, r0, r_step, pc_range, bev_hw):
    grid = torch.empty(BV, R, W, 2, device=cam.device, dtype=torch.float32)
    rng = (ctypes.c_float * 6)(*[float(v) for v in pc_range])
    _call('di_polar_grid_f32', _ptr(cam), _ptr(grid), BV, R, W, h_feat, float(im_scale), float(r0), float(r_step), rng,
          bev_hw[0], bev_hw[1], _stream())
    return grid


def add_rows_mod(x, pos):
    """x [M, C] + pos[m % mod] (pos [mod, C])."""
    assert x.is_contiguous() and pos.is_contiguous() and x.shape[1] == pos.shape[1]
    out = torch.empty_like(x)
    _call('di_add_rows_mod_f32', _ptr(x), _ptr(pos), _ptr(out), x.shape[0], x.shape[1], pos.shape[0], _stream(),
          nbytes=8 * x.numel())
    return out


def seq_attn(q, k, v, G, Wn, Lq, Lk, heads):
    """Attention over column sequences: q [G*Lq*Wn, C] row views, k / v [G*Lk*Wn, C] row views -> [G*Lq*Wn, C]."""
    C = q.shape[1]
    out = torch.empty(G * Lq * Wn, C, device=q.device, dtype=torch.float32)
    (pq, lq), (pk, lk), (pv, lv) = _rows(q), _rows(k), _rows(v)
    _call('di_seq_attn_f32', pq, lq, pk, lk, pv, lv, _ptr(out), C, G, Wn, Lq, Lk, heads, C // heads, _stream(),
          flops=4 * G * Wn * Lq * Lk * C)
    return out


def polar_gather(rays, lidar, proj, undo, camc, V, in_hw, pc_range, r0, r_count):
    BV, R, W, C = rays.shape
    B, Y, X, _ = lidar.shape
    out = torch.empty_like(lidar)
    rng = (ctypes.c_float * 6)(*[float(v) for v in pc_range])
    _call('di_polar_gather_f32', _ptr(rays), _ptr(lidar), _ptr(proj), _ptr(undo), _ptr(camc), _ptr(out), B, V, R, W, Y, X,
          C, in_hw[0], in_hw[1], rng, float(r0), float(r_count), _stream(), nbytes=4 * (rays.numel() + 2 * lidar.numel()))
    return out


def axpy(a, b, scale):
    """a + scale[0] * b; scale: 1-element device tensor."""
    assert a.is_contiguous() and b.is_contiguous() and a.shape == b.shape
    out = torch.empty_like(a)
    _call('di_axpy_f32', _ptr(a), _ptr(b), _ptr(scale), _ptr(out), a.numel(), _stream(), nbytes=12 * a.numel())
    return out


def msdeform_bwd(values, raw, dout, B, hq, wq, heads=8, points=4):
    """Gradient of msdeform: dout [B*hq*wq, C] -> (d_raw [B*hq*wq, heads*L*P*3] in raw's layout (offsets | logits),
    [d value_l [B, H_l, W_l, C]])."""
    L = len(values)
    C = values[0].shape[-1]
    assert all(v.is_contiguous() and v.shape[0] == B for v in values) and raw.shape[0] == B * hq * wq
    d_raw = torch.empty(raw.shape[0], heads * L * points * 3, device=raw.device, dtype=torch.float32)
    d_vals = [torch.zeros_like(v) for v in values]
    sh = (ctypes.c_int * (2 * L))(*[d for v in values for d in v.shape[1:3]])
    (pr, ldr), (pd, ldd) = _rows(raw), _rows(dout)
    _call('di_msdeform_bwd_f32', _ptr(values[0]), _ptr(values[1]) if L > 1 else None, pr, ldr, pd, ldd, _ptr(d_raw),
          d_raw.stride(0), _ptr(d_vals[0]), _ptr(d_vals[1]) if L > 1 else None, B, hq * wq, hq, wq, heads, C // heads, L,
          points, sh, _stream(), nbytes=4 * (2 * sum(v.numel() for v in values) + raw.numel() + d_raw.numel() + dout.numel()))
    return d_raw, d_vals


def seq_attn_bwd(q, k, v, out, dout, G, Wn, Lq, Lk, heads, dq, dk, dv):
    """Gradient of seq_attn from its saved output `out`: dout [G*Lq*Wn, C] -> dq, dk, dv written into the given row views
    (e.g. the three column blocks of one packed [M, 3C] buffer)."""
    C = q.shape[1]
    args = []
    for t in (q, k, v, out, dout, dq, dk, dv):
        args += list(_rows(t))
    _call('di_seq_attn_bwd_f32', *args, G, Wn, Lq, Lk, heads, C // heads, _stream(), flops=10 * G * Wn * Lq * Lk * C)
    return dq, dk, dv


def polar_gather_bwd(d_out, rays_shape, proj, undo, camc, V, in_hw, pc_range, r0, r_count):
    """Adjoint of polar_gather w.r.t. the rays: d_out [B, Y, X, C] -> d_rays of shape rays_shape [B*V, R, W, C]."""
    BV, R, W, C = rays_shape
    B, Y, X, _ = d_out.shape
    assert d_out.is_contiguous()
    d_rays = torch.zeros(BV, R, W, C, device=d_out.device, dtype=torch.float32)
    rng = (ctypes.c_float * 6)(*[float(v) for v in pc_range])
    _call('di_polar_gather_bwd_f32', _ptr(d_out), _ptr(proj), _ptr(undo), _ptr(camc), _ptr(d_rays), B, V, R, W, Y, X, C,
          in_hw[0], in_hw[1], rng, float(r0), float(r_count), _stream(), nbytes=4 * (2 * d_rays.numel() + d_out.numel()))
    return d_rays


def axpy_bwd(dout, b, scale):
    """Gradient of axpy(a, b, scale) w.r.t. b and scale: -> (s * dout, d scale [1] = sum dout . b); d a is dout."""
    assert dout.is_contiguous() and b.is_contiguous() and dout.shape == b.shape
    n = _lib.check(_lib.lib().di_axpy_bwd_workspace(), 'di_axpy_bwd_workspace')
    work = torch.empty(n, device=b.device, dtype=torch.float64)
    db = torch.empty_like(b)
    ds = torch.empty(1, device=b.device, dtype=torch.float32)
    _call('di_axpy_bwd_f32', _ptr(dout), _ptr(b), _ptr(scale), _ptr(db), _ptr(ds), _ptr(work), b.numel(), _stream(),
          nbytes=12 * b.numel(), launches=2)
    return db, ds


def i2p_attend(qk, pillars, npts, coors, proj, img_nhwc, V, in_hw, n_dev=None, dropout=None):
    """dropout = (p, seed): training-mode attention dropout (mask = hash(seed, pillar, key), see i2p_dropout_mask); s is then
    [P, C + 4] with rho = sum_j a_j m_j in column C (fold.i2p_fold(split_bias=True) gives the matching [C, C + 4] weight)."""
    P, C = qk.shape
    _, T, pdim = pillars.shape
    BV, h, w, Ci = img_nhwc.shape
    assert Ci == C and pillars.is_contiguous() and img_nhwc.is_contiguous()
    drop = dropout is not None and dropout[0] > 0
    s = torch.empty(P, C + 4 if drop else C, device=qk.device, dtype=torch.float32)
    cnt = torch.empty(P, device=qk.device, dtype=torch.int32)
    if n_dev is not None:
        s.zero_()                       # rows beyond the live count feed a dense layer: keep them finite
    nb = 4 * (2 * P * C + pillars.numel() + img_nhwc.numel())
    if drop:
        _call('di_i2p_attend_dropout_f32', _ptr(qk), _ptr(pillars), _ptr(npts), _ptr(coors), _ptr(proj), _ptr(img_nhwc), _ptr(s),
              _ptr(cnt), P, T, pdim, V, h, w, C, in_hw[0], in_hw[1], _ptr(n_dev), float(dropout[0]), int(dropout[1]) & 0xFFFFFFFF,
              _stream(), nbytes=nb)
        return s, cnt
    _call('di_i2p_attend_f32', _ptr(qk), _ptr(pillars), _ptr(npts), _ptr(coors), _ptr(proj), _ptr(img_nhwc), _ptr(s),
          _ptr(cnt), P, T, pdim, V, h, w, C, in_hw[0], in_hw[1], _ptr(n_dev), _stream(), nbytes=nb, flops=0)
    return s, cnt


def i2p_dropout_mask(P, S, pdrop, seed, device):
    """[P, S] factors (0 or 1 / (1 - pdrop)) that i2p_attend / i2p_attend_bwd apply with dropout = (pdrop, seed)."""
    mask = torch.empty(P, S, device=device, dtype=torch.float32)
    _call('di_i2p_dropout_mask_f32', _ptr(mask), P, S, float(pdrop), int(seed) & 0xFFFFFFFF, _stream())
    return mask


def depth_scatter(pts, proj_b, keys_b, in_hw, n_dev=None):
    """pts (n, >=3) row-major; proj_b (V,12); keys_b (V,h,w) int64 view of zeroed uint64 keys."""
    V, h, w = keys_b.shape
    if pts.shape[0] == 0:                 # a sample without lidar points: its depth maps stay empty
        return
    assert pts.stride(1) == 1
    _call('di_depth_scatter', _ptr(pts), pts.stride(0), pts.shape[0], _ptr(proj_b), _ptr(keys_b), V, h, w, in_hw[0],
          in_hw[1], _ptr(n_dev), _stream())


def depth_complete(keys, want_sparse=False):
    n_img, h, w = keys.shape
    dev = keys.device
    scratch = torch.empty(3 * n_img * h * w, device=dev, dtype=torch.float32)
    dense = torch.empty(n_img, h, w, device=dev, dtype=torch.float32)
    sparse = torch.empty(n_img, h, w, device=dev, dtype=torch.float32) if want_sparse else None
    _call('di_depth_complete', _ptr(keys), _ptr(scratch), _ptr(dense), _ptr(sparse), n_img, h, w, _stream())
    return (dense, sparse) if want_sparse else dense


def lift_grid(dense, i2l, in_hw, bev_hw, pc_range):
    n_img, h, w = dense.shape
    grid = torch.empty(n_img, h, w, 2, device=dense.device, dtype=torch.float32)
    rng = (ctypes.c_float * 6)(*[float(v) for v in pc_range])
    _call('di_lift_grid', _ptr(dense), _ptr(i2l), _ptr(grid), n_img, h, w, in_hw[0], in_hw[1], bev_hw[0], bev_hw[1],
          rng, _stream())
    return grid


def bev_sample(bev_nhwc, grid, V):
    B, Yb, Xb, C = bev_nhwc.shape
    n_img, h, w, _ = grid.shape
    out = torch.empty(n_img, h, w, C, device=grid.device, dtype=torch.float32)
    _call('di_bev_sample_f32', _ptr(bev_nhwc), _ptr(grid), _ptr(out), B, V, h * w, Yb, Xb, C, _stream(),
          nbytes=4 * (bev_nhwc.numel() + grid.numel() + out.numel()))
    return out


def heatmap_nms(a, b, K, ks, no_nms_mask, want_dense=True):
    """a, b: pixel-major logits [B,H,W,ld] (ld >= K).  -> masked heat [B,K,H*W], dense_b [B,K,H,W]."""
    B, H, W, ld = a.shape
    assert a.is_contiguous() and b.is_contiguous() and b.shape == a.shape
    out = torch.empty(B, K, H * W, device=a.device, dtype=torch.float32)
    dense = torch.empty(B, K, H, W, device=a.device, dtype=torch.float32) if want_dense else None
    _call('di_heatmap_nms_f32', _ptr(a), _ptr(b), ld, _ptr(out), _ptr(dense), B, K, H, W, ks, no_nms_mask, _stream())
    return out, dense


def topk(scores, k):
    B, n = scores.shape
    assert scores.is_contiguous()
    idx = torch.empty(B, k, device=scores.device, dtype=torch.int32)
    slices = 64 if n >= 64 * 1024 else 0
    work = torch.empty(B * slices * k * 2, device=scores.device, dtype=torch.float32) if slices else None
    _call('di_topk_f32', _ptr(scores), _ptr(idx), B, n, k, _ptr(work), slices, _stream())
    return idx


def query_init(feat_nhwc, top, heat, wce_t, bce, W):
    B, HW, C = feat_nhwc.shape
    K = heat.shape[1]
    P = top.shape[1]
    dev = top.device
    qfeat = torch.empty(B * P, C, device=dev, dtype=torch.float32)
    qpos = torch.empty(B * P, 2, device=dev, dtype=torch.float32)
    labels = torch.empty(B, P, device=dev, dtype=torch.int32)
    qscore = torch.empty(B, K, P, device=dev, dtype=torch.float32)
    _call('di_query_init_f32', _ptr(feat_nhwc), _ptr(top), _ptr(heat), _ptr(wce_t), _ptr(bce), _ptr(qfeat), _ptr(qpos),
          _ptr(labels), _ptr(qscore), B, HW, W, C, K, P, _stream())
    return qfeat, qpos, labels, qscore


def query_init_bwd(dq, top, labels, d_feat, K):
    """Backward of query_init's rows q0 = feat[b, pix] + class encoding: adds the dq [B*P, C] rows into d_feat [B, HW, C]
    in place at the selected pixels -> (d class_encoding.weight [C, K], d bias [C])."""
    B, HW, C = d_feat.shape
    P = top.shape[1]
    assert dq.is_contiguous() and d_feat.is_contiguous() and top.is_contiguous() and labels.is_contiguous()
    assert dq.shape == (B * P, C) and top.dtype == torch.int32 and labels.dtype == torch.int32
    d_w = torch.empty(C, K, device=dq.device, dtype=torch.float32)
    d_b = torch.empty(C, device=dq.device, dtype=torch.float32)
    _call('di_query_init_bwd_f32', _ptr(_f32(dq)), _ptr(top), _ptr(labels), _ptr(_f32(d_feat)), _ptr(d_w), _ptr(d_b), B, HW,
          C, K, P, _stream(), nbytes=4 * (3 * B * P * C + K * C), launches=2)
    return d_w, d_b


def mha_small(q, k, v, B, P, heads, onbits=None, win=None):
    C = q.shape[1]
    out = torch.empty(B * P, C, device=q.device, dtype=torch.float32)
    (pq, lq), (pk, lk), (pv, lv) = _rows(q), _rows(k), _rows(v)
    _call('di_mha_small_f32', pq, lq, pk, lk, pv, lv, _ptr(out), C, _ptr(onbits), _ptr(win), B, P, heads, C // heads,
          _stream())
    return out


def cross_attn(q, kv, B, P, HW, heads, nsplit=32):
    C = q.shape[1]
    assert q.is_contiguous() and kv.is_contiguous() and kv.shape == (B * HW, 2 * C)
    part = torch.empty(B * heads * P * nsplit * 18, device=q.device, dtype=torch.float32)
    out = torch.empty(B * P, C, device=q.device, dtype=torch.float32)
    _call('di_cross_attn_f32', _ptr(q), _ptr(kv), _ptr(part), _ptr(out), B, P, HW, C, heads, nsplit, _stream(),
          nbytes=4 * (kv.numel() + 2 * q.numel()), flops=4 * B * P * HW * C, launches=2)
    return out


def rows_finish(x, bias=None, res=None, gamma=None, beta=None, act=ACT_NONE, zero_if_neg=None, eps=1e-5):
    """x: [M,C] or split-K partials [S,M,C].  y = act(LN(sum_s x[s] + bias + res))."""
    if x.dim() == 2:
        S, M, C = 1, x.shape[0], x.shape[1]
        stride, ldp = 0, x.stride(0)
    else:
        S, M, C = x.shape
        assert x.is_contiguous()
        stride, ldp = M * C, C
    out = torch.empty(M, C, device=x.device, dtype=torch.float32)
    pr, ldr = (None, 0) if res is None else _rows(res)
    _call('di_rows_finish_f32', _ptr(x), S, stride, ldp, _ptr(bias), pr, ldr, _ptr(gamma), _ptr(beta), _ptr(out), C,
          _ptr(zero_if_neg), M, C, act, eps, _stream())
    return out


ROWS_MLP = [os.environ.get('DI_B200_ROWS_MLP', '1') != '0']   # query-row dense layers on the fused FFMA kernel (M <= 2048)


def can_rows_mlp(M, K, N1, N2=0):
    return bool(ROWS_MLP[0] and M <= 2048 and K <= 1024 and N1 <= 512 and N2 <= 512 and N1 % 4 == 0 and N2 % 4 == 0 and
                K + N1 + N2 <= 1800)


def rows_mlp(srcs, W1, b1=None, act1=ACT_NONE, W2=None, b2=None, res=None, gamma=None, beta=None, act_out=ACT_NONE,
             zero_if_neg=None, eps=1e-5):
    """act_out(LN(act1(cat(srcs) W1^T + b1) [W2^T + b2] + res)) on a few hundred rows in one launch (W*: fold.Weight)."""
    srcs = list(srcs)
    M = srcs[0].shape[0]
    N1 = W1.shape[0]
    N2 = W2.shape[0] if W2 is not None else 0
    assert len(srcs) <= 2 and sum(s.shape[1] for s in srcs) == W1.shape[1]
    (p0, l0) = _rows(srcs[0])
    (p1, l1) = _rows(srcs[1]) if len(srcs) > 1 else (None, 0)
    K1 = srcs[1].shape[1] if len(srcs) > 1 else 0
    out = torch.empty(M, N2 or N1, device=srcs[0].device, dtype=torch.float32)
    pr, ldr = (None, 0) if res is None else _rows(res)
    _call('di_rows_mlp_f32', p0, l0, srcs[0].shape[1], p1, l1, K1, _ptr(W1.wt), _ptr(b1), N1, act1,
          _ptr(W2.wt) if W2 is not None else None, _ptr(b2), N2, pr, ldr, _ptr(gamma), _ptr(beta), float(eps), act_out,
          _ptr(zero_if_neg), _ptr(out), out.shape[1], M, _stream(),
          nbytes=4 * (W1.shape[0] * W1.shape[1] + (N2 * N1 if N2 else 0) + M * (W1.shape[1] + (N2 or N1))),
          flops=2 * M * (W1.shape[0] * W1.shape[1] + N2 * N1))
    return out


def pred_finish(pred, qpos, first=None, win=None):
    M, NP = pred.shape
    _call('di_pred_finish_f32', _ptr(pred), _ptr(qpos), _ptr(first), _ptr(win), M, NP, _stream())


def pred_finish_pp(pred, qpos, look, first, win, keep, first_layer):
    M, NP = pred.shape
    _call('di_pred_finish_pp_f32', _ptr(pred), _ptr(qpos), _ptr(look), _ptr(first), _ptr(win), _ptr(keep),
          1 if first_layer else 0, M, NP, _stream())


def rcnn_leaders(onbits, B, P, V):
    lead_row = torch.empty(B * V, device=onbits.device, dtype=torch.int32)
    lead_win = torch.empty(B * V, device=onbits.device, dtype=torch.int32)
    _call('di_rcnn_leaders', _ptr(onbits), _ptr(lead_row), _ptr(lead_win), B, P, V, _stream())
    return lead_row, lead_win


def mha_small_rows(q, k, v, B, P, heads, onbits, rows, rwin):
    C, R = q.shape[1], rows.shape[0]
    out = torch.empty(R, C, device=q.device, dtype=torch.float32)
    (pq, lq), (pk, lk), (pv, lv) = _rows(q), _rows(k), _rows(v)
    _call('di_mha_small_rows_f32', pq, lq, pk, lk, pv, lv, _ptr(out), C, _ptr(onbits), _ptr(rows), _ptr(rwin), R, R // B, B,
          P, heads, C // heads, _stream())
    return out


def take_rows(src, idx):
    R, C = idx.shape[0], src.shape[1]
    out = torch.empty(R, C, device=src.device, dtype=torch.float32)
    p, ld = _rows(src)
    _call('di_take_rows_f32', p, ld, _ptr(idx), _ptr(out), R, C, _stream())
    return out


def branch_mix(a, lead, win, scale, self_scale, P, V, zero_off):
    M, C = a.shape
    assert a.is_contiguous() and lead.is_contiguous() and lead.shape == (M // P * V, C)
    out = torch.empty(M, C, device=a.device, dtype=torch.float32)
    _call('di_branch_mix_f32', _ptr(a), _ptr(lead), _ptr(win), _ptr(scale), _ptr(self_scale), _ptr(out), M, C, P, V,
          1 if zero_off else 0, _stream())
    return out


def branch_mix_bwd(dout, a, lead, win, scale, self_scale, P, V, zero_off):
    """Gradient of branch_mix: dout [M, C] -> (da [M, C], dlead [M / P * V, C], d scale [1], d self_scale [1])."""
    M, C = a.shape
    assert dout.is_contiguous() and a.is_contiguous() and lead.is_contiguous() and lead.shape == (M // P * V, C)
    dev_ = a.device
    da, dlead = torch.empty(M, C, device=dev_), torch.empty(M // P * V, C, device=dev_)
    ds, dt, work = torch.empty(1, device=dev_), torch.empty(1, device=dev_), torch.empty(2 * M, device=dev_)
    _call('di_branch_mix_bwd_f32', _ptr(dout), _ptr(a), _ptr(lead), _ptr(win), _ptr(scale), _ptr(self_scale), _ptr(da),
          _ptr(dlead), _ptr(ds), _ptr(dt), _ptr(work), M, C, P, V, 1 if zero_off else 0, _stream(), launches=3)
    return da, dlead, ds, dt


def mha_small_rows_bwd(q, k, v, dout, B, P, heads, onbits, rows, rwin, dk, dv):
    """Gradient of mha_small_rows: dout [R, C] -> dq [R, C] (rows[r] = -1: zero row); the key and value gradients are
    ADDED to the rows of dk / dv [B*P, C] (views with one leading dimension, e.g. columns of mha_small_bwd's dqkv)."""
    C, R = q.shape[1], rows.shape[0]
    dq = torch.empty(R, C, device=q.device, dtype=torch.float32)
    work = torch.empty(2 * B * heads * P * (R // B), device=q.device, dtype=torch.float32)
    (pq, lq), (pk, lk), (pv, lv), (pd, ld), (pgk, lg), (pgv, lgv) = (_rows(t) for t in (q, k, v, dout, dk, dv))
    assert lg == lgv and dk.shape == dv.shape == (B * P, C)
    _call('di_mha_small_rows_bwd_f32', pq, lq, pk, lk, pv, lv, pd, ld, _ptr(dq), C, pgk, pgv, lg, _ptr(work), _ptr(onbits),
          _ptr(rows), _ptr(rwin), R, R // B, B, P, heads, C // heads, _stream(), launches=2)
    return dq


def rows_scatter_add(src, idx, dst):
    """dst[idx[r]] += src[r] in place (r ascending; idx[r] = -1 skipped): the adjoint of take_rows.  dst: rows view."""
    R, C = src.shape
    (ps, ls), (pd, ld) = _rows(src), _rows(dst)
    assert dst.shape[1] == C and idx.shape[0] == R
    _call('di_rows_scatter_add_f32', ps, ls, _ptr(idx), pd, ld, R, C, _stream())
    return dst


def pred_finish_pp_bwd(dpred, keep):
    """Gradient of the L layers' pred_finish_pp: dpred [L, M, NP], keep [L, M] int32 (each layer's mask) -> (d_delta
    [L, M, NP], the gradient of each prediction head's output rows; d_first [M, NP])."""
    L, M, NP = dpred.shape
    assert dpred.is_contiguous() and keep.is_contiguous() and keep.shape == (L, M) and keep.dtype == torch.int32
    d_delta, d_first = torch.empty_like(dpred), torch.empty(M, NP, device=dpred.device)
    _call('di_pred_finish_pp_bwd_f32', _ptr(dpred), _ptr(keep), _ptr(d_delta), _ptr(d_first), L, M, NP, _stream())
    return d_delta, d_first


def rcnn_rois(pred, B, P, V, mode, params10, proj=None, aux=None):
    dev = pred.device
    rois = torch.empty(B * P, 5, device=dev, dtype=torch.float32)
    win = torch.empty(B * P, device=dev, dtype=torch.int32)
    onbits = torch.empty(B * P, device=dev, dtype=torch.int32)
    prm = (ctypes.c_float * 10)(*[float(v) for v in params10])
    _call('di_rcnn_rois_f32', _ptr(pred), pred.shape[1], _ptr(proj), _ptr(aux), _ptr(rois), _ptr(win), _ptr(onbits), B,
          P, V, mode, prm, _stream())
    return rois, win, onbits


def roi_align(maps_nhwc, rois, scale):
    n_maps, H, W, C = maps_nhwc.shape
    n = rois.shape[0]
    out = torch.empty(n, 49, C, device=rois.device, dtype=torch.float32)
    _call('di_roi_align_f32', _ptr(maps_nhwc), _ptr(rois), _ptr(out), n, H, W, C, float(scale), _stream(),
          nbytes=4 * (out.numel() * 5))
    return out


def dynconv(roi, params, g1, b1, g2, b2, eps=1e-5):
    n = roi.shape[0]
    assert roi.shape[1:] == (49, 128) and params.shape == (n, 2 * 128 * 128) and params.is_contiguous()
    out = torch.empty(n, 49 * 128, device=roi.device, dtype=torch.float32)
    _call('di_dynconv_f32', _ptr(roi), _ptr(params), _ptr(g1), _ptr(b1), _ptr(g2), _ptr(b2), _ptr(out), n, float(eps),
          _stream(), nbytes=4 * (roi.numel() + params.numel() + out.numel()), flops=2 * 2 * n * 49 * 128 * 128)
    return out


def roi_align_bwd(d_out, rois, n_maps, H, W, scale):
    """Gradient of roi_align w.r.t. the maps: d_out [n, 49, C] -> d_maps [n_maps, H, W, C] (every pixel written)."""
    n, _, C = d_out.shape
    assert d_out.is_contiguous() and rois.is_contiguous() and d_out.shape[1] == 49 and rois.shape == (n, 5)
    d_maps = torch.empty(n_maps, H, W, C, device=d_out.device, dtype=torch.float32)
    _call('di_roi_align_bwd_f32', _ptr(rois), _ptr(d_out), _ptr(d_maps), n, n_maps, H, W, C, float(scale), _stream(),
          nbytes=4 * (d_out.numel() + d_maps.numel()))
    return d_maps


def dynconv_bwd(roi, params, g1, b1, g2, b2, d_out, eps=1e-5):
    """Gradient of dynconv: -> (d_roi [n, 49, 128], d_params [n, 32768], d_norm [n, 512] per-query partials of
    dgamma1 | dbeta1 | dgamma2 | dbeta2)."""
    n = roi.shape[0]
    assert roi.shape[1:] == (49, 128) and params.shape == (n, 2 * 128 * 128) and d_out.shape == (n, 49 * 128)
    assert roi.is_contiguous() and params.is_contiguous() and d_out.is_contiguous()
    d_roi = torch.empty(n, 49, 128, device=roi.device, dtype=torch.float32)
    d_params = torch.empty(n, 2 * 128 * 128, device=roi.device, dtype=torch.float32)
    d_norm = torch.empty(n, 4 * 128, device=roi.device, dtype=torch.float32)
    _call('di_dynconv_bwd_f32', _ptr(roi), _ptr(params), _ptr(g1), _ptr(b1), _ptr(g2), _ptr(b2), _ptr(d_out), _ptr(d_roi),
          _ptr(d_params), _ptr(d_norm), n, float(eps), _stream(),
          nbytes=4 * (2 * roi.numel() + 2 * params.numel() + d_out.numel() + d_norm.numel()),
          flops=6 * 2 * 2 * n * 49 * 128 * 128)
    return d_roi, d_params, d_norm


def gelu_bwd(dy, h):
    assert dy.is_contiguous() and h.is_contiguous() and dy.shape == h.shape
    dx = torch.empty_like(dy)
    _call('di_gelu_bwd_f32', _ptr(dy), _ptr(h), _ptr(dx), dy.numel(), _stream(), nbytes=12 * dy.numel())
    return dx


def nchw_to_nhwc(x):
    N, C, H, W = x.shape
    assert x.is_contiguous()
    out = torch.empty(N, H, W, C, device=x.device, dtype=torch.float32)
    _call('di_nchw_to_nhwc_f32', _ptr(_f32(x)), _ptr(out), N, C, H * W, _stream())
    return out


def nhwc_to_nchw(x):
    N, H, W, C = x.shape
    assert x.is_contiguous()
    out = torch.empty(N, C, H, W, device=x.device, dtype=torch.float32)
    _call('di_nhwc_to_nchw_f32', _ptr(_f32(x)), _ptr(out), N, C, H * W, _stream())
    return out


def bbox_decode(heat, rot, dim, center, height, vel, sx, sy, ox, oy, post_range=None, score_thr=None, qscore=None,
                qlabel=None):
    """TransFusionBBoxCoder.decode on [B,k,P] tensors -> boxes [B,P,7|9], scores [B,P], labels [B,P] int32,
    keep [B,P] bool (range + score filter).  With qscore/qlabel the get_bboxes score composition is applied first."""
    B, K, P = heat.shape
    heat, rot, dim, center, height = (t.contiguous() for t in (heat, rot, dim, center, height))
    vel = None if vel is None else vel.contiguous()
    qscore = None if qscore is None else qscore.contiguous()
    qlabel = None if qlabel is None else qlabel.to(torch.int32).contiguous()
    dev = heat.device
    boxes = torch.empty(B, P, 9 if vel is not None else 7, device=dev, dtype=torch.float32)
    scores = torch.empty(B, P, device=dev, dtype=torch.float32)
    labels = torch.empty(B, P, device=dev, dtype=torch.int32)
    keep = torch.empty(B, P, device=dev, dtype=torch.uint8)
    rng = None if post_range is None else (ctypes.c_float * 6)(*[float(v) for v in post_range])
    use_thr = bool(score_thr)                       # the reference tests `if self.score_threshold:` (coder :110)
    _call('di_bbox_decode_f32', _ptr(heat), _ptr(qscore), _ptr(qlabel), _ptr(rot), _ptr(dim), _ptr(center), _ptr(height),
          _ptr(vel), B, K, P, float(sx), float(sy), float(ox), float(oy), rng, float(score_thr or 0.0), int(use_thr),
          _ptr(boxes), _ptr(scores), _ptr(labels), _ptr(keep), _stream())
    return boxes, scores, labels, keep.bool()


def bbox_encode(boxes, code_size, sx, sy, ox, oy):
    boxes = boxes.contiguous()
    _f32(boxes)
    n, nb = boxes.shape
    out = torch.empty(n, code_size, device=boxes.device, dtype=torch.float32)
    if n:
        _call('di_bbox_encode_f32', _ptr(boxes), nb, _ptr(out), code_size, n, float(sx), float(sy), float(ox), float(oy),
              _stream())
    return out


def circle_nms(boxes, scores, labels, keep, class_mask, thresh, post_max=83):
    """In-place per-task circle NMS on keep [B,P] (bool)."""
    B, P, nb = boxes.shape
    k8 = keep.to(torch.uint8).contiguous()
    _call('di_circle_nms_f32', _ptr(boxes), nb, _ptr(scores), _ptr(labels), _ptr(k8), B, P, int(class_mask), float(thresh),
          int(post_max), _stream())
    return k8.bool()


# ---- backward of the window attention (csrc/lcab_bwd.cu; composition in backward.py) ---------------------------------
def win_dot(a, b, N, H, W, ks):
    P, C = a.shape
    out = torch.empty(P, ks * ks, device=a.device, dtype=torch.float32)
    (pa, la), (pb, lb) = _rows(a), _rows(b)
    _call('di_win_dot_f32', pa, la, pb, lb, _ptr(out), N, H, W, C, ks, _stream(), nbytes=4 * (2 * P * C + P * ks * ks),
          flops=2 * P * C * ks * ks)
    return out


def _win_apply(name, w, b, N, H, W, ks):
    P, C = b.shape
    out = torch.empty(P, C, device=b.device, dtype=torch.float32)
    pb, lb = _rows(b)
    _call(name, _ptr(w), pb, lb, _ptr(out), C, N, H, W, C, ks, _stream(), nbytes=4 * (2 * P * C + P * ks * ks),
          flops=2 * P * C * ks * ks)
    return out


def win_gather(w, b, N, H, W, ks):
    return _win_apply('di_win_gather_f32', w, b, N, H, W, ks)


def win_scatter(w, b, N, H, W, ks):
    return _win_apply('di_win_scatter_f32', w, b, N, H, W, ks)


def win_softmax(S, scale):
    A = torch.empty_like(S)
    _call('di_win_softmax_f32', _ptr(S), _ptr(A), S.shape[0], S.shape[1], float(scale), _stream(), nbytes=8 * S.numel())
    return A


def win_softmax_bwd(A, dA, scale):
    dS = torch.empty_like(A)
    _call('di_win_softmax_bwd_f32', _ptr(A), _ptr(dA), _ptr(dS), A.shape[0], A.shape[1], float(scale), _stream(),
          nbytes=12 * A.numel())
    return dS


def relu_bwd(dy, y):
    assert dy.is_contiguous() and y.is_contiguous() and dy.shape == y.shape
    dx = torch.empty_like(dy)
    _call('di_relu_bwd_f32', _ptr(dy), _ptr(y), _ptr(dx), dy.numel(), _stream(), nbytes=12 * dy.numel())
    return dx


def shift_map(x_nhwc, dy, dx):
    """out[n, y, x] = in[n, y + dy, x + dx] (zeros outside)."""
    N, H, W, C = x_nhwc.shape
    assert x_nhwc.is_contiguous()
    out = torch.empty_like(x_nhwc)
    _call('di_shift_map_f32', _ptr(x_nhwc), _ptr(out), N, H, W, C, dy, dx, _stream(), nbytes=8 * x_nhwc.numel())
    return out


def col_sum(x):
    M, C = x.shape
    p, ld = _rows(x)
    work = torch.empty(256 * C, device=x.device, dtype=torch.float32)
    out = torch.empty(C, device=x.device, dtype=torch.float32)
    _call('di_col_sum_f32', p, ld, M, C, _ptr(work), _ptr(out), _stream(), nbytes=4 * M * C, launches=2)
    return out


# ---- train-mode BatchNorm over rows (csrc/bn_train.cu; composition in train.py) ----------------------------------------
def bn_stats(y, run_mean=None, run_var=None, momentum=0.1):
    """y [M, C] -> (mean [C], biased var [C]); running statistics updated in place when given."""
    M, C = y.shape
    assert y.is_contiguous()
    work = torch.empty(592 * C * 3, device=y.device, dtype=torch.float32)
    mean = torch.empty(C, device=y.device, dtype=torch.float32)
    var = torch.empty(C, device=y.device, dtype=torch.float32)
    _call('di_bn_stats_f32', _ptr(y), M, C, _ptr(work), _ptr(mean), _ptr(var), _ptr(run_mean), _ptr(run_var), float(momentum),
          _stream(), nbytes=4 * M * C, launches=2)
    return mean, var


def bn_apply(y, mean, var, gamma, beta, eps, relu):
    M, C = y.shape
    assert y.is_contiguous()
    z = torch.empty_like(y)
    _call('di_bn_apply_f32', _ptr(y), M, C, _ptr(mean), _ptr(var), _ptr(gamma), _ptr(beta), float(eps), int(relu), _ptr(z),
          _stream(), nbytes=8 * M * C)
    return z


def bn_bwd(dz, z, y, mean, var, gamma, eps):
    """-> (dy [M, C], dgamma [C], dbeta [C]); z = the saved output when the layer ends in ReLU, else None."""
    M, C = y.shape
    assert y.is_contiguous() and dz.is_contiguous() and (z is None or z.is_contiguous())
    work = torch.empty(592 * C * 2, device=y.device, dtype=torch.float32)
    dy = torch.empty_like(y)
    dg = torch.empty(C, device=y.device, dtype=torch.float32)
    db = torch.empty(C, device=y.device, dtype=torch.float32)
    _call('di_bn_bwd_f32', _ptr(dz), _ptr(z), _ptr(y), M, C, _ptr(mean), _ptr(var), _ptr(gamma), float(eps), _ptr(work), _ptr(dy),
          _ptr(dg), _ptr(db), _stream(), nbytes=4 * M * C * 7, launches=3)
    return dy, dg, db


def i2p_attend_bwd(qk, ds, pillars, npts, coors, proj, img_nhwc, d_img, V, in_hw, dropout=None):
    """Gradient of i2p_attend: -> dqk [P, C]; d_img (same shape as img_nhwc) is accumulated into."""
    P, C = qk.shape
    _, T, pdim = pillars.shape
    BV, h, w, Ci = img_nhwc.shape
    assert Ci == C and d_img.shape == img_nhwc.shape and d_img.is_contiguous() and ds.is_contiguous()
    dqk = torch.empty(P, C, device=qk.device, dtype=torch.float32)
    nb = 4 * (3 * P * C + pillars.numel() + 2 * img_nhwc.numel())
    if dropout is not None and dropout[0] > 0:
        assert ds.shape == (P, C + 4), ds.shape
        _call('di_i2p_attend_bwd_dropout_f32', _ptr(qk), _ptr(ds), _ptr(pillars), _ptr(npts), _ptr(coors), _ptr(proj),
              _ptr(img_nhwc), _ptr(d_img), _ptr(dqk), P, T, pdim, V, h, w, C, in_hw[0], in_hw[1], None, float(dropout[0]),
              int(dropout[1]) & 0xFFFFFFFF, _stream(), nbytes=nb)
        return dqk
    _call('di_i2p_attend_bwd_f32', _ptr(qk), _ptr(ds), _ptr(pillars), _ptr(npts), _ptr(coors), _ptr(proj), _ptr(img_nhwc),
          _ptr(d_img), _ptr(dqk), P, T, pdim, V, h, w, C, in_hw[0], in_hw[1], None, _stream(), nbytes=nb)
    return dqk


def gather_rows_masked(map_nhwc, cnt, coors):
    B, Y, X, C = map_nhwc.shape
    P = coors.shape[0]
    rows = torch.empty(P, C, device=map_nhwc.device, dtype=torch.float32)
    _call('di_gather_rows_masked_f32', _ptr(map_nhwc), _ptr(cnt), _ptr(coors), _ptr(rows), P, Y, X, C, _stream())
    return rows


def bev_sample_bwd(d_out, grid, V, bev_shape):
    """Gradient of bev_sample w.r.t. the BEV map: d_out [B*V, h, w, C] -> [B, Yb, Xb, C]."""
    B, Yb, Xb, C = bev_shape
    n_img, h, w, _ = grid.shape
    d_bev = torch.zeros(B, Yb, Xb, C, device=d_out.device, dtype=torch.float32)
    assert d_out.is_contiguous()
    _call('di_bev_sample_bwd_f32', _ptr(d_out), _ptr(grid), _ptr(d_bev), B, V, h * w, Yb, Xb, C, _stream(),
          nbytes=4 * (d_bev.numel() + grid.numel() + d_out.numel()))
    return d_bev


# ---- tensor-core query x BEV cross attention (csrc/xattn_tc.cu) ----------------------------------------------------------
XATTN_TC = [os.environ.get('DI_B200_XATTN_TC', '1') != '0']   # tensor-core query x BEV cross attention (xattn_tc.cu)


def can_xattn_tc(P, C, heads, M_keys):
    return bool(XATTN_TC[0] and USE_TC[0] and C == 128 and heads == 8 and P <= 256 and M_keys >= TC_MIN_M[0])


def _xattn_planes(q, kv, B, P, HW):
    assert kv.is_contiguous() and kv.shape == (B * HW, 256) and q.shape == (B * P, 128)
    dev_ = q.device
    qp = torch.empty(B * P, 192, device=dev_, dtype=torch.float32)
    kp = torch.empty(B * HW, 192, device=dev_, dtype=torch.float32)
    vp = torch.empty(B * HW, 128, device=dev_, dtype=torch.float32)
    pq, lq = _rows(q)
    _call('di_attn_planes_f32', pq, lq, _ptr(qp), B * P, _ptr(kv), 256, _ptr(kp), _ptr(vp), B * HW, _stream(),
          nbytes=4 * (kv.numel() + kp.numel() + vp.numel()), launches=2)
    return qp, kp, vp


def xattn_tc(q, kv, B, P, HW, heads):
    """q [B*P, 128] fp32 (pre-scaled queries), kv [B*HW, 256] fp32 (K | V) -> softmax(q k^T) v per head, [B*P, 128] fp32:
    operand planes (di_attn_planes_f32) + the mma.sync attention kernel + the split merge."""
    qp, kp, vp = _xattn_planes(q, kv, B, P, HW)
    nsplit = _lib.lib().di_xattn_tc_splits(B, HW)
    part = torch.empty(B * heads * nsplit * 18 * P, device=q.device, dtype=torch.float32)
    out = torch.empty(B * P, 128, device=q.device, dtype=torch.float32)
    _call('di_xattn_tc_f32', _ptr(qp), _ptr(kp), _ptr(vp), _ptr(part), _ptr(out), B, P, HW, heads, _stream(),
          nbytes=4 * (kp.numel() + vp.numel() + 2 * q.numel()), flops=4 * B * P * HW * 128, launches=2)
    return out


def xattn_tc_lse(q, kv, B, P, HW, heads):
    """xattn_tc plus the row log-sum-exp of the logits: -> (out [B*P, 128] (bit-identical to xattn_tc), lse [B, heads, P],
    planes (q, k, v operand planes, the inputs of xattn_bwd))."""
    planes = _xattn_planes(q, kv, B, P, HW)
    nsplit = _lib.check(_lib.lib().di_xattn_tc_splits(B, HW), 'di_xattn_tc_splits')
    part = torch.empty(B * heads * nsplit * 18 * P, device=q.device, dtype=torch.float32)
    out = torch.empty(B * P, 128, device=q.device, dtype=torch.float32)
    lse = torch.empty(B, heads, P, device=q.device, dtype=torch.float32)
    _call('di_xattn_tc_lse_f32', *(_ptr(t) for t in planes), _ptr(part), _ptr(out), _ptr(lse), B, P, HW, heads, _stream(),
          nbytes=4 * (planes[1].numel() + planes[2].numel() + 2 * q.numel()), flops=4 * B * P * HW * 128, launches=2)
    return out, lse, planes


def xattn_bwd(planes, out, lse, dout, B, P, HW, heads, dkv=None):
    """Gradient of xattn_tc_lse (csrc/xattn_bwd.cu): dout [B*P, 128] -> (dq [B*P, 128] w.r.t. the pre-scaled queries,
    dkv [B*HW, 256] = dK | dV).  dkv may be given (rows [B*HW, >= 256]); only its first 256 columns are written."""
    qp, kp, vp = planes
    dev_ = out.device
    if dkv is None:
        dkv = torch.empty(B * HW, 256, device=dev_, dtype=torch.float32)
    assert dkv.shape[0] == B * HW and dkv.stride(1) == 1 and dkv.stride(0) >= 256
    pd, ld = _rows(dout)
    n = _lib.check(_lib.lib().di_xattn_bwd_workspace(B, P, HW), 'di_xattn_bwd_workspace')
    work = torch.empty(n, device=dev_, dtype=torch.float32)
    dq = torch.empty(B * P, 128, device=dev_, dtype=torch.float32)
    _call('di_xattn_bwd_f32', _ptr(qp), _ptr(kp), _ptr(vp), _ptr(out), pd, ld, _ptr(lse), _ptr(work), _ptr(dq), _ptr(dkv),
          ctypes.c_void_p(dkv.data_ptr() + 128 * 4), dkv.stride(0), B, P, HW, heads, _stream(),
          nbytes=4 * (kp.numel() + vp.numel() + 2 * B * HW * 128), flops=10 * B * P * HW * 128, launches=3)
    return dq, dkv


def mha_small_bwd(q, k, v, dout, B, P, heads, onbits=None, win=None):
    """Gradient of mha_small, with the same optional group mask (onbits, win): -> dqkv [B*P, 3C] = dq | dk | dv."""
    C = q.shape[1]
    dqkv = torch.empty(B * P, 3 * C, device=q.device, dtype=torch.float32)
    work = torch.empty(2 * B * heads * P * P, device=q.device, dtype=torch.float32)
    (pq, lq), (pk, lk), (pv, lv), (pd, ld) = _rows(q), _rows(k), _rows(v), _rows(dout)
    base = dqkv.data_ptr()
    _call('di_mha_small_bwd_f32', pq, lq, pk, lk, pv, lv, pd, ld, ctypes.c_void_p(base), ctypes.c_void_p(base + 4 * C),
          ctypes.c_void_p(base + 8 * C), 3 * C, _ptr(work), _ptr(onbits), _ptr(win), B, P, heads, C // heads, _stream(), launches=2)
    return dqkv


def ln_bwd(dy, z, gamma, eps=1e-5):
    """Backward of y = LayerNorm(z) * gamma + beta over [M, C] rows (z: the pre-norm sum) -> (dz, dgamma, dbeta)."""
    M, C = z.shape
    dz = torch.empty(M, C, device=z.device, dtype=torch.float32)
    dg = torch.empty(C, device=z.device, dtype=torch.float32)
    db = torch.empty(C, device=z.device, dtype=torch.float32)
    work = torch.empty(M * C + 256 * C, device=z.device, dtype=torch.float32)
    (py, ly), (pz, lz) = _rows(dy), _rows(z)
    _call('di_ln_bwd_f32', py, ly, pz, lz, _ptr(gamma), _ptr(dz), C, _ptr(dg), _ptr(db), _ptr(work), M, C, float(eps), _stream(),
          nbytes=4 * 4 * M * C, launches=5)
    return dz, dg, db
