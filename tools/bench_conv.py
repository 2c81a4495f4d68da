"""Times the tensor-core 3x3 convolutions at the shapes of the base forward, through their C entry points, L2 flushed.

    python tools/bench_conv.py [--lib LABEL=PATH ...] [--reps 30]

Each --lib is a built libdi_b200.so (default: the in-tree library); with several, the libraries are called in turn for
every repetition so that they see the same clocks.  Per shape and library it prints the median time, and per shape the
MMA floor of the issued split products at the data-sheet rate (H100 SXM dense: 989 TFLOP/s bf16, 495 TFLOP/s tf32),
the bytes the conv kernel moves from L2 into shared memory (this tree's kernel, and the parent's one A box per tap
with 128-column tiles) and the HBM floor (input, weights and output once, 3.35 TB/s).  Data-sheet floors are not
measurements.
"""
import argparse
import ctypes
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
from deepinteraction_b200 import _lib, fold

# (label, images, Cin, H, W, Cout, act, bf16 split) -- the base forward's calls (calls per frame in the comment)
SHAPES = [('shared_conv_img', 6, 256, 112, 200, 128, 0, True),      # 1
          ('shared_conv_pts', 1, 512, 180, 180, 128, 0, True),      # 1
          ('heatmap_conv0', 1, 128, 180, 180, 128, 1, False),       # 2
          ('heatmap_conv1', 1, 128, 180, 180, 12, 0, False)]        # 2
PEAK = {True: 989e12, False: 495e12}
HBM = 3.35e12


def conv_model(n, cin, H, W, cout, bf):
    """(issued MMA FLOP, L2 -> shared bytes of this tree's kernel, of the parent's kernel, HBM bytes)."""
    ke = 64 if bf else 32                       # input channels per chunk
    wb = 2 if bf else 4                         # bytes per weight value (hi and lo / mid planes)
    nt = 16 if cout <= 16 else 128              # column tile
    tiles = n * -(-H // 8) * -(-W // 16)        # 8 x 16-pixel tiles
    col_tiles = -(-cout // nt)
    chunks = cin // ke
    flop = 3 * 2 * tiles * 128 * col_tiles * nt * 9 * cin
    a = 10 * 18 * ke * 4 if not bf else 9 * 128 * ke * 4     # 3xTF32: one halo per chunk; bf16: one box per tap
    fill = tiles * col_tiles * chunks * (a + 9 * nt * ke * wb * 2)
    fill_parent = tiles * -(-cout // 128) * chunks * 9 * (128 * ke * 4 + 128 * ke * wb * 2)
    hbm = 4 * n * H * W * (cin + cout) + 9 * cin * cout * wb * 2
    return flop, fill, fill_parent, hbm


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--lib', action='append', default=[], help='LABEL=PATH of a libdi_b200.so (repeatable)')
    ap.add_argument('--reps', type=int, default=30)
    args = ap.parse_args()
    libs = []
    for spec in args.lib or ['tree=' + _lib.LIB_PATH]:
        label, path = spec.split('=', 1)
        L = ctypes.CDLL(os.path.abspath(path), mode=ctypes.RTLD_LOCAL)
        for name in ('di_conv3x3_tc_f32', 'di_conv3x3_tcb_f32'):
            getattr(L, name).argtypes = _lib.SIGNATURES[name]
            getattr(L, name).restype = ctypes.c_int
        libs.append((label, L))
    dev = torch.device('cuda:0')
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = torch.cuda.get_device_name(0) + ', power limit not read'
    print('device: %s' % q)
    flush = torch.empty(256 << 20 >> 2, device=dev)
    stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    g = torch.Generator().manual_seed(7)
    for label, n, cin, H, W, cout, act, bf in SHAPES:
        x = torch.randn(n, H, W, cin, generator=g).to(dev)
        wk = fold.Weight(fold.pack_conv3x3(torch.randn(cout, cin, 3, 3, generator=g) / (3 * cin ** 0.5)), dev)
        bias = torch.randn(cout, generator=g).to(dev)
        y = torch.empty(n, H, W, cout, device=dev)
        name = 'di_conv3x3_tcb_f32' if bf else 'di_conv3x3_tc_f32'
        w0, w1 = (wk.bh, wk.bm) if bf else (wk.hi, wk.lo)
        ptr = lambda t: ctypes.c_void_p(t.data_ptr())

        def call(L):
            rc = getattr(L, name)(ptr(x), ptr(w0), ptr(w1), ptr(bias), ptr(y), n, cin, H, W, cout, act, stream)
            if rc != 0:
                raise RuntimeError('%s returned %d' % (name, rc))

        times = {lb: [] for lb, _ in libs}
        outs = {}
        for lb, L in libs:                               # warm-up (module load, first launch)
            call(L)
            call(L)
            torch.cuda.synchronize()
            outs[lb] = y.clone()
        for _ in range(args.reps):
            for lb, L in libs:
                flush.zero_()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                call(L)
                e1.record()
                torch.cuda.synchronize()
                times[lb].append(e0.elapsed_time(e1) * 1e3)
        flop, fill, fill_parent, hbm = conv_model(n, cin, H, W, cout, bf)
        print('%s  %dx%dx%dx%d -> %d  %s' % (label, n, cin, H, W, cout, 'bf16 split' if bf else '3xTF32'))
        print('    MMA floor %.1f us (%.1f GFLOP issued)   L2->smem %.2f GB (parent %.2f GB)   HBM floor %.1f us' % (
            flop / PEAK[bf] * 1e6, flop / 1e9, fill / 1e9, fill_parent / 1e9, hbm / HBM * 1e6))
        ref = outs[libs[0][0]]
        for lb, _ in libs:
            ts = np.array(times[lb])
            d = float(((outs[lb] - ref).abs().max() / ref.abs().max()).item())
            print('    %-12s median %8.1f us  (min %8.1f, max %8.1f)   max rel diff vs %s %.2e' % (
                lb, np.median(ts), ts.min(), ts.max(), libs[0][0], d))


if __name__ == '__main__':
    main()
