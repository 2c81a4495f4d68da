"""Writes tests/golden/locatt_ref.pt: the outputs of the reference's own CUDA extension `localattention` (compiled
unmodified into oracle/_ref/ by oracle/build_ref.py) on the inputs of tests/locatt_cases.py.  Needs a GPU and the
built extension; the tests then compare against the stored outputs and need neither.

    python oracle/build_ref.py && python tools/make_goldens_locatt.py
"""
import os
import sys

import numpy as np
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, 'tests'))
sys.path.insert(0, os.path.join(ROOT, 'oracle'))
import build_ref  # noqa: E402
import locatt_cases as lc  # noqa: E402


def main():
    ref = build_ref.load()
    assert ref is not None, 'oracle/_ref/localattention.so is not built (python oracle/build_ref.py)'
    dev = torch.device('cuda:0')
    d = lambda *ts: [t.to(dev) for t in ts]
    out = {}
    for case in lc.DROP_IN:
        N, C, H, W, kH, kW = case
        outs = lc.drop_in_calls(ref, *d(*lc.drop_in_inputs(*case)), kH, kW)
        for name, t in outs.items():
            out[lc.key('drop_in', *case, name)] = lc.take(t)
    for N, H, W in lc.FUSED:
        q, kk, v = d(*lc.fused_inputs(N, H, W))
        sim = ref.similar_forward(q, kk, 9, 9)
        want = ref.weighting_forward(v, F.softmax(sim / np.sqrt(128), -1), 9, 9)
        out[lc.key('fused', N, H, W)] = lc.take(want)
    q, kk, v, k = lc.oracle_inputs()
    C = q.shape[1]
    sim_r = ref.similar_forward(q.to(dev), kk.to(dev), k, k).cpu()
    w = F.softmax(sim_r / np.sqrt(C), -1)
    out[lc.key('oracle', 'sim')] = sim_r.clone()                   # full: the test's softmax input
    out[lc.key('oracle', 'out')] = lc.take(ref.weighting_forward(v.to(dev), w.to(dev), k, k))
    for case in lc.BACKWARD:
        ks = case[-1]
        a, b, w = d(*lc.backward_inputs(*case))
        calls = {'similar_forward(a,b)': ref.similar_forward(a, b, ks, ks),
                 'weighting_forward(b,w)': ref.weighting_forward(b, w, ks, ks),
                 'similar_backward(b,w,ori)': ref.similar_backward(b, w, ks, ks, True),
                 'similar_backward(a,w,loc)': ref.similar_backward(a, w, ks, ks, False),
                 'weighting_backward_ori(w,a)': ref.weighting_backward_ori(w, a, ks, ks),
                 'weighting_backward_weight(b,a)': ref.weighting_backward_weight(b, a, ks, ks)}
        for name, t in calls.items():
            out[lc.key('backward', *case, name)] = lc.take(t)
    dst = os.path.join(ROOT, 'tests', 'golden', lc.GOLDEN)
    os.makedirs(os.path.dirname(dst), exist_ok=True)
    torch.save(out, dst)
    print(dst, len(out), 'arrays', os.path.getsize(dst), 'bytes')


if __name__ == '__main__':
    main()
