"""Writes tests/golden/ref_configs.pt: the reference's UNCHANGED configs Fusion_0075_refactor.py and
Fusion_0075_plusplus.py as parsed by the plug-in's load_config (name -> config dict; `gpu_ids` as a list so that the
file loads with torch.load(weights_only=True)).  tests/test_host_cpu.py builds the plug-in modules from them.

    python tools/make_goldens_configs.py [--ref /root/reference] [--out tests/golden]
"""
import argparse
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAMES = ('Fusion_0075_refactor', 'Fusion_0075_plusplus')


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--ref', default='/root/reference')
    ap.add_argument('--out', default=os.path.join(ROOT, 'tests', 'golden'))
    args = ap.parse_args()
    sys.path.insert(0, ROOT)
    from projects.mmdet3d_plugin.registry import load_config
    cfgs = {}
    for n in NAMES:
        cfg = load_config(os.path.join(args.ref, 'projects', 'configs', 'nuscenes', n + '.py'))
        cfg['gpu_ids'] = list(cfg['gpu_ids'])
        cfgs[n] = cfg
    dst = os.path.join(args.out, 'ref_configs.pt')
    torch.save(cfgs, dst)
    print(dst, os.path.getsize(dst), 'bytes')


if __name__ == '__main__':
    main()
