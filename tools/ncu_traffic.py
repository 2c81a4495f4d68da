#!/usr/bin/env python
"""DRAM traffic per launch from an `ncu --set full` report -> profiles/r2_traffic.json (read by bench.py: roofline.traffic).

    python tools/ncu_traffic.py gpurun_out/r2_ncu_full.ncu-rep [profiles/r2_traffic.json]

For every kernel of the report: mean over its captured launches of dram__bytes_read.sum + dram__bytes_write.sum, keyed by
the C-ABI entry point that launches it (the names bench.py's kernel table uses)."""
import collections
import csv
import json
import subprocess
import sys

ENTRY = [('lcab_window_tc_kernel', 'di_lcab_window_tc_f32'), ('lcab_proj_kernel', 'di_lcab_proj_f32'),
         ('lcab_window_pre_kernel', 'di_lcab_window_pre_f32'), ('msdeform_kernel', 'di_msdeform_f32'),
         ('i2p_attend_kernel', 'di_i2p_attend_f32'), ('bev_sample_kernel', 'di_bev_sample_f32'),
         ('cross_attn', 'di_cross_attn_f32'), ('dynconv_kernel', 'di_dynconv_f32'), ('seq_attn_kernel', 'di_seq_attn_f32'),
         ('gemm_tc_kernel_v3', 'gemm_tc_kernel_v3 (di_linear_tc*/di_conv3x3_tc*_nchw)'),
         ('conv3x3_tc_kernel', 'conv3x3_tc_kernel (di_conv3x3_tc*_f32)'), ('rows_mlp_kernel', 'di_rows_mlp_f32'),
         ('depth_complete_kernel', 'di_depth_complete')]


def main(rep, out):
    raw = subprocess.run(['ncu', '-i', rep, '--page', 'raw', '--csv'], capture_output=True, text=True).stdout
    rows = list(csv.reader(raw.splitlines()))
    hdr, units = rows[0], rows[1]
    ik, ir, iw = hdr.index('Kernel Name'), hdr.index('dram__bytes_read.sum'), hdr.index('dram__bytes_write.sum')
    scale = {'byte': 1.0, 'Kbyte': 1e3, 'Mbyte': 1e6, 'Gbyte': 1e9}
    acc = collections.defaultdict(list)
    for r in rows[2:]:
        name = next((e for k, e in ENTRY if k in r[ik]), None)
        if name is None:
            continue
        acc[name].append(float(r[ir].replace(',', '')) * scale[units[ir]] + float(r[iw].replace(',', '')) * scale[units[iw]])
    res = {k: sum(v) / len(v) for k, v in acc.items()}
    if 'di_lcab_proj_f32' in res and 'di_lcab_window_tc_f32' in res:      # the one-call module = both kernels
        res['di_lcab_forward_f32'] = res['di_lcab_proj_f32'] + res['di_lcab_window_tc_f32']
    res['_source'] = dict(report=rep, launches={k: len(v) for k, v in acc.items()},
                          metric='dram__bytes_read.sum + dram__bytes_write.sum per launch (ncu --set full, --clock-control none)')
    json.dump(res, open(out, 'w'), indent=1)
    print(json.dumps(res, indent=1))


if __name__ == '__main__':
    main(sys.argv[1], sys.argv[2] if len(sys.argv) > 2 else 'profiles/r2_traffic.json')
