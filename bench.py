#!/usr/bin/env python
"""Benchmark of the MMRI encoder + MMPI decoder forward (BASELINE.json metric: frames/sec).

    python bench.py --gpus N --steps K --warmup W            # this repository's sm_90a kernels
    python bench.py --impl reference --steps K --warmup W     # the reference's PyTorch math on the host CPU

Workload = BASELINE.json configs[1]: DeepInteraction-base (Fusion_0075_refactor.py) full MMRI+MMPI forward,
bs=1 per GPU: 6 x (256,112,200) camera FPN maps + (512,180,180) BEV map + ~250k LiDAR points / ~12.3k
pillars, 200 queries; synthetic seeded inputs (deepinteraction_b200/synth.py), random-init weights.

A step = one forward of imgpts_neck + pts_bbox_head over one batch.  `value` is measured with the inputs
resident in HBM; `e2e` goes through the plug-in modules' public forward with HOST (pinned) inputs: every
step copies the step's inputs host->device and the result dict device->host inside the timed region.
Inputs are 204 MB/frame (> 50 MB L2 of the H100), so iterations do not hit in L2 ("inputs larger than L2").
One process per GPU; frames are independent, so N GPUs = N independent shards (weak scaling), NCCL is
used only for the barrier / max-over-ranks of the device times.
"""
import argparse
import json
import os
import subprocess
import sys
import threading
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

METRIC = 'frames/sec MMRI+MMPI forward, 180x180 BEV / 6 cams / 200 q'
WORKLOAD = 'DeepInteraction-base Fusion_0075_refactor full MMRI+MMPI fwd, bs=1/GPU'
CFG = os.path.join(ROOT, 'projects', 'configs', 'nuscenes', 'di_b200_base_hotpath.py')
SEED = 1236


def usable_cores():
    """Host cores this process may really use: affinity mask and cgroup CPU quota (a box can report 128 CPUs
    while the container is capped at a few), capped at 32 threads (beyond that the small torch CPU ops of the
    oracle only lose time to synchronisation)."""
    n = len(os.sched_getaffinity(0)) if hasattr(os, 'sched_getaffinity') else (os.cpu_count() or 1)
    try:
        q, per = open('/sys/fs/cgroup/cpu.max').read().split()
        if q != 'max':
            n = min(n, max(1, int(float(q) / float(per))))
    except Exception:
        pass
    return max(1, min(n, 32))


class Deadline:
    """Raise TimeoutError in the main thread after `seconds` (between torch ops) -- keeps the CPU legs bounded."""

    def __init__(self, seconds):
        self.seconds = seconds

    def __enter__(self):
        import signal

        def _raise(signum, frame):
            raise TimeoutError('cpu baseline exceeded its time budget')
        self.old = signal.signal(signal.SIGALRM, _raise)
        signal.alarm(int(self.seconds))

    def __exit__(self, *a):
        import signal
        signal.alarm(0)
        signal.signal(signal.SIGALRM, self.old)
        return False


def peaks():
    p = os.path.join(ROOT, 'MEASURED_PEAKS.json')
    if os.path.exists(p):
        d = json.load(open(p))
        return dict(hbm=d['hbm_gbs'], tf=d['bf16_tflops'], tf_sus=d.get('bf16_tflops_sustained', d['bf16_tflops']),
                    src='measured')
    return dict(hbm=3350.0, tf=989.0, tf_sus=989.0, src='fallback: H100 SXM data sheet (700 W), dense BF16')


def build_models(device):
    import projects.mmdet3d_plugin  # noqa: F401  (registers the plug-in classes)
    from projects.mmdet3d_plugin.registry import load_config, build_hot_path
    from deepinteraction_b200 import synth
    torch.manual_seed(SEED)
    neck, head = build_hot_path(load_config(CFG))
    synth.randomize_norm_stats(neck, SEED)
    synth.randomize_norm_stats(head, SEED + 1)
    return neck.to(device).eval(), head.to(device).eval()


def build_oracle(neck_sd=None, head_sd=None):
    import oracle.mmri as om
    import oracle.mmpi as omp
    from projects.mmdet3d_plugin.registry import load_config
    from deepinteraction_b200 import synth
    cfg = load_config(CFG)['model']
    torch.manual_seed(SEED)
    ncfg = {k: v for k, v in cfg['imgpts_neck'].items() if k != 'type'}
    hcfg = {k: v for k, v in cfg['pts_bbox_head'].items() if k != 'type'}
    neck = om.DeepInteractionEncoder(**ncfg).eval()
    head = omp.DeepInteractionDecoder(test_cfg=cfg['test_cfg']['pts'], **hcfg).eval()
    synth.randomize_norm_stats(neck, SEED)
    synth.randomize_norm_stats(head, SEED + 1)
    if neck_sd is not None:          # check the product's weights, not a re-draw
        neck.load_state_dict({k: v.detach().cpu() for k, v in neck_sd.items()}, strict=True)
        head.load_state_dict({k: v.detach().cpu() for k, v in head_sd.items()}, strict=True)
    return neck, head


def host_frame(batch, cloud, seed, n_points=250000):
    from deepinteraction_b200 import synth
    fr = synth.make_frame_batch(seed, batch=batch, cloud=cloud, n_points=n_points)
    pin = lambda t: t.contiguous().pin_memory() if torch.cuda.is_available() else t
    pm = fr['pts_metas']
    fr['img_feats'], fr['pts_feats'] = pin(fr['img_feats']), pin(fr['pts_feats'])
    pm['pillars'], pm['pillar_coors'], pm['pillars_num_points'] = pin(pm['pillars']), pin(pm['pillar_coors']), \
        pin(pm['pillars_num_points'])
    pm['pts'] = [pin(p) for p in pm['pts']]
    return fr


def h2d(fr, device):
    pm = fr['pts_metas']
    nb = lambda t: t.to(device, non_blocking=True)
    out = dict(img_feats=nb(fr['img_feats']), pts_feats=nb(fr['pts_feats']), img_metas=fr['img_metas'],
               pts_metas=dict(pillars=nb(pm['pillars']), pillar_coors=nb(pm['pillar_coors']),
                              pillars_num_points=nb(pm['pillars_num_points']), pts=[nb(p) for p in pm['pts']]))
    return out


def h2d_bytes(fr):
    pm = fr['pts_metas']
    ts = [fr['img_feats'], fr['pts_feats'], pm['pillars'], pm['pillar_coors'], pm['pillars_num_points']] + list(pm['pts'])
    return int(sum(t.numel() * t.element_size() for t in ts))


def ncu_traffic():
    """dram__bytes_read.sum + dram__bytes_write.sum per launch of the dominant kernels, measured by `ncu --set full`
    on the bench command of this build and written by tools/ncu_traffic.py (kernel -> average bytes per launch)."""
    p = os.path.join(ROOT, 'profiles', 'r2_traffic.json')
    if os.path.exists(p):
        return json.load(open(p)), 'profiles/r2_traffic.json'
    return {}, None


def forward(neck, head, fr):
    img, pts = neck(fr['img_feats'], fr['pts_feats'], fr['img_metas'], fr['pts_metas'])
    return head(pts, img, fr['img_metas'])[0][0]


class ClockSampler:
    """nvidia-smi clocks / throttle reasons sampled every 200 ms while the timed region runs."""
    Q = ('index,clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.hw_slowdown,'
         'clocks_event_reasons.hw_thermal_slowdown,clocks_event_reasons.sw_thermal_slowdown,'
         'clocks_event_reasons.sw_power_cap')

    def __init__(self, index):
        self.index, self.rows, self.proc = index, [], None

    def __enter__(self):
        try:
            self.proc = subprocess.Popen(['nvidia-smi', f'--query-gpu={self.Q}', '--format=csv,noheader,nounits',
                                          '-lms', '200', '-i', str(self.index)], stdout=subprocess.PIPE,
                                         stderr=subprocess.DEVNULL, text=True)
            self.th = threading.Thread(target=self._read, daemon=True)
            self.th.start()
        except Exception:
            self.proc = None
        return self

    def _read(self):
        for line in self.proc.stdout:
            self.rows.append([c.strip() for c in line.split(',')])

    def __exit__(self, *a):
        if self.proc is not None:
            time.sleep(0.25)
            self.proc.terminate()
            self.th.join(timeout=2)

    def summary(self):
        sm, mx, reasons = [], [], set()
        for r in self.rows:
            try:
                sm.append(float(r[1]))
                mx.append(float(r[2]))
            except Exception:
                continue
            for name, v in zip(('hw_slowdown', 'hw_thermal_slowdown', 'sw_thermal_slowdown', 'sw_power_cap'), r[4:8]):
                if v.lower().startswith('active'):
                    reasons.add(name)
        if not sm:
            return dict(sm_mhz=None, sm_max_mhz=None, reasons=[], samples=0)
        return dict(sm_mhz=float(np.median(sm)), sm_max_mhz=float(max(mx)), reasons=sorted(reasons), samples=len(sm))


def run_reference(args):
    """The reference's own PyTorch math (oracle port; locatt window ops as 81 shifted MACs, OpenCV depth
    completion as in the reference) on the box's host cores, same workload/config/metric."""
    rank = int(os.environ.get('RANK', '0'))
    if rank != 0:
        return
    cores = usable_cores()
    torch.set_num_threads(cores)
    try:
        import cv2
        cv2.setNumThreads(cores)
    except Exception:
        pass
    torch.set_grad_enabled(False)
    neck, head = build_oracle()
    fr = host_frame(args.batch, args.cloud, SEED)
    fr = dict(img_feats=fr['img_feats'].clone(), pts_feats=fr['pts_feats'].clone(), img_metas=fr['img_metas'],
              pts_metas=fr['pts_metas'])
    t0 = time.perf_counter()
    try:
        with Deadline(170):
            forward(neck, head, fr)                  # warm-up step (also sizes the bounded sample)
    except TimeoutError:
        print(json.dumps(dict(impl='reference', unavailable='oracle frame did not finish within 170 s on this host')))
        return
    steps = max(1, args.steps)
    warm = 1
    t0 = time.perf_counter()
    for _ in range(steps):
        forward(neck, head, fr)
    dt = (time.perf_counter() - t0) / steps
    fps = args.batch / dt
    line = dict(metric=METRIC, value=fps, unit='frames/s', n_gpus=args.gpus, steps=steps, warmup=warm,
                ms_per_step=dt * 1e3, higher_is_better=True, scaling='weak', vs_baseline=None, dtype='fp32',
                data='synthetic', impl='reference',
                config=dict(workload=WORKLOAD, global_batch=args.batch, cloud=args.cloud, device='host CPU',
                            note='reference math restated in PyTorch (oracle/), all host threads'),
                cpu_baseline=dict(value=fps, unit='frames/s', cores=cores, kind='port',
                                  sample=f'{steps} full frame(s) of the same workload (bounded to ~{budget:.0f} s)'),
                e2e=dict(value=fps, unit='frames/s', h2d_bytes_per_step=0, d2h_bytes_per_step=0), gpu_launches=0)
    print(json.dumps(line), flush=True)


def randomize_deform(model, seed):
    """mmcv initialises sampling_offsets.weight / attention_weights to zero (query-independent sampling): draw them, the
    LayerNorm affines and the layer scales so that every path of the ++ encoder is exercised."""
    g = torch.Generator().manual_seed(seed + 17)
    for m in model.modules():
        if hasattr(m, 'sampling_offsets') and hasattr(m, 'attention_weights'):
            m.sampling_offsets.weight.data = torch.randn(m.sampling_offsets.weight.shape, generator=g) * 0.05
            m.attention_weights.weight.data = torch.randn(m.attention_weights.weight.shape, generator=g) * 0.1
            m.attention_weights.bias.data = torch.randn(m.attention_weights.bias.shape, generator=g) * 0.1
        if isinstance(m, torch.nn.LayerNorm):
            m.weight.data = 1 + 0.2 * torch.randn(m.weight.shape, generator=g)
            m.bias.data = 0.1 * torch.randn(m.bias.shape, generator=g)
    for n, p_ in model.named_parameters():
        if n.endswith('scale'):
            p_.data.fill_(0.7)


def pp_host_frame(batch, seed, n_points=250000):
    """Config 4 inputs (SURVEY.md 8(d)): image levels (B*6,256,112,200), (B*6,256,56,100); BEV maps [(B,512,180,180),
    (B,256,180,180), (B,256,180,180)]; the base frame's cloud / pillars / camera rig."""
    from deepinteraction_b200 import synth
    fr = synth.make_frame_batch(seed, batch=batch, cloud='lidar', n_points=n_points, c_pts=256)
    g = torch.Generator().manual_seed(seed + 3)
    p1, p2 = fr['pts_feats'], torch.randn(batch, 256, 180, 180, generator=g)
    pin = lambda t: t.contiguous().pin_memory() if torch.cuda.is_available() else t
    fr['img_levels'] = [pin(fr['img_feats']), pin(torch.randn(batch * 6, 256, 56, 100, generator=g))]
    fr['pts_levels'] = [pin(torch.cat([p1, p2], 1)), pin(p1), pin(p2)]
    pm = fr['pts_metas']
    for k in ('pillars', 'pillar_coors', 'pillars_num_points'):
        pm[k] = pin(pm[k])
    pm['pts'] = [pin(p) for p in pm['pts']]
    return fr


def run_plusplus(args):
    """BASELINE.json config 4: the ++ ("deformable") encoder FusionTransformerv4 (Fusion_0075_plusplus.py imgpts_neck),
    bs = --batch per GPU (default 2: bs=4 on 2 GPUs).  One JSON line like the base workload: `value` with the inputs
    resident in HBM, `e2e` with host buffers (H2D of the five input maps + pillars / points and D2H of the three output
    maps inside the timed region), per-kernel table, CPU oracle of the same module for ONE sample as cpu_baseline."""
    world = int(os.environ.get('WORLD_SIZE', '1'))
    rank = int(os.environ.get('RANK', '0'))
    local = int(os.environ.get('LOCAL_RANK', '0'))
    assert torch.cuda.is_available(), 'bench.py needs a CUDA device: the product path has no CPU fallback'
    torch.cuda.set_device(local)
    device = torch.device('cuda', local)
    if world > 1:
        import torch.distributed as dist
        os.environ.setdefault('MASTER_ADDR', '127.0.0.1')
        dist.init_process_group('nccl', device_id=device)
    torch.set_grad_enabled(False)
    import projects.mmdet3d_plugin  # noqa: F401
    from projects.mmdet3d_plugin.registry import load_config, build_hot_path
    from deepinteraction_b200 import ops, synth, graph as di_graph
    cfg = load_config(os.path.join(ROOT, 'projects', 'configs', 'nuscenes', 'di_b200_plusplus_hotpath.py'))
    torch.manual_seed(SEED)
    neck, head = build_hot_path(cfg)
    synth.randomize_norm_stats(neck, SEED)
    randomize_deform(neck, SEED)
    synth.randomize_norm_stats(head, SEED + 1)
    neck = neck.to(device).eval()
    head = head.to(device).eval() if args.with_decoder else None      # --with-decoder: + DeepInteractionPlusPlusDecoder
    B = args.batch
    NF = 3
    hosts = [pp_host_frame(B, SEED + 1000 * rank + i, n_points=int(250000 * (0.9 + 0.05 * i))) for i in range(NF)]
    nb = lambda t: t.to(device, non_blocking=True)

    def to_dev(fr):
        pm = fr['pts_metas']
        return dict(img=[nb(t) for t in fr['img_levels']], pts=[nb(t) for t in fr['pts_levels']], img_metas=fr['img_metas'],
                    pts_metas=dict(pillars=nb(pm['pillars']), pillar_coors=nb(pm['pillar_coors']),
                                   pillars_num_points=nb(pm['pillars_num_points']), pts=[nb(p) for p in pm['pts']]))
    devs = [to_dev(f) for f in hosts]
    enc = lambda d: neck(d['img'], d['pts'], d['img_metas'], d['pts_metas'])

    def fwd(d):
        o = enc(d)
        return o if head is None else head(o[1], o[0], d['img_metas'])
    results = lambda o: (o[0], o[1][0], o[1][1]) if head is None else tuple(o[0][0].values())
    W, K = max(args.warmup, 3), args.steps
    for _ in range(3):
        for d in devs:
            out = fwd(d)
    torch.cuda.synchronize()

    def barrier():
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()

    def max_over_ranks(ms):
        if world > 1:
            t = torch.tensor([ms], device=device, dtype=torch.float64)
            dist.all_reduce(t, op=dist.ReduceOp.MAX)
            return float(t.item())
        return ms
    for i in range(W):
        fwd(devs[i % NF])
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    with ClockSampler(local) as clk:
        barrier()
        l0 = ops.LAUNCHES[0]
        e0.record()
        for i in range(K):
            out = fwd(devs[i % NF])
        e1.record()
        barrier()
        launches = ops.LAUNCHES[0] - l0
        ms = max_over_ranks(e0.elapsed_time(e1))
        # end to end: host -> device copies of every input of the step, forward, device -> host of the three outputs
        flat = lambda fr: list(fr['img_levels']) + list(fr['pts_levels'])
        dset = dict(img=[torch.empty_like(t) for t in devs[0]['img']], pts=[torch.empty_like(t) for t in devs[0]['pts']])
        outs_host = [torch.empty(o.shape, dtype=o.dtype).pin_memory() for o in results(out)]
        h2d_b = int(np.mean([sum(t.numel() * 4 for t in flat(f)) + sum(v.numel() * v.element_size() for k_, v in
                             f['pts_metas'].items() if k_ != 'pts') + sum(p.numel() * 4 for p in f['pts_metas']['pts'])
                             for f in hosts]))

        def e2e_step(i):
            fh = hosts[i % NF]
            for dst, src in zip(dset['img'] + dset['pts'], flat(fh)):
                dst.copy_(src, non_blocking=True)
            pm = fh['pts_metas']
            o = fwd(dict(img=dset['img'], pts=dset['pts'], img_metas=fh['img_metas'],
                         pts_metas=dict(pillars=nb(pm['pillars']), pillar_coors=nb(pm['pillar_coors']),
                                        pillars_num_points=nb(pm['pillars_num_points']), pts=[nb(p) for p in pm['pts']])))
            for dst, src in zip(outs_host, results(o)):
                dst.copy_(src, non_blocking=True)
        for i in range(3):
            e2e_step(i)
        barrier()
        e2, e3 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e2.record()
        for i in range(K):
            e2e_step(i)
        e3.record()
        barrier()
        ms_e2e = max_over_ranks(e2.elapsed_time(e3))
    clocks = clk.summary()
    if rank != 0:
        if world > 1:
            dist.destroy_process_group()
        return
    frames = B * world * K
    pk = peaks()
    di_graph.ENABLED[0] = False
    neck._graphs.clear()
    if head is not None:
        head._graphs.clear()
    ops.PROFILE_FLUSH[0] = torch.empty(256 * 1024 * 1024 // 4, device=device)   # cold-cache, queue-full kernel timing
    ops.PROFILE[0] = []
    for _ in range(2):
        fwd(devs[0])
    torch.cuda.synchronize()
    agg = {}
    for name, a, b, nbytes, flops, mod in ops.PROFILE[0]:
        d = agg.setdefault(name.split(' ')[0], dict(ms=0.0, n=0, bytes=0, flops=0))
        d['ms'] += a.elapsed_time(b)
        d['n'] += 1
        d['bytes'] += nbytes
        d['flops'] += flops
    ops.PROFILE[0] = None
    ops.PROFILE_FLUSH[0] = None
    di_graph.ENABLED[0] = True
    tot = sum(d['ms'] for d in agg.values())
    kernels = [dict(name=n, launches_per_step=d['n'] / 2, ms_per_step=d['ms'] / 2, share=d['ms'] / tot,
                    avg_us=d['ms'] / d['n'] * 1e3, gbs=d['bytes'] / max(d['ms'], 1e-9) / 1e6)
               for n, d in sorted(agg.items(), key=lambda kv: -kv[1]['ms'])]
    top = kernels[0]
    roof = dict(bound='hbm', achieved=top['gbs'], peak=pk['hbm'], unit='GB/s', frac=top['gbs'] / pk['hbm'], kernel=top['name'],
                traffic=None, peak_source=pk['src'], share_of_step=top['share'], avg_launch_us=top['avg_us'])
    cpu = None
    if not args.no_cpu_baseline and world == 1:
        import oracle.mmri_pp as opp
        cores = usable_cores()
        torch.set_num_threads(cores)
        try:
            with Deadline(170):
                o = opp.FusionTransformerv4(**{k: v for k, v in cfg['model']['imgpts_neck'].items() if k != 'type'}).eval()
                o.load_state_dict({k: v.detach().cpu() for k, v in neck.state_dict().items()}, strict=True)
                f1 = pp_host_frame(1, SEED + 77, n_points=120000)
                t0 = time.perf_counter()
                r_img, r_pts = o(list(f1['img_levels']), list(f1['pts_levels']), f1['img_metas'], f1['pts_metas'])
                dt = time.perf_counter() - t0
            d1 = to_dev(f1)
            g_img, g_pts = enc(d1)
            rel = lambda a, b: float((a.cpu() - b).abs().max() / b.abs().max().clamp_min(1e-12))
            cpu = dict(value=1.0 / dt, unit='frames/s', cores=cores, kind='port',
                       sample='1 sample (6 cameras) of the same workload through oracle/mmri_pp.py (reference math, fp32)',
                       max_rel_err_vs_gpu=max(rel(g_img, r_img), rel(g_pts[1], r_pts[1])))
        except TimeoutError:
            cpu = dict(value=None, unit='frames/s', cores=cores, kind='port', sample='1 sample did not finish within 170 s')
    what = '++ MMRI encoder (FusionTransformerv4)' + (' + ++ MMPI decoder' if head is not None else '')
    line = dict(metric='frames/sec %s, 180x180 BEV / 6 cams x 2 levels' % what, value=frames / (ms * 1e-3),
                unit='frames/s', n_gpus=world, steps=K, warmup=W, ms_per_step=ms / K, higher_is_better=True, scaling='weak',
                vs_baseline=None, dtype='fp32', data='synthetic',
                config=dict(workload='DeepInteraction++ Fusion_0075_plusplus imgpts_neck%s (deformable variant), bs=%d/GPU'
                            % (' + pts_bbox_head' if head is not None else '', B),
                            global_batch=B * world, parallelism=f'dp{world} (independent frames, no data-path collective)',
                            l2='inputs (%.0f MB/step) larger than L2; %d distinct frames cycled' % (h2d_b / 1e6, NF)),
                clocks=clocks, e2e=dict(value=frames / (ms_e2e * 1e-3), unit='frames/s', h2d_bytes_per_step=h2d_b,
                                        d2h_bytes_per_step=int(sum(t.numel() * 4 for t in outs_host)), ms_per_step=ms_e2e / K),
                gpu_launches=launches, launches_per_step=launches / K, roofline=roof, cpu_baseline=cpu, kernels=kernels[:12])
    print(json.dumps(line), flush=True)
    if world > 1:
        dist.destroy_process_group()


def run_large(args):
    """BASELINE.json config 5 ("large" sweep): MMRI encoder at a 256x256 BEV grid with 6 camera maps of 128x352
    (512x1408 inputs, stride 4) and hidden width C = --channels in {128, 256, 512}; for C = 128 the MMPI decoder with 300
    queries follows (C != 128 cannot be built: DynamicConv is hard-coded to 128 channels, decoder_utils.py:589-591).
    Pillars are generated on the GPU from the raw points inside the forward (pts_metas carries `pts` only).  Same JSON
    contract as the base workload; frames run one after the other (no frames in flight)."""
    world = int(os.environ.get('WORLD_SIZE', '1'))
    rank = int(os.environ.get('RANK', '0'))
    local = int(os.environ.get('LOCAL_RANK', '0'))
    assert torch.cuda.is_available(), 'bench.py needs a CUDA device: the product path has no CPU fallback'
    torch.cuda.set_device(local)
    device = torch.device('cuda', local)
    if world > 1:
        import torch.distributed as dist
        os.environ.setdefault('MASTER_ADDR', '127.0.0.1')
        dist.init_process_group('nccl', device_id=device)
    torch.set_grad_enabled(False)
    import projects.mmdet3d_plugin  # noqa: F401
    from projects.mmdet3d_plugin.registry import load_config, build_hot_path
    from deepinteraction_b200 import ops, synth, graph as di_graph
    C, B, BEV, IN_HW = args.channels, args.batch, 256, (512, 1408)
    cfg = load_config(CFG)
    cfg['model']['imgpts_neck']['hidden_channel'] = C
    cfg['model']['pts_bbox_head']['num_proposals'] = 300
    cfg['model']['test_cfg']['pts']['grid_size'] = [BEV * 8, BEV * 8, 40]
    torch.manual_seed(SEED)
    if C == 128:
        neck, head = build_hot_path(cfg)
        synth.randomize_norm_stats(head, SEED + 1)
        head = head.to(device).eval()
    else:
        from projects.mmdet3d_plugin.registry import build_neck
        neck, head = build_neck(cfg), None
    synth.randomize_norm_stats(neck, SEED)
    neck = neck.to(device).eval()
    NF = 3
    pin = lambda t: t.contiguous().pin_memory()

    def mk(seed, n_points):
        fr = synth.make_frame_batch(seed, batch=B, in_hw=IN_HW, bev_hw=(BEV, BEV), n_points=n_points)
        return dict(img=pin(fr['img_feats']), pts=pin(fr['pts_feats']), img_metas=fr['img_metas'],
                    cloud=[pin(p) for p in fr['pts_metas']['pts']])
    hosts = [mk(SEED + 1000 * rank + i, int(250000 * (0.9 + 0.05 * i))) for i in range(NF)]
    nb = lambda t: t.to(device, non_blocking=True)
    devs = [dict(img=nb(f['img']), pts=nb(f['pts']), img_metas=f['img_metas'], cloud=[nb(p) for p in f['cloud']]) for f in hosts]

    def fwd(d):
        img, pts = neck(d['img'], d['pts'], d['img_metas'], dict(pts=d['cloud']))
        return (img, pts[0], pts[1]) if head is None else tuple(head(pts, img, d['img_metas'])[0][0].values())
    W, K = max(args.warmup, 3), args.steps
    for _ in range(3):
        for d in devs:
            out = fwd(d)
    torch.cuda.synchronize()

    def barrier():
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()

    def max_over_ranks(ms):
        if world > 1:
            t = torch.tensor([ms], device=device, dtype=torch.float64)
            dist.all_reduce(t, op=dist.ReduceOp.MAX)
            return float(t.item())
        return ms
    for i in range(W):
        fwd(devs[i % NF])
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    with ClockSampler(local) as clk:
        barrier()
        l0 = ops.LAUNCHES[0]
        e0.record()
        for i in range(K):
            out = fwd(devs[i % NF])
        e1.record()
        barrier()
        launches = ops.LAUNCHES[0] - l0
        ms = max_over_ranks(e0.elapsed_time(e1))
        dset = dict(img=torch.empty_like(devs[0]['img']), pts=torch.empty_like(devs[0]['pts']))
        outs_host = [torch.empty(o.shape, dtype=o.dtype).pin_memory() for o in out]
        h2d_b = int(np.mean([sum(t.numel() * 4 for t in [f['img'], f['pts']] + f['cloud']) for f in hosts]))

        def e2e_step(i):
            fh = hosts[i % NF]
            dset['img'].copy_(fh['img'], non_blocking=True)
            dset['pts'].copy_(fh['pts'], non_blocking=True)
            o = fwd(dict(img=dset['img'], pts=dset['pts'], img_metas=fh['img_metas'], cloud=[nb(p) for p in fh['cloud']]))
            for dst, src in zip(outs_host, o):
                dst.copy_(src, non_blocking=True)
        for i in range(3):
            e2e_step(i)
        barrier()
        e2, e3 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e2.record()
        for i in range(K):
            e2e_step(i)
        e3.record()
        barrier()
        ms_e2e = max_over_ranks(e2.elapsed_time(e3))
    clocks = clk.summary()
    if rank != 0:
        if world > 1:
            dist.destroy_process_group()
        return
    frames = B * world * K
    pk = peaks()
    di_graph.ENABLED[0] = False
    neck._graphs.clear()
    if head is not None:
        head._graphs.clear()
    ops.PROFILE_FLUSH[0] = torch.empty(256 * 1024 * 1024 // 4, device=device)   # cold-cache, queue-full kernel timing
    ops.PROFILE[0] = []
    for _ in range(2):
        fwd(devs[0])
    torch.cuda.synchronize()
    agg = {}
    for name, a, b, nbytes, flops, mod in ops.PROFILE[0]:
        d = agg.setdefault(name.split(' ')[0], dict(ms=0.0, n=0, bytes=0, flops=0))
        d['ms'] += a.elapsed_time(b)
        d['n'] += 1
        d['bytes'] += nbytes
        d['flops'] += flops
    ops.PROFILE[0] = None
    ops.PROFILE_FLUSH[0] = None
    di_graph.ENABLED[0] = True
    tot = sum(d['ms'] for d in agg.values())
    kernels = [dict(name=n, launches_per_step=d['n'] / 2, ms_per_step=d['ms'] / 2, share=d['ms'] / tot,
                    avg_us=d['ms'] / d['n'] * 1e3, gbs=d['bytes'] / max(d['ms'], 1e-9) / 1e6,
                    tflops=d['flops'] / max(d['ms'], 1e-9) / 1e9)
               for n, d in sorted(agg.items(), key=lambda kv: -kv[1]['ms'])]
    top = kernels[0]
    roof = dict(bound='hbm', achieved=top['gbs'], peak=pk['hbm'], unit='GB/s', frac=top['gbs'] / pk['hbm'], kernel=top['name'],
                traffic=None, peak_source=pk['src'], share_of_step=top['share'], avg_launch_us=top['avg_us'])
    what = 'MMRI encoder' + (' + MMPI decoder (300 q)' if head is not None else ' (decoder needs C = 128)')
    line = dict(metric='frames/sec %s, 256x256 BEV / 6 cams 128x352 / C=%d' % (what, C), value=frames / (ms * 1e-3),
                unit='frames/s', n_gpus=world, steps=K, warmup=W, ms_per_step=ms / K, higher_is_better=True, scaling='weak',
                vs_baseline=None, dtype='fp32', data='synthetic',
                config=dict(workload='BASELINE config 5 large sweep: DeepInteraction-base modules, 256x256 BEV, 6 x 128x352 maps, '
                                     'C=%d, bs=%d/GPU' % (C, B), global_batch=B * world,
                            parallelism=f'dp{world} (independent frames, no data-path collective)',
                            l2='inputs (%.0f MB/step) larger than L2; %d distinct frames cycled' % (h2d_b / 1e6, NF)),
                clocks=clocks, e2e=dict(value=frames / (ms_e2e * 1e-3), unit='frames/s', h2d_bytes_per_step=h2d_b,
                                        d2h_bytes_per_step=int(sum(t.numel() * t.element_size() for t in outs_host)),
                                        ms_per_step=ms_e2e / K),
                gpu_launches=launches, launches_per_step=launches / K, roofline=roof, cpu_baseline=None, kernels=kernels[:12])
    print(json.dumps(line), flush=True)
    if world > 1:
        dist.destroy_process_group()


def dump_outputs(d, out, budget=64 << 20):
    """out: name -> CPU tensor.  Each array gets an equal share of the byte budget; a larger one is replaced by a sorted
    sample of its flattened elements drawn with a fixed seed (same positions from run to run)."""
    os.makedirs(d, exist_ok=True)
    share = budget // max(1, len(out))
    for k, v in sorted(out.items()):
        a = v.float().numpy()
        if a.nbytes > share:
            idx = np.sort(np.random.default_rng(0).choice(a.size, share // 4, replace=False))
            a = a.reshape(-1)[idx]
        np.save(os.path.join(d, '%s.npy' % k), np.ascontiguousarray(a, dtype=np.float32))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--workload', default='base', choices=['base', 'plusplus', 'large'],
                    help='base = BASELINE.json config 2 (the headline metric); plusplus = config 4 (++ encoder); '
                         'large = config 5 (256x256 BEV, 128x352 maps, --channels C)')
    ap.add_argument('--channels', type=int, default=128, choices=[128, 256, 512], help='large workload: hidden width C')
    ap.add_argument('--gpus', type=int, default=1)
    ap.add_argument('--steps', type=int, default=30)
    ap.add_argument('--warmup', type=int, default=5)
    ap.add_argument('--impl', default='ours', choices=['ours', 'reference'])
    ap.add_argument('--batch', type=int, default=1, help='frames per GPU per step')
    ap.add_argument('--cloud', default='lidar', choices=['lidar', 'dense'])
    ap.add_argument('--no-cpu-baseline', action='store_true')
    ap.add_argument('--with-decoder', action='store_true',
                    help='plusplus workload: run DeepInteractionPlusPlusDecoder after the ++ encoder (default: encoder only, '
                         'as BASELINE.json config 4 is quoted)')
    ap.add_argument('--profile-steps', type=int, default=3)
    ap.add_argument('--inflight', type=int, default=5, help='independent frames in flight per GPU (CUDA streams)')
    ap.add_argument('--dump-outputs', metavar='DIR', default=None,
                    help='after the timed steps, write what the last timed step returned as DIR/<name>.npy (float32; '
                         'at most 64 MB in all, larger arrays as a fixed seeded sample) for output-by-output comparison')
    ap.add_argument('--frames', type=int, default=9, help='distinct synthetic frames (different point / pillar counts) cycled '
                    'through the timed regions, each in its own device buffers')
    args = ap.parse_args()
    if args.dump_outputs and (args.impl != 'ours' or args.workload != 'base'):
        ap.error('--dump-outputs is supported for the base workload of impl=ours')
    if args.impl == 'reference':
        return run_reference(args)
    if args.workload == 'plusplus':
        if args.batch == 1:
            args.batch = 2                       # config 4: bs=4 on 2 GPUs
        return run_plusplus(args)
    if args.workload == 'large':
        return run_large(args)

    world = int(os.environ.get('WORLD_SIZE', '1'))
    rank = int(os.environ.get('RANK', '0'))
    local = int(os.environ.get('LOCAL_RANK', '0'))
    assert torch.cuda.is_available(), 'bench.py (impl=ours) needs a CUDA device: the product path has no CPU fallback'
    torch.cuda.set_device(local)
    device = torch.device('cuda', local)
    if world > 1:
        import torch.distributed as dist
        os.environ.setdefault('MASTER_ADDR', '127.0.0.1')
        dist.init_process_group('nccl', device_id=device)
    assert world == args.gpus or world == 1, f'--gpus {args.gpus} but WORLD_SIZE={world}'
    torch.set_grad_enabled(False)
    from deepinteraction_b200 import ops

    neck, head = build_models(device)
    W, K = max(args.warmup, 3), args.steps
    from deepinteraction_b200.pipeline import FramePipeline
    depth = max(args.inflight, 1)
    pipe = FramePipeline(neck, head, depth=depth, device=device)
    # NF distinct frames (different seeds, point counts and therefore pillar counts), each in its own device buffers;
    # NF is a multiple of the pipeline depth so that a frame always runs on the same stream (one graph per frame set).
    NF = max(1, args.frames // depth) * depth if args.frames >= depth else args.frames
    frames_host = [host_frame(args.batch, args.cloud, SEED + 1000 * rank + i, n_points=int(250000 * (0.86 + 0.035 * i)))
                   for i in range(NF)]
    frames_dev = [h2d(f, device) for f in frames_host]
    fr_host, fr_dev = frames_host[0], frames_dev[0]
    n_pillars = [int(f['pts_metas']['pillars'].shape[0]) for f in frames_host]
    n_points = [int(sum(p.shape[0] for p in f['pts_metas']['pts'])) for f in frames_host]
    torch.cuda.synchronize()
    out = forward(neck, head, fr_dev)                   # one plain call (default stream), then per-stream graph capture
    for _ in range(3):                                  # every (frame set, stream) pair captures its graphs
        for i in range(NF):
            pipe.submit(frames_dev[i], stream_index=i % depth)
    pipe.join()
    for i in range(W):
        out = pipe.submit(frames_dev[i % NF], stream_index=i % depth)[0]
    pipe.join()
    torch.cuda.synchronize()

    def barrier():
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()

    def max_over_ranks(ms):
        if world > 1:
            t = torch.tensor([ms], device=device, dtype=torch.float64)
            dist.all_reduce(t, op=dist.ReduceOp.MAX)
            return float(t.item())
        return ms

    # ---- timed region 1: inputs resident in HBM (NF distinct frames cycled) ------------------------------
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    with ClockSampler(local) as clk:
        barrier()
        l0 = ops.LAUNCHES[0]
        e0.record()
        for i in range(K):
            out = pipe.submit(frames_dev[i % NF], stream_index=i % depth)[0]
        pipe.join()
        e1.record()
        barrier()
        launches = ops.LAUNCHES[0] - l0
        ms = max_over_ranks(e0.elapsed_time(e1))
        # the last timed step's result (the pipeline's buffers are reused by the next region)
        last_out = {k: v.detach().cpu() for k, v in out.items()} if args.dump_outputs else None
        # ---- timed region 2: end to end through the plug-in API, host buffers ------------------------------
        # NSETS device input sets; the host->device copy of a later step runs on a copy stream while earlier steps
        # compute on the pipeline's streams; every step's result goes back to pinned host memory on its own stream.
        # The feature maps land in persistent per-set buffers; the per-frame pillar / point arrays (their sizes change
        # from frame to frame) land in the leading rows of per-set capacity buffers and are passed as exact-size views.
        NSETS = depth + 1
        outs_host = [{k: torch.empty(v.shape, dtype=v.dtype).pin_memory() for k, v in out.items()} for _ in range(depth)]
        copy_stream = torch.cuda.Stream()
        cap_p, cap_n = max(n_pillars), max(max(int(p.shape[0]) for p in f['pts_metas']['pts']) for f in frames_host)
        pm0 = fr_host['pts_metas']
        mk = lambda t, n: torch.empty((n,) + tuple(t.shape[1:]), dtype=t.dtype, device=device)
        sets = [dict(img_feats=torch.empty_like(fr_dev['img_feats']), pts_feats=torch.empty_like(fr_dev['pts_feats']),
                     pillars=mk(pm0['pillars'], cap_p), pillar_coors=mk(pm0['pillar_coors'], cap_p),
                     pillars_num_points=mk(pm0['pillars_num_points'], cap_p),
                     pts=[mk(p, cap_n) for p in pm0['pts']]) for _ in range(NSETS)]
        torch.cuda.synchronize()
        done = [None] * NSETS
        ready = [torch.cuda.Event() for _ in range(NSETS)]
        views = [None] * NSETS

        def issue_copy(i):
            bi, fh = i % NSETS, frames_host[i % NF]
            st, pm = sets[bi], fh['pts_metas']
            with torch.cuda.stream(copy_stream):
                if done[bi] is not None:
                    copy_stream.wait_event(done[bi])          # the forward that read this set has finished
                st['img_feats'].copy_(fh['img_feats'], non_blocking=True)
                st['pts_feats'].copy_(fh['pts_feats'], non_blocking=True)
                npl = pm['pillars'].shape[0]
                v = dict(pillars=st['pillars'][:npl], pillar_coors=st['pillar_coors'][:npl],
                         pillars_num_points=st['pillars_num_points'][:npl], pts=[])
                for k_ in ('pillars', 'pillar_coors', 'pillars_num_points'):
                    v[k_].copy_(pm[k_], non_blocking=True)
                for dst, src in zip(st['pts'], pm['pts']):
                    d = dst[:src.shape[0]]
                    d.copy_(src, non_blocking=True)
                    v['pts'].append(d)
                views[bi] = dict(img_feats=st['img_feats'], pts_feats=st['pts_feats'], img_metas=fh['img_metas'], pts_metas=v)
                ready[bi].record(copy_stream)

        def step(i):
            bi = i % NSETS
            o, ev, s_ = pipe.submit(views[bi], wait_event=ready[bi], stream_index=i % depth)
            done[bi] = ev
            with torch.cuda.stream(s_):
                for k_, v in o.items():
                    outs_host[i % depth][k_].copy_(v, non_blocking=True)

        for r in range(3):                                       # every (input set, stream) pair owns its graphs
            for i in range(NSETS * depth):
                issue_copy(i)
                step(i)
        pipe.join()
        barrier()
        e2, e3 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e2.record()
        issue_copy(0)
        host_fwd = 0.0
        for i in range(K):
            if i + 1 < K:
                issue_copy(i + 1)
            t_h = time.perf_counter()
            step(i)
            host_fwd += time.perf_counter() - t_h
        pipe.join()
        e3.record()
        barrier()
        ms_e2e = max_over_ranks(e2.elapsed_time(e3))
    clocks = clk.summary()

    if rank != 0:
        if world > 1:
            dist.destroy_process_group()
        return
    frames = args.batch * world * K
    value = frames / (ms * 1e-3)
    e2e_value = frames / (ms_e2e * 1e-3)
    pk = peaks()

    # ---- encoder / decoder split of the step (graph replay, device-resident inputs) -----
    def stage_ms(fn, n=10):
        fn(); fn()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        a.record()
        for _ in range(n):
            fn()
        b.record()
        torch.cuda.synchronize()
        return a.elapsed_time(b) / n
    enc_out = neck(fr_dev['img_feats'], fr_dev['pts_feats'], fr_dev['img_metas'], fr_dev['pts_metas'])
    enc_out = (enc_out[0].clone(), [t.clone() for t in enc_out[1]])
    stages = dict(encoder_ms=stage_ms(lambda: neck(fr_dev['img_feats'], fr_dev['pts_feats'], fr_dev['img_metas'],
                                                   fr_dev['pts_metas'])),
                  decoder_ms=stage_ms(lambda: head(enc_out[1], enc_out[0], fr_dev['img_metas'])))

    # ---- per-kernel device times (separate pass so the event pairs do not perturb the timed regions) -----
    from deepinteraction_b200 import graph as di_graph
    di_graph.ENABLED[0] = False                  # event-instrumented pass: launch kernel by kernel
    neck._graphs.clear()
    head._graphs.clear()
    ops.PROFILE_FLUSH[0] = torch.empty(256 * 1024 * 1024 // 4, device=device)   # cold-cache, queue-full kernel timing
    ops.PROFILE[0] = []
    for _ in range(max(args.profile_steps, 1)):
        forward(neck, head, fr_dev)
    args.profile_steps = max(args.profile_steps, 1)
    torch.cuda.synchronize()
    agg = {}
    shapes = {}
    mods = {}
    for name, a, b, nbytes, flops, mod in ops.PROFILE[0]:
        if mod is not None:
            md = mods.setdefault(mod[0], dict(ms=0.0, bytes=0, flops=0, launches=0, seen=set()))
            md['ms'] += a.elapsed_time(b)
            md['launches'] += 1
            md['bytes'], md['flops'] = mod[1], mod[2]
        sd = shapes.setdefault((name, nbytes, flops), [0, 0.0])
        sd[0] += 1
        sd[1] += a.elapsed_time(b)
        name = name.split(' ')[0]                    # drop the shape tag for the per-kernel totals
        d = agg.setdefault(name, dict(ms=0.0, n=0, bytes=0, flops=0))
        d['ms'] += a.elapsed_time(b)
        d['n'] += 1
        d['bytes'] += nbytes
        d['flops'] += flops
    ops.PROFILE[0] = None
    ops.PROFILE_FLUSH[0] = None
    di_graph.ENABLED[0] = True
    if os.environ.get('DI_B200_SHAPES'):             # per-shape table (stderr), for kernel work
        for (name, nbytes, flops), (n, t) in sorted(shapes.items(), key=lambda kv: -kv[1][1]):
            print('%-44s n/step=%5.1f  avg=%8.1f us  total=%7.3f ms/step  %8.2f MB %8.3f GFLOP' % (
                name, n / args.profile_steps, t / n * 1e3, t / args.profile_steps, nbytes / 1e6, flops / 1e9),
                file=sys.stderr)
    total_ms = sum(d['ms'] for d in agg.values())
    kernels = []
    for name, d in sorted(agg.items(), key=lambda kv: -kv[1]['ms']):
        per = d['ms'] / d['n']
        kernels.append(dict(name=name, launches_per_step=d['n'] / args.profile_steps,
                            ms_per_step=d['ms'] / args.profile_steps, share=d['ms'] / total_ms,
                            avg_us=per * 1e3, gbs=(d['bytes'] / d['n']) / (per * 1e-3) / 1e9 if per > 0 else 0.0,
                            tflops=(d['flops'] / d['n']) / (per * 1e-3) / 1e12 if per > 0 else 0.0))
    top = kernels[0]
    intensity = (agg[top['name']]['flops'] / max(agg[top['name']]['bytes'], 1))
    if intensity > pk['tf'] * 1e12 / (pk['hbm'] * 1e9):
        roof = dict(bound='tensor', achieved=top['tflops'], peak=pk['tf'], unit='TFLOP/s', frac=top['tflops'] / pk['tf'])
    else:
        roof = dict(bound='hbm', achieved=top['gbs'], peak=pk['hbm'], unit='GB/s', frac=top['gbs'] / pk['hbm'])
    traffic, traffic_src = ncu_traffic()
    roof.update(kernel=top['name'], traffic=traffic.get(top['name']), traffic_source=traffic_src, peak_source=pk['src'],
                share_of_step=top['share'], avg_launch_us=top['avg_us'])
    # per-MODULE roofline with the module-boundary numerators of SURVEY.md 8(d): time = sum of the module's kernel
    # durations (eager, serialised pass), calls = instances per frame
    calls = {'MMRI_I2P': 2, 'LCAB_self_bev': 2, 'P_out_proj+P_integration': 2, 'MMRI_P2I': 2, 'LCAB_self_img': 2,
             'I_out_proj+I_integration': 2, 'ImageRCNNBlock': 2, 'PointRCNNBlock': 2, 'prediction_heads': 5}
    modules = []
    for name, md in mods.items():
        n = calls.get(name, 1) * args.profile_steps
        us = md['ms'] / n * 1e3
        gbs = md['bytes'] / (us * 1e-6) / 1e9 if us > 0 else 0.0
        tfl = md['flops'] / (us * 1e-6) / 1e12 if us > 0 else 0.0
        modules.append(dict(module=name, calls_per_frame=calls.get(name, 1), us_per_call=us, launches_per_call=md['launches'] / n,
                            bytes_mb=md['bytes'] / 1e6, gflop=md['flops'] / 1e9, gbs=gbs, frac_of_hbm_peak=gbs / pk['hbm'],
                            tflops=tfl, frac_of_bf16_peak=tfl / pk['tf']))
    modules.sort(key=lambda m: -m['us_per_call'] * m['calls_per_frame'])

    cpu = None
    if not args.no_cpu_baseline and world == 1:
        cores = usable_cores()
        torch.set_num_threads(cores)
        try:
            with Deadline(150):
                o_neck, o_head = build_oracle(neck.state_dict(), head.state_dict())
                # the check frame of the workload definition (250 000 draws, seed SEED + rank), not one of the cycled ones
                fr_chk = host_frame(args.batch, args.cloud, SEED + rank)
                frc = dict(img_feats=fr_chk['img_feats'], pts_feats=fr_chk['pts_feats'],
                           img_metas=fr_chk['img_metas'], pts_metas=fr_chk['pts_metas'])
                t0 = time.perf_counter()
                ref_out = forward(o_neck, o_head, frc)
                dt = time.perf_counter() - t0
            # The ORDER of the proposals is defined only up to the fp32 rounding of the heat-map scores (top-k over 324 000
            # values that agree to ~1e-6 between the two implementations: neighbouring ranks can swap).  The decoder is
            # equivariant to that order, so the proposals are matched by their heat-map score vectors before comparing.
            got = {k: v.float().cpu().clone() for k, v in forward(neck, head, h2d(fr_chk, device)).items()}   # the SAME frame
            labels = head.query_labels.cpu().clone()
            P_ = got['query_heatmap_score'].shape[-1]
            moved, unmatched = 0, 0
            errs, lab_ok = {k: 0.0 for k in ref_out}, True
            for b in range(got['query_heatmap_score'].shape[0]):
                dist = torch.cdist(ref_out['query_heatmap_score'][b].t().double(), got['query_heatmap_score'][b].t().double())
                # a BEV cell can be proposed for two classes (same score vector): the class label completes the key
                dist = dist + 1e3 * (o_head.query_labels[b][:, None] != labels[b][None, :]).double()
                perm = dist.argmin(1)
                ok = dist.min(1).values <= 1e-5                      # a near tie AT the cut swaps one proposal for another:
                unmatched += int((~ok).sum())                        # those columns are counted, not compared
                moved += int((perm != torch.arange(P_))[ok].sum())
                lab_ok = lab_ok and bool(torch.equal(labels[b][perm][ok], o_head.query_labels[b][ok]))
                for k, r in ref_out.items():
                    if k == 'dense_heatmap':
                        errs[k] = max(errs[k], float((got[k][b] - r[b]).abs().max() / r[b].abs().max().clamp_min(1e-12)))
                        continue
                    L_ = r.shape[-1] // P_
                    cols = torch.cat([perm + c * P_ for c in range(L_)])
                    keep = ok.repeat(L_)
                    d_ = (got[k][b][..., cols] - r[b])[..., keep]
                    errs[k] = max(errs[k], float(d_.abs().max() / r[b].abs().max().clamp_min(1e-12)))
            cpu = dict(value=args.batch / dt, unit='frames/s', cores=cores, kind='port',
                       sample='1 full frame of the same workload (oracle = reference PyTorch math, fp32)',
                       max_rel_err_vs_gpu=max(errs.values()), labels_equal=lab_ok,
                       proposals_reordered=moved, proposals_unmatched=unmatched,
                       note='proposal ORDER / the membership at the top-k cut depend on fp32 rounding of heat-map scores that '
                            'agree to ~1e-6 between the two implementations; proposals are matched by their score vectors, '
                            'unmatched ones (near tie at the cut) are counted and excluded from max_rel_err')
        except TimeoutError:
            cpu = dict(value=None, unit='frames/s', cores=cores, kind='port',
                       sample='1 full frame did not finish within 150 s on this host')

    line = dict(metric=METRIC, value=value, unit='frames/s', n_gpus=world, steps=K, warmup=W, ms_per_step=ms / K,
                higher_is_better=True, scaling='weak', vs_baseline=None, dtype='fp32', data='synthetic',
                config=dict(workload=WORKLOAD, global_batch=args.batch * world, cloud=args.cloud,
                            parallelism=f'dp{world} (independent frames, no data-path collective)',
                            frames_in_flight=pipe.depth,
                            arithmetic='fp32 in/out and accumulate; dense products as error-compensated splits on wgmma '
                                       '(bf16 hi+mid x3 in the encoder, 3xTF32 in the decoder), mma.sync bf16 hi+mid x3 in the '
                                       'window attention; measured vs the fp32 oracle: see cpu_baseline.max_rel_err_vs_gpu',
                            l2='inputs (204 MB/frame, %d distinct frames in their own buffers) larger than L2; no flush' % NF,
                            frames=dict(distinct=NF, pillars=n_pillars, points=n_points,
                                        note='frames differ in seed, point and pillar counts; CUDA graphs are keyed on '
                                             'bucketed capacities, live counts are read from device memory')),
                clocks=clocks,
                e2e=dict(value=e2e_value, unit='frames/s', h2d_bytes_per_step=int(np.mean([h2d_bytes(f) for f in frames_host])),
                         bound='PCIe host->device copies (%.0f MB/frame of fp32 feature maps)' % (h2d_bytes(fr_host) / 1e6),
                         d2h_bytes_per_step=int(sum(v.numel() * v.element_size() for v in out.values())),
                         ms_per_step=ms_e2e / K, host_launch_ms_per_step=host_fwd / K * 1e3,
                         overlap='H2D of step i+1 on a copy stream (depth+1 device input sets) while earlier steps compute'),
                gpu_launches=launches, launches_per_step=launches / K, stages=stages, cuda_graph=bool(di_graph.ENABLED[0] and os.environ.get('DI_B200_GRAPH', '1') != '0'),
                roofline=roof, modules=modules, cpu_baseline=cpu,
                kernels=kernels[:12])
    print(json.dumps(line), flush=True)
    if last_out is not None and rank == 0:
        dump_outputs(args.dump_outputs, last_out)
    if world > 1:
        dist.destroy_process_group()


if __name__ == '__main__':
    main()
