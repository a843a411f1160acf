#!/usr/bin/env python
"""Per-iteration scene switch of training with the PCG cache (`pcg_cache: True`): PCGCache.sample_world through the hook
(read-ahead on a worker thread, pinned upload on a copy stream, sdb_scene_scatter into the truncated volume) against the
reference's body (the same hooked class with SDB200_SCENECACHE=0), in one process, arms alternating block by block.

    python bench_scene_cache.py [--worlds 3] [--steps 8] [--warmup 2] [--rounds 2]

One iteration = sample_world -> a 262x262 raycast of the new volume -> the C5 recording forward + backward of the per-pixel
path as bench_train.py builds it (the GPU work the next load overlaps).  A synthetic cache of 1024^2 worlds in the layout
scripts/pcg_cache.py writes goes to a temporary directory; the files are read once before timing, so the page cache is warm
(disk speed is not what this measures).  Prints ONE JSON line: per arm the median and min..max iteration time (CUDA events),
the host time per iteration (a host clock around each arm's block, ending in a synchronise), the host time inside
sample_world, peak allocated memory and prefetch hits; with the GPU name and power limit.
"""
import argparse
import json
import os
import random
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

VIEW, PAD, SPP = 256, 6, 24


def gpu_info():
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [s.strip() for s in out.split(',')]
        return name, power
    except Exception:
        return torch.cuda.get_device_name(0), 'unknown'


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--worlds', type=int, default=3)
    ap.add_argument('--steps', type=int, default=8, help='timed iterations per arm and round')
    ap.add_argument('--warmup', type=int, default=2)
    ap.add_argument('--rounds', type=int, default=2)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_scene_cache.py: no CUDA device (no CPU fallback)')
    staged = os.path.join(ROOT, 'oracle', '_ref', 'py')
    if not os.path.isdir(os.path.join(staged, 'imaginaire')):
        raise SystemExit('bench_scene_cache.py: PCGCache is taken from the reference Python staged by oracle/build_ref.py '
                         '(oracle/_ref/py), which is missing')
    import oracle                                      # synthetic weights only
    from oracle import refgen
    from scenedreamer_b200 import ops, render, synth, worldgen
    refgen.setup('dropin')
    import imaginaire.model_utils.pcg_gen as pcg
    worldgen.install(pcg.PCGCache)
    dev = torch.device('cuda', 0)

    tmp = tempfile.mkdtemp(prefix='sdb_scene_cache_')
    for k in range(a.worlds):
        synth.write_cache_world(os.path.join(tmp, 'w%d' % k), seed=11 + k)
    nnz = [int(np.load(os.path.join(tmp, 'w%d' % k, 'voxel_sparse.npy'), mmap_mode='r').shape[1]) for k in range(a.worlds)]
    cache_bytes = sum(os.path.getsize(os.path.join(tmp, d, f)) for d in os.listdir(tmp) for f in os.listdir(os.path.join(tmp, d)))

    P0 = oracle.make_params(seed=0, stress=True)
    g = torch.Generator().manual_seed(8888)
    z0 = oracle.style_mlp(torch.randn(1, 128, generator=g), P0)
    genc0 = torch.tanh(torch.randn(1, 2, generator=g))
    lut = render.reduced_label_lut(np.load(os.path.join(ROOT, 'tests', 'golden', 'ref_python_ops.npz'))['mc2reduced_lut']).to(dev)
    _, pls = oracle.grid_offsets()
    P = {k: v.to(dev).requires_grad_(True) for k, v in P0.items()}
    z, genc = z0.to(dev).requires_grad_(True), genc0.to(dev).requires_grad_(True)
    H = W = VIEW + PAD
    uni = torch.rand(1, H, W, SPP + 1, 1, device=dev)
    G = torch.randn(1, H, W, 64, device=dev)
    cam_d = torch.tensor([-0.45, 1.0, 0.8])
    cam_d = cam_d / cam_d.norm()
    cam_up = torch.tensor([1.0, 0.0, 0.0])

    arms = {'fused': pcg.PCGCache(tmp), 'reference': pcg.PCGCache(tmp)}
    rngs = {}
    for name in arms:
        random.seed(1234)                              # the same sequence of worlds in both arms
        rngs[name] = random.getstate()
    res = {name: {'iter_ms': [], 'load_host_ms': [], 'host_ms_per_iter': [], 'peak_gb': 0.0, 'live': []} for name in arms}

    def iteration(cache, rec, ev):
        ev[0].record()
        t0 = time.perf_counter()
        cache.sample_world(dev)
        t1 = time.perf_counter()
        vox = cache.voxel_t
        ori = torch.tensor([float(vox.shape[0]) + 8.0, 200.0, 230.0])
        vid, dep, rd = ops.ray_voxel_intersection_perspective(vox, ori, cam_d, cam_up, 220.0, [(H - 1) / 2, (W - 1) / 2], [H, W], 6)
        out = render.render_rays_train(P, vid.unsqueeze(0), dep.unsqueeze(0), rd.unsqueeze(0), ori.unsqueeze(0).to(dev), z, genc,
                                       [float(v) for v in vox.shape], lut, pls, num_samples=SPP, uniforms=uni)
        (out['net_out'] * G).sum().backward()
        ev[1].record()
        for t in list(P.values()) + [z, genc]:
            t.grad = None
        if rec is not None:
            rec['load_host_ms'].append(1e3 * (t1 - t0))
            rec['live'].append(vid[..., 0, 0] != 0)

    def block(name, steps, rec):
        os.environ['SDB200_SCENECACHE'] = '1' if name == 'fused' else '0'
        random.setstate(rngs[name])
        evs = [[torch.cuda.Event(enable_timing=True) for _ in range(2)] for _ in range(steps)]
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats(dev)
        t0 = time.perf_counter()
        for k in range(steps):
            iteration(arms[name], rec, evs[k])
        torch.cuda.synchronize()
        wall = time.perf_counter() - t0
        rngs[name] = random.getstate()
        if rec is not None:
            rec['iter_ms'] += [e[0].elapsed_time(e[1]) for e in evs]
            rec['host_ms_per_iter'].append(1e3 * wall / steps)
            rec['peak_gb'] = max(rec['peak_gb'], torch.cuda.max_memory_allocated(dev) / 1e9)

    order = ['fused', 'reference']
    for name in order:
        block(name, a.warmup + a.worlds, None)         # warms the page cache (every world read) and every shape
    base = dict(worldgen.stats)
    for r in range(a.rounds):
        for name in (order if r % 2 == 0 else order[::-1]):
            block(name, a.steps, res[name])
    st = {k: worldgen.stats[k] - base[k] for k in base}

    gpu, power = gpu_info()
    line = {'metric': 'training iteration with a PCG-cache scene switch: sample_world + 262x262 raycast + C5 recording '
                      'forward/backward', 'unit': 'ms', 'gpu': gpu, 'power_limit': power,
            'worlds': a.worlds, 'world': '1024x1024x256', 'nnz_per_world': nnz, 'cache_bytes': cache_bytes,
            'page_cache': 'warm (every world read before timing)', 'steps_per_arm': a.steps * a.rounds,
            'rounds': a.rounds, 'order': 'arms alternate block by block'}
    for name in order:
        rec = res[name]
        it = rec['iter_ms']
        line[name] = {'iter_ms_median': round(float(np.median(it)), 2), 'iter_ms_min': round(min(it), 2),
                      'iter_ms_max': round(max(it), 2), 'host_ms_per_iter': [round(v, 2) for v in rec['host_ms_per_iter']],
                      'sample_world_host_ms_median': round(float(np.median(rec['load_host_ms'])), 2),
                      'sample_world_host_ms_max': round(max(rec['load_host_ms']), 2),
                      'peak_allocated_gb': round(rec['peak_gb'], 2),
                      'live_ray_fraction': round(float(torch.stack(rec['live']).float().mean()), 3)}
    line['fused']['prefetch_hits'] = st['prefetch_hits']
    line['fused']['prefetch_misses'] = st['prefetch_misses']
    line['reference']['reference_loads'] = st['reference_loads']
    line['speedup_median'] = round(line['reference']['iter_ms_median'] / line['fused']['iter_ms_median'], 3)
    for s in worldgen._states.values():
        worldgen._shutdown(s)
    import shutil
    shutil.rmtree(tmp, ignore_errors=True)
    print(json.dumps(line))


if __name__ == '__main__':
    main()
