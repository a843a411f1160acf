"""Training step of the fused per-pixel path over a batch of N views of one scene, with the per-sample record kept from
forward to backward (record mode, render_rays_train's default) against the record rebuilt one view at a time in the
backward (recompute=True, what the generator hook runs with SDB200_TRAIN_RECOMPUTE=1), in the same process, alternating.
Both arms take the batch in one pass.  Prints one JSON line.

    python bench_train_recompute.py [--steps 5] [--warmup 2] [--views 1,2,4,8]

Workload: 262 x 262 views (training crop 256 + pad 6) at 24 samples per ray, stratified sampling, distinct cameras and
style codes -- the batch of the C5 training workload is 8 such views.  A step is forward + backward of sum(net_out * G).
Times are CUDA-event medians with L2 flushed between steps; each arm's peak allocated memory is reported.  Record mode
holds about 6.9 GB of render record per view; a batch it cannot allocate is reported as not fitting rather than
shrunk.  Recompute mode holds one view's record whatever the batch, and pays one more recording forward per view."""
import argparse
import gc
import json
import statistics
import subprocess

import torch

import oracle
from scenedreamer_b200 import _lib, ops, render, synth

H = W = 262
S = 24


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=5)
    ap.add_argument('--warmup', type=int, default=2)
    ap.add_argument('--views', default='1,2,4,8')
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_train_recompute.py needs a CUDA GPU')
    dev = 'cuda:0'
    res = {'gpu': torch.cuda.get_device_name(0), 'size': '%dx%d' % (H, W), 'samples': S,
           'record_gb_per_view': round(_lib.lib().sdb_render_train_record_bytes(1, H, W, S) / 1e9, 2)}
    try:
        res['power_limit_w'] = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader,nounits', '-i', '0'],
                                              capture_output=True, text=True).stdout.strip()
    except OSError:
        res['power_limit_w'] = None
    flush = torch.empty(64 << 20, dtype=torch.float32, device=dev)          # 256 MB > L2
    world = synth.SyntheticVoxelWorld(size=512, seed=7)
    poses = synth.eval_camera_poses(world, maxstep=16, pattern=0)
    P = {k: v.to(dev).requires_grad_(True) for k, v in oracle.make_params(seed=1, stress=True).items()}
    lut = render.reduced_label_lut(_lut(), 0, 3)
    _, pls = oracle.grid_offsets()
    nmax = max(int(n) for n in a.views.split(','))
    cams = []
    for k in range(nmax):
        o, d, u, f, c, r = synth.frame_camera(world, poses[1 + k % (len(poses) - 1)], resolution_hw=(H - 6, W - 6), pad=6)
        vid, dep, rd = ops.ray_voxel_intersection_perspective(world.voxel_t.to(dev), o, d, u, f, c, r, 6)
        cams.append((vid, dep, rd, o))
    g = torch.Generator().manual_seed(3)
    z_all = oracle.style_mlp(torch.randn(nmax, 128, generator=g), {k: v.detach().cpu() for k, v in P.items()}).to(dev)
    genc = torch.tanh(torch.randn(1, 2, generator=g)).to(dev)
    vdims = list(world.voxel_t.shape)

    for n in (int(v) for v in a.views.split(',')):
        vid = torch.stack([c[0] for c in cams[:n]])
        dep = torch.stack([c[1] for c in cams[:n]])
        rd = torch.stack([c[2] for c in cams[:n]])
        ori = torch.stack([c[3] for c in cams[:n]]).to(dev)
        z = z_all[:n].clone().requires_grad_(True)
        uni = torch.rand(n, H, W, S + 1, 1, device=dev)
        G = torch.randn(n, H, W, 64, device=dev)

        def step(recompute):
            out = render.render_rays_train(P, vid, dep, rd, ori, z, genc, vdims, lut, pls, num_samples=S, uniforms=uni,
                                           recompute=recompute)
            (out['net_out'] * G).sum().backward()

        r = {}
        for rnd in range(2):                                               # alternate the arms
            for name, recompute in (('record', False), ('recompute', True)):
                if r.get(name + '_step_ms') == 'does not fit':
                    continue
                render.clear_scratch()
                for q in list(P.values()) + [z]:
                    q.grad = None
                gc.collect()                                               # graphs of the other arm: freed before, not during
                torch.cuda.empty_cache()
                torch.cuda.reset_peak_memory_stats()
                try:
                    for _ in range(a.warmup):
                        step(recompute)
                    ts = []
                    for _ in range(a.steps):
                        flush.zero_()
                        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                        e0.record()
                        step(recompute)
                        e1.record()
                        torch.cuda.synchronize()
                        ts.append(e0.elapsed_time(e1))
                    r.setdefault(name + '_step_ms', []).append(statistics.median(ts))
                    r[name + '_peak_gb'] = round(torch.cuda.max_memory_allocated() / 1e9, 2)
                except torch.OutOfMemoryError:
                    r[name + '_step_ms'] = 'does not fit'
                    r[name + '_peak_gb'] = 'does not fit'
                    render.clear_scratch()
                    torch.cuda.empty_cache()
        out = {k: (v if isinstance(v, str) else (round(min(v), 2) if isinstance(v, list) else v)) for k, v in r.items()}
        out['live_rays'] = int((vid[..., 0, 0] != 0).sum())
        res['views_%d' % n] = out
    print(json.dumps(res))


def _lut():
    import os
    import numpy as np
    return np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), 'tests', 'golden', 'ref_python_ops.npz'))['mc2reduced_lut']


if __name__ == '__main__':
    main()
