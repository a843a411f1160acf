#!/usr/bin/env python
"""Mixed-precision training step of the per-pixel path: what a user who turns AMP on gets.

    python bench_amp.py [--steps 7] [--warmup 3]

Workload: BASELINE config C5's per-pixel stage, one 262x262 view (256 + 6 px pad) at 24 samples per ray, stratified
sampling, forward + backward of sum(net_out * G), the harness of bench_train.py.  Three arms, alternating step by step in
one process, CUDA-event medians with L2 flushed between steps:
  (a) fused, under torch.autocast(fp16): the recording forward in one fp16 pass (precision 0), bf16 x3 backward;
  (b) fused, autocast off: the fp16 x3 recording forward (the default training step);
  (c) the unfused composition (torch ops + the reference's GridEncoder) under torch.autocast(fp16): what an AMP step cost
      before the fused path took autocast calls (needs the reference's Python staged by oracle/build_ref.py).
Also the recording-forward kernel alone (sdb_render_rays_train_forward) at precision 0 and 2 on the same rays.
Prints one JSON line with the GPU name and power limit."""
import argparse
import ctypes
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'dropin'))      # `_gridencoder` for the reference's own gridencoder package (arm c)

import bench_train  # noqa: E402

VIEW, PAD, SPP = bench_train.VIEW, bench_train.PAD, bench_train.SPP


def _power_limit():
    try:
        return subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader,nounits', '-i', '0'],
                              capture_output=True, text=True).stdout.strip()
    except OSError:
        return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=7)
    ap.add_argument('--warmup', type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_amp.py: no CUDA device (no CPU fallback)')
    import oracle
    from scenedreamer_b200 import _lib, ops, render, synth
    dev = torch.device('cuda', 0)
    world = synth.SyntheticVoxelWorld(bench_train.SCENE, 3407)
    pose = synth.eval_camera_poses(world, maxstep=40, pattern=0)[5]
    P0 = oracle.make_params(seed=0, stress=True)
    g = torch.Generator().manual_seed(8888)
    z0 = oracle.style_mlp(torch.randn(1, 128, generator=g), P0)
    genc0 = torch.tanh(torch.randn(1, 2, generator=g))
    lut = render.reduced_label_lut(np.load(os.path.join(ROOT, 'tests', 'golden', 'ref_python_ops.npz'))['mc2reduced_lut']).to(dev)
    _, pls = oracle.grid_offsets()
    P = {k: v.to(dev).requires_grad_(True) for k, v in P0.items()}
    z, genc = z0.to(dev).requires_grad_(True), genc0.to(dev).requires_grad_(True)
    vdims = [float(v) for v in world.voxel_t.shape]
    o, d, u, f, c, res = synth.frame_camera(world, pose, (VIEW, VIEW), PAD)
    vid, dep, rd = ops.ray_voxel_intersection_perspective(world.voxel_t.to(dev), o, d, u, f, c, res, 6)
    vid, dep, rd, ori = vid.unsqueeze(0), dep.unsqueeze(0), rd.unsqueeze(0), o.unsqueeze(0).to(dev)
    H = W = VIEW + PAD
    torch.manual_seed(0)
    uni = torch.rand(1, H, W, SPP + 1, 1, device=dev)
    G = torch.randn(1, H, W, 64, device=dev)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)

    def zero_grads():
        for t in list(P.values()) + [z, genc]:
            t.grad = None

    def fused(prec, amp):
        def step():
            with torch.autocast('cuda', torch.float16, enabled=amp):
                out = render.render_rays_train(P, vid, dep, rd, ori, z, genc, vdims, lut, pls, num_samples=SPP, uniforms=uni,
                                               precision=prec)
                loss = (out['net_out'] * G).sum()
            loss.backward()
        return step
    arms = {'a_fused_fp16_amp': fused(render.PRECISION_FP16, True), 'b_fused_fp16x3': fused(render.PRECISION_FP16X3, False)}
    from oracle import refgen
    ref_py = refgen.reference_python_root()
    if ref_py is not None:
        sys.path.insert(1, ref_py)
        from gridencoder import GridEncoder
        ge = GridEncoder(input_dim=5, num_levels=16, level_dim=8, base_resolution=16, log2_hashmap_size=19,
                         desired_resolution=2048).to(dev)
        ge.embeddings = torch.nn.Parameter(P['hash_encoder.embeddings'].detach().clone())

        def comp_step():
            with torch.autocast('cuda', torch.float16):
                bench_train.composition_step(P, ge, vid, dep, rd, ori, z, genc, vdims, lut, uni, G)
            ge.embeddings.grad = None
        arms['c_composition_amp'] = comp_step

    times = {k: [] for k in arms}
    for it in range(a.warmup + a.steps):
        for name, fn in arms.items():
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            fn()
            e1.record()
            zero_grads()
            flush.zero_()
            torch.cuda.synchronize()
            if it >= a.warmup:
                times[name].append(e0.elapsed_time(e1))
    render.clear_scratch()

    # the recording forward kernel alone (plus its tiny pre-pass), same rays, both precisions over one record buffer
    Lb = _lib.lib()
    st = render._stream(dev)
    kern = {}
    with torch.no_grad():
        wh, bh = render.modulated_weights(P, z[0])
        W1 = P['render_net.fc_1.weight'].detach().contiguous()
        ins = dict(b1=P['render_net.fc_1.bias'], emb=P['render_net.fc_m_a.weight'].t(), wsig=P['render_net.fc_sigma.weight'].reshape(-1),
                   bsig=P['render_net.fc_sigma.bias'].reshape(-1), wout=P['render_net.fc_out_c.weight'], bout=P['render_net.fc_out_c.bias'])
        ins = {k: v.detach().contiguous() for k, v in ins.items()}
        table3 = render.preblend_table(P['hash_encoder.embeddings'].detach(), genc.detach(), 19, pls, 16, 16)
        sky = torch.zeros(1, H, W, 64, device=dev)
        sky_avg = torch.zeros(1, 64, device=dev)
        outs = [torch.empty(1, H, W, 64, device=dev), torch.empty(1, H, W, device=dev), torch.empty(1, H, W, device=dev),
                torch.empty(1, H, W, SPP, 1, device=dev), torch.empty(1, H, W, SPP, 1, device=dev)]
        ws = torch.empty(int(Lb.sdb_render_workspace_bytes(1, H, W)), dtype=torch.uint8, device=dev)
        record = torch.empty(int(Lb.sdb_render_train_record_bytes(1, H, W, SPP)), dtype=torch.uint8, device=dev)
        p = render._ptr
        prms = {}
        for prec in (render.PRECISION_FP16, render.PRECISION_FP16X3):
            pack = torch.empty(1, int(Lb.sdb_mlp_pack_bytes(prec)), dtype=torch.uint8, device=dev)
            _lib.check(Lb.sdb_pack_mlp(p(W1), p(ins['b1']), p(ins['emb']), int(ins['emb'].shape[0]), p(wh), p(bh), p(ins['wsig']),
                                       p(ins['bsig']), p(ins['wout']), p(ins['bout']), prec, p(pack), st), 'sdb_pack_mlp')
            prm, keep = render._RenderParams(), [pack]
            render._fill_render_params(prm, keep, vid, dep, rd, ori, genc.detach().reshape(1, 2).contiguous(), vdims, lut, pack, sky,
                                       sky_avg, table3=table3, S=SPP, sample_depth=3.0, dists_scale=0.25, uniforms=uni,
                                       precision=prec, per_level_scale=pls, base_res=16, log2_T=19, L=16, net_out=outs[0],
                                       depth=outs[1], tw=outs[2], wts=outs[3], rdp=outs[4], ws=ws)
            prms[prec] = (prm, keep)
            kern[prec] = []
        for it in range(a.warmup + 2 * a.steps):
            for prec, (prm, _) in prms.items():
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                _lib.check(Lb.sdb_render_rays_train_forward(ctypes.byref(prm), p(record), st), 'sdb_render_rays_train_forward')
                e1.record()
                flush.zero_()
                torch.cuda.synchronize()
                if it >= a.warmup:
                    kern[prec].append(e0.elapsed_time(e1))

    med = {k: float(np.median(v)) for k, v in times.items()}
    line = {'metric': 'AMP train step of the per-pixel path: forward(record)+backward, 262x262 rays x 24 spp, stratified',
            'unit': 'ms', 'gpu': torch.cuda.get_device_name(0), 'power_limit_w': _power_limit(),
            'step_ms_median': med, 'step_ms_all': {k: [round(t, 2) for t in v] for k, v in times.items()},
            'train_forward_kernel_ms_median': {'precision0_fp16': float(np.median(kern[0])), 'precision2_fp16x3': float(np.median(kern[2]))},
            'train_forward_kernel_ms_all': {str(k): [round(t, 2) for t in v] for k, v in kern.items()},
            'aggregate': 'median, arms alternating step by step, CUDA events, L2 flushed between steps', 'steps': a.steps}
    if 'c_composition_amp' not in med:
        line['c_composition_amp'] = 'skipped: reference Python not staged (oracle/build_ref.py)'
    print(json.dumps(line))


if __name__ == '__main__':
    main()
