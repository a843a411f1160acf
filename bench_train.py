#!/usr/bin/env python
"""Train-step benchmark of the per-pixel path (BASELINE.json config 5, per-GPU share): one 256x256 view
(+6 px pad -> 262x262 rays), 24 samples/ray, scene_size 1024, stratified sampling; renderer forward WITH
the training record + full backward (all parameter gradients of hash table, scene code, LightningMLP,
style code, sky net).  Not the headline metric (bench.py is); this is the measurement for row a7 /
config C5 (BASELINE.md).

    python bench_train.py [--steps K] [--warmup W] [--no-composition]

Prints ONE JSON line: fused forward+backward ms per view and Msamples/s, and next to it the same step
through the UNFUSED composition on the same GPU (torch autograd MLP / compositing in fp32 via cuBLAS +
this library's stand-alone hash-grid forward/backward kernels = the structure of the reference's
train step), inputs resident, CUDA events, L2 flushed between steps.
"""
import argparse
import json
import os
import sys

import numpy as np
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'dropin'))      # `_gridencoder` for the reference's own gridencoder package (composition leg)

VIEW, PAD, SPP, SCENE = 256, 6, 24, 1024


def composition_step(P, ge, vid, dep, rd, ori, z, genc, vdims, lut, uni, G):
    """Unfused train step on the GPU (reference structure): torch ops + GridEncoder autograd.Function."""
    from scenedreamer_b200 import render
    N, H, W, M = vid.shape[:4]
    S = SPP
    with torch.no_grad():
        d2 = dep[:, 1] - dep[:, 0]
        d2[torch.isnan(d2)] = 0
        accu = torch.cumsum(d2, -2)
        total = accu[..., [-1], :].clamp(max=3.0)
        r = uni / (S + 1) + torch.linspace(0, 1, S + 2, device=vid.device)[:-1].view(1, 1, 1, -1, 1)
        r = torch.sort(r * total, dim=-2)[0]
        mid = (r[..., 1:, :] + r[..., :-1, :]) / 2
        nd = r[..., 1:, :] - r[..., :-1, :]
        idx = torch.sum(mid.unsqueeze(-3) > accu.unsqueeze(-2), dim=-3)
        dd = torch.cumsum(dep[:, 0, :, :, 1:, :] - dep[:, 1, :, :, :-1, :], -2)
        heads = torch.cat([dep[:, 0, :, :, [0], :], dd + dep[:, 0, :, :, [0], :]], -2)
        rdp = torch.gather(heads, -2, idx) + mid
        rdp[torch.isnan(rdp) | torch.isinf(rdp)] = 0
        wc = rd * rdp + ori[:, None, None, None, :]
        lab = torch.gather(lut.long()[vid.long()], -2, idx).squeeze(-1)
        nrm = wc / torch.tensor(vdims, device=vid.device) * 2 - 1
        sky_only = vid[:, :, :, [0], :] == 0
        sky_mask = vid[:, :, :, [-1], :] == 0
    x5 = torch.cat([nrm, genc[:, None, None, None, :].expand(-1, H, W, S, -1)], -1)
    feat = ge(x5.reshape(-1, 5))
    p = 'render_net.'
    f = F.linear(feat, P[p + 'fc_1.weight'], P[p + 'fc_1.bias']) + P[p + 'fc_m_a.weight'].t()[lab.reshape(-1)]
    f = F.leaky_relu(f, 0.2)
    wh, bh = render.modulated_weights(P, z[0])
    sig = None
    for k in range(5):
        f = F.leaky_relu(F.linear(f, wh[k], bh[k]), 0.2)
        if k == 2:
            sig = F.linear(f, P[p + 'fc_sigma.weight'], P[p + 'fc_sigma.bias'])
    col = F.linear(f, P[p + 'fc_out_c.weight'], P[p + 'fc_out_c.bias']).reshape(N, H, W, S, 64)
    sig = sig.reshape(N, H, W, S, 1)
    sky = render.sky_features(P, rd, z).unsqueeze(-2)
    e = F.relu(sig) * (nd * 0.25)
    wts = (1 - torch.exp(-e)) * torch.exp(-(torch.cumsum(e, -2) - e)) * (~sky_only).float()
    tw = wts.sum(-2, keepdim=True)
    is_gnd = (wc[..., [0]] <= 1.0).any(-2, keepdim=True)
    nosky = (~sky_mask | is_gnd).float()
    sky_used = sky * (1 - nosky) + sky.mean(dim=[1, 2], keepdim=True) * nosky
    out = (wts * (col.clamp(-1, 1) + 1)).sum(-2, keepdim=True) + (1 - tw) * (sky_used.clamp(-1, 1) + 1)
    out = out.squeeze(-2) - 1
    (out * G).sum().backward()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=10)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--no-composition', action='store_true')
    ap.add_argument('--views', type=int, default=8, help='number of distinct camera poses cycled through')
    ap.add_argument('--profile', action='store_true', help='host/device time of the autograd Functions (diagnostics, stderr)')
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_train.py: no CUDA device (no CPU fallback)')
    import oracle                      # synthetic weights only
    from scenedreamer_b200 import ops, render, synth
    dev = torch.device('cuda', 0)
    world = synth.SyntheticVoxelWorld(SCENE, 3407)
    poses = synth.eval_camera_poses(world, maxstep=40, pattern=0)
    P0 = oracle.make_params(seed=0, stress=True)
    g = torch.Generator().manual_seed(8888)
    z0 = oracle.style_mlp(torch.randn(1, 128, generator=g), P0)
    genc0 = torch.tanh(torch.randn(1, 2, generator=g))
    lut = render.reduced_label_lut(np.load(os.path.join(ROOT, 'tests', 'golden', 'ref_python_ops.npz'))['mc2reduced_lut']).to(dev)
    _, pls = oracle.grid_offsets()
    P = {k: v.to(dev).requires_grad_(True) for k, v in P0.items()}
    z, genc = z0.to(dev).requires_grad_(True), genc0.to(dev).requires_grad_(True)
    voxel = world.voxel_t.to(dev)
    vdims = [float(v) for v in world.voxel_t.shape]
    views = []
    for k in range(a.views):
        o, d, u, f, c, res = synth.frame_camera(world, poses[(5 * k) % 40], (VIEW, VIEW), PAD)
        vid, dep, rd = ops.ray_voxel_intersection_perspective(voxel, o, d, u, f, c, res, 6)
        views.append((vid.unsqueeze(0), dep.unsqueeze(0), rd.unsqueeze(0), o.unsqueeze(0).to(dev)))
    H = W = VIEW + PAD
    uni = torch.rand(1, H, W, SPP + 1, 1, device=dev)
    G = torch.randn(1, H, W, 64, device=dev)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    samples = H * W * SPP

    def zero_grads():
        for t in list(P.values()) + [z, genc]:
            t.grad = None

    def fused_step(k, ev=None):
        vid, dep, rd, ori = views[k % len(views)]
        if ev:
            ev[0].record()
        out = render.render_rays_train(P, vid, dep, rd, ori, z, genc, vdims, lut, pls, num_samples=SPP, uniforms=uni)
        if ev:
            ev[1].record()
        (out['net_out'] * G).sum().backward()
        if ev:
            ev[2].record()

    def timed(fn, steps, warmup):
        for w in range(warmup):
            fn(w)
            zero_grads()
            flush.zero_()
        torch.cuda.synchronize()
        evs = [[torch.cuda.Event(enable_timing=True) for _ in range(3)] for _ in range(steps)]
        for k in range(steps):
            fn(k, evs[k])
            zero_grads()
            flush.zero_()
        torch.cuda.synchronize()
        fwds = [e[0].elapsed_time(e[1]) for e in evs]
        tots = [e[0].elapsed_time(e[2]) for e in evs]
        timed.last_steps = [round(t, 2) for t in tots]              # every step, for the reader: a mean hides a host hiccup
        return float(np.median(fwds)), float(np.median(tots))

    if a.profile:
        import time
        stats = {}

        def wrap(cls, name):
            orig = getattr(cls, name)

            def f(ctx, *args):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                r = orig(ctx, *args)
                e1.record()
                t1 = time.perf_counter()
                torch.cuda.synchronize()
                stats.setdefault(cls.__name__ + '.' + name, []).append((1e3 * (t1 - t0), e0.elapsed_time(e1)))
                return r
            setattr(cls, name, staticmethod(f))
        for cls in (render._FusedRenderTrainFn, render._SkyTrainFn):
            wrap(cls, 'forward')
            wrap(cls, 'backward')
        for k in range(6):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            fused_step(k)
            torch.cuda.synchronize()
            stats.setdefault('whole step (synchronous)', []).append((1e3 * (time.perf_counter() - t0), 0.0))
            zero_grads()
        for k, v in stats.items():
            v = v[2:]
            print('%-40s host %.2f ms   device %.2f ms' % (k, np.mean([x[0] for x in v]), np.mean([x[1] for x in v])), file=sys.stderr)
        return
    fwd_ms, tot_ms = timed(fused_step, a.steps, max(3, a.warmup))
    live = float(np.mean([float((v[0][..., 0, 0] != 0).float().mean()) for v in views]))
    line = {'metric': 'train-step per-pixel path: forward(record)+backward, 262x262 rays x 24 spp, per GPU', 'unit': 'ms',
            'fused': {'forward_ms': fwd_ms, 'backward_ms': tot_ms - fwd_ms, 'total_ms': tot_ms,
                      'msamples_per_s_fwd_bwd': samples / (tot_ms * 1e-3) / 1e6},
            'aggregate': 'median over the timed steps (CUDA events around forward / forward+backward)',
            'total_ms_per_step': timed.last_steps,
            'samples_per_view': samples, 'live_ray_fraction': live, 'steps': a.steps, 'data': 'synthetic',
            'l2': 'flushed between steps', 'record_bytes': int(render._lib.lib().sdb_render_train_record_bytes(1, H, W, SPP)),
            'backward_workspace_bytes': int(render._lib.lib().sdb_render_backward_workspace_bytes(1, H, W, SPP, 16, 19))}
    ref_py = None
    if not a.no_composition:
        from oracle import refgen                     # where the reference's own Python is staged (baseline leg only)
        ref_py = refgen.reference_python_root()
        if ref_py is None:
            line['unfused_composition'] = {'skipped': 'reference Python not staged (oracle/build_ref.py)'}
    if ref_py is not None:
        sys.path.insert(1, ref_py)
        from gridencoder import GridEncoder
        ge = GridEncoder(input_dim=5, num_levels=16, level_dim=8, base_resolution=16, log2_hashmap_size=19,
                         desired_resolution=2048).to(dev)
        ge.embeddings = torch.nn.Parameter(P['hash_encoder.embeddings'].detach().clone())
        Pc = dict(P)

        def comp_step(k, ev=None):
            vid, dep, rd, ori = views[k % len(views)]
            if ev:
                ev[0].record()
            composition_step(Pc, ge, vid, dep, rd, ori, z, genc, vdims, lut, uni, G)
            if ev:
                ev[1].record()
                ev[2].record()
            ge.embeddings.grad = None
        _, comp_ms = timed(comp_step, max(3, a.steps // 2), 2)
        line['unfused_composition'] = {'total_ms': comp_ms, 'what': 'torch fp32 autograd (cuBLAS SGEMM MLP, ATen compositing) + '
                                       'stand-alone sdb grid_encode fwd/bwd kernels, same GPU', 'speedup_fused': comp_ms / tot_ms}
    print(json.dumps(line))


if __name__ == '__main__':
    main()
