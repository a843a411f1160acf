#!/usr/bin/env python
"""Timings of the ops either side of the fused per-pixel kernel, each next to the
reference's own implementation of the same op on the same GPU / host.  Not the headline metric (bench.py is); this is the
measurement for rows a1, a6/a7 (stand-alone), f1, f2, f3, f4 and the `voxlib` surface.

    python tests/ops_timing.py     # one JSON line, needs a CUDA device; reference legs need oracle/_ref (oracle/build_ref.py)

Lives under tests/ because it uses oracle/ (parameter builders, the reference's prebuilt extensions and staged Python) as the
comparison arm; the product package never does.

Every number: median of several runs, CUDA events (device work) or wall clock around a synchronised call (host-inclusive work:
scene build, camera sampler), inputs resident.
"""
import json
import os
import random
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
DEV = 'cuda:0'


def dev_ms(fn, reps=7, warm=2):
    for _ in range(warm):
        fn()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    return float(np.median(ts))


def wall_ms(fn, reps=3, warm=1):
    for _ in range(warm):
        fn()
    ts = []
    for _ in range(reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ts.append(1e3 * (time.perf_counter() - t0))
    return float(np.median(ts))


def main():
    if not torch.cuda.is_available():
        raise SystemExit('ops_timing.py: no CUDA device')
    import oracle
    from oracle import refgen
    from scenedreamer_b200 import ops, optim, rendercnn, synth
    sys.path.insert(0, os.path.join(ROOT, 'tests'))
    from _ref_ext import load as load_ref
    rv, rg = load_ref('ref_voxlib'), load_ref('ref_gridencoder')
    out = {'metric': 'boundary / next-row ops: ours vs the reference implementation on the same box', 'unit': 'ms'}
    g = torch.Generator().manual_seed(0)

    # ---- a1: raycast of the C2 frame ----
    world = synth.SyntheticVoxelWorld(1024, 3407)
    vox = world.voxel_t.to(DEV)
    o, d, u, f, c, res = synth.frame_camera(world, synth.eval_camera_poses(world, maxstep=40, pattern=0)[3], (540, 960), 30)
    r = {'ours': dev_ms(lambda: ops.ray_voxel_intersection_perspective(vox, o, d, u, f, c, res, 6))}
    if rv is not None:
        r['reference_cuda'] = dev_ms(lambda: rv.ray_voxel_intersection_perspective(vox, o, d, u, float(f), [float(c[0]), float(c[1])],
                                                                                   [int(res[0]), int(res[1])], 6))
    out['a1_raycast_570x990'] = r

    # ---- a6 / a7: stand-alone hash-grid encode, one reference tile (158 x 158 x 24 samples) ----
    B, L, C, D = 158 * 158 * 24, 16, 8, 5
    offsets, pls = oracle.grid_offsets()
    emb = ((torch.rand(int(offsets[-1]), C, generator=g) * 2 - 1) * 0.1).to(DEV)
    x = torch.rand(B, D, generator=g).to(DEV)
    offs = offsets.to(DEV)
    outp = torch.empty(L, B, C, device=DEV)
    dydx = torch.empty(B, L * D * C, device=DEV)
    S = float(np.log2(pls))
    grad = torch.randn(L, B, C, generator=g).to(DEV)
    ge, gi = torch.zeros_like(emb), torch.zeros_like(x)
    r = {'ours_fwd': dev_ms(lambda: ops.grid_encode_forward(x, emb, offs, outp, B, D, C, L, S, 16, True, dydx, 0, False)),
         'ours_bwd': dev_ms(lambda: ops.grid_encode_backward(grad, x, emb, offs, ge, B, D, C, L, S, 16, True, dydx, gi, 0, False))}
    if rg is not None:
        r['reference_cuda_fwd'] = dev_ms(lambda: rg.grid_encode_forward(x, emb, offs, outp, B, D, C, L, S, 16, True, dydx, 0, False))
        r['reference_cuda_bwd'] = dev_ms(lambda: rg.grid_encode_backward(grad, x, emb, offs, ge, B, D, C, L, S, 16, True, dydx, gi, 0, False))
    out['a6_a7_grid_encode_tile_599k_samples'] = r
    del outp, dydx, grad, ge, gi, x

    # ---- f1: RenderCNN + tanh on the padded C2 frame ----
    P = {k: v.to(DEV) for k, v in oracle.make_cnn_params(1).items()}
    net = (torch.rand(1, 570, 990, 64, generator=g) * 2 - 1).to(DEV)
    z = torch.randn(1, 256, generator=g).to(DEV)
    e3, e1 = rendercnn.RenderCNNEngine(P, rendercnn.PRECISION_FP16X3), rendercnn.RenderCNNEngine(P, rendercnn.PRECISION_FP16)
    r = {'ours_fp16x3': dev_ms(lambda: e3.forward(net, z, want_raw=False)), 'ours_fp16x1': dev_ms(lambda: e1.forward(net, z, want_raw=False))}
    with torch.no_grad():
        for tf32 in (True, False):
            torch.backends.cudnn.allow_tf32 = tf32
            r['torch_cudnn_%s_whole_frame' % ('tf32' if tf32 else 'fp32')] = dev_ms(lambda: oracle.render_cnn(net, z, P), reps=3, warm=1)
        torch.backends.cudnn.allow_tf32 = True
    out['f1_rendercnn_570x990'] = r
    del e3, e1, net

    # ---- f2: Adam step of the hash table ----
    p = torch.nn.Parameter(emb.clone())
    opt = torch.optim.Adam([p], lr=1e-4, eps=1e-7, betas=(0.0, 0.999))
    gsp = torch.zeros_like(emb)
    idx = torch.randint(0, emb.shape[0], (emb.shape[0] // 25,), generator=g).to(DEV)
    gsp[idx] = torch.randn(idx.numel(), C, generator=g).to(DEV)

    def torch_step():
        p.grad = gsp
        opt.step()
    m, v, pp = torch.zeros_like(emb), torch.zeros_like(emb), emb.clone()
    step = [0]

    def ours_step():
        step[0] += 1
        optim.adam_step_(pp, gsp, m, v, step[0], 1e-4, 0.0, 0.999, 1e-7)
    out['f2_adam_step_67M_entries_4pct_touched'] = {'ours': dev_ms(ours_step), 'torch_optim_adam': dev_ms(torch_step)}
    del p, opt, gsp, m, v, pp, emb

    # ---- f3 / f4 need the reference's Python ----
    if refgen.reference_python_root() is not None:
        refgen.setup('dropin')
        import cv2
        import imaginaire.model_utils.pcg_gen as pcg
        from scenedreamer_b200 import integration
        gen, _ = refgen.build_generator(1024, DEV)
        integration.ensure_installed()
        size = 1024
        h, sem, tree = synth.make_bev(size, seed=5)
        dd = tempfile.mkdtemp()
        np.save(os.path.join(dd, 'heightmap.npy'), h)
        cv2.imwrite(os.path.join(dd, 'semanticmap.png'), sem)
        cv2.imwrite(os.path.join(dd, 'treemap.png'), tree)
        assets = {'assets': [torch.from_numpy(mm) for mm in synth.make_tree_models()]}

        def ref_world():
            random.seed(1)
            vg = pcg.PCGVoxelGenerator(size)
            pcg.PCGVoxelGenerator._sdb200_reference_next_world(vg, torch.device(DEV), dd, assets)     # CPU build + upload, as shipped

        def our_world():
            random.seed(1)
            pcg.PCGVoxelGenerator(size).next_world(torch.device(DEV), dd, assets)
        stdout = sys.stdout
        sys.stdout = open(os.devnull, 'w')
        try:
            out['f3_next_world_1024'] = {'ours': wall_ms(our_world, reps=3, warm=1), 'reference_cpu_plus_upload': wall_ms(ref_world, reps=1, warm=0)}
            refgen.set_world(gen, world, DEV)
            gen.cam_res, gen.crop_size, gen.pad = [360, 640], [256, 256], 6
            gen.voxel.sample_world = lambda device: None
            cls = type(gen)

            def sampler(fn):
                def run():
                    torch.manual_seed(7)
                    np.random.seed(7)
                    fn(gen, 8, torch.device(DEV))
                return run
            out['f4_get_batch_8_views'] = {'ours': wall_ms(sampler(cls._get_batch), reps=3, warm=1),
                                           'reference': wall_ms(sampler(cls._sdb200_reference_get_batch), reps=3, warm=1)}
        finally:
            sys.stdout.close()
            sys.stdout = stdout

    # ---- a9 boundary op: positional encoding of the C2 frame's ray directions (pe degree 5 + original, the sky branch's input) ----
    rdirs = torch.nn.functional.normalize(torch.randn(1, 570, 990, 1, 3, generator=g), dim=-1).to(DEV)
    r = {'ours': dev_ms(lambda: ops.positional_encoding(rdirs, 5, -1, True))}
    if rv is not None:
        r['reference_cuda'] = dev_ms(lambda: rv.positional_encoding(rdirs, 5, -1, True))
    out['a9_positional_encoding_564k_rays'] = r

    # ---- voxlib surface: sp_trilinear ----
    lut = torch.randint(0, 200000, (64, 256, 256), generator=g, dtype=torch.int32).to(DEV)
    feat = torch.randn(200000, 64, generator=g).to(DEV)
    wc = (torch.rand(1, 256, 256, 24, 3, generator=g) * torch.tensor([62.0, 254.0, 254.0])).to(DEV)
    r = {'ours': dev_ms(lambda: ops.sp_trilinear_worldcoord(feat, lut, wc, True, -1))}
    if rv is not None:
        r['reference_cuda'] = dev_ms(lambda: rv.sp_trilinear_worldcoord(feat, lut, wc, True, -1))
    out['voxlib_sp_trilinear_1.57M_points_64ch'] = r
    print(json.dumps(out))


if __name__ == '__main__':
    main()
