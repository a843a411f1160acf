"""The REAL reference `Generator` as checker and GPU baseline -- TEST / BENCH-BASELINE INFRASTRUCTURE ONLY.

Imports the reference's own, unmodified Python (`imaginaire.generators.scenedreamer.Generator`, resolved through
`cfg.gen.type` exactly like imaginaire/utils/trainer.py:94-95) from where `oracle/build_ref.py` staged it
(oracle/_ref/py/, git-ignored; /root/reference when that exists) and runs its `inference_givenstyle`
(imaginaire/generators/scenedreamer.py:479-631) in one of two environments:

  backend='ref'     `voxlib` / `_gridencoder` are the reference's own CUDA extensions compiled unmodified into
                    oracle/_ref/*.so: the reference renderer as it ships (unfused tile loop, cuBLAS fp32, ATen).
  backend='dropin'  `dropin/` first on sys.path -- what a user does (INTEGRATION.md): the same Python, zero edits, on
                    libsdb200; importing dropin/voxlib arms the class-level fused hook.

A process can hold only one of the two (the top-level module names collide), so comparisons run the 'ref' arm in a
subprocess (`python -m oracle.refgen --backend ref ...`) that leaves its frames in an .npz.

Nothing on the product path imports this file.
"""
import argparse
import importlib
import importlib.util
import os
import sys
import time
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
STAGED = os.path.join(HERE, '_ref', 'py')
STUBS = os.path.join(HERE, 'stubs')


def reference_python_root():
    if os.path.isdir(os.path.join(STAGED, 'imaginaire')):
        return STAGED
    ref = os.environ.get('SD_REFERENCE_ROOT', '/root/reference')
    if os.path.isdir(os.path.join(ref, 'imaginaire')):
        return ref
    return None


def _load_ext(name):
    path = os.path.join(HERE, '_ref', name, name + '.so')
    if not os.path.exists(path):
        raise RuntimeError('%s is not built (oracle/build_ref.py)' % path)
    spec = importlib.util.spec_from_file_location(name, path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def setup(backend):
    """Arrange sys.path / sys.modules for one backend.  Call once per process, before importing imaginaire."""
    root = reference_python_root()
    if root is None:
        raise RuntimeError('the reference Python is not staged (oracle/_ref/py) and /root/reference is absent')
    if ROOT not in sys.path:
        sys.path.insert(0, ROOT)
    if backend == 'dropin':
        sys.path.insert(0, os.path.join(ROOT, 'dropin'))
    elif backend == 'ref':
        sys.modules['voxlib'] = _load_ext('ref_voxlib')
        sys.modules['_gridencoder'] = _load_ext('ref_gridencoder')
        for name in ('upfirdn2d_cuda', 'bias_act_cuda'):       # import-time only; dropin/ ships the product's stand-ins
            sys.modules.setdefault(name, types.ModuleType(name))
    else:
        raise ValueError(backend)
    sys.path.insert(1 if backend == 'dropin' else 0, root)
    sys.path.append(STUBS)                                     # LAST: real imageio / matplotlib win when installed
    return root


def build_generator(scene_size=1024, device='cuda', weights_seed=0, stress=True, quiet=True):
    """-> (generator in eval mode on `device`, cfg).  Weights: seeded module init (torch.manual_seed(0), CPU) and, for the
    three networks of the per-pixel path, the oracle's "stress" set under the reference's own state-dict names."""
    from oracle import ref_ops
    root = reference_python_root()
    stdout = sys.stdout
    if quiet:
        sys.stdout = open(os.devnull, 'w')
    try:
        from imaginaire.config import Config
        cfg = Config(os.path.join(root, 'configs', 'scenedreamer_inference.yaml'))
        cfg.gen.scene_size = scene_size
        torch.manual_seed(0)
        lib = importlib.import_module(cfg.gen.type)            # imaginaire/utils/trainer.py:94-95
        gen = lib.Generator(cfg.gen, cfg.data)
        gen.custom_init()
    finally:
        if quiet:
            sys.stdout.close()
            sys.stdout = stdout
    P = ref_ops.make_params(seed=weights_seed, stress=stress)
    sd = gen.state_dict()
    sub = {k: v for k, v in P.items() if k.split('.')[0] in ('render_net', 'sky_net', 'hash_encoder', 'style_net')}
    for k, v in sub.items():
        assert k in sd and tuple(sd[k].shape) == tuple(v.shape), (k, tuple(v.shape))
    gen.load_state_dict(sub, strict=False)
    g = torch.Generator().manual_seed(weights_seed + 1)
    with torch.no_grad():                                      # denoiser / world encoder: O(1) outputs instead of ~1e-3
        for name, p in gen.denoiser.named_parameters():
            if name.endswith('weight') and p.dim() > 1:
                fan_in = p[0].numel()
                p.copy_(torch.randn(p.shape, generator=g) * (1.4 / np.sqrt(fan_in)))
            elif name.endswith('bias'):
                p.copy_(torch.randn(p.shape, generator=g) * 0.1)
        gen.denoiser.conv4.weight.mul_(0.2)                    # raw image O(1): tanh not saturated
    gen = gen.to(device).eval()
    for p in gen.parameters():
        p.requires_grad = False
    return gen, cfg


def set_world(gen, world, device='cuda'):
    """Give the generator's PCGVoxelGenerator the state `next_world` (pcg_gen.py:83-174) would have left."""
    v = gen.voxel
    v.voxel_t = world.voxel_t.to(device)
    v.heightmap = world.heightmap
    v.trans_mat = world.trans_mat.clone()
    v.current_height_map = world.current_height_map.to(device)
    v.current_semantic_map = world.current_semantic_map.to(device)
    v.total_size = tuple(world.heightmap.shape)
    return gen


def default_style(gen, seed=8888, device='cuda'):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(1, gen.style_dims, generator=g).to(device)


def run_inference(gen, style, outdir, camera_mode=0, cam_maxstep=40, frames=1, num_samples=24, resolution_hw=(540, 960),
                  pad=30, keep=True, referee=False):
    """Run the reference's own `inference_givenstyle` for the first `frames` poses of the trajectory and collect, per
    frame, the stitched per-pixel feature map, the depth map sum(w * t) and the RGB image, plus GPU-timeline
    durations: `perpix_ms` = raycast + sky pre-pass + all `_forward_perpix` calls, `cnn_ms` = all `_forward_global`
    calls (CUDA events around the calls; the PNG write between frames is outside both).

    referee=True (reference composition only): every tile's LightningMLP is re-evaluated in FLOAT64 on the fp32 hash-grid
    features the reference computed (a double copy of `render_net`), followed by `volum_rendering_relu` and the depth sum in
    float64 -> `depth64` per frame: the arbiter for the 1e-3 depth bar (depth = sum w*t with t of several hundred voxels,
    where fp32 rounding of either implementation is of the order of the bar itself)."""
    import imaginaire.model_utils.gancraft.camctl as camctl
    smod = sys.modules[type(gen).__module__]
    vox_pkg = smod.voxlib
    tiles, frames_out = [], []
    marks = []                                                  # (kind, event)

    def mark(kind):
        e = torch.cuda.Event(enable_timing=True)
        e.record()
        marks.append((kind, e))

    real_dda = vox_pkg.ray_voxel_intersection_perspective
    real_ctl = camctl.EvalCameraController

    class FirstFrames(real_ctl):                                # same controller; the `for` over it stops after `frames` poses
        def __len__(self):
            return min(frames, super().__len__())

        def __getitem__(self, idx):
            if idx >= frames:
                raise IndexError(idx)
            return super().__getitem__(idx)

    def dda(*a, **k):
        mark('frame')
        return real_dda(*a, **k)

    cls = type(gen)
    net64, captured, hook = None, [], None
    if referee:
        import copy
        import imaginaire.model_utils.gancraft.mc_utils as mc_utils
        net64 = copy.deepcopy(gen.render_net).double()
        hook = gen.render_net.register_forward_hook(lambda m, inp, out: captured.append(inp))

    def perpix(*a, **k):
        out = cls._forward_perpix(gen, *a, **k)
        d64 = None
        if referee:
            x, raydir, zz, onehot = captured.pop()
            sig64, _ = net64(x.double(), None, zz.double(), onehot.double())
            w64 = mc_utils.volum_rendering_relu(sig64, out[1].double() * gen.dists_scale, dim=-2)
            w64 = w64 * torch.logical_not(out[10]).double()
            d64 = torch.sum(w64 * out[4].double(), -2)
            del sig64, w64, x, onehot
        tiles.append([out[0], torch.sum(out[2] * out[4], -2) if keep else None, None, d64])
        return out

    def glob(net_out, z):
        mark('cnn0')
        out = cls._forward_global(gen, net_out, z)
        mark('cnn1')
        tiles[-1][2] = out[0]
        return out

    gen._forward_perpix, gen._forward_global = perpix, glob     # instance attributes shadow the (possibly patched) class methods
    vox_pkg.ray_voxel_intersection_perspective = dda
    smod.camctl.EvalCameraController = FirstFrames
    t0 = time.perf_counter()
    try:
        with torch.no_grad():
            gen.inference_givenstyle(style, outdir, camera_mode=camera_mode, cam_maxstep=cam_maxstep, num_samples=num_samples,
                                     resolution_hw=list(resolution_hw), pad=pad)
        mark('end')
        torch.cuda.synchronize()
    finally:
        if hook is not None:
            hook.remove()
        del gen._forward_perpix, gen._forward_global
        vox_pkg.ray_voxel_intersection_perspective = real_dda
        smod.camctl.EvalCameraController = real_ctl
    wall = time.perf_counter() - t0
    # ---- stitch (scenedreamer.py:600-628: strips of tile_size=128, crop pad/2 on every side) ----
    nh = (resolution_hw[0] + 127) // 128
    nw = (resolution_hw[1] + 127) // 128
    per = nh * nw
    assert len(tiles) == frames * per, (len(tiles), frames, per)
    c = pad // 2

    def crop(t, chan_last):
        if pad == 0:
            return t
        return t[:, c:-c, c:-c] if chan_last else t[:, :, c:-c, c:-c]

    for f in range(frames):
        rows_n, rows_d, rows_i, rows_r = [], [], [], []
        for i in range(nh):
            tl = tiles[f * per + i * nw: f * per + (i + 1) * nw]
            rows_n.append(torch.cat([crop(t[0], True) for t in tl], 2))
            if keep:
                rows_d.append(torch.cat([crop(t[1], True) for t in tl], 2))
            if referee:
                rows_r.append(torch.cat([crop(t[3], True) for t in tl], 2))
            rows_i.append(torch.cat([crop(t[2], False) for t in tl], 3))
        frames_out.append(dict(net_out=torch.cat(rows_n, 1)[0], depth=torch.cat(rows_d, 1)[0, ..., 0] if keep else None,
                               depth64=torch.cat(rows_r, 1)[0, ..., 0] if referee else None,
                               rgb=torch.cat(rows_i, 2)[0]))
    # ---- timeline segments ----
    perpix_ms, cnn_ms = [0.0] * frames, [0.0] * frames
    f, prev = -1, None
    for kind, e in marks:
        if kind == 'frame':
            f += 1
            prev = e
        elif kind == 'cnn0':
            perpix_ms[f] += prev.elapsed_time(e)
            prev = e
        elif kind == 'cnn1':
            cnn_ms[f] += prev.elapsed_time(e)
            prev = e
    return dict(frames=frames_out, perpix_ms=perpix_ms, cnn_ms=cnn_ms, wall_s=wall)


def synthetic_world(scene_size=1024, seed=3407):
    from scenedreamer_b200 import synth                        # host-side scene generator (numpy), shared with bench.py
    return synth.SyntheticVoxelWorld(scene_size, seed)


def main():
    ap = argparse.ArgumentParser(description='run the reference Generator.inference_givenstyle in one backend')
    ap.add_argument('--backend', required=True, choices=['ref', 'dropin'])
    ap.add_argument('--out', required=True, help='.npz: frame 0 (net_out, depth, rgb) + timings of all frames')
    ap.add_argument('--scene', type=int, default=1024)
    ap.add_argument('--frames', type=int, default=1)
    ap.add_argument('--warm', type=int, default=0, help='untimed leading frames (same poses) before the measured run')
    ap.add_argument('--hw', type=int, nargs=2, default=[540, 960])
    ap.add_argument('--spp', type=int, default=24)
    ap.add_argument('--camera-mode', type=int, default=0)
    ap.add_argument('--workdir', default='/tmp/sdb_refgen')
    ap.add_argument('--referee', action='store_true', help="also leave depth64 (float64 re-evaluation of frame 0's MLP + compositing)")
    args = ap.parse_args()
    setup(args.backend)
    dev = 'cuda'
    gen, _ = build_generator(args.scene, dev)
    set_world(gen, synthetic_world(args.scene), dev)
    style = default_style(gen, device=dev)
    os.makedirs(args.workdir, exist_ok=True)
    kw = dict(camera_mode=args.camera_mode, num_samples=args.spp, resolution_hw=tuple(args.hw))
    if args.warm:
        run_inference(gen, style, args.workdir, frames=args.warm, keep=False, **kw)
    extra = {}
    if args.referee:
        rr = run_inference(gen, style, args.workdir, frames=1, referee=True, **kw)
        extra['depth64'] = rr['frames'][0]['depth64'].cpu().numpy()
        del rr
    r = run_inference(gen, style, args.workdir, frames=args.frames, **kw)
    f0 = r['frames'][0]
    np.savez(args.out, net_out=f0['net_out'].cpu().numpy(), depth=f0['depth'].cpu().numpy(), rgb=f0['rgb'].cpu().numpy(),
             perpix_ms=np.array(r['perpix_ms']), cnn_ms=np.array(r['cnn_ms']), wall_s=r['wall_s'], **extra)
    print('[refgen:%s] frames %d  perpix ms %s  cnn ms %s' % (args.backend, args.frames,
                                                              ' '.join('%.1f' % v for v in r['perpix_ms']),
                                                              ' '.join('%.1f' % v for v in r['cnn_ms'])))


if __name__ == '__main__':
    main()
