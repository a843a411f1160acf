"""GPU parity tests for the fused per-pixel renderer (sdb_render_rays_forward) through the C ABI:
CUDA path vs the CPU oracle on the same seeded inputs, vs the committed reference-generated golden
frame, plus size-independent properties.  Tolerance: 1e-3 max-abs on net_out / depth (north star);
sampling indices are covered bit-exactly by the oracle tests."""
import numpy as np
import pytest
import torch

import oracle
from scenedreamer_b200 import ops, render, synth

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(300)]
DEV = 'cuda:0'
TOL = 1e-3


def to_dev(P):
    return {k: v.to(DEV) for k, v in P.items()}


def device_level_scales(L, pls, base):
    S = torch.tensor(float(np.float32(np.log2(pls))), device=DEV)
    lv = torch.arange(L, device=DEV, dtype=torch.float32)
    return (torch.exp2(lv * S) * float(base) - 1.0).cpu()


@pytest.fixture(scope='module')
def lut(golden_ops):
    return render.reduced_label_lut(golden_ops['mc2reduced_lut'], 0, 3)


@pytest.fixture(scope='module')
def scene():
    world = synth.SyntheticVoxelWorld(size=128, seed=7)
    pose = synth.eval_camera_poses(world, maxstep=8, pattern=0)[1]
    o, d, u, f, c, res = synth.frame_camera(world, pose, resolution_hw=(44, 60), pad=4)
    vid, dep, rd = ops.ray_voxel_intersection_perspective(world.voxel_t.to(DEV), o, d, u, f, c, res, 6)
    return dict(world=world, o=o, vid=vid.unsqueeze(0), dep=dep.unsqueeze(0), rd=rd.unsqueeze(0))


def run_oracle(P, sc, z, genc, lut_raw, S=24, uniforms=None):
    offsets, pls = oracle.grid_offsets()
    return oracle.forward_perpix(P, sc['vid'].cpu(), sc['dep'].cpu(), sc['rd'].cpu(), sc['o'].unsqueeze(0), z, genc,
                                 list(sc['world'].voxel_t.shape), lut_raw, offsets, pls, num_samples=S,
                                 deterministic=uniforms is None, uniforms=uniforms,
                                 level_scales=device_level_scales(16, pls, 16))


def run_fused(P, sc, z, genc, lut, precision, preblend, S=24, uniforms=None):
    _, pls = oracle.grid_offsets()
    r = render.FusedPerPixelRenderer(to_dev(P), sc['world'].voxel_t.shape, lut, pls, precision=precision, preblend=preblend)
    out = r.forward(sc['vid'], sc['dep'], sc['rd'], sc['o'].unsqueeze(0), z.to(DEV), genc.to(DEV), num_samples=S,
                    uniforms=uniforms)
    torch.cuda.synchronize()
    return out


@pytest.mark.parametrize('stress', [False, True])
@pytest.mark.parametrize('preblend', [False, True])
@pytest.mark.parametrize('precision', [render.PRECISION_FP16X3, render.PRECISION_BF16X3])
def test_fused_vs_oracle_x3(scene, lut, golden_ops, stress, preblend, precision):
    P = oracle.make_params(seed=21, stress=stress)
    g = torch.Generator().manual_seed(8888)
    z = oracle.style_mlp(torch.randn(1, 128, generator=g), P)
    genc = torch.tanh(torch.randn(1, 2, generator=g))
    ref = run_oracle(P, scene, z, genc, torch.from_numpy(golden_ops['mc2reduced_lut']))
    out = run_fused(P, scene, z, genc, lut, precision, preblend)
    err = (out['net_out'].cpu() - ref['net_out']).abs()
    derr = (out['depth'].cpu() - ref['depth_map'].squeeze(-1)).abs()
    werr = (out['total_weight'].cpu() - ref['total_weights'].reshape(out['total_weight'].shape)).abs()
    print('prec=%d stress=%s preblend=%s: net_out max err %.3e (|ref| max %.2f), depth err %.3e (max depth %.1f), '
          'weight err %.3e (max %.3f), live %.2f'
          % (precision, stress, preblend, float(err.max()), float(ref['net_out'].abs().max()), float(derr.max()),
             float(ref['depth_map'].abs().max()), float(werr.max()), float(ref['total_weights'].max()),
             float((scene['vid'][..., 0, 0] != 0).float().mean())))
    assert float(err.max()) <= TOL
    assert float(werr.max()) <= TOL
    if precision == render.PRECISION_FP16X3:
        assert float(derr.max()) <= TOL                       # depth (values up to ~100 voxels): 1e-3 ABSOLUTE
    else:                                                     # bf16 split: ~2^-16 relative on the weights
        assert float(derr.max()) <= 1e-4 * max(1.0, float(ref['depth_map'].abs().max()))
    if stress:
        assert float(ref['net_out'].abs().max()) > 0.5 and float(ref['total_weights'].max()) > 0.9


def test_fused_vs_reference_golden_frame(lut, golden_fpp, golden_ops):
    """The committed frame produced by the reference's own _forward_perpix (tests/golden)."""
    g = golden_fpp
    dims = [int(v) for v in g['fpp_voxel_dims']]
    cam = g['fpp_cam']
    _, pls = oracle.grid_offsets()
    for tag, stress in (('spec', False), ('stress', True)):
        P = oracle.make_params(seed=9, stress=stress)
        r = render.FusedPerPixelRenderer(to_dev(P), dims, lut, pls, precision=render.PRECISION_BF16X3, preblend=False)
        vid = torch.from_numpy(g['fpp_voxel_id']).to(DEV).unsqueeze(0).contiguous()
        dep = torch.from_numpy(g['fpp_depth2']).to(DEV).unsqueeze(0).contiguous()
        rd = torch.from_numpy(g['fpp_raydirs']).to(DEV).unsqueeze(0).contiguous()
        out = r.forward(vid, dep, rd, torch.from_numpy(cam[0:3]).float().unsqueeze(0),
                        torch.from_numpy(g['fpp_%s_z' % tag]).to(DEV), torch.from_numpy(g['fpp_%s_genc' % tag]).to(DEV))
        torch.cuda.synchronize()
        err = np.abs(out['net_out'].cpu().numpy() - g['fpp_%s_net_out' % tag])
        werr = np.abs(out['total_weight'].cpu().numpy() - g['fpp_%s_total_weights_raw' % tag].reshape(out['total_weight'].shape))
        print('golden frame %s: net_out max err %.3e, total weight err %.3e' % (tag, err.max(), werr.max()))
        assert err.max() <= TOL and werr.max() <= TOL


def test_fused_fp16_single_pass_error_budget(scene, lut, golden_ops):
    """precision 0 (one fp16 pass) is the fast mode: documents its error; must stay within 1e-2."""
    P = oracle.make_params(seed=21, stress=True)
    g = torch.Generator().manual_seed(8888)
    z = oracle.style_mlp(torch.randn(1, 128, generator=g), P)
    genc = torch.tanh(torch.randn(1, 2, generator=g))
    ref = run_oracle(P, scene, z, genc, torch.from_numpy(golden_ops['mc2reduced_lut']))
    out = run_fused(P, scene, z, genc, lut, render.PRECISION_FP16, True)
    err = (out['net_out'].cpu() - ref['net_out']).abs()
    print('fp16x1 stress: net_out max err %.3e mean %.3e' % (float(err.max()), float(err.mean())))
    assert float(err.max()) <= 1e-2


def test_fused_stratified_sampling_and_small_S(scene, lut, golden_ops):
    P = oracle.make_params(seed=5, stress=True)
    g = torch.Generator().manual_seed(1)
    z = oracle.style_mlp(torch.randn(1, 128, generator=g), P)
    genc = torch.tanh(torch.randn(1, 2, generator=g))
    N, H, W = scene['vid'].shape[:3]
    for S in (24, 4):
        u = torch.rand(N, H, W, S + 1, 1, generator=g)
        ref = run_oracle(P, scene, z, genc, torch.from_numpy(golden_ops['mc2reduced_lut']), S=S, uniforms=u)
        out = run_fused(P, scene, z, genc, lut, render.PRECISION_BF16X3, False, S=S, uniforms=u)
        err = (out['net_out'].cpu() - ref['net_out']).abs()
        print('stratified S=%d: net_out max err %.3e' % (S, float(err.max())))
        assert float(err.max()) <= TOL


def test_fused_batch_of_views_two_styles(scene, lut, golden_ops):
    """N=2 images with different style codes / scene codes (the train.py shape): per-image packs."""
    P = oracle.make_params(seed=33, stress=True)
    g = torch.Generator().manual_seed(3)
    z = oracle.style_mlp(torch.randn(2, 128, generator=g), P)
    genc = torch.tanh(torch.randn(2, 2, generator=g))
    sc2 = dict(scene)
    sc2['vid'] = torch.cat([scene['vid'], scene['vid'].flip(2)], 0).contiguous()
    sc2['dep'] = torch.cat([scene['dep'], scene['dep'].flip(3)], 0).contiguous()
    sc2['rd'] = torch.cat([scene['rd'], scene['rd'].flip(2)], 0).contiguous()
    offsets, pls = oracle.grid_offsets()
    ref = oracle.forward_perpix(P, sc2['vid'].cpu(), sc2['dep'].cpu(), sc2['rd'].cpu(), scene['o'].repeat(2, 1), z, genc,
                                list(scene['world'].voxel_t.shape), torch.from_numpy(golden_ops['mc2reduced_lut']), offsets,
                                pls, level_scales=device_level_scales(16, pls, 16))
    r = render.FusedPerPixelRenderer(to_dev(P), scene['world'].voxel_t.shape, lut, pls, preblend=False)
    out = r.forward(sc2['vid'], sc2['dep'], sc2['rd'], scene['o'].repeat(2, 1), z.to(DEV), genc.to(DEV))
    torch.cuda.synchronize()
    err = (out['net_out'].cpu() - ref['net_out']).abs()
    print('batch of 2 views: net_out max err %.3e' % float(err.max()))
    assert float(err.max()) <= TOL


def test_fused_properties_all_sky_and_determinism(scene, lut):
    """Sky-only frame -> output is exactly the clamped sky feature; two runs are bit-identical."""
    P = oracle.make_params(seed=2, stress=True)
    _, pls = oracle.grid_offsets()
    r = render.FusedPerPixelRenderer(to_dev(P), scene['world'].voxel_t.shape, lut, pls)
    g = torch.Generator().manual_seed(4)
    z = oracle.style_mlp(torch.randn(1, 128, generator=g), P).to(DEV)
    genc = torch.tanh(torch.randn(1, 2, generator=g)).to(DEV)
    vid0 = torch.zeros_like(scene['vid'])
    dep0 = torch.full_like(scene['dep'], float('nan'))
    out = r.forward(vid0, dep0, scene['rd'], scene['o'].unsqueeze(0), z, genc)
    sky = out['sky']
    expect = (torch.clamp(sky, -1, 1) + 1) - 1
    assert torch.equal(out['net_out'], expect)
    assert float(out['total_weight'].abs().max()) == 0.0
    a = r.forward(scene['vid'], scene['dep'], scene['rd'], scene['o'].unsqueeze(0), z, genc)['net_out'].clone()
    b = r.forward(scene['vid'], scene['dep'], scene['rd'], scene['o'].unsqueeze(0), z, genc)['net_out']
    torch.cuda.synchronize()
    assert torch.equal(a, b)
    assert bool(torch.isfinite(a).all())


def test_sky_forward_vs_oracle(scene):
    """a9 on the tensor-core engine: PE + SKYMLP + frame mean vs the oracle (and vs the cuBLAS path)."""
    P = oracle.make_params(seed=12, stress=True)
    Pd = to_dev(P)
    g = torch.Generator().manual_seed(6)
    z = oracle.style_mlp(torch.randn(2, 128, generator=g), P)
    rd = torch.cat([scene['rd'], scene['rd'].flip(1)], 0).contiguous()
    N, H, W = rd.shape[:3]
    pe = oracle.positional_encoding_pt(rd.cpu(), 5, -1, True)
    ref = oracle.sky_mlp(pe.reshape(N, H * W, -1), z, P).reshape(N, H, W, 64)
    for prec, tol in ((render.PRECISION_FP16X3, 2e-4), (render.PRECISION_BF16X3, 1e-3), (render.PRECISION_FP16, 2e-2)):
        sky, avg = render.sky_forward(rd, render.pack_sky_mlp(Pd, z.to(DEV), prec), prec)
        torch.cuda.synchronize()
        err = float((sky.cpu() - ref).abs().max())
        aerr = float((avg.cpu() - ref.mean(dim=(1, 2))).abs().max())
        print('sky precision %d: max err %.3e (|ref| max %.2f), mean err %.3e' % (prec, err, float(ref.abs().max()), aerr))
        assert err <= tol and aerr <= tol
    t = render.sky_features(Pd, rd, z.to(DEV))
    assert float((t.cpu() - ref).abs().max()) <= 1e-4


def test_early_termination_error_bound_and_savings(scene, lut, golden_ops):
    """Tile-level early termination (render.EARLY_STOP_T): outputs stay within 2*T of the exact march, the samples not
    shaded report weight 0 and were below T in the exact march, and with T = 0 the kernel is the exact march."""
    P = oracle.make_params(seed=21, stress=True)
    P['render_net.fc_sigma.bias'] = torch.full((1,), 150.0)      # dense medium: rays saturate within a few samples
    g = torch.Generator().manual_seed(8888)
    z = oracle.style_mlp(torch.randn(1, 128, generator=g), P)
    genc = torch.tanh(torch.randn(1, 2, generator=g))
    _, pls = oracle.grid_offsets()
    r = render.FusedPerPixelRenderer(to_dev(P), scene['world'].voxel_t.shape, lut, pls)
    args = (scene['vid'], scene['dep'], scene['rd'], scene['o'].unsqueeze(0), z.to(DEV), genc.to(DEV))
    outs = {}
    for T in (0.0, 1e-7, 1e-3):
        r.early_stop = T
        o = r.forward(*args, want_samples=True)
        torch.cuda.synchronize()
        outs[T] = {k: o[k].clone() for k in ('net_out', 'depth', 'total_weight', 'weights', 'rand_depth')}
    exact = outs[0.0]
    for T in (1e-7, 1e-3):
        d = outs[T]
        assert float((d['net_out'] - exact['net_out']).abs().max()) <= 2.5 * T + 1e-7
        assert float((d['total_weight'] - exact['total_weight']).abs().max()) <= T + 1e-7
        assert torch.equal(d['rand_depth'], exact['rand_depth'])
        skipped = (d['weights'] == 0) & (exact['weights'] != 0)
        assert float(exact['weights'][skipped].max() if bool(skipped.any()) else 0.0) <= T
        same = ~skipped
        assert torch.equal(d['weights'][same], exact['weights'][same])
        dmax = float(exact['rand_depth'].abs().max())
        assert float((d['depth'] - exact['depth']).abs().max()) <= T * dmax + 1e-4
        print('early stop T=%g: %.1f %% of the non-zero sample weights skipped, max |d net_out| %.2e'
              % (T, 100.0 * float(skipped.float().sum() / max(1.0, float((exact['weights'] != 0).sum()))),
                 float((d['net_out'] - exact['net_out']).abs().max())))
    assert bool(((outs[1e-3]['weights'] == 0) & (exact['weights'] != 0)).any())       # something was skipped


def test_ray_slots_equal_the_tile_kernel(scene, lut, golden_ops, monkeypatch):
    """The ray-slot kernel (every MMA row a ray with its own cursor, the inference default) against the tile kernel
    (SDB_RAY_SLOTS=0): bit-identical with early termination off -- every ray's arithmetic is the same, only its row and
    its companions differ -- and within the termination threshold otherwise."""
    P = oracle.make_params(seed=21, stress=True)
    P['render_net.fc_sigma.bias'] = torch.full((1,), 60.0)
    g = torch.Generator().manual_seed(8888)
    z = oracle.style_mlp(torch.randn(1, 128, generator=g), P)
    genc = torch.tanh(torch.randn(1, 2, generator=g))
    _, pls = oracle.grid_offsets()
    r = render.FusedPerPixelRenderer(to_dev(P), scene['world'].voxel_t.shape, lut, pls)
    args = (scene['vid'], scene['dep'], scene['rd'], scene['o'].unsqueeze(0), z.to(DEV), genc.to(DEV))
    keys = ('net_out', 'depth', 'total_weight', 'weights', 'rand_depth')
    res = {}
    for T in (0.0, None):
        r.early_stop = T
        for variant in ('1', '0'):
            monkeypatch.setenv('SDB_RAY_SLOTS', variant)
            o = r.forward(*args, want_samples=True)
            torch.cuda.synchronize()
            ws = o['workspace'][:16].view(torch.int32).cpu()
            assert int(ws[3]) == int(variant)
            res[(T, variant)] = ({k: o[k].clone() for k in keys}, int(ws[1]))
    for k in keys:
        assert torch.equal(res[(0.0, '1')][0][k], res[(0.0, '0')][0][k]), k
    a, b = res[(None, '1')][0], res[(None, '0')][0]
    assert float((a['net_out'] - b['net_out']).abs().max()) <= 5 * render.EARLY_STOP_T
    assert torch.equal(a['rand_depth'], b['rand_depth'])
    steps_rq, steps_tile = res[(None, '1')][1], res[(None, '0')][1]
    print('steps of 128 rows: ray slots %d, tiles %d (early termination on); %d / %d with it off'
          % (steps_rq, steps_tile, res[(0.0, '1')][1], res[(0.0, '0')][1]))
    assert steps_rq > 0 and steps_tile > 0          # (fewer steps only on frame-sized inputs, tools/ray_stats.py; here the
                                                    #  per-CTA drain of a 3,000-ray window dominates: 603 vs 576 steps measured)
