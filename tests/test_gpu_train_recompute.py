"""Recompute mode of the fused training path (render.render_rays_train(recompute=True): a forward that keeps no record and
sdb_render_rays_backward_recompute, which rebuilds one view's record at a time) against record mode on the same inputs:
forward outputs, the rebuilt record, every gradient, peak memory at the training size, and through the Generator hook."""
import gc
import os

import numpy as np
import pytest
import torch

import oracle
from _train_record import Record, layout
from scenedreamer_b200 import _lib, ops, render, synth
from test_gpu_train import GRAD_KEYS

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1500)]
DEV = 'cuda:0'
GRAD_TOL = 1e-2          # against the float64 oracle, as tests/test_gpu_train.py
# recompute vs record mode: the same arithmetic, only the order of the fp32 red.add differs.  That order alone moves a gradient
# by up to a few 1e-5 rel-L2 where terms cancel (the style code, the sky's first layers; tests/test_gpu_train_views.py), and a
# pair of identical runs under-samples that spread, so the bound is the larger of MODE_TOL and 4x the largest difference
# between identical record-mode runs (two pairs)
MODE_TOL = 1e-5
N_VIEWS, S = 3, 24


def _rel(a, b):
    return float((a.double() - b.double()).norm() / max(float(b.double().norm()), 1e-30))


@pytest.fixture(scope='module')
def views():
    world = synth.SyntheticVoxelWorld(size=128, seed=7)
    poses = synth.eval_camera_poses(world, maxstep=8, pattern=0)
    vids, deps, rds, oris = [], [], [], []
    for k in (1, 3, 5):
        o, d, u, f, c, res = synth.frame_camera(world, poses[k], resolution_hw=(36, 52), pad=4)
        vid, dep, rd = ops.ray_voxel_intersection_perspective(world.voxel_t.to(DEV), o, d, u, f, c, res, 6)
        vids.append(vid), deps.append(dep), rds.append(rd), oris.append(o)
    return dict(world=world, vid=torch.stack(vids), dep=torch.stack(deps), rd=torch.stack(rds), o=torch.stack(oris))


@pytest.fixture(scope='module')
def setup(views, golden_ops):
    P0 = oracle.make_params(seed=21, stress=True)
    g = torch.Generator().manual_seed(8888)
    z0 = oracle.style_mlp(torch.randn(N_VIEWS, 128, generator=g), P0)
    genc0 = torch.tanh(torch.randn(1, 2, generator=g))
    N, H, W = views['vid'].shape[:3]
    uni = torch.rand(N, H, W, S + 1, 1, generator=torch.Generator().manual_seed(5)).to(DEV)
    G = torch.randn(N, H, W, 64, generator=torch.Generator().manual_seed(9)).to(DEV)
    lut = render.reduced_label_lut(golden_ops['mc2reduced_lut'], 0, 3)
    _, pls = oracle.grid_offsets()
    return dict(P0=P0, z0=z0, genc0=genc0, uni=uni, G=G, lut=lut, pls=pls, vdims=list(views['world'].voxel_t.shape))


def _run(v, s, n, recompute, precision=render.PRECISION_FP16X3, stratified=True, backward=True):
    """One training pass over the first n views -> (detached outputs, gradients of every leaf)."""
    P = {k: t.detach().clone().to(DEV).requires_grad_(True) for k, t in s['P0'].items()}
    z = s['z0'][:n].clone().to(DEV).requires_grad_(True)
    genc = s['genc0'].clone().to(DEV).requires_grad_(True)
    with torch.set_grad_enabled(backward):
        out = render.render_rays_train(P, v['vid'][:n], v['dep'][:n], v['rd'][:n], v['o'][:n].to(DEV), z, genc, s['vdims'], s['lut'],
                                       s['pls'], num_samples=S, uniforms=s['uni'][:n] if stratified else None, precision=precision,
                                       recompute=recompute)
        if backward:
            (out['net_out'] * s['G'][:n]).sum().backward()
    torch.cuda.synchronize()
    outs = {k: out[k].detach() for k in ('net_out', 'depth', 'total_weight', 'weights', 'rand_depth')}
    grads = {k: q.grad for k, q in P.items() if q.grad is not None}
    if backward:
        grads['z'], grads['global_enc'] = z.grad, genc.grad
    return outs, grads


@pytest.mark.parametrize('n', [1, N_VIEWS])
@pytest.mark.parametrize('precision', [render.PRECISION_FP16X3, render.PRECISION_FP16])
@pytest.mark.parametrize('stratified', [True, False])
def test_forward_outputs_equal_record_mode(views, setup, n, precision, stratified):
    rec, _ = _run(views, setup, n, False, precision, stratified, backward=False)
    rcp, _ = _run(views, setup, n, True, precision, stratified, backward=False)
    assert float(rec['total_weight'].max()) > 0
    for k in rec:
        assert torch.equal(rec[k], rcp[k]), (k, float((rec[k] - rcp[k]).abs().max()))


def _pooled_record():
    return render._scratch_pool[(DEV, 'record')].clone()


def test_rebuilt_record_equals_the_views_slice(views, setup):
    """After a recompute backward over N views the one-view record holds the last view's items, bit for bit those of that
    view in the N-view record of record mode (items matched by tile: the live-tile list is filled in no fixed order)."""
    L = _lib.lib()
    n = N_VIEWS
    H, W = views['vid'].shape[1:3]
    render.clear_scratch()
    _run(views, setup, n, False)
    rec_n = Record(layout(L, n, H, W, S), _pooled_record(), n, H, W, S)
    _run(views, setup, n, True)
    rec_1 = Record(layout(L, 1, H, W, S), _pooled_record(), 1, H, W, S)
    i = n - 1
    first_n, count = rec_n.views[i]
    assert rec_1.views[0] == (0, count) and rec_1.n_live == count and count > 0
    tiles_n = rec_n.tile_list[first_n:first_n + count] - i * rec_n.tpi
    tiles_1 = rec_1.tile_list[:count]
    order_n, order_1 = torch.argsort(tiles_n), torch.argsort(tiles_1)
    assert torch.equal(tiles_n[order_n], tiles_1[order_1])
    work_n, work_1 = (first_n + order_n).tolist(), order_1.tolist()

    def rows(per_work, works):
        return torch.cat([torch.arange(w * per_work, (w + 1) * per_work, device=DEV) for w in works])

    sn, s1 = rows(S * 128, work_n), rows(S * 128, work_1)
    fn, f1 = rows(128, work_n), rows(128, work_1)
    bits = lambda t: t.view(torch.int32) if t.dtype == torch.float32 else (t.view(torch.int16) if t.dtype == torch.bfloat16 else t)
    for name in ('x3', 'x0', 'sig', 'nds', 'c'):
        a, b = getattr(rec_n, name)[sn], getattr(rec_1, name)[s1]
        assert torch.equal(bits(a), bits(b)), name
    for k in range(6):
        assert torch.equal(bits(rec_n.act[k][sn]), bits(rec_1.act[k][s1])), 'act %d' % k
        assert torch.equal(rec_n.mask[k][sn], rec_1.mask[k][s1]), 'mask %d' % k
    for name in ('live', 'nosky', 'valid'):
        assert torch.equal(getattr(rec_n, name)[fn], getattr(rec_1, name)[f1]), name
    # the sky-only tiles of the view are the same too
    assert torch.equal(rec_n.sky_only_rays(i), rec_1.sky_only_rays(0))


@pytest.mark.parametrize('n', [1, N_VIEWS])
@pytest.mark.parametrize('precision', [render.PRECISION_FP16X3, render.PRECISION_FP16])
def test_gradients_equal_record_mode(views, setup, n, precision):
    _, g_rec = _run(views, setup, n, False, precision)
    _, g_rcp = _run(views, setup, n, True, precision)
    reps = [_run(views, setup, n, False, precision)[1] for _ in range(2)]
    assert set(g_rcp) == set(g_rec) and set(GRAD_KEYS) <= set(g_rec) and {'z', 'global_enc'} <= set(g_rec)
    worst = worst_spread = 0.0
    for k in g_rec:
        spread = max(_rel(r[k], g_rec[k]) for r in reps)
        e = _rel(g_rcp[k], g_rec[k])
        worst, worst_spread = max(worst, e), max(worst_spread, spread)
        assert float(g_rec[k].abs().max()) > 0, k
        assert e <= max(MODE_TOL, 4.0 * spread), (k, e, spread)
    print('recompute vs record mode, %d views, precision %d: worst gradient rel-L2 %.2e over %d tensors; record vs record up '
          'to %.2e' % (n, precision, worst, len(g_rec), worst_spread))


def test_gradients_match_oracle(views, setup):
    v, s = views, setup
    _, g = _run(v, s, N_VIEWS, True)
    Pc = {k: t.detach().clone().requires_grad_(True) for k, t in s['P0'].items()}
    zc, gc = s['z0'].clone().requires_grad_(True), s['genc0'].clone().requires_grad_(True)
    offsets, pls = oracle.grid_offsets()
    ls = (torch.exp2(torch.arange(16, device=DEV, dtype=torch.float32) * torch.tensor(float(np.float32(np.log2(pls))), device=DEV))
          * 16.0 - 1.0).cpu()
    lut_raw = torch.from_numpy(_golden_lut())
    for i in range(N_VIEWS):
        ref = oracle.forward_perpix_autograd(Pc, v['vid'][i:i + 1].cpu(), v['dep'][i:i + 1].cpu(), v['rd'][i:i + 1].cpu(),
                                             v['o'][i:i + 1], zc[i:i + 1], gc, s['vdims'], lut_raw, offsets, pls, num_samples=S,
                                             deterministic=False, uniforms=s['uni'][i:i + 1].cpu(), level_scales=ls)
        (ref * s['G'][i:i + 1].cpu().to(ref.dtype)).sum().backward()
    ref_g = {k: q.grad for k, q in Pc.items() if q.grad is not None}
    ref_g['z'], ref_g['global_enc'] = zc.grad, gc.grad
    for k in GRAD_KEYS + ['z', 'global_enc']:
        assert float(ref_g[k].norm()) > 0, k
        e = _rel(g[k].cpu(), ref_g[k])
        assert e <= GRAD_TOL, (k, e)


def _golden_lut():
    root = os.path.abspath(os.path.join(os.path.dirname(__file__), '..'))
    return np.load(os.path.join(root, 'tests', 'golden', 'ref_python_ops.npz'))['mc2reduced_lut']


def _one_pass(views, s, recompute, sky_impl, uniforms=None):
    P = {k: t.detach().clone().to(DEV).requires_grad_(True) for k, t in s['P0'].items()}
    z = s['z0'][:2].clone().to(DEV).requires_grad_(True)
    out = render.render_rays_train(P, views['vid'][:2], views['dep'][:2], views['rd'][:2], views['o'][:2].to(DEV), z,
                                   s['genc0'].to(DEV), s['vdims'], s['lut'], s['pls'], num_samples=S,
                                   uniforms=s['uni'][:2] if uniforms is None else uniforms, sky_impl=sky_impl, recompute=recompute)
    return (out['net_out'] * s['G'][:2]).sum()


@pytest.mark.parametrize('sky_impl', ['native', 'torch'])
@pytest.mark.parametrize('recompute', [True, False])
def test_second_backward_raises(views, setup, recompute, sky_impl):
    """A second backward through the same graph (retain_graph) raises in recompute mode as in record mode, with the native
    sky branch (what the Generator hook runs) and with the torch one: the render path refuses it first."""
    loss = _one_pass(views, setup, recompute, sky_impl)
    loss.backward(retain_graph=True)
    with pytest.raises(RuntimeError, match='released by its first backward'):
        loss.backward()


def test_inputs_modified_in_place_are_refused(views, setup):
    """Recompute mode reads the rays, uniforms, camera origins and sky features again in the backward: changing one of them in
    place after the forward makes the backward raise (autograd's version check) instead of differentiating another pass."""
    uni = setup['uni'][:2].clone()
    loss = _one_pass(views, setup, True, 'native', uniforms=uni)
    uni.mul_(0.5)
    with pytest.raises(RuntimeError, match='modified by an inplace operation'):
        loss.backward()
    torch.cuda.synchronize()


def test_memory_does_not_grow_with_the_batch(golden_ops):
    """262 x 262 views at 24 spp: with 4 views recompute mode peaks at least three records below record mode, and grows by
    less than one record from 1 view to 4."""
    L = _lib.lib()
    H = W = 262
    rec1 = int(L.sdb_render_train_record_bytes(1, H, W, S))
    world = synth.SyntheticVoxelWorld(size=512, seed=7)
    poses = synth.eval_camera_poses(world, maxstep=16, pattern=0)
    cams = []
    for k in range(4):
        o, d, u, f, c, r = synth.frame_camera(world, poses[1 + k], resolution_hw=(H - 6, W - 6), pad=6)
        cams.append(tuple(ops.ray_voxel_intersection_perspective(world.voxel_t.to(DEV), o, d, u, f, c, r, 6)) + (o,))
    P = {k: t.to(DEV).requires_grad_(True) for k, t in oracle.make_params(seed=1, stress=True).items()}
    g = torch.Generator().manual_seed(3)
    z_all = oracle.style_mlp(torch.randn(4, 128, generator=g), {k: t.detach().cpu() for k, t in P.items()}).to(DEV)
    genc = torch.tanh(torch.randn(1, 2, generator=g)).to(DEV)
    lut = render.reduced_label_lut(golden_ops['mc2reduced_lut'], 0, 3)
    _, pls = oracle.grid_offsets()
    uni = torch.rand(4, H, W, S + 1, 1, device=DEV)
    G = torch.randn(4, H, W, 64, device=DEV)

    def peak(n, recompute):
        vid, dep, rd, ori = (torch.stack([c[j] for c in cams[:n]]) for j in range(4))
        z = z_all[:n].clone().requires_grad_(True)
        for q in P.values():
            q.grad = None
        render.clear_scratch()
        # unreachable graphs of earlier passes (reference cycles, e.g. through a caught exception's traceback) would otherwise
        # be collected during the measured step and lower its peak above `base`
        gc.collect()
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        out = render.render_rays_train(P, vid, dep, rd, ori.to(DEV), z, genc, list(world.voxel_t.shape), lut, pls, num_samples=S,
                                       uniforms=uni[:n], recompute=recompute)
        torch.cuda.synchronize()
        fwd = torch.cuda.max_memory_allocated() - base
        (out['net_out'] * G[:n]).sum().backward()
        torch.cuda.synchronize()
        print('262x262, %d views, recompute %s: peak above the inputs %.2f GB after the forward, %.2f GB after the backward' %
              (n, recompute, fwd / 1e9, (torch.cuda.max_memory_allocated() - base) / 1e9))
        return torch.cuda.max_memory_allocated() - base

    r4, c4, c1 = peak(4, False), peak(4, True), peak(1, True)
    render.clear_scratch()
    print('262x262 peak above the inputs: record mode 4 views %.2f GB, recompute mode 4 views %.2f GB, 1 view %.2f GB '
          '(one record %.2f GB): recompute saves %.2f records at 4 views' % (r4 / 1e9, c4 / 1e9, c1 / 1e9, rec1 / 1e9, (r4 - c4) / rec1))
    # besides the records the two peaks hold the same tensors up to a few MB (2 MB measured on an H100)
    assert r4 - c4 >= 3 * rec1 - (32 << 20)
    assert c4 - c1 < rec1


# ---- through the Generator hook -------------------------------------------------------------------------------------------
def _have_reference():
    from oracle import refgen
    root = os.path.abspath(os.path.join(os.path.dirname(__file__), '..'))
    return (refgen.reference_python_root() is not None and
            os.path.exists(os.path.join(root, 'oracle', '_ref', 'ref_voxlib', 'ref_voxlib.so')) and
            os.path.exists(os.path.join(root, 'oracle', '_ref', 'ref_gridencoder', 'ref_gridencoder.so')))


@pytest.fixture(scope='module')
def generator():
    from oracle import refgen
    if not _have_reference():
        pytest.skip('reference Python / extensions not staged in oracle/_ref (oracle/build_ref.py)')
    refgen.setup('dropin')
    gen, _ = refgen.build_generator(1024, DEV)
    refgen.set_world(gen, refgen.synthetic_world(1024), DEV)
    from scenedreamer_b200 import integration
    integration.ensure_installed()
    return gen


PARAMS = ('render_net.fc_1.weight', 'render_net.fc_4.weight_alpha', 'render_net.fc_out_c.weight', 'hash_encoder.embeddings',
          'sky_net.fc3.weight', 'sky_net.fc_z_a.weight')


def _gen_step(gen, n_views, monkeypatch, env):
    import imaginaire.model_utils.gancraft.camctl as camctl
    from scenedreamer_b200 import integration
    for k, val in env.items():
        monkeypatch.setenv(k, val)
    vox = gen.voxel.voxel_t
    ctl = camctl.EvalCameraController(gen.voxel, maxstep=8, pattern=0, cam_ang=72)
    H = W = 64 + gen.pad
    vids, deps, rds, oris = [], [], [], []
    for k in range(n_views):
        pose = ctl[1 + 2 * k]
        vid, dep, rd = ops.ray_voxel_intersection_perspective(vox, pose[0], pose[1], pose[2], pose[3] * (W - 1),
                                                              [(H - 1) / 2, (W - 1) / 2], [H, W], 6)
        vids.append(vid), deps.append(dep), rds.append(rd), oris.append(pose[0].to(DEV))
    data = dict(images=torch.zeros(n_views, 3, 64, 64, device=DEV), voxel_id=torch.stack(vids), depth2=torch.stack(deps),
                raydirs=torch.stack(rds), cam_ori_t=torch.stack(oris))
    mods = dict(gen.named_parameters())
    params = [mods[k] for k in PARAMS]
    for q in params:
        q.requires_grad_(True)
        q.grad = None
    if hasattr(gen, 'sky_avg'):
        del gen.sky_avg
    st = integration._state(gen).stats
    before = (st['train_calls'], st['train_recompute_calls'], st['reference_calls'])
    try:
        gen.coarse_deterministic_sampling = False
        gen.num_samples = 24
        torch.manual_seed(5)
        out = gen(data, random_style=True)
        out['fake_images'].square().mean().backward()
        torch.cuda.synchronize()
        after = (st['train_calls'], st['train_recompute_calls'], st['reference_calls'])
        return {k: q.grad.clone() for k, q in zip(PARAMS, params)}, tuple(a - b for a, b in zip(after, before))
    finally:
        for q in params:
            q.requires_grad_(False)
            q.grad = None
        for k in env:
            monkeypatch.delenv(k)


@pytest.mark.parametrize('one_pass', ['1', '0'])
def test_generator_recompute_switch(generator, monkeypatch, one_pass):
    """SDB200_TRAIN_RECOMPUTE=1 gives the gradients of the default, for the one-pass batch and for the per-view loop."""
    g_on, calls_on = _gen_step(generator, 2, monkeypatch, {'SDB200_TRAIN_VIEWS': one_pass, 'SDB200_TRAIN_RECOMPUTE': '1'})
    assert calls_on == (1, 1, 0)
    g_off, calls_off = _gen_step(generator, 2, monkeypatch, {'SDB200_TRAIN_VIEWS': one_pass})
    assert calls_off == (1, 0, 0)
    reps = [_gen_step(generator, 2, monkeypatch, {'SDB200_TRAIN_VIEWS': one_pass, 'SDB200_TRAIN_RECOMPUTE': '0'})[0] for _ in range(2)]
    for k in PARAMS:
        assert float(g_off[k].abs().max()) > 0, k
        spread = max(_rel(r[k], g_off[k]) for r in reps)
        e = _rel(g_on[k], g_off[k])
        print('SDB200_TRAIN_VIEWS=%s, recompute vs record: %s rel-L2 %.2e (record vs record %.2e)' % (one_pass, k, e, spread))
        assert e <= max(MODE_TOL, 4.0 * spread), (k, e, spread)
