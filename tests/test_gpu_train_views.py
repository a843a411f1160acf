"""A batch of views of one scene in ONE recorded pass of the fused training path (render.render_rays_train with N views:
sdb_render_rays_train_forward over n_img images, sdb_render_rays_backward_views, sdb_sky_*_views), against N single-view
passes, the float64 oracle under torch.autograd, and through the Generator hook."""
import os

import numpy as np
import pytest
import torch

import oracle
from scenedreamer_b200 import _lib, ops, render, synth

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1500)]
DEV = 'cuda:0'
GRAD_TOL = 1e-2          # against the float64 oracle, as tests/test_gpu_train.py
SUM_TOL = 1e-5           # against the sum of single-view passes: only the order of fp32 atomics differs (see below)
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


def _leaf(P, dev):
    return {k: v.detach().clone().to(dev).requires_grad_(True) for k, v in P.items()}


def test_batch_equals_single_views_and_oracle(views, golden_ops):
    v = views
    P0 = oracle.make_params(seed=21, stress=True)
    g = torch.Generator().manual_seed(8888)
    z0 = oracle.style_mlp(torch.randn(N_VIEWS, 128, generator=g), P0)
    genc0 = torch.tanh(torch.randn(1, 2, generator=g))
    N, H, W = v['vid'].shape[:3]
    assert N == N_VIEWS and bool((v['vid'] != 0).any())
    uni = torch.rand(N, H, W, S + 1, 1, generator=torch.Generator().manual_seed(5)).to(DEV)
    G = torch.randn(N, H, W, 64, generator=torch.Generator().manual_seed(9)).to(DEV)
    lut_raw = torch.from_numpy(golden_ops['mc2reduced_lut'])
    lut = render.reduced_label_lut(golden_ops['mc2reduced_lut'], 0, 3)
    offsets, pls = oracle.grid_offsets()
    vdims = list(v['world'].voxel_t.shape)

    def run(sl):
        Pg = _leaf(P0, DEV)
        z, genc = z0.clone().to(DEV).requires_grad_(True), genc0.clone().to(DEV).requires_grad_(True)
        outs = []
        for a, b in sl:
            out = render.render_rays_train(Pg, v['vid'][a:b], v['dep'][a:b], v['rd'][a:b], v['o'][a:b].to(DEV), z[a:b], genc,
                                           vdims, lut, pls, num_samples=S, uniforms=uni[a:b])
            (out['net_out'] * G[a:b]).sum().backward()
            outs.append(out)
        torch.cuda.synchronize()
        cat = {k: torch.cat([o[k].detach() for o in outs], 0) for k in ('net_out', 'depth', 'total_weight', 'weights',
                                                                        'rand_depth', 'sky')}
        grads = {k: q.grad for k, q in Pg.items() if q.grad is not None}
        grads['z'], grads['global_enc'] = z.grad, genc.grad
        return cat, grads

    bo, bg = run([(0, N)])
    so, sg = run([(i, i + 1) for i in range(N)])
    # the weight-gradient kernels add their CTAs' partial sums with red.add, in no fixed order; where the views' gradients
    # cancel (the style-code terms of the sky's layer-0 bias) that order alone moves a tensor by more than 1e-5.  The bound is
    # therefore also held to 4x the largest difference between identical single-view runs (two pairs: one pair alone
    # under-samples that spread)
    reps = [run([(i, i + 1) for i in range(N)])[1] for _ in range(2)]
    spread = {k: max(_rel(r[k], sg[k]) for r in reps) for k in sg}
    for k in bo:
        assert torch.equal(bo[k], so[k]), (k, float((bo[k] - so[k]).abs().max()))
    assert set(bg) == set(sg) and len(bg) > 20
    worst = 0.0
    for k in bg:
        e = _rel(bg[k], sg[k])
        worst = max(worst, e)
        assert e <= max(SUM_TOL, 4.0 * spread[k]), (k, e, spread[k])
    print('batch vs single views: worst gradient rel-L2 %.2e over %d tensors; single vs single up to %.2e' %
          (worst, len(bg), max(spread.values())))

    # the oracle's torch composition under torch.autograd, view by view (the gradients of the views add up in the leaves)
    Pc = _leaf(P0, 'cpu')
    zc, gc = z0.clone().requires_grad_(True), genc0.clone().requires_grad_(True)
    ls = (torch.exp2(torch.arange(16, device=DEV, dtype=torch.float32) * torch.tensor(float(np.float32(np.log2(pls))), device=DEV))
          * 16.0 - 1.0).cpu()
    for i in range(N):
        ref = oracle.forward_perpix_autograd(Pc, v['vid'][i:i + 1].cpu(), v['dep'][i:i + 1].cpu(), v['rd'][i:i + 1].cpu(),
                                             v['o'][i:i + 1], zc[i:i + 1], gc, vdims, lut_raw, offsets, pls, num_samples=S,
                                             deterministic=False, uniforms=uni[i:i + 1].cpu(), level_scales=ls)
        (ref * G[i:i + 1].cpu().to(ref.dtype)).sum().backward()
    ref_g = {k: q.grad for k, q in Pc.items() if q.grad is not None}
    ref_g['z'], ref_g['global_enc'] = zc.grad, gc.grad
    for k in bg:
        if k in ref_g and float(ref_g[k].norm()) > 0:
            e = _rel(bg[k].cpu(), ref_g[k])
            assert e <= GRAD_TOL, (k, e)


def test_batch_workspace_is_one_view():
    L = _lib.lib()
    for H, W in ((262, 262), (36, 52)):
        assert L.sdb_render_backward_workspace_bytes(8, H, W, S, 16, 19) == L.sdb_render_backward_workspace_bytes(1, H, W, S, 16, 19)
        assert L.sdb_sky_backward_workspace_bytes(8, H, W) == L.sdb_sky_backward_workspace_bytes(1, H, W)
        assert L.sdb_render_train_record_bytes(8, H, W, S) > 7 * L.sdb_render_train_record_bytes(1, H, W, S)


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


def _gen_step(gen, n_views, monkeypatch, env, sky_avg=None):
    from scenedreamer_b200 import ops
    import imaginaire.model_utils.gancraft.camctl as camctl
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
    if sky_avg is not None:
        gen.sky_avg = sky_avg
    from scenedreamer_b200 import integration
    st = integration._state(gen).stats
    before = (st['train_calls'], st['reference_calls'])
    try:
        gen.coarse_deterministic_sampling = False
        gen.num_samples = 24
        torch.manual_seed(5)
        out = gen(data, random_style=True)
        out['fake_images'].square().mean().backward()
        torch.cuda.synchronize()
        return {k: q.grad.clone() for k, q in zip(PARAMS, params)}, (st['train_calls'] - before[0], st['reference_calls'] - before[1])
    finally:
        for q in params:
            q.requires_grad_(False)
            q.grad = None
        if hasattr(gen, 'sky_avg'):
            del gen.sky_avg
        for k in env:
            monkeypatch.delenv(k)


def test_generator_two_views_one_pass(generator, monkeypatch):
    gb, (tc, rc) = _gen_step(generator, 2, monkeypatch, {'SDB200_TRAIN_VIEWS': '1'})
    assert (tc, rc) == (1, 0)
    gl, (tc2, _) = _gen_step(generator, 2, monkeypatch, {'SDB200_TRAIN_VIEWS': '0'})
    assert tc2 == 1
    for k in PARAMS:
        assert float(gb[k].abs().max()) > 0, k
        assert _rel(gb[k], gl[k]) <= SUM_TOL, (k, _rel(gb[k], gl[k]))


def test_generator_preset_sky_avg_matches_reference(generator, monkeypatch):
    sky_avg = (torch.randn(1, 1, 1, 1, 64, generator=torch.Generator().manual_seed(3)) * 0.3).to(DEV)
    # one view: the reference's own composition (SDB200_FUSED=0) takes one scene code per ray batch
    gf, (tc, rc) = _gen_step(generator, 1, monkeypatch, {'SDB200_TRAIN_VIEWS': '1'}, sky_avg=sky_avg)
    assert tc == 1 and rc == 0
    tf32 = (torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32)
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    try:
        gr, _ = _gen_step(generator, 1, monkeypatch, {'SDB200_FUSED': '0'}, sky_avg=sky_avg)
    finally:
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = tf32
    for k in PARAMS:
        e = _rel(gf[k], gr[k])
        print('preset sky_avg, fused vs reference: %s rel-L2 %.2e' % (k, e))
        assert e <= 1e-2, (k, e)
