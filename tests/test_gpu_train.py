"""GPU parity tests of the fused training path (sdb_render_rays_train_forward / sdb_render_rays_backward)
through the C ABI: every parameter gradient of the per-pixel stage against the CPU oracle under
torch.autograd (oracle.forward_perpix_autograd: the reference's _grid_encode autograd.Function
restated on oracle.c + the torch fp32 MLP / compositing) on the same seeded inputs.

Tolerances (no gradient tolerance is stated by the north star; these are the ones asserted here):
  * forward of the recording kernel: 1e-3 max-abs on net_out like the inference kernel;
  * gradients: relative L2 error per tensor <= 1e-2 -- the data-gradient chain runs bf16x3 (2^-16
    relative per product) and the weight-gradient GEMMs take bf16 operands (2^-9 per element,
    fp32 accumulation over >= 10^4 samples); observed errors are printed per tensor.
"""
import os

import numpy as np
import pytest
import torch

import oracle
from scenedreamer_b200 import ops, render, synth

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), '..'))

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(600)]
DEV = 'cuda:0'
GRAD_TOL = 1e-2


def device_level_scales(L, pls, base):
    S = torch.tensor(float(np.float32(np.log2(pls))), device=DEV)
    lv = torch.arange(L, device=DEV, dtype=torch.float32)
    return (torch.exp2(lv * S) * float(base) - 1.0).cpu()


def make_scene(M=6):
    world = synth.SyntheticVoxelWorld(size=128, seed=7)
    pose = synth.eval_camera_poses(world, maxstep=8, pattern=0)[1]
    o, d, u, f, c, res = synth.frame_camera(world, pose, resolution_hw=(36, 52), pad=4)
    vid, dep, rd = ops.ray_voxel_intersection_perspective(world.voxel_t.to(DEV), o, d, u, f, c, res, M)
    return dict(world=world, o=o, vid=vid.unsqueeze(0), dep=dep.unsqueeze(0), rd=rd.unsqueeze(0))


@pytest.fixture(scope='module')
def scene():
    return make_scene()


def _leaf(P, dev):
    return {k: v.detach().clone().to(dev).requires_grad_(True) for k, v in P.items()}


GRAD_KEYS = ['hash_encoder.embeddings', 'render_net.fc_1.weight', 'render_net.fc_1.bias', 'render_net.fc_m_a.weight',
             'render_net.fc_sigma.weight', 'render_net.fc_sigma.bias', 'render_net.fc_out_c.weight', 'render_net.fc_out_c.bias',
             'sky_net.fc1.weight', 'sky_net.fc1.bias', 'sky_net.fc_z_a.weight', 'sky_net.fc2.weight', 'sky_net.fc3.bias',
             'sky_net.fc5.weight', 'sky_net.fc_out_c.weight', 'sky_net.fc_out_c.bias'] + \
            ['render_net.fc_%d.%s' % (k, n) for k in (2, 3, 4, 5, 6) for n in ('weight', 'weight_alpha', 'bias_alpha',
                                                                                'weight_beta', 'bias_beta')]


@pytest.mark.parametrize('stress,S,stratified,M', [(True, 24, True, 6), (False, 12, False, 6), (True, 64, True, 8)])
def test_fused_backward_vs_oracle_autograd(scene, golden_ops, stress, S, stratified, M):
    sc = scene if M == 6 else make_scene(M)
    P0 = oracle.make_params(seed=21, stress=stress)
    g = torch.Generator().manual_seed(8888)
    z0 = oracle.style_mlp(torch.randn(1, 128, generator=g), P0)
    genc0 = torch.tanh(torch.randn(1, 2, generator=g))
    N, H, W = sc['vid'].shape[:3]
    uni = torch.rand(N, H, W, S + 1, 1, generator=torch.Generator().manual_seed(5)) if stratified else None
    G = torch.randn(N, H, W, 64, generator=torch.Generator().manual_seed(9))
    if not stress:
        G = G * 100.0          # spec init: outputs ~1e-3; keep the gradients in a comfortable range
    lut_raw = torch.from_numpy(golden_ops['mc2reduced_lut'])
    offsets, pls = oracle.grid_offsets()

    # ---- oracle (CPU, torch.autograd) ----
    Pc = _leaf(P0, 'cpu')
    zc, gc = z0.clone().requires_grad_(True), genc0.clone().requires_grad_(True)
    ref = oracle.forward_perpix_autograd(Pc, sc['vid'].cpu(), sc['dep'].cpu(), sc['rd'].cpu(), sc['o'].unsqueeze(0), zc, gc,
                                         list(sc['world'].voxel_t.shape), lut_raw, offsets, pls, num_samples=S,
                                         deterministic=uni is None, uniforms=uni,
                                         level_scales=device_level_scales(16, pls, 16))
    (ref * G).sum().backward()

    # ---- fused (GPU) ----
    Pg = _leaf(P0, DEV)
    zg, gg = z0.clone().to(DEV).requires_grad_(True), genc0.clone().to(DEV).requires_grad_(True)
    lut = render.reduced_label_lut(golden_ops['mc2reduced_lut'], 0, 3)
    out = render.render_rays_train(Pg, sc['vid'], sc['dep'], sc['rd'], sc['o'].unsqueeze(0), zg, gg,
                                   list(sc['world'].voxel_t.shape), lut, pls, num_samples=S,
                                   uniforms=None if uni is None else uni.to(DEV))
    (out['net_out'] * G.to(DEV)).sum().backward()
    torch.cuda.synchronize()

    ferr = float((out['net_out'].detach().cpu() - ref.detach()).abs().max())
    print('forward (recording kernel) max abs err %.3e (|ref| max %.3f)' % (ferr, float(ref.abs().max())))
    assert ferr <= 1e-3
    worst = 0.0
    rows = [('z', zg.grad, zc.grad), ('global_enc', gg.grad, gc.grad)] + [(k, Pg[k].grad, Pc[k].grad) for k in GRAD_KEYS]
    for name, a, b in rows:
        assert a is not None, 'no gradient reached %s' % name
        a, b = a.detach().cpu().double(), b.detach().double()
        rel = float((a - b).norm() / (b.norm() + 1e-30))
        print('%-36s rel-L2 %.3e   max|diff| %.3e   max|ref| %.3e' % (name, rel, float((a - b).abs().max()), float(b.abs().max())))
        assert float(b.abs().max()) > 0, 'oracle gradient of %s is identically zero: vacuous test' % name
        worst = max(worst, rel)
    assert worst <= GRAD_TOL, worst


def test_train_forward_equals_inference_forward(scene, golden_ops):
    """The recording variant of the kernel computes exactly what the inference kernel computes."""
    sc = scene
    P = {k: v.to(DEV) for k, v in oracle.make_params(seed=3, stress=True).items()}
    g = torch.Generator().manual_seed(1)
    z = oracle.style_mlp(torch.randn(1, 128, generator=g), {k: v.cpu() for k, v in P.items()}).to(DEV)
    genc = torch.tanh(torch.randn(1, 2, generator=g)).to(DEV)
    lut = render.reduced_label_lut(golden_ops['mc2reduced_lut'], 0, 3)
    _, pls = oracle.grid_offsets()
    with torch.no_grad():
        tr = render.render_rays_train(P, sc['vid'], sc['dep'], sc['rd'], sc['o'].unsqueeze(0), z, genc,
                                      list(sc['world'].voxel_t.shape), lut, pls)
    r = render.FusedPerPixelRenderer(P, sc['world'].voxel_t.shape, lut, pls)
    r.early_stop = 0            # the recording kernel never terminates early: compare like with like
    inf = r.forward(sc['vid'], sc['dep'], sc['rd'], sc['o'].unsqueeze(0), z, genc, want_samples=True)
    torch.cuda.synchronize()
    for k in ('depth', 'total_weight', 'weights', 'rand_depth'):
        assert torch.equal(tr[k], inf[k]), k
    assert torch.equal(tr['sky'], inf['sky'])                # recording and plain sky kernels: same arithmetic
    # net_out additionally sees the frame mean of the sky features (torch reduction here, sky_mean_kernel there)
    assert float((tr['net_out'] - inf['net_out']).abs().max()) <= 1e-5


@pytest.mark.parametrize('sky_impl', ['torch'])
def test_train_sky_torch_crosscheck(scene, golden_ops, sky_impl):
    """The torch/cuBLAS sky branch stays available as an independent cross-check of the native one."""
    sc = scene
    P = {k: v.to(DEV).requires_grad_(True) for k, v in oracle.make_params(seed=3, stress=True).items()}
    g = torch.Generator().manual_seed(1)
    z = oracle.style_mlp(torch.randn(1, 128, generator=g), {k: v.detach().cpu() for k, v in P.items()}).to(DEV).requires_grad_(True)
    genc = torch.tanh(torch.randn(1, 2, generator=g)).to(DEV)
    lut = render.reduced_label_lut(golden_ops['mc2reduced_lut'], 0, 3)
    _, pls = oracle.grid_offsets()
    G = torch.randn(1, *sc['vid'].shape[1:3], 64, generator=torch.Generator().manual_seed(3)).to(DEV)
    grads = {}
    for impl in ('native', sky_impl):
        for t in list(P.values()) + [z]:
            t.grad = None
        out = render.render_rays_train(P, sc['vid'], sc['dep'], sc['rd'], sc['o'].unsqueeze(0), z, genc,
                                       list(sc['world'].voxel_t.shape), lut, pls, sky_impl=impl)
        (out['net_out'] * G).sum().backward()
        grads[impl] = {k: P[k].grad.clone() for k in P if k.startswith('sky_net.')}
        grads[impl]['z'] = z.grad.clone()
    for k in grads['native']:
        a, b = grads['native'][k].double(), grads[sky_impl][k].double()
        rel = float((a - b).norm() / (b.norm() + 1e-30))
        print('sky %-28s native vs %s rel-L2 %.3e' % (k, sky_impl, rel))
        assert rel <= 1e-2, k


def test_fused_style_modulation_matches_torch_autograd(monkeypatch):
    """ModLinear's fold for one style code (layers.py:247-260) as one fused forward / backward (csrc/modulate.cu) against the same
    algebra in torch ops under autograd: W', beta, and the gradients of all 25 tensors and of z."""
    P = {k: v.to(DEV).requires_grad_(True) for k, v in oracle.make_params(seed=5, stress=True, table_entries=64).items()
         if k.startswith('render_net.fc_') and '.' in k}
    g = torch.Generator().manual_seed(2)
    z = torch.randn(256, generator=g).to(DEV).requires_grad_(True)
    gw, gb = torch.randn(5, 256, 256, generator=g).to(DEV), torch.randn(5, 256, generator=g).to(DEV)
    res = {}
    for fused in ('1', '0'):
        monkeypatch.setenv('SDB200_FUSED_MOD', fused)
        for t in list(P.values()) + [z]:
            t.grad = None
        wh, bh = render.modulated_weights(P, z)
        assert (wh.grad_fn is not None) and (('Modulate' in type(wh.grad_fn).__name__) == (fused == '1'))
        ((wh * gw).sum() + (bh * gb).sum()).backward()
        res[fused] = (wh.detach().clone(), bh.detach().clone(), z.grad.clone(),
                      {k: v.grad.clone() for k, v in P.items() if v.grad is not None})
    a, b = res['1'], res['0']
    for x, y, name in ((a[0], b[0], 'wh'), (a[1], b[1], 'bh'), (a[2], b[2], 'dz')):
        assert float((x - y).abs().max()) <= 2e-5 * float(y.abs().max()) + 1e-7, name
    names = [k for k in b[3] if any(k.endswith(f) for f in ('.weight', '.weight_alpha', '.bias_alpha', '.weight_beta', '.bias_beta'))
             and k.split('.')[1] in ('fc_2', 'fc_3', 'fc_4', 'fc_5', 'fc_6')]
    assert len(names) == 25 and set(names) <= set(a[3])
    for k in names:
        assert float((a[3][k] - b[3][k]).abs().max()) <= 2e-5 * float(b[3][k].abs().max()) + 1e-7, k


@pytest.mark.parametrize('betas', [(0.0, 0.999), (0.9, 0.999)])
def test_fused_adam_step_matches_torch_adam(betas):
    """f2: sdb_adam_step == torch.optim.Adam (reference: trainer.py:297-323, scenedreamer_train.yaml:36-61) over several
    steps with the sparse gradients a hash table sees (most rows exactly zero); parameters AND optimizer state."""
    from scenedreamer_b200 import optim
    g = torch.Generator().manual_seed(0)
    rows = 50000
    p0 = (torch.rand(rows, 8, generator=g) * 2e-4 - 1e-4).to(DEV)
    pa = torch.nn.Parameter(p0.clone())
    ref = torch.optim.Adam([pa], lr=1e-4, eps=1e-7, betas=betas)
    pb = p0.clone()
    m, v = torch.zeros_like(pb), torch.zeros_like(pb)
    for t in range(1, 7):
        grad = torch.zeros(rows, 8, device=DEV)
        idx = torch.randint(0, rows, (rows // 20,), generator=g).to(DEV)
        grad[idx] = torch.randn(idx.numel(), 8, generator=g).to(DEV) * 10 ** float(torch.randint(-6, 1, (1,), generator=g))
        pa.grad = grad.clone()
        ref.step()
        optim.adam_step_(pb, grad, m, v, t, 1e-4, betas[0], betas[1], 1e-7)
    st = ref.state[pa]
    np.testing.assert_allclose(pb.cpu().numpy(), pa.detach().cpu().numpy(), rtol=2e-6, atol=1e-10)
    np.testing.assert_allclose(m.cpu().numpy(), st['exp_avg'].cpu().numpy(), rtol=2e-6, atol=1e-30)
    np.testing.assert_allclose(v.cpu().numpy(), st['exp_avg_sq'].cpu().numpy(), rtol=2e-6, atol=1e-30)


def test_adam_step_hook_takes_over_tagged_table_only():
    """Zero-edit route of f2: a plain torch.optim.Adam over (table, other); the tagged table is stepped by the fused kernel
    with the optimizer's own hyper-parameters and state, everything else by torch -- same result as untouched torch Adam."""
    from scenedreamer_b200 import optim
    g = torch.Generator().manual_seed(1)
    t0, o0 = torch.randn(4096, 8, generator=g).to(DEV), torch.randn(33, generator=g).to(DEV)
    table, other = torch.nn.Parameter(t0.clone()), torch.nn.Parameter(o0.clone())
    table_r, other_r = torch.nn.Parameter(t0.clone()), torch.nn.Parameter(o0.clone())
    kw = dict(lr=1e-3, eps=1e-7, betas=(0.0, 0.999))
    opt = torch.optim.Adam([{'params': [table], 'lr': 5e-4}, {'params': [other]}], **kw)
    opt_r = torch.optim.Adam([{'params': [table_r], 'lr': 5e-4}, {'params': [other_r]}], **kw)
    optim.tag_table(table)
    optim.install_step_hook()
    before = optim.stats['fused_steps']
    try:
        for _ in range(3):
            gt = torch.zeros_like(t0)
            gt[::7] = torch.randn(gt[::7].shape, generator=g).to(DEV)
            go = torch.randn(33, generator=g).to(DEV)
            table.grad, other.grad = gt.clone(), go.clone()
            table_r.grad, other_r.grad = gt.clone(), go.clone()
            opt.step()
            assert table.grad is None                                  # cleared by the hook: torch skipped it
            optim.remove_step_hook()
            opt_r.step()
            optim.install_step_hook()
    finally:
        optim.remove_step_hook()
    assert optim.stats['fused_steps'] == before + 3
    np.testing.assert_allclose(table.detach().cpu().numpy(), table_r.detach().cpu().numpy(), rtol=2e-6, atol=1e-9)
    assert torch.equal(other, other_r)
    assert float(opt.state[table]['step']) == 3.0 and set(opt.state[table]) == {'step', 'exp_avg', 'exp_avg_sq'}
    sd = opt.state_dict()                                              # interchangeable with a plain Adam
    opt_r.load_state_dict(sd)


def test_c5_size_gradients_vs_unfused_composition(golden_ops):
    """BASELINE C5 size: one 262x262 view, 24 samples/ray, stratified sampling (record 6.9 GB, workspace 7.1 GB).  The fused
    forward(record) + backward against the UNFUSED composition on the same GPU (torch fp32 autograd for MLP / compositing / sky
    on cuBLAS + the reference's own GridEncoder autograd.Function over the stand-alone grid kernels): output and every gradient."""
    import sys
    import bench_train
    from oracle import refgen
    ref_py = refgen.reference_python_root()
    if ref_py is None:
        pytest.skip('reference Python not staged (gridencoder package)')
    for pth in (os.path.join(ROOT, 'dropin'), ref_py):
        if pth not in sys.path:
            sys.path.append(pth)
    from gridencoder import GridEncoder
    world = synth.SyntheticVoxelWorld(1024, 3407)
    pose = synth.eval_camera_poses(world, maxstep=40, pattern=0)[5]
    o, d, u, f, c, res = synth.frame_camera(world, pose, (256, 256), 6)
    vid, dep, rd = ops.ray_voxel_intersection_perspective(world.voxel_t.to(DEV), o, d, u, f, c, res, 6)
    vid, dep, rd, ori = vid.unsqueeze(0), dep.unsqueeze(0), rd.unsqueeze(0), o.unsqueeze(0).to(DEV)
    P0 = oracle.make_params(seed=3, stress=True)
    g = torch.Generator().manual_seed(8888)
    z0 = oracle.style_mlp(torch.randn(1, 128, generator=g), P0)
    genc0 = torch.tanh(torch.randn(1, 2, generator=g))
    lut = render.reduced_label_lut(golden_ops['mc2reduced_lut']).to(DEV)
    _, pls = oracle.grid_offsets()
    H = W = 262
    uni = torch.rand(1, H, W, 25, 1, generator=g).to(DEV)
    G = torch.randn(1, H, W, 64, generator=g).to(DEV)
    vdims = [float(v) for v in world.voxel_t.shape]

    def leaves():
        P = {k: v.to(DEV).clone().requires_grad_(True) for k, v in P0.items()}
        return P, z0.to(DEV).clone().requires_grad_(True), genc0.to(DEV).clone().requires_grad_(True)
    P, z, genc = leaves()
    out = render.render_rays_train(P, vid, dep, rd, ori, z, genc, vdims, lut, pls, num_samples=24, uniforms=uni)
    (out['net_out'] * G).sum().backward()
    Pc, zc, gc = leaves()
    ge = GridEncoder(input_dim=5, num_levels=16, level_dim=8, base_resolution=16, log2_hashmap_size=19, desired_resolution=2048).to(DEV)
    ge.embeddings = torch.nn.Parameter(Pc['hash_encoder.embeddings'].detach().clone())
    ref_out = bench_train.composition_step(Pc, ge, vid, dep, rd, ori, zc, gc, vdims, lut, uni, G)
    Pc['hash_encoder.embeddings'].grad = ge.embeddings.grad
    torch.cuda.synchronize()
    e_out = float((out['net_out'].detach() - ref_out.detach()).abs().max())
    print('C5 size (262x262x24): forward max|fused - composition| %.3e' % e_out)
    assert e_out <= 1e-3
    worst = 0.0
    for name in list(P0.keys()) + ['z', 'global_enc']:
        a = (z.grad if name == 'z' else genc.grad if name == 'global_enc' else P[name].grad)
        b = (zc.grad if name == 'z' else gc.grad if name == 'global_enc' else Pc[name].grad)
        if name.startswith('style_net') or b is None:
            continue
        rel = float((a.double() - b.double()).norm() / (b.double().norm() + 1e-30))
        worst = max(worst, rel)
        assert rel <= 1e-2, (name, rel)
    print('C5 size: worst parameter-gradient rel-L2 vs the unfused composition %.3e' % worst)
    render.clear_scratch()
