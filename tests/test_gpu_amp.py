"""The fused per-pixel path under torch.autocast: the single-pass fp16 recording forward (precision 0) and the generator hook
that routes AMP calls onto it (integration.precision_for).

  * the precision-0 recording forward computes what the precision-0 inference kernel computes;
  * every stage of the (unchanged, bf16 x3) backward holds its DESIGN.md section 4 bound on a record the precision-0
    forward wrote (tests/test_gpu_train_stages.py run with the fp16 x1 pack and params);
  * render_rays_train at precision 0 against the CPU oracle under torch.autograd, and against the unfused composition
    under torch.autocast where the reference's gridencoder is staged;
  * the real Generator under autocast stays on the fused kernels, with the reference's output dtypes, and trains under
    torch.amp.GradScaler, which still skips a step whose gradients hold an inf.
Bounds are at most 4x the worst value measured on an NVIDIA H100 80GB HBM3 (power limit 700 W); DESIGN.md section 4."""
import ctypes

import pytest
import torch

import oracle
import test_gpu_train_stages as stages
from scenedreamer_b200 import _lib, integration, optim, render
from test_gpu_train import GRAD_KEYS, device_level_scales, make_scene
from test_gpu_train_stages import base  # noqa: F401  (module fixture)
from test_gpu_train_views import PARAMS, _rel, generator  # noqa: F401  (module fixture)

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1800)]
DEV = 'cuda:0'
NET_OUT_TOL = 1e-2            # max-abs budget of one fp16 pass (DESIGN.md section 4)
GRAD_TOL = 0.5                # render_rays_train at precision 0 vs the oracle, rel-L2 per gradient tensor (worst measured
                              # 0.225, fc_sigma.bias; the unfused composition under autocast: 0.276 on the same tensor)
GEN_GRAD_TOL = 0.35           # Generator under autocast, fused vs SDB200_FUSED=0, rel-L2 per parameter (worst measured 9.4e-2,
                              # hash_encoder.embeddings; 3e-3 .. 1.8e-2 on the others)
DSIG_DW_TERMS = 0.9           # dsig32 in units of 2^-24 x the _composite_ref_dw_terms scale (worst measured 0.234)
VS_COMPOSITION = 2.0          # fused distance to the oracle <= this x the unfused composition's own under autocast
AMP = dict(device_type='cuda', dtype=torch.float16)


def test_fp16_train_forward_equals_inference_forward(golden_ops):
    sc = make_scene()
    P = {k: v.to(DEV) for k, v in oracle.make_params(seed=3, stress=True).items()}
    g = torch.Generator().manual_seed(1)
    z = oracle.style_mlp(torch.randn(1, 128, generator=g), {k: v.cpu() for k, v in P.items()}).to(DEV)
    genc = torch.tanh(torch.randn(1, 2, generator=g)).to(DEV)
    lut = render.reduced_label_lut(golden_ops['mc2reduced_lut'], 0, 3)
    _, pls = oracle.grid_offsets()
    args = (P, sc['vid'], sc['dep'], sc['rd'], sc['o'].unsqueeze(0), z, genc, list(sc['world'].voxel_t.shape), lut, pls)
    with torch.no_grad():
        tr = render.render_rays_train(*args, precision=render.PRECISION_FP16)
        tr3 = render.render_rays_train(*args)
    r = render.FusedPerPixelRenderer(P, sc['world'].voxel_t.shape, lut, pls, precision=render.PRECISION_FP16)
    r.early_stop = 0
    # the recording path's sky branch is fp16 x3 in both modes: hand it to the inference kernel so that the MLP is compared
    inf = r.forward(sc['vid'], sc['dep'], sc['rd'], sc['o'].unsqueeze(0), z, genc, want_samples=True, sky=tr['sky'],
                    sky_avg=tr['sky_avg'])
    torch.cuda.synchronize()
    for k in ('depth', 'total_weight', 'weights', 'rand_depth'):
        assert torch.equal(tr[k], inf[k]), k
    e = float((tr['net_out'] - inf['net_out']).abs().max())
    e3 = float((tr['net_out'] - tr3['net_out']).abs().max())
    print('precision 0 recording vs inference net_out max abs %.3e; vs the fp16 x3 recording forward %.3e' % (e, e3))
    assert e <= 1e-5
    assert e3 > 0.0, 'the precision-0 recording forward computed the fp16 x3 result: the mode did not take effect'


class _Fp16Lib:
    """The library with every render MLP pack made at precision 0 (what a precision-0 caller hands the recording forward)."""

    def __init__(self, L):
        self._L, self.seen = L, set()

    def __getattr__(self, name):
        return getattr(self._L, name)

    def sdb_mlp_pack_bytes(self, precision):
        return self._L.sdb_mlp_pack_bytes(render.PRECISION_FP16)

    def sdb_pack_mlp(self, *a):
        return self._L.sdb_pack_mlp(*a[:10], render.PRECISION_FP16, *a[11:])

    def sdb_render_rays_train_forward(self, prm, record, stream):
        self.seen.add(prm._obj.precision)
        return self._L.sdb_render_rays_train_forward(prm, record, stream)


_composite_ref = stages.tr.composite_backward_ref


def _dw_parts(sig, nds, c, live, g, sky_used):
    """Float64 pieces of dL/dw_s = g . (clamp(c_s) + 1) - g . (clamp(sky) + 1): (dw, dot, gsky, dw_mag), dw_mag = the sum
    of the magnitudes of both 64-term dot products, which bounds the kernel's fp32 evaluation of each of them."""
    c, g, sky_used = c.double(), g.double(), sky_used.double()
    livef = live.double()[:, None]
    dot = (g[:, None, :] * (c.clamp(-1, 1) + 1)).sum(-1)
    gsky = (g * (sky_used.clamp(-1, 1) + 1)).sum(-1)[:, None]
    dw_mag = ((g.abs()[:, None, :] * (c.clamp(-1, 1) + 1)).sum(-1) + (g.abs() * (sky_used.clamp(-1, 1) + 1)).sum(-1)[:, None])
    return (dot - gsky) * livef, dot, gsky, dw_mag * livef


def _composite_ref_dw_terms(sig, nds, c, live, g, sky_used):
    """tests/_train_record.composite_backward_ref with the magnitude of dL/dw_s taken from its two dot products instead of
    from |dL/dw_s|.  The kernel forms dw_s = dot - gsky in fp32 and each dot product errs by a few 2^-24 of its own
    magnitude: where the two nearly cancel, |dw_s| is far below that error and the scale of the other stages' model
    (|dw|) under-counts it.  Only dsig32 (and the dsig of every earlier sample of the ray, through the suffix sums) reads
    dw; the other scales are unchanged."""
    ref, (sdc, _, sdsky) = _composite_ref(sig, nds, c, live, g, sky_used)
    sig_, nds_ = sig.double(), nds.double()
    e = sig_.clamp(min=0) * nds_
    E = torch.cumsum(e, 1) - e
    T = torch.exp(-E) * live.double()[:, None]
    Tb = T * (1 + torch.arange(1, e.shape[1] + 1, dtype=torch.float64, device=e.device) * E)
    _, _, _, dw_mag = _dw_parts(sig, nds, c, live, g, sky_used)
    suffix = lambda v: v.flip(1).cumsum(1).flip(1) - v
    sdsig = (dw_mag * Tb * torch.exp(-e) + suffix(dw_mag * Tb)) * (sig_ > 0).double() * nds_
    return ref, (sdc, sdsig, sdsky)


def _dsig_diagnosis(rec, i, G, sky, sky_avg, ws):
    """The slot of view i where dsig32 is worst against the |dw| scale, and its error against both scales."""
    S, HW = rec.S, rec.H * rec.W
    first, count = rec.views[i]
    if count == 0:
        return None
    sl, rs = rec.view_slots(i), slice(first * 128, (first + count) * 128)
    ray, _ = rec.rays(i)
    ray = ray.reshape(-1)
    live, nosky, valid = rec.live[rs], rec.nosky[rs], rec.valid[rs]
    Gi, skyi = G[i].reshape(HW, 64).double(), sky[i].reshape(HW, 64).double()
    g = Gi[ray] * valid[:, None]
    sky_used = torch.where(nosky[:, None], sky_avg[i].double()[None, :], skyi[ray] * valid[:, None])
    per_ray = lambda t, *tail: t.reshape(count, S, 128, *tail).transpose(1, 2).reshape(count * 128, S, *tail)
    args = (per_ray(rec.sig[sl]), per_ray(rec.nds[sl]), per_ray(rec.c[sl], 64), live, g, sky_used)
    (_, dsig, _), (_, s_old, _) = _composite_ref(*args)
    _, (_, s_new, _) = _composite_ref_dw_terms(*args)
    dw, dot, gsky, dw_mag = _dw_parts(*args)
    err = (per_ray(ws.dsig32[:count * S * 128]).double() - dsig).abs()
    r_old, r_new = err / (stages.EPS * s_old + stages.tr.FP32_TINY), err / (stages.EPS * s_new + stages.tr.FP32_TINY)
    k = int(torch.argmax(r_old))
    r, t = divmod(k, S)
    cancel = float((dw_mag[r] / (dw[r].abs() + stages.tr.FP32_TINY)).max())
    return dict(ray=r, sample=t, err_old_scale=float(r_old.max()), err_new_scale_same_slot=float(r_new.reshape(-1)[k]),
                err_new_scale=float(r_new.max()), dw=float(dw[r, t]), dot=float(dot[r, t]), gsky=float(gsky[r, 0]),
                dw_mag=float(dw_mag[r, t]), worst_cancellation_on_ray=cancel)


@pytest.mark.parametrize('case', list(stages.CASES))
def test_fp16_record_backward_stages(base, golden_ops, case, monkeypatch):  # noqa: F811
    """Every stage check of tests/test_gpu_train_stages.py, at its DESIGN.md section 4 bound, on a record the precision-0
    forward wrote, except dsig32, which is normalised by the dot-product magnitudes of dL/dw (_composite_ref_dw_terms) and
    held to DSIG_DW_TERMS of that scale.  Against the |dw| scale a precision-0 record of views_empty_first gave 3771 x
    2^-24 (bound 350) at one slot where g . (clamp(c) + 1) = -8.859053 and g . (clamp(sky) + 1) = -8.859057 cancel to
    dw = 4.2e-6 (2.4e7 times below the magnitude of its terms): the fp32 sum is as exact as its terms allow, |dw| was the
    wrong yardstick there, and an fp16 x3 record can meet such a near-tie just as well.  The worst slot of each view is
    printed with its error against both scales."""
    lib = _Fp16Lib(_lib.lib())
    monkeypatch.setattr(_lib, 'lib', lambda: lib)
    fill = render._fill_render_params
    monkeypatch.setattr(render, '_fill_render_params', lambda *a, **k: fill(*a, **dict(k, precision=render.PRECISION_FP16)))
    monkeypatch.setattr(stages.tr, 'composite_backward_ref', _composite_ref_dw_terms)

    class Report(stages.Report):
        def check(self, stage, err, bound, sens=None):
            super().check(stage, err, DSIG_DW_TERMS if stage == 'dsig32' else bound, sens)
    monkeypatch.setattr(stages, 'Report', Report)
    checks = stages._composite_checks

    def composite_checks(rep, rec, i, G, sky, sky_avg, cam_x, gr, ws):
        checks(rep, rec, i, G, sky, sky_avg, cam_x, gr, ws)
        if ws is not None:
            print('  %-10s dsig32 worst slot of view %d: %s' % (rep.case, i, _dsig_diagnosis(rec, i, G, sky, sky_avg, ws)))
    monkeypatch.setattr(stages, '_composite_checks', composite_checks)
    stages.test_backward_stages_vs_float64(base, golden_ops, case)
    assert lib.seen == {render.PRECISION_FP16}


def test_fp16_render_rays_train_vs_oracle(golden_ops):
    import os
    import sys
    import bench_train
    from oracle import refgen
    sc = make_scene()
    S = 24
    P0 = oracle.make_params(seed=21, stress=True)
    g = torch.Generator().manual_seed(8888)
    z0 = oracle.style_mlp(torch.randn(1, 128, generator=g), P0)
    genc0 = torch.tanh(torch.randn(1, 2, generator=g))
    N, H, W = sc['vid'].shape[:3]
    uni = torch.rand(N, H, W, S + 1, 1, generator=torch.Generator().manual_seed(5))
    G = torch.randn(N, H, W, 64, generator=torch.Generator().manual_seed(9))
    lut_raw = torch.from_numpy(golden_ops['mc2reduced_lut'])
    offsets, pls = oracle.grid_offsets()
    vdims = list(sc['world'].voxel_t.shape)
    leaf = lambda dev: ({k: v.detach().clone().to(dev).requires_grad_(True) for k, v in P0.items()},
                        z0.clone().to(dev).requires_grad_(True), genc0.clone().to(dev).requires_grad_(True))

    Pc, zc, gc = leaf('cpu')
    ref = oracle.forward_perpix_autograd(Pc, sc['vid'].cpu(), sc['dep'].cpu(), sc['rd'].cpu(), sc['o'].unsqueeze(0), zc, gc, vdims,
                                         lut_raw, offsets, pls, num_samples=S, deterministic=False, uniforms=uni,
                                         level_scales=device_level_scales(16, pls, 16))
    (ref * G).sum().backward()
    grads = lambda P, z, gg: dict({k: P[k].grad for k in GRAD_KEYS}, z=z.grad, global_enc=gg.grad)
    rg = grads(Pc, zc, gc)

    Pg, zg, gg = leaf(DEV)
    lut = render.reduced_label_lut(golden_ops['mc2reduced_lut'], 0, 3)
    with torch.autocast(**AMP):
        out = render.render_rays_train(Pg, sc['vid'], sc['dep'], sc['rd'], sc['o'].unsqueeze(0), zg, gg, vdims, lut, pls,
                                       num_samples=S, uniforms=uni.to(DEV), precision=render.PRECISION_FP16)
    assert out['net_out'].dtype == torch.float32
    (out['net_out'] * G.to(DEV)).sum().backward()
    fg = grads(Pg, zg, gg)
    ferr = float((out['net_out'].detach().cpu() - ref.detach()).abs().max())

    comp = None
    if refgen.reference_python_root() is not None:
        for pth in (os.path.join(bench_train.ROOT, 'dropin'), refgen.reference_python_root()):
            if pth not in sys.path:
                sys.path.append(pth)
        from gridencoder import GridEncoder
        Pr, zr, gr = leaf(DEV)
        ge = GridEncoder(input_dim=5, num_levels=16, level_dim=8, base_resolution=16, log2_hashmap_size=19,
                         desired_resolution=2048).to(DEV)
        ge.embeddings = torch.nn.Parameter(Pr['hash_encoder.embeddings'].detach().clone())
        with torch.autocast(**AMP):
            cout = bench_train.composition_step(Pr, ge, sc['vid'], sc['dep'], sc['rd'], sc['o'].unsqueeze(0).to(DEV), zr, gr, vdims,
                                                lut.to(DEV), uni.to(DEV), G.to(DEV))
        Pr['hash_encoder.embeddings'].grad = ge.embeddings.grad
        comp = (float((cout.detach().float().cpu() - ref.detach()).abs().max()), grads(Pr, zr, gr))
    torch.cuda.synchronize()
    print('net_out max abs vs oracle: fused precision 0 %.3e%s' % (
        ferr, '' if comp is None else ', unfused composition under autocast %.3e' % comp[0]))
    assert ferr <= NET_OUT_TOL
    if comp is not None:
        assert ferr <= VS_COMPOSITION * comp[0]
    worst = 0.0
    for k in rg:
        assert fg[k] is not None, 'no gradient reached %s' % k
        e = _rel(fg[k].cpu(), rg[k])
        worst = max(worst, e)
        ec = None if comp is None else _rel(comp[1][k].float().cpu(), rg[k])
        print('%-36s rel-L2 to the oracle: fused %.3e%s' % (k, e, '' if ec is None else ', composition under autocast %.3e' % ec))
        if ec is not None:
            assert e <= VS_COMPOSITION * ec, (k, e, ec)
    assert worst <= GRAD_TOL, worst


# ---- the real Generator through the zero-edit hook, under autocast ----------------------------------------------------
def _data(gen, n_views):
    from scenedreamer_b200 import ops
    import imaginaire.model_utils.gancraft.camctl as camctl
    ctl = camctl.EvalCameraController(gen.voxel, maxstep=8, pattern=0, cam_ang=72)
    H = W = 64 + gen.pad
    vids, deps, rds, oris = [], [], [], []
    for k in range(n_views):
        pose = ctl[1 + 2 * k]
        vid, dep, rd = ops.ray_voxel_intersection_perspective(gen.voxel.voxel_t, pose[0], pose[1], pose[2], pose[3] * (W - 1),
                                                              [(H - 1) / 2, (W - 1) / 2], [H, W], 6)
        vids.append(vid), deps.append(dep), rds.append(rd), oris.append(pose[0].to(DEV))
    return dict(images=torch.zeros(n_views, 3, 64, 64, device=DEV), voxel_id=torch.stack(vids), depth2=torch.stack(deps),
                raydirs=torch.stack(rds), cam_ori_t=torch.stack(oris))


@pytest.fixture
def amp_gen(generator, monkeypatch):  # noqa: F811
    """The generator with PARAMS trainable, its _forward_perpix wrapped to note the dtypes of the tuple entries callers use
    (0, 2, 3, 4) and, when `inject` is set, to put an inf into dL/d net_out at one pixel."""
    gen = generator
    cls = type(gen)
    fused = cls.__dict__['_forward_perpix']
    seen = {'dtypes': [], 'inject': False}

    def inf_at_one_pixel(g):
        g = g.clone()
        g[0, g.shape[1] // 2, g.shape[2] // 2] = float('inf')
        return g

    def wrapped(self, *a):
        out = fused(self, *a)
        seen['dtypes'].append(tuple(out[i].dtype for i in (0, 2, 3, 4)))
        if seen['inject'] and out[0].requires_grad:
            out[0].register_hook(inf_at_one_pixel)
        return out
    monkeypatch.setattr(cls, '_forward_perpix', wrapped)
    mods = dict(gen.named_parameters())
    params = [mods[k] for k in PARAMS]
    saved = [q.detach().clone() for q in params]
    for q in params:
        q.requires_grad_(True)
        q.grad = None
    if hasattr(gen, 'sky_avg'):
        del gen.sky_avg
    gen.coarse_deterministic_sampling = False
    gen.num_samples = 24
    try:
        yield gen, params, seen
    finally:
        with torch.no_grad():
            for q, s in zip(params, saved):
                q.copy_(s)
                q.requires_grad_(False)
                q.grad = None


def _stats(gen):
    st = integration._state(gen).stats
    return {k: st[k] for k in ('train_calls', 'reference_calls', 'fused_calls', 'cnn_reference_calls')}


def _delta(gen, before):
    return {k: v - before[k] for k, v in _stats(gen).items()}


def _amp_step(gen, params, n_views, monkeypatch, env):
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    try:
        data = _data(gen, n_views)
        before = _stats(gen)
        torch.manual_seed(5)
        with torch.autocast(**AMP):
            out = gen(data, random_style=True)
            loss = out['fake_images'].float().square().mean()
        loss.backward()
        torch.cuda.synchronize()
        grads = {k: q.grad.clone() for k, q in zip(PARAMS, params)}
        for q in params:
            q.grad = None
        return grads, _delta(gen, before)
    finally:
        for k in env:
            monkeypatch.delenv(k)


def test_generator_under_autocast_stays_fused(amp_gen, monkeypatch):
    gen, params, seen = amp_gen
    res = {}
    for name, env in (('views', {'SDB200_TRAIN_VIEWS': '1'}), ('loop', {'SDB200_TRAIN_VIEWS': '0'}), ('reference', {'SDB200_FUSED': '0'})):
        seen['dtypes'].clear()
        # one view: the reference's own composition takes one scene code per ray batch (tests/test_gpu_train_views.py)
        grads, d = _amp_step(gen, params, 1, monkeypatch, env)
        res[name] = (grads, d, list(seen['dtypes']))
        print('%-9s hook stats %s, tuple dtypes %s' % (name, d, seen['dtypes']))
    for name in ('views', 'loop'):
        grads, d, dt = res[name]
        assert d['train_calls'] == 1 and d['reference_calls'] == 0, (name, d)
        assert d['cnn_reference_calls'] >= 1, (name, d)          # RenderCNN with gradients under autocast: the reference's
        assert dt == res['reference'][2], (name, dt, res['reference'][2])
        for k in PARAMS:
            assert bool(torch.isfinite(grads[k]).all()) and float(grads[k].abs().max()) > 0, (name, k)
            e = _rel(grads[k], res['reference'][0][k])
            print('%-9s %-32s rel-L2 to the SDB200_FUSED=0 arm under autocast %.3e' % (name, k, e))
            assert e <= GEN_GRAD_TOL, (name, k, e)
    assert res['reference'][1]['reference_calls'] == 1
    # no gradients: dis_update's generator call and inference under autocast take the precision-0 inference kernels
    before = _stats(gen)
    seen['dtypes'].clear()
    with torch.no_grad(), torch.autocast(**AMP):
        torch.manual_seed(5)
        gen(_data(gen, 1), random_style=True)
    d = _delta(gen, before)
    assert d['fused_calls'] == 1 and d['reference_calls'] == 0, d
    assert seen['dtypes'] and all(t == torch.float32 for t in seen['dtypes'][0])
    assert integration._state(gen).renderer.precision == render.PRECISION_FP16


def test_gradscaler_steps_and_skips(amp_gen, monkeypatch):
    gen, params, seen = amp_gen
    optim.install_step_hook()
    data = _data(gen, 1)
    results = {}
    for arm, env in (('fused', {}), ('reference', {'SDB200_FUSED': '0'})):
        for k, v in env.items():
            monkeypatch.setenv(k, v)
        opt = torch.optim.Adam(params, lr=1e-4, eps=1e-7, betas=(0.0, 0.999))
        scaler = torch.amp.GradScaler('cuda')
        start = [q.detach().clone() for q in params]
        fused0 = optim.stats['fused_steps']
        before = _stats(gen)

        def step():
            opt.zero_grad(set_to_none=True)
            with torch.autocast(**AMP):
                loss = gen(data, random_style=True)['fake_images'].float().square().mean()
            scaler.scale(loss).backward()
            scaler.step(opt)
            scaler.update()
        for _ in range(3):
            step()
        torch.cuda.synchronize()
        d = _delta(gen, before)
        fused_steps = optim.stats['fused_steps'] - fused0
        after3 = [q.detach().clone() for q in params]
        scale = scaler.get_scale()
        seen['inject'] = True
        try:
            step()
        finally:
            seen['inject'] = False
        torch.cuda.synchronize()
        unchanged = all(torch.equal(a, q.detach()) for a, q in zip(after3, params))
        results[arm] = (d, fused_steps, optim.stats['fused_steps'] - fused0 - fused_steps, unchanged, scaler.get_scale() < scale)
        print('%-9s hook stats %s, fused table Adam steps %d (+%d on the inf step), inf step skipped %s, scale lowered %s' % (
            (arm, d) + results[arm][1:]))
        for a, b, k in zip(start, after3, PARAMS):
            assert bool(torch.isfinite(b).all()), (arm, k)
            assert not torch.equal(a, b), (arm, k, 'did not change over three steps')
        with torch.no_grad():
            for q, s in zip(params, start):
                q.copy_(s)
        for k in env:
            monkeypatch.delenv(k)
    fd, fsteps, finf, fskip, flow = results['fused']
    assert fd['train_calls'] == 3 and fd['reference_calls'] == 0, fd
    assert fsteps == 3 and finf == 0                 # the table is stepped by the fused Adam hook, and not on the skipped step
    assert fskip and flow
    rd, _, _, rskip, rlow = results['reference']
    assert rd['reference_calls'] == 3 and rskip and rlow


def test_gradscaler_fused_adam_keeps_the_table():
    """Adam(fused=True) under GradScaler unscales and skips inside its own kernel, with the gradients still scaled when it is
    called: the table hook leaves a tagged table to it, so the table follows torch's fused Adam exactly and stays finite
    (and unchanged) on a step with an inf gradient."""
    g = torch.Generator().manual_seed(4)
    t0 = (torch.randn(4096, 8, generator=g) * 1e-2).to(DEV)
    w = torch.randn(4096, 8, generator=g).to(DEV)
    table, twin = optim.tag_table(torch.nn.Parameter(t0.clone())), torch.nn.Parameter(t0.clone())     # twin: not tagged
    kw = dict(lr=1e-3, eps=1e-7, betas=(0.0, 0.999), fused=True)
    arms = [(table, torch.optim.Adam([table], **kw), torch.amp.GradScaler('cuda')),
            (twin, torch.optim.Adam([twin], **kw), torch.amp.GradScaler('cuda'))]
    had_hook = optim._hook_handle is not None
    optim.install_step_hook()
    fused0 = optim.stats['fused_steps']
    try:
        for k in range(4):
            wk = w.clone()
            if k == 3:
                wk[7, 3] = float('inf')
            for t, opt, scaler in arms:
                before = t.detach().clone()
                opt.zero_grad(set_to_none=True)
                scaler.scale((t * wk).sum()).backward()
                scaler.step(opt)
                scaler.update()
                if k == 3:
                    assert torch.equal(t.detach(), before), 'a step with an inf gradient changed the parameter'
                else:
                    assert not torch.equal(t.detach(), before)
            torch.cuda.synchronize()
            assert torch.equal(table.detach(), twin.detach()), k
            st = arms[0][1].state[table]
            assert all(bool(torch.isfinite(v).all()) for v in (table, st['exp_avg'], st['exp_avg_sq'])), k
    finally:
        if not had_hook:
            optim.remove_step_hook()
    assert optim.stats['fused_steps'] == fused0
