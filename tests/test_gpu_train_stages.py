"""Each stage of the fused training backward (sdb_render_rays_train_forward + sdb_render_rays_backward_views) against a
float64 reference fed the library's own recorded inputs of that stage (tests/_train_record.py decodes them), over the
shapes the path accepts: S from 1 to 64, M 1 and 8, frames from one ray to several waves of work items, 15 labels, a
ground-level camera, all-sky and dense frames, and 3-view batches with an empty view.

The record, the workspace and every backward output start as NaN (0xFF bytes), and NaN follows the stratified
uniforms, so a value the pass does not write in this call, or a read past an input, fails the test instead of reading a
previous pass's data.  Per stage (each bound is at most 4x the worst error
measured on an NVIDIA H100 80GB HBM3, power limit 700 W, over all cases; every error is normalised elementwise and
2^-126 is added to every scale, since the kernels flush subnormals):
  compositing   dc32, dsig32, g_sky, g_sky_avg: |err| <= COMP * 2^-24 * scale, the scale being the same expression with
                every weight w_t replaced by a bound of its transmittance and every term by its magnitude (fp32 cancels
                in 1 - exp(-e), in dsig and in 1 - sum w).  Bound 350, measured 88.7 (dsig32, S = 64).  dc16 / dsig16 are
                bit-equal to round-to-nearest bf16 of the kernel's own dc32 / dsig32.
  chain         from the recorded dc32 / dsig32 / sign words and the fp32 weights: dx0 |err| <= DX0 * 2^-16 * (|dZ1| @ |W1|),
                bound 4, measured 1.06; dx0 rel-L2 <= 8e-5, measured 2.1e-5; every bf16 dZ within DZ * (1 bf16 ulp +
                2^-16 * the magnitude of its products), bound 1, measured 0.72.
  weights       g_w1ext, g_wh, g_wsig, g_wout: |err| <= WGRAD * 2^-24 * sum |dZ| |A| over the recorded bf16 tiles
                (bf16 x bf16 products are exact in fp32; only the accumulation errs).  Bound 280, measured 77.
                Rows 1..7 of g_wsig are exactly 0.
  table         dt3: |err| <= TABLE * 2^-24 * sum |w dx0|, bound 85, measured 25.6; g_table = the transpose of the
                pre-blend applied to dt3, through the adjoint identity <g_table, E> = sum <dx0, enc_E(x)> with the
                oracle's 5-D grid forward for two random tables E: |err| <= ADJ * 2^-24 * sum |dx0| enc_|E|(x), bound
                0.11, measured 0.031.
Every elementwise stage also reports the error its check would see if the reference lacked one ray at one step, one ray
or one 128-row item -- the one typical of where the gradient's mass lies -- and requires it to exceed the bound at least
10x: a bound too loose to see that fails the test.  The whole file takes about a minute on that GPU.
"""
import ctypes
import time

import numpy as np
import pytest
import torch

import _train_record as tr
import oracle
from scenedreamer_b200 import _lib, ops, render, synth

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1800)]
DEV = 'cuda:0'
EPS = 2.0 ** -24
COMP, DX0, DX0_L2, DZ, WGRAD, TABLE, ADJ = 350.0, 4.0, 8e-5, 1.0, 280.0, 85.0, 0.11
BF16X3 = 2.0 ** -16          # relative error of one product split into bf16 hi + lo parts (three passes)
SENSITIVITY = 10.0


@pytest.fixture(scope='module')
def base():
    """One 160x224 frame of the synthetic world (8 voxel hits per ray); cases crop windows out of it."""
    world = synth.SyntheticVoxelWorld(size=128, seed=7)
    pose = synth.eval_camera_poses(world, maxstep=8, pattern=0)[1]
    o, d, u, f, c, res = synth.frame_camera(world, pose, resolution_hw=(156, 220), pad=4)
    vid, dep, rd = ops.ray_voxel_intersection_perspective(world.voxel_t.to(DEV), o, d, u, f, c, res, 8)
    return dict(world=world, o=o, vid=vid, dep=dep, rd=rd, ids=torch.unique(vid.cpu()).tolist())


def _frame(b, y0, x0, h, w, M=8, sky_cols=0, empty=False):
    """[H, W, M, 1] / [2, H, W, M, 1] / [H, W, 1, 3] window of the base frame; the first `sky_cols` columns hit nothing."""
    vid = b['vid'][y0:y0 + h, x0:x0 + w, :M].clone()
    dep = b['dep'][:, y0:y0 + h, x0:x0 + w, :M].contiguous()
    rd = b['rd'][y0:y0 + h, x0:x0 + w].contiguous()
    if sky_cols:
        vid[:, :sky_cols] = 0
    if empty:
        vid.zero_()
    return vid.contiguous(), dep, rd


# id: (windows [(y0, x0, h, w, sky_cols, empty)], S, M, options)
CASES = {
    'ray1_S1': ([(80, 100, 1, 1, 0, False)], 1, 8, {}),
    'tile8x16_S64_M8': ([(64, 96, 8, 16, 3, False)], 64, 8, {}),
    '9x17_S33_M1_strat': ([(70, 50, 9, 17, 0, False)], 33, 1, dict(stratified=True)),
    '36x52_S64_waves': ([(40, 60, 36, 52, 0, False)], 64, 8, {}),
    'wide8x220_S32': ([(90, 2, 8, 220, 5, False)], 32, 8, {}),
    'tall150x9_S31_strat': ([(4, 120, 150, 9, 0, False)], 31, 8, dict(stratified=True)),
    'labels15_S12': ([(40, 60, 36, 52, 6, False)], 12, 8, dict(nlabels=15)),
    'ground_cam_S33': ([(40, 60, 24, 40, 20, False)], 33, 8, dict(ground=True)),
    'all_sky_S24': ([(40, 60, 20, 36, 0, True)], 24, 8, dict(ground=True)),
    'dense_S33': ([(40, 60, 24, 40, 0, False)], 33, 8, dict(sigma_bias=150.0)),
    'negative_sigma_S24': ([(40, 60, 24, 40, 0, False)], 24, 8, dict(sigma_bias=-1e4)),
    'views_empty_first': ([(0, 0, 20, 36, 0, True), (40, 60, 20, 36, 4, False), (90, 120, 20, 36, 0, False)], 33, 8, {}),
    'views_empty_middle': ([(40, 60, 20, 36, 0, False), (0, 0, 20, 36, 0, True), (90, 120, 20, 36, 0, False)], 24, 8,
                           dict(stratified=True)),
    'views_empty_last': ([(40, 60, 20, 36, 0, False), (90, 120, 20, 36, 6, False), (0, 0, 20, 36, 0, True)], 64, 8, {}),
}


def _weights(seed, nlabels, sigma_bias, n_views):
    P = {k: v.to(DEV) for k, v in oracle.make_params(seed=seed, stress=True, nlabels=nlabels).items()}
    if sigma_bias is not None:
        P['render_net.fc_sigma.bias'] = torch.full((1,), float(sigma_bias), device=DEV)
    g = torch.Generator().manual_seed(seed + 1)
    z = oracle.style_mlp(torch.randn(n_views, 128, generator=g), {k: v.cpu() for k, v in P.items()}).to(DEV)
    genc = torch.tanh(torch.randn(1, 2, generator=g)).to(DEV)
    with torch.no_grad():
        mods = [render.modulated_weights(P, z[i]) for i in range(n_views)]
    W = dict(w1=P['render_net.fc_1.weight'].contiguous(), b1=P['render_net.fc_1.bias'].contiguous(),
             emb=P['render_net.fc_m_a.weight'].t().contiguous(), wsig=P['render_net.fc_sigma.weight'].reshape(-1).contiguous(),
             bsig=P['render_net.fc_sigma.bias'].reshape(-1).contiguous(), wout=P['render_net.fc_out_c.weight'].contiguous(),
             bout=P['render_net.fc_out_c.bias'].contiguous(), wh=torch.stack([m[0] for m in mods]).contiguous(),
             bh=torch.stack([m[1] for m in mods]).contiguous(), table=P['hash_encoder.embeddings'].contiguous())
    return W, genc


def _run(W, genc, frames, ori, lut, S, uni, sky, sky_avg, G, views=None):
    """One recorded pass and its backward through the C ABI over test-owned, NaN-filled buffers; `views` selects a
    subset of the batch (the same per-view weights)."""
    Lb = _lib.lib()
    views = list(range(len(frames))) if views is None else views
    vid = torch.stack([frames[i][0] for i in views]).contiguous()
    dep = torch.stack([frames[i][1] for i in views]).contiguous()
    rd = torch.stack([frames[i][2] for i in views]).contiguous()
    N, H, W_, M = vid.shape[:4]
    st = render._stream(DEV)
    _, pls = oracle.grid_offsets()
    pack = torch.empty(N, int(Lb.sdb_mlp_pack_bytes(2)), dtype=torch.uint8, device=DEV)
    bpack = torch.empty(N, int(Lb.sdb_mlp_backward_pack_bytes()), dtype=torch.uint8, device=DEV)
    p = render._ptr
    for j, i in enumerate(views):
        _lib.check(Lb.sdb_pack_mlp(p(W['w1']), p(W['b1']), p(W['emb']), int(W['emb'].shape[0]), p(W['wh'][i]), p(W['bh'][i]),
                                   p(W['wsig']), p(W['bsig']), p(W['wout']), p(W['bout']), 2, p(pack[j]), st), 'pack')
        _lib.check(Lb.sdb_pack_mlp_backward(p(W['w1']), p(W['wh'][i]), p(W['wsig']), p(W['wout']), p(bpack[j]), st), 'bpack')
    genc_n = genc.reshape(1, 2).expand(N, 2).contiguous()
    table3 = render.preblend_table(W['table'], genc_n[0], 19, pls, 16, 16)
    nan = lambda *shape: torch.full(shape, float('nan'), device=DEV)
    out = dict(net_out=nan(N, H, W_, 64), depth=nan(N, H, W_), tw=nan(N, H, W_), wts=nan(N, H, W_, S, 1), rdp=nan(N, H, W_, S, 1))
    ws = torch.empty(int(Lb.sdb_render_workspace_bytes(N, H, W_)), dtype=torch.uint8, device=DEV)
    lay = tr.layout(Lb, N, H, W_, S)
    record = torch.full((lay['record_bytes'],), 255, dtype=torch.uint8, device=DEV)
    prm, keep = render._RenderParams(), []
    cam = ori[views].to(DEV).contiguous()
    u = None
    if uni is not None:                     # followed by NaN: a read past the end of the uniforms shows in the outputs
        buf = torch.full((2 * uni[views].numel(),), float('nan'), device=DEV)
        u = buf[:uni[views].numel()].view(uni[views].shape)
        u.copy_(uni[views])
    sky_v, sky_avg_v = sky[views].contiguous(), sky_avg[views].contiguous()      # read again by the backward
    render._fill_render_params(prm, keep, vid, dep, rd, cam, genc_n, list(frames[0][3]), lut, pack, sky_v, sky_avg_v,
                               table3=table3, S=S, sample_depth=3.0, dists_scale=0.25, uniforms=u, precision=2,
                               per_level_scale=pls, base_res=16, log2_T=19, L=16, net_out=out['net_out'],
                               depth=out['depth'], tw=out['tw'], wts=out['wts'], rdp=out['rdp'], ws=ws)
    _lib.check(Lb.sdb_render_rays_train_forward(ctypes.byref(prm), p(record), st), 'train forward')
    gr = dict(table=torch.full_like(W['table'], float('nan')), genc=nan(2), w1ext=nan(N, 256, 144), wh=nan(N, 5, 256, 272),
              wsig=nan(N, 8, 272), wout=nan(N, 64, 272), sky=nan(N, H, W_, 64), sky_avg=nan(N, 64))
    wsb = torch.full((lay['workspace_bytes'],), 255, dtype=torch.uint8, device=DEV)
    Gv = G[views].contiguous()
    vg = render._RenderViewGrads()
    g = vg.g
    g.d_grad_net_out, g.d_bwd_pack, g.bwd_pack_stride = p(Gv), p(bpack), int(bpack.stride(0))
    g.d_table = p(W['table'])
    g.d_grad_table, g.d_grad_global_enc, g.d_grad_w1ext = p(gr['table']), p(gr['genc']), p(gr['w1ext'])
    g.d_grad_wh, g.d_grad_wsig, g.d_grad_wout = p(gr['wh']), p(gr['wsig']), p(gr['wout'])
    g.d_grad_sky, g.d_grad_sky_avg, g.d_workspace = p(gr['sky']), p(gr['sky_avg']), p(wsb)
    vg.w1ext_stride, vg.wh_stride, vg.wsig_stride = gr['w1ext'].stride(0), gr['wh'].stride(0), gr['wsig'].stride(0)
    vg.wout_stride, vg.sky_avg_stride = gr['wout'].stride(0), gr['sky_avg'].stride(0)
    _lib.check(Lb.sdb_render_rays_backward_views(ctypes.byref(prm), p(record), ctypes.byref(vg), st), 'backward')
    torch.cuda.synchronize()
    rec = tr.Record(lay, record, N, H, W_, S, wsb)
    bad = [k for k, v in list(out.items()) + list(gr.items()) if not bool(torch.isfinite(v).all())]
    assert not bad, 'outputs %s not (fully) written or not finite; views %s; %s' % (bad, rec.views, _nonfinite(rec, gr))
    return rec, out, gr


def _nonfinite(rec, gr):
    """Where the record / workspace of a pass holds non-finite values (by 128-row item) and which gradient rows / columns do."""
    n = rec.n_live * rec.S * 128
    wn = max(c for _, c in rec.views) * rec.S * 128
    arrays = [('x0', rec.x0), ('x3', rec.x3), ('sig', rec.sig), ('nds', rec.nds), ('c', rec.c)]
    arrays += [('act%d' % k, a) for k, a in enumerate(rec.act)]
    arrays += [('ws.dz%d' % k, d[:wn]) for k, d in enumerate(rec.dz)]
    arrays += [('ws.dc32', rec.dc32[:wn]), ('ws.dc16', rec.dc16[:wn]), ('ws.dsig32', rec.dsig32[:wn]),
               ('ws.dsig16', rec.dsig16[:wn]), ('ws.dx0', rec.dx0[:wn])]
    msg = ['live slots %d' % n]
    for name, a in arrays:
        bad = ~torch.isfinite(a.float().reshape(a.shape[0], -1))
        if bool(bad.any()):
            rows = torch.nonzero(bad.any(1)).reshape(-1)
            cols = torch.nonzero(bad.any(0)).reshape(-1)
            msg.append('%s: %d slots in items %s, columns %s, values %s' % (
                name, rows.numel(), sorted(set((rows // 128).tolist()))[:12], cols.tolist()[:20],
                a.float().reshape(a.shape[0], -1)[bad][:4].tolist()))
    for name in ('w1ext', 'wh', 'wsig', 'wout'):
        bad = ~torch.isfinite(gr[name])
        if bool(bad.any()):
            msg.append('g_%s: %d non-finite of %d, rows %s, columns %s' % (
                name, int(bad.sum()), bad.numel(), torch.nonzero(bad.any(-1).reshape(-1)).reshape(-1).tolist()[:12],
                torch.nonzero(bad.reshape(-1, bad.shape[-1]).any(0)).reshape(-1).tolist()[:12]))
    return '; '.join(msg)


class Report:
    """Prints and checks every stage of a case; the case fails at its end with the list of every stage that failed."""

    def __init__(self, case):
        self.case, self.worst, self.failed = case, {}, []

    def check(self, stage, err, bound, sens=None):
        """err <= bound, and the error of a reference missing one item / ray-step (sens) >= SENSITIVITY * bound."""
        self.worst[stage] = max(self.worst.get(stage, 0.0), err)
        print('  %-10s %-28s err %.3e  bound %.3e  dropped-one %s' % (self.case, stage, err, bound,
                                                                     '-' if sens is None else '%.3e' % sens))
        if not err <= bound:
            self.failed.append((stage, err, bound))
        if sens is not None and not sens >= SENSITIVITY * bound:
            self.failed.append((stage, 'insensitive', sens, bound))


def _typical(b, group):
    """The group of `group` consecutive flat elements of b that is typical of where b's mass lies: sorted by norm, the
    groups before it hold less than half of the squared norm of b, those after it less than half too.  None if b is 0."""
    norms = b.double().reshape(-1, group).norm(dim=1)
    if norms.numel() == 0 or float(norms.max()) == 0.0:
        return None
    order = torch.argsort(norms, descending=True)
    mass = torch.cumsum(norms[order] ** 2, 0)
    return int(order[int(torch.searchsorted(mass, 0.5 * mass[-1]))])


def _drop(b, k, group):
    """b with its k-th group of `group` consecutive flat elements (one ray, one ray-step or one 128-row item) zeroed."""
    d = b.clone().reshape(-1)
    d[k * group:(k + 1) * group] = 0
    return d.reshape(b.shape)


def _sens(a, b, scale, group):
    """The error a check of a against b would report if b lacked its typical group."""
    k = _typical(b, group)
    return None if k is None else tr.ratio(a, _drop(b, k, group), scale)


class Slots:
    """A view's workspace arrays (dz, dc16, dsig16, dx0) taken from a pass over that view alone, in the item order of the
    batch record: the live-tile list of a pass is in no fixed order, so items are matched by their tile."""

    def __init__(self, own, batch, i):
        S, n = own.S, own.views[0][1] * own.S * 128
        pos = torch.full((own.tpi,), -1, dtype=torch.long, device=DEV)
        pos[own.tile_list] = torch.arange(own.n_live, device=DEV)
        first, count = batch.views[i]
        p = pos[batch.tile_list[first:first + count] - i * batch.tpi]
        assert bool((p >= 0).all()) and count == own.n_live, 'the batch and the single view differ in their live tiles'
        idx = (p[:, None] * S * 128 + torch.arange(S * 128, device=DEV)[None, :]).reshape(-1)
        self.dz = [d[:n][idx] for d in own.dz]
        self.dc16, self.dsig16, self.dx0 = own.dc16[:n][idx], own.dsig16[:n][idx], own.dx0[:n][idx]
        self.dc32, self.dsig32 = own.dc32[:n][idx], own.dsig32[:n][idx]


def _composite_checks(rep, rec, i, G, sky, sky_avg, cam_x, gr, ws):
    """Compositing backward of view i from its recorded sigma / nds / c / rayflags; dL/dsky over every ray of the view,
    and (ws: this record's own workspace holds view i) dc32 / dsig32 / dc16 / dsig16."""
    S, HW = rec.S, rec.H * rec.W
    first, count = rec.views[i]
    sl = rec.view_slots(i)
    rs = slice(first * 128, (first + count) * 128)
    ray, inside = rec.rays(i)
    ray, inside = ray.reshape(-1), inside.reshape(-1)
    live, nosky, valid = rec.live[rs], rec.nosky[rs], rec.valid[rs]
    assert torch.equal(valid, inside), 'valid flags disagree with the tile geometry'
    Gi, skyi = G[i].reshape(HW, 64).double(), sky[i].reshape(HW, 64).double()
    g = Gi[ray] * valid[:, None]
    sky_used = torch.where(nosky[:, None], sky_avg[i].double()[None, :], skyi[ray] * valid[:, None])
    per_ray = lambda t, *tail: t.reshape(count, S, 128, *tail).transpose(1, 2).reshape(count * 128, S, *tail)
    (dc, dsig, dsky), (sdc, sdsig, sdsky) = tr.composite_backward_ref(per_ray(rec.sig[sl]), per_ray(rec.nds[sl]),
                                                                       per_ray(rec.c[sl], 64), live, g, sky_used)
    # dL/dsky per ray (live tiles: (1 - W) g; sky-only tiles: g), routed to sky_avg where the ray blends it
    ref_sky, sc_sky = torch.zeros(HW, 64, dtype=torch.float64, device=DEV), torch.zeros(HW, 64, dtype=torch.float64, device=DEV)
    keep = valid & ~nosky
    ref_sky[ray[keep]], sc_sky[ray[keep]] = dsky[keep], sdsky[keep]
    to_avg = valid & nosky
    ref_avg, sc_avg = dsky[to_avg].sum(0), sdsky[to_avg].sum(0)
    dead = rec.sky_only_rays(i)
    if bool(dead.any()):
        sk = sky_avg[i].double()[None, :].expand(int(dead.sum()), 64) if cam_x <= 1.0 else skyi[dead]
        d = Gi[dead] * tr.in_clamp(sk).double()
        if cam_x <= 1.0:
            ref_avg, sc_avg = ref_avg + d.sum(0), sc_avg + d.abs().sum(0)
        else:
            ref_sky[dead], sc_sky[dead] = d, d.abs()
    a_sky = gr['sky'][i].reshape(HW, 64)
    rep.check('g_sky', tr.ratio(a_sky, ref_sky, EPS * sc_sky), COMP, _sens(a_sky, ref_sky, EPS * sc_sky, 64))
    rep.check('g_sky_avg', tr.ratio(gr['sky_avg'][i], ref_avg, EPS * sc_avg), COMP)
    if ws is None:
        return
    n = count * S * 128
    a_dc, a_dsig = per_ray(ws.dc32[:n], 64), per_ray(ws.dsig32[:n])
    rep.check('dsig32', tr.ratio(a_dsig, dsig, EPS * sdsig), COMP, _sens(a_dsig, dsig, EPS * sdsig, 1))
    rep.check('dc32', tr.ratio(a_dc, dc, EPS * sdc), COMP, _sens(a_dc, dc, EPS * sdc, 64))
    assert torch.equal(ws.dc16[:n].view(torch.int16), tr.bf16_bits(ws.dc32[:n])), 'dc16 != bf16(dc32)'
    assert torch.equal(ws.dsig16[:n, 0].view(torch.int16), tr.bf16_bits(ws.dsig32[:n])), 'dsig16 != bf16(dsig32)'
    assert bool((ws.dsig16[:n, 1:].view(torch.int16) == 0).all()), 'dsig16 padding columns not zero'


def _chain_checks(rep, rec, W, wh):
    """Data-gradient chain of a one-view record from its own dc32 / dsig32 / sign words and the fp32 weights."""
    n = rec.n_live * rec.S * 128
    if n == 0:
        return
    bits = [tr.sign_bits(rec.mask[k]) for k in range(6)]
    dz, dx0, mag, mag0 = tr.chain_ref(rec.dc32[:n], rec.dsig32[:n], bits, W['w1'], wh, W['wsig'], W['wout'])
    item = _typical(dx0, 128 * 128)
    sens = lambda a, b, scale: None if item is None else tr.ratio(a, _drop(b, item, 128 * b.shape[1]), scale)
    a = rec.dx0[:n]
    rep.check('dx0', tr.ratio(a, dx0, BF16X3 * mag0), DX0, sens(a, dx0, BF16X3 * mag0))
    rep.check('dx0 rel-L2', tr.rel_l2(a, dx0) if float(dx0.abs().max()) > 0 else float(a.abs().max()), DX0_L2)
    for k in range(6):
        scale = tr.bf16_ulp(dz[k]) + BF16X3 * mag[k]
        a = rec.dz[k][:n]
        rep.check('dZ%d (bf16 ulps)' % (k + 1), tr.ratio(a, dz[k], scale), DZ, sens(a, dz[k], scale))


def _wgrad_checks(rep, rec, i, gr, ws):
    """Weight gradients of view i from its recorded bf16 tiles: A from the record, dZ / dc16 / dsig16 from ws."""
    n = rec.views[i][1] * rec.S * 128
    sl = rec.view_slots(i)
    jobs = [('g_w1ext', gr['w1ext'][i], ws.dz[0][:n], rec.x0[sl])]
    jobs += [('g_wh[%d]' % k, gr['wh'][i][k], ws.dz[k + 1][:n], rec.act[k][sl]) for k in range(5)]
    jobs += [('g_wout', gr['wout'][i], ws.dc16[:n], rec.act[5][sl]),
             ('g_wsig', gr['wsig'][i][:1], ws.dsig16[:n, :1], rec.act[3][sl])]
    assert bool((gr['wsig'][i][1:] == 0).all()), 'rows 1..7 of g_wsig must be exactly 0'
    for name, a, Z, A in jobs:
        ref, mag = tr.wgrad_ref(Z, A)
        item = _typical(Z, 128 * Z.shape[1])
        sens = None
        if item is not None:
            part, _ = tr.wgrad_ref(Z[item * 128:item * 128 + 128], A[item * 128:item * 128 + 128])
            sens = tr.ratio(a, ref - part, EPS * mag)
        rep.check(name, tr.ratio(a, ref, EPS * mag), WGRAD, sens)


def _table_checks(rep, rec, dx0s, dt3, gr, genc):
    """dt3, the pre-blended table gradient of the batch, from every view's dx0 (in record order) at its recorded grid
    positions; g_table, the transpose of the pre-blend applied to dt3, through the adjoint identity."""
    _, pls = oracle.grid_offsets()
    scales = tr.level_scales(16, float(np.log2(pls)), 16, DEV)
    x3 = torch.cat([rec.x3[rec.view_slots(i)] for i in range(rec.n_img)])
    dx0 = torch.cat(dx0s)
    ref, mag = tr.table_scatter_ref(x3, dx0, scales, 19)
    a = dt3.reshape(-1, 8)
    inside = torch.nonzero(x3[:, 3] > 0).reshape(-1)
    sens = None
    j = _typical(dx0 * (x3[:, 3:] > 0), 128)
    if j is not None:
        one, _ = tr.table_scatter_ref(x3[j:j + 1], dx0[j:j + 1], scales, 19)
        sens = tr.ratio(a, ref - one, EPS * mag)
        del one
    rep.check('dt3', tr.ratio(a, ref, EPS * mag), TABLE, sens)
    del ref, mag
    # <g_table, E> = sum over the inside samples of <dx0, enc_E(x, genc)>, with the oracle's 5-D hash-grid forward (CPU); one
    # item more or less is the dt3 check's to see -- this one holds the transpose of the pre-blend to the 5-D encoding
    offsets, _ = oracle.grid_offsets()
    x5 = torch.cat([x3[inside, :3], ((genc.reshape(1, 2) + 1) * 0.5).expand(inside.numel(), 2)], 1).cpu()
    gi = dx0[inside].double().cpu().reshape(-1, 16, 8).transpose(0, 1)                      # [L, B, 8]
    for probe in range(2):
        E = torch.randn(tuple(gr['table'].shape), generator=torch.Generator().manual_seed(100 + probe))
        lhs = float((gr['table'].double().cpu() * E.double()).sum())
        rhs = scale = 0.0
        if inside.numel():
            enc, _ = oracle.grid_encode_forward(x5, E, offsets, pls, 16, level_scales=scales.cpu())
            encm, _ = oracle.grid_encode_forward(x5, E.abs(), offsets, pls, 16, level_scales=scales.cpu())
            rhs, scale = float((gi * enc.double()).sum()), float((gi.abs() * encm.double()).sum())
        rep.check('<g_table,E%d>' % probe, abs(lhs - rhs) / (EPS * scale + tr.FP32_TINY), ADJ)


_WORST = {}


@pytest.mark.parametrize('case', list(CASES))
def test_backward_stages_vs_float64(base, golden_ops, case):
    t0 = time.time()
    windows, S, M, opt = CASES[case]
    n_views = len(windows)
    frames = [_frame(base, y0, x0, h, w, M, sky_cols, empty) + (list(base['world'].voxel_t.shape),)
              for y0, x0, h, w, sky_cols, empty in windows]
    H, W_ = frames[0][0].shape[:2]
    nlabels = opt.get('nlabels', 12)
    W, genc = _weights(21 + len(case), nlabels, opt.get('sigma_bias'), n_views)
    lut = render.reduced_label_lut(golden_ops['mc2reduced_lut'], 0, 3)
    if nlabels == 15:                       # labels 0 .. 14 over the voxel ids the frame hits: the first gets 0, the last 14
        ids = [v for v in torch.unique(torch.cat([f[0].reshape(-1) for f in frames])).tolist() if v != 0]
        assert len(ids) >= 2
        lut = torch.zeros(max(lut.numel(), max(ids) + 1), dtype=torch.int32)
        lut[torch.tensor(ids)] = torch.arange(len(ids), dtype=torch.int32) * 14 // (len(ids) - 1)
    lut = lut.to(DEV)
    g = torch.Generator().manual_seed(7)
    ori = base['o'].reshape(1, 3).repeat(n_views, 1)
    if opt.get('ground'):
        ori[:, 0] = 0.5                     # camera at ground level: sky-only rays blend the frame's mean sky feature
    sky = (torch.randn(n_views, H, W_, 64, generator=g) * 0.8).to(DEV)
    sky_avg = (torch.randn(n_views, 64, generator=g) * 0.8).to(DEV)
    G = torch.randn(n_views, H, W_, 64, generator=g).to(DEV)
    uni = torch.rand(n_views, H, W_, S + 1, 1, generator=g).to(DEV) if opt.get('stratified') else None
    rep = Report(case)
    print()
    rec, out, gr = _run(W, genc, frames, ori, lut, S, uni, sky, sky_avg, G)
    assert rec.n_live == sum(c for _, c in rec.views)
    assert all(rec.views[i][0] == sum(c for _, c in rec.views[:i]) for i in range(n_views)), rec.views
    if n_views == 1:
        own = [(rec, gr)]
        slots = [rec]
    else:                                   # the batch keeps only its last view's workspace: each view alone for the others
        own = [_run(W, genc, frames, ori, lut, S, uni, sky, sky_avg, G, views=[i])[::2] for i in range(n_views)]
        slots = [Slots(o, rec, i) for i, (o, _) in enumerate(own)]
        n = rec.views[-1][1] * S * 128
        for name in ('dc32', 'dsig32', 'dx0', 'dc16'):
            assert torch.equal(getattr(rec, name)[:n], getattr(slots[-1], name)), name
        for k in range(6):
            assert torch.equal(rec.dz[k][:n], slots[-1].dz[k]), 'dz%d' % (k + 1)
    for i in range(n_views):
        own_rec, own_gr = own[i]
        _composite_checks(rep, rec, i, G, sky, sky_avg, float(ori[i, 0]), gr, rec if i == n_views - 1 else None)
        if n_views > 1:
            _composite_checks(rep, own_rec, 0, G[i:i + 1], sky[i:i + 1], sky_avg[i:i + 1], float(ori[i, 0]), own_gr, own_rec)
        _chain_checks(rep, own_rec, W, W['wh'][i])
        _wgrad_checks(rep, rec, i, gr, slots[i])
    _table_checks(rep, rec, [s_.dx0[:rec.views[i][1] * S * 128] for i, s_ in enumerate(slots)], rec.dt3, gr, genc)
    if nlabels == 15:                       # the one-hot columns of labels 0 and 14 (x0 columns 128 and 142) were trained
        assert float(gr['w1ext'][:, :, 128].abs().sum()) > 0 and float(gr['w1ext'][:, :, 142].abs().sum()) > 0
    if rec.n_live == 0:
        assert float(gr['w1ext'].abs().sum() + gr['wh'].abs().sum() + gr['wout'].abs().sum() + gr['table'].abs().sum()) == 0.0
    if opt.get('sigma_bias', 0) < 0:        # no sample has opacity: no sigma gradient anywhere
        assert float(rec.dsig32[:rec.n_live * S * 128].abs().max()) == 0.0
    for k, v in rep.worst.items():
        _WORST[k] = max(_WORST.get(k, 0.0), v)
    print('  %s: %d views, %dx%d, S=%d, M=%d, live items %s, %.1f s; worst so far %s' % (
        case, n_views, H, W_, S, M, [c * S for _, c in rec.views], time.time() - t0,
        ', '.join('%s %.2e' % kv for kv in sorted(_WORST.items()))))
    assert not rep.failed, (case, rep.failed)
