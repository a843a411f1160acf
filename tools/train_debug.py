"""Stage-by-stage diagnostics of the fused training path on the GPU (not a test; prints a table).

Every stage of sdb_render_rays_train_forward / sdb_render_rays_backward is compared with plain torch fp32 on the
GPU, using the library's OWN recorded inputs of that stage, so a wrong stage is visible in isolation:
  record:  A_{k+1} = lrelu(A_k W^T + b), sign words, sigma, colour head, constant columns
  backward: compositing (torch autograd on the recorded sigma / c), every dZ_k of the chain, d(features),
            the weight-gradient GEMMs, the table scatter.
Usage: python tools/train_debug.py [--stress] [--S 24]
"""
import argparse
import ctypes
import os
import sys

import numpy as np
import torch
import torch.nn.functional as F

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), '..'))
sys.path.insert(0, ROOT)
import oracle  # noqa: E402  (synthetic weights only)
from scenedreamer_b200 import _lib, ops, render, synth  # noqa: E402

DEV = 'cuda:0'


def rel(a, b):
    a, b = a.double(), b.double()
    return float((a - b).norm() / (b.norm() + 1e-30)), float((a - b).abs().max()), float(b.abs().max())


def report(name, a, b):
    r, m, s = rel(a, b)
    print('  %-34s rel-L2 %.3e   max|diff| %.3e   max|ref| %.3e' % (name, r, m, s), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--stress', action='store_true')
    ap.add_argument('--S', type=int, default=24)
    ap.add_argument('--res', type=int, nargs=2, default=[44, 60])
    a = ap.parse_args()
    torch.manual_seed(0)
    Lb = _lib.lib()
    world = synth.SyntheticVoxelWorld(size=128, seed=7)
    pose = synth.eval_camera_poses(world, maxstep=8, pattern=0)[1]
    o, d, u, f, c, res = synth.frame_camera(world, pose, resolution_hw=tuple(a.res), pad=4)
    vid, dep, rd = ops.ray_voxel_intersection_perspective(world.voxel_t.to(DEV), o, d, u, f, c, res, 6)
    vid, dep, rd = vid.unsqueeze(0), dep.unsqueeze(0), rd.unsqueeze(0)
    N, H, W = vid.shape[:3]
    S = a.S
    P = {k: v.to(DEV) for k, v in oracle.make_params(seed=21, stress=a.stress).items()}
    g = torch.Generator().manual_seed(8888)
    z = oracle.style_mlp(torch.randn(1, 128, generator=g), {k: v.cpu() for k, v in P.items()}).to(DEV)
    genc = torch.tanh(torch.randn(1, 2, generator=g)).to(DEV)
    lut_raw = np.load(os.path.join(ROOT, 'tests', 'golden', 'ref_python_ops.npz'))['mc2reduced_lut']
    lut = render.reduced_label_lut(lut_raw)
    _, pls = oracle.grid_offsets()
    for k in P:
        P[k].requires_grad_(True)
    z.requires_grad_(True)
    genc.requires_grad_(True)
    uni = torch.rand(N, H, W, S + 1, 1, generator=torch.Generator().manual_seed(5)).to(DEV)

    # keep handles on the autograd Function's context through a hook on apply
    holder = {}
    orig_fwd = render._FusedRenderTrainFn.forward

    def fwd(ctx, *args):
        holder['ctx'] = ctx
        return orig_fwd(ctx, *args)
    render._FusedRenderTrainFn.forward = staticmethod(fwd)
    out = render.render_rays_train(P, vid, dep, rd, o.unsqueeze(0), z, genc, list(world.voxel_t.shape), lut, pls,
                                   num_samples=S, uniforms=uni)
    torch.cuda.synchronize()
    print('train forward done: net_out', tuple(out['net_out'].shape), 'finite', bool(torch.isfinite(out['net_out']).all()))
    # same frame through the inference kernel
    r = render.FusedPerPixelRenderer({k: v.detach() for k, v in P.items()}, world.voxel_t.shape, lut, pls)
    r.sky_impl = 'torch'
    inf = r.forward(vid, dep, rd, o.unsqueeze(0), z.detach(), genc.detach(), num_samples=S, uniforms=uni)
    report('net_out train vs inference kernel', out['net_out'].detach(), inf['net_out'])

    ctx = holder['ctx']
    record = ctx.record
    lay = (ctypes.c_int64 * 20)()
    _lib.check(Lb.sdb_debug_train_layout(N, H, W, S, 16, 19, lay), 'layout')
    lay = list(lay)
    tiles_x, tiles_y = (W + 15) // 16, (H + 7) // 8
    ntiles = N * tiles_x * tiles_y
    cap, steps = ntiles * S * 128, ntiles * S

    def rv(off, nbytes, dtype):
        return record[off:off + nbytes].view(dtype)

    def untile(t, cols):
        """bf16 records are MMA-ready tiles [item][chunk of 8 columns][128 rows][8] (rf_common.cuh: rec_chunk) -> [slots, cols]"""
        items = t.numel() // (128 * cols)
        return t.reshape(items, cols // 8, 128, 8).permute(0, 2, 1, 3).reshape(items * 128, cols)
    n_live = int(rv(lay[0], 4, torch.int32)[0])
    nsl = n_live * S * 128
    print('tiles %d live %d slots %d' % (ntiles, n_live, nsl))
    tile_list = rv(lay[1], ntiles * 4, torch.int32)[:n_live].long()
    rayflags = rv(lay[3], ntiles * 128 * 4, torch.int32)[:n_live * 128]
    x3 = rv(lay[4], cap * 16, torch.float32).reshape(cap, 4)[:nsl]
    x0 = untile(rv(lay[5], cap * 288, torch.bfloat16), 144)[:nsl].float()
    act = torch.stack([untile(a_, 272) for a_ in rv(lay[6], 6 * cap * 544, torch.bfloat16).reshape(6, cap * 272)])[:, :nsl].float()
    mask = rv(lay[7], steps * 6 * 128 * 8 * 4, torch.int32).reshape(steps, 6, 128, 8)[:n_live * S]
    sig = rv(lay[8], cap * 4, torch.float32)[:nsl]
    nds = rv(lay[9], cap * 4, torch.float32)[:nsl]
    cc = rv(lay[10], cap * 256, torch.float32).reshape(cap, 64)[:nsl]

    Pd = {k: v.detach() for k, v in P.items()}
    wh, bh = render.modulated_weights(Pd, z.detach()[0])
    w1, b1 = Pd['render_net.fc_1.weight'], Pd['render_net.fc_1.bias']
    fcm = Pd['render_net.fc_m_a.weight']
    w0ext = torch.zeros(256, 144, device=DEV)
    w0ext[:, :128] = w1
    w0ext[:, 128:128 + fcm.shape[1]] = fcm
    w0ext[:, 143] = b1
    wsig, bsig = Pd['render_net.fc_sigma.weight'].reshape(-1), Pd['render_net.fc_sigma.bias']
    wout, bout = Pd['render_net.fc_out_c.weight'], Pd['render_net.fc_out_c.bias']
    lre = lambda t: F.leaky_relu(t, 0.2)
    print('--- forward record ---')
    report('A1 = lrelu(X0 W0ext^T)', act[0][:, :256], lre(x0 @ w0ext.t()))
    for k in range(5):
        report('A%d = lrelu(A%d W^T + b)' % (k + 2, k + 1), act[k + 1][:, :256], lre(act[k][:, :256] @ wh[k].t() + bh[k]))
    report('sigma', sig, act[3][:, :256] @ wsig + bsig)
    report('colour head', cc, act[5][:, :256] @ wout.t() + bout)
    print('  ones column ok:', bool((act[:, :, 256] == 1).all()), ' zero pad ok:', bool((act[:, :, 257:] == 0).all()),
          ' x0 col 143 ones:', bool((x0[:, 143] == 1).all()))
    bits = torch.arange(32, device=DEV)
    for k in range(6):
        m = mask[:, k].reshape(nsl, 8)
        mb = ((m.unsqueeze(-1) >> bits) & 1).reshape(nsl, 256).bool()
        print('  sign words layer %d: mismatches vs (A>0): %d of %d' % (k + 1, int((mb != (act[k][:, :256] > 0)).sum()), mb.numel()))

    # ---------------- backward ----------------
    G = torch.randn(out['net_out'].shape, generator=torch.Generator().manual_seed(9)).to(DEV)
    orig_bwd = render._FusedRenderTrainFn.backward

    def bwd(ctx2, *gs):
        res_ = orig_bwd(ctx2, *gs)
        holder['grads'] = res_
        return res_
    render._FusedRenderTrainFn.backward = staticmethod(bwd)
    # keep the backward workspace alive for inspection: wrap torch.empty?  simpler: re-run the C call by hand below
    (out['net_out'] * G).sum().backward()
    torch.cuda.synchronize()
    print('backward done')
    grads = holder['grads']
    # re-run the backward by hand to keep the workspace
    prm = ctx.prm
    embeddings_, w1_, wh_, wsig_, wout_ = ctx.saved
    bpack = torch.empty(int(Lb.sdb_mlp_backward_pack_bytes()), dtype=torch.uint8, device=DEV)
    _lib.check(Lb.sdb_pack_mlp_backward(render._ptr(w1_), render._ptr(wh_), render._ptr(wsig_), render._ptr(wout_),
                                        render._ptr(bpack), render._stream(DEV)), 'pack bwd')
    g_table = torch.empty_like(embeddings_)
    g_genc = torch.empty(2, device=DEV)
    g_w1ext = torch.empty(256, 144, device=DEV)
    g_wh = torch.empty(5, 256, 272, device=DEV)
    g_wsig = torch.empty(8, 272, device=DEV)
    g_wout = torch.empty(64, 272, device=DEV)
    g_sky = torch.zeros(N, H, W, 64, device=DEV)
    g_sky_avg = torch.empty(N, 64, device=DEV)
    wsb = torch.empty(lay[19], dtype=torch.uint8, device=DEV)
    gr = render._RenderGrads()
    Gc = G.contiguous()
    gr.d_grad_net_out, gr.d_bwd_pack, gr.bwd_pack_stride = render._ptr(Gc), render._ptr(bpack), 0
    gr.d_table = render._ptr(embeddings_)
    gr.d_grad_table, gr.d_grad_global_enc, gr.d_grad_w1ext = render._ptr(g_table), render._ptr(g_genc), render._ptr(g_w1ext)
    gr.d_grad_wh, gr.d_grad_wsig, gr.d_grad_wout = render._ptr(g_wh), render._ptr(g_wsig), render._ptr(g_wout)
    gr.d_grad_sky, gr.d_grad_sky_avg, gr.d_workspace = render._ptr(g_sky), render._ptr(g_sky_avg), render._ptr(wsb)
    _lib.check(Lb.sdb_render_rays_backward(ctypes.byref(prm), render._ptr(record), ctypes.byref(gr), render._stream(DEV)), 'bwd')
    torch.cuda.synchronize()

    def wv(off, nbytes, dtype):
        return wsb[off:off + nbytes].view(dtype)
    dc32 = wv(lay[11], cap * 256, torch.float32).reshape(cap, 64)[:nsl]
    dc16 = untile(wv(lay[12], cap * 128, torch.bfloat16), 64)[:nsl].float()
    dsig32 = wv(lay[13], cap * 4, torch.float32)[:nsl]
    dsig16 = wv(lay[14], cap * 16, torch.bfloat16).reshape(cap, 8)[:nsl].float()
    dz = torch.stack([untile(d_, 256) for d_ in wv(lay[15], 6 * cap * 512, torch.bfloat16).reshape(6, cap * 256)])[:, :nsl].float()
    dx0 = wv(lay[16], cap * 512, torch.float32).reshape(cap, 128)[:nsl]

    print('--- compositing backward (torch autograd on the recorded sigma / c) ---')
    ty, tx = (tile_list // tiles_x) * 8, (tile_list % tiles_x) * 16                      # N == 1
    rows = torch.arange(128, device=DEV)
    yy = ty[:, None] + (rows >> 4)[None, :]
    xx = tx[:, None] + (rows & 15)[None, :]
    valid = (yy < H) & (xx < W)
    ray = (yy * W + xx).clamp(max=H * W - 1)
    live = (rayflags & 1).bool().reshape(n_live, 128)
    nosky = (rayflags & 2).bool().reshape(n_live, 128)
    print('  valid flag consistent:', bool((((rayflags & 4) != 0).reshape(n_live, 128) == valid).all()))
    sig_t = sig.reshape(n_live, S, 128).clone().requires_grad_(True)
    c_t = cc.reshape(n_live, S, 128, 64).clone().requires_grad_(True)
    nds_t = nds.reshape(n_live, S, 128)
    e = F.relu(sig_t) * nds_t
    Eex = torch.cumsum(e, 1) - e
    wgt = (1 - torch.exp(-e)) * torch.exp(-Eex) * live[:, None, :].float()
    Wt = wgt.sum(1)
    sky = out['sky'].detach().reshape(H * W, 64)
    sky_avg = out['sky_avg'].detach().reshape(64)
    sky_leaf = sky[ray].clone().requires_grad_(True)                                        # [n_live,128,64]
    avg_leaf = sky_avg.clone().requires_grad_(True)
    sky_used = torch.where(nosky[..., None], avg_leaf.expand(n_live, 128, 64), sky_leaf)
    o_ref = (wgt[..., None] * (c_t.clamp(-1, 1) + 1)).sum(1) + (1 - Wt)[..., None] * (sky_used.clamp(-1, 1) + 1) - 1
    Gr = G.reshape(H * W, 64)[ray] * valid[..., None].float()
    report('net_out (recomputed from the record)', out['net_out'].detach().reshape(H * W, 64)[ray][valid], o_ref.detach()[valid])
    (o_ref * Gr).sum().backward()
    report('dL/dc', dc32.reshape(n_live, S, 128, 64), c_t.grad)
    report('dL/dsigma', dsig32.reshape(n_live, S, 128), sig_t.grad)
    report('dc16 vs dc32', dc16, dc32)
    report('dsig16[:,0] vs dsig32', dsig16[:, 0], dsig32)
    gsk = torch.zeros(H * W, 64, device=DEV)
    gsk.index_put_((ray[valid],), (sky_leaf.grad * (~nosky)[..., None].float())[valid], accumulate=True)
    live_rays = torch.zeros(H * W, dtype=torch.bool, device=DEV)
    live_rays[ray[valid]] = True
    report('dL/dsky (rays of live tiles)', g_sky.reshape(H * W, 64)[live_rays], gsk[live_rays])
    print('  (dsky_avg from live tiles: ref norm %.3e, ours total norm %.3e)' % (float(avg_leaf.grad.norm()), float(g_sky_avg.norm())))

    print('--- data-gradient chain (each layer from the RECORDED input of that layer) ---')
    def slope(k):
        m = mask[:, k].reshape(nsl, 8)
        mb = ((m.unsqueeze(-1) >> bits) & 1).reshape(nsl, 256).float()
        return mb + 0.2 * (1 - mb)
    report('dZ6 = (dC Wc) * m6', dz[5], (dc32 @ wout) * slope(5))
    report('dZ5 = (dZ6 W6) * m5', dz[4], (dz[5] @ wh[4]) * slope(4))
    report('dZ4 = (dZ5 W5 + dsig wsig) * m4', dz[3], (dz[4] @ wh[3] + dsig32[:, None] * wsig[None, :]) * slope(3))
    report('dZ3 = (dZ4 W4) * m3', dz[2], (dz[3] @ wh[2]) * slope(2))
    report('dZ2 = (dZ3 W3) * m2', dz[1], (dz[2] @ wh[1]) * slope(1))
    report('dZ1 = (dZ2 W2) * m1', dz[0], (dz[1] @ wh[0]) * slope(0))
    report('dX0 = dZ1 W1', dx0, dz[0] @ w1)
    print('--- weight-gradient GEMMs (vs torch matmul of the same bf16 records) ---')
    report('w1ext', g_w1ext, dz[0].t() @ x0)
    for k in range(5):
        report('wh[%d] (fc_%d)' % (k, k + 2), g_wh[k], dz[k + 1].t() @ act[k])
    report('wout', g_wout, dc16.t() @ act[5])
    report('wsig', g_wsig[0], dsig16[:, 0] @ act[3])
    print('--- table ---')
    print('  |g_table| %.4e  nonzero rows %d   g_genc %s' % (float(g_table.norm()), int((g_table.abs().sum(1) > 0).sum()),
                                                            g_genc.tolist()))
    # table scatter vs the stand-alone 3-D grid backward on the recorded coordinates + un-blend
    inb = x3[:, 3] > 0
    B = int(inb.sum())
    if B > 0:
        offs = torch.arange(17, device=DEV, dtype=torch.int32) * (1 << 19)
        gl = dx0[inb].reshape(B, 16, 8).permute(1, 0, 2).contiguous()
        gt3 = torch.zeros_like(embeddings_)
        xin = x3[inb][:, :3].contiguous()
        one = torch.zeros(1, device=DEV)
        ops.grid_encode_backward(gl, xin, embeddings_, offs, gt3, B, 3, 8, 16, float(np.log2(pls)), 16, False, one, one, 0, False)
        ref_tab = render.preblend_table(gt3, genc.detach(), 19, pls, 16, 16)
        report('g_table vs stand-alone 3-D scatter', g_table, ref_tab)


if __name__ == '__main__':
    main()
