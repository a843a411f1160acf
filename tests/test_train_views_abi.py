"""Argument checks of the multi-view training entry points (include/sdb200.h: sdb_render_rays_backward_views,
sdb_sky_train_forward_views, sdb_sky_backward_views, and sdb_render_rays_train_forward with n_img > 1), and the record /
workspace sizes of a batch.  The checks come before any CUDA call, so they run without a GPU; the pointers handed over are
never dereferenced."""
import ctypes

from scenedreamer_b200 import _lib, render

EINVAL, EUNSUPPORTED = -1, -2
D = 0x1000


def _params(n_img, raw5d=False, pack_stride=0):
    p = render._RenderParams()
    p.n_img, p.H, p.W, p.M, p.S = n_img, 20, 36, 4, 12
    for f in ('d_voxel_id', 'd_depth2', 'd_raydirs', 'd_cam_ori', 'd_global_enc', 'd_fractions', 'd_label_lut', 'd_mlp_pack',
              'd_sky', 'd_sky_avg', 'd_net_out', 'd_workspace'):
        setattr(p, f, D)
    p.n_lut, p.L, p.log2_T, p.base_res, p.level_S, p.precision = 15, 16, 19, 16, 0.5, 2
    if raw5d:
        p.d_table = D
    else:
        p.d_table3 = D
    p.mlp_pack_stride = pack_stride
    return p


def _view_grads(**strides):
    L = _lib.lib()
    vg = render._RenderViewGrads()
    for f in ('d_grad_net_out', 'd_bwd_pack', 'd_table', 'd_grad_table', 'd_grad_global_enc', 'd_grad_w1ext', 'd_grad_wh',
              'd_grad_wsig', 'd_grad_wout', 'd_grad_sky', 'd_grad_sky_avg', 'd_workspace'):
        setattr(vg.g, f, D)
    vg.g.bwd_pack_stride = L.sdb_mlp_backward_pack_bytes()
    vg.w1ext_stride, vg.wh_stride, vg.wsig_stride, vg.wout_stride, vg.sky_avg_stride = 256 * 144, 5 * 256 * 272, 8 * 272, 64 * 272, 64
    for k, v in strides.items():
        setattr(vg, k, v)
    return vg


def _old_layout(n_img, H, W, S, L, log2_T):
    """The single-view record / workspace layout of sdb_debug_train_layout, restated (20 values)."""
    up = lambda v: (v + 255) // 256 * 256
    tiles = n_img * -(-H // 8) * -(-W // 16)
    cap, steps = tiles * S * 128, tiles * S
    r, o = [0], 16
    for size in (tiles * 4, tiles * 4, tiles * 128 * 4, cap * 16, cap * 144 * 2, 6 * cap * 272 * 2, steps * 6 * 128 * 8 * 4,
                 cap * 4, cap * 4, cap * 64 * 4):
        r.append(o)
        o = up(o + size)
    b, q = [], 0
    for size in (cap * 64 * 4, cap * 64 * 2, cap * 4, cap * 8 * 2, 6 * cap * 256 * 2, cap * 128 * 4, (L << log2_T) * 32):
        b.append(q)
        q = up(q + size)
    return r + b + [o, q]


def test_one_view_layout_is_unchanged():
    L = _lib.lib()
    for H, W, S in ((262, 262, 24), (20, 36, 12), (570, 990, 24)):
        out = (ctypes.c_int64 * 20)()
        assert L.sdb_debug_train_layout(1, H, W, S, 16, 19, out) == 0
        assert list(out) == _old_layout(1, H, W, S, 16, 19)
        assert L.sdb_render_train_record_bytes(1, H, W, S) == out[18]
        assert L.sdb_render_backward_workspace_bytes(1, H, W, S, 16, 19) == out[19]


def test_batch_record_grows_and_workspace_does_not():
    L = _lib.lib()
    one = L.sdb_render_train_record_bytes(1, 262, 262, 24)
    for n in (2, 3, 8):
        assert L.sdb_render_train_record_bytes(n, 262, 262, 24) >= n * one - n * 4096
        assert L.sdb_render_backward_workspace_bytes(n, 262, 262, 24, 16, 19) == L.sdb_render_backward_workspace_bytes(1, 262, 262, 24, 16, 19)
        assert L.sdb_sky_backward_workspace_bytes(n, 262, 262) == L.sdb_sky_backward_workspace_bytes(1, 262, 262)
        out = (ctypes.c_int64 * 20)()
        assert L.sdb_debug_train_layout(n, 262, 262, 24, 16, 19, out) == 0
        assert out[1] >= 4 + 8 * n                              # header: total + {first, count} per image
        assert out[18] == L.sdb_render_train_record_bytes(n, 262, 262, 24)


def test_render_backward_views_refuses_bad_arguments():
    L = _lib.lib()
    bw = L.sdb_render_rays_backward_views
    p3, vg = _params(3), _view_grads()
    assert bw(None, D, ctypes.byref(vg), None) == EINVAL
    assert bw(ctypes.byref(p3), None, ctypes.byref(vg), None) == EINVAL
    assert bw(ctypes.byref(p3), D, None, None) == EINVAL
    for f in ('d_grad_net_out', 'd_bwd_pack', 'd_grad_table', 'd_grad_wh', 'd_grad_sky_avg', 'd_workspace'):
        v = _view_grads()
        setattr(v.g, f, None)
        assert bw(ctypes.byref(p3), D, ctypes.byref(v), None) == EINVAL, f
    for n in (0, -2):
        assert bw(ctypes.byref(_params(n)), D, ctypes.byref(vg), None) == EINVAL
    assert bw(ctypes.byref(_params(3, raw5d=True)), D, ctypes.byref(vg), None) == EUNSUPPORTED
    for k, bad in (('w1ext_stride', 256 * 144 - 1), ('wh_stride', -1), ('wsig_stride', 8), ('wout_stride', 64 * 271),
                   ('sky_avg_stride', 63)):
        assert bw(ctypes.byref(p3), D, ctypes.byref(_view_grads(**{k: bad})), None) == EINVAL, k
    v = _view_grads()
    v.g.bwd_pack_stride = -8
    assert bw(ctypes.byref(p3), D, ctypes.byref(v), None) == EINVAL
    v.g.bwd_pack_stride = L.sdb_mlp_backward_pack_bytes() - 256
    assert bw(ctypes.byref(p3), D, ctypes.byref(v), None) == EINVAL
    # the single-view entry keeps refusing batches: it has one set of weight gradients
    assert L.sdb_render_rays_backward(ctypes.byref(p3), D, ctypes.byref(vg.g), None) == EUNSUPPORTED


def test_train_forward_batch_refuses_bad_arguments():
    L = _lib.lib()
    fw = L.sdb_render_rays_train_forward
    assert fw(ctypes.byref(_params(3, raw5d=True)), D, None) == EUNSUPPORTED
    assert fw(ctypes.byref(_params(0)), D, None) == EINVAL
    assert fw(ctypes.byref(_params(3, pack_stride=-64)), D, None) == EINVAL
    assert fw(ctypes.byref(_params(3, pack_stride=L.sdb_mlp_pack_bytes(2) - 256)), D, None) == EINVAL
    assert fw(ctypes.byref(_params(3)), None, None) == EINVAL


def test_sky_views_refuse_bad_arguments():
    L = _lib.lib()
    fw, bw = L.sdb_sky_train_forward_views, L.sdb_sky_backward_views
    sb = L.sdb_sky_pack_bytes(2)
    assert fw(D, 3, 8, 8, D, sb, D, D, D, None, None) == EINVAL                # no record
    assert fw(None, 3, 8, 8, D, sb, D, D, D, D, None) == EINVAL
    assert fw(D, 0, 8, 8, D, sb, D, D, D, D, None) == EINVAL
    assert fw(D, 3, 8, 8, D, -1, D, D, D, D, None) == EINVAL
    assert fw(D, 3, 8, 8, D, sb - 16, D, D, D, D, None) == EINVAL
    good = lambda **kw: render._SkyViewGrads(D, kw.get('a', 256 * 48), D, kw.get('b', 4 * 256 * 272), D, kw.get('c', 64 * 272))
    g = good()
    bb = L.sdb_sky_backward_pack_bytes()
    assert bw(3, 8, 8, None, D, D, 0, ctypes.byref(g), D, None) == EINVAL
    assert bw(3, 8, 8, D, D, D, 0, None, D, None) == EINVAL
    assert bw(3, 8, 8, D, D, D, 0, ctypes.byref(render._SkyViewGrads(None, 256 * 48, D, 4 * 256 * 272, D, 64 * 272)), D, None) == EINVAL
    assert bw(-1, 8, 8, D, D, D, 0, ctypes.byref(g), D, None) == EINVAL
    assert bw(3, 8, 8, D, D, D, -bb, ctypes.byref(g), D, None) == EINVAL
    assert bw(3, 8, 8, D, D, D, bb - 16, ctypes.byref(g), D, None) == EINVAL
    for kw in (dict(a=-1), dict(b=4 * 256 * 272 - 1), dict(c=0)):
        assert bw(3, 8, 8, D, D, D, 0, ctypes.byref(good(**kw)), D, None) == EINVAL, kw
    # the single-view entry points keep refusing batches
    assert L.sdb_sky_backward(3, 8, 8, D, D, D, D, D, D, D, None) == EUNSUPPORTED
    assert L.sdb_sky_train_forward(D, 3, 8, 8, D, D, D, D, D, None) == EUNSUPPORTED
