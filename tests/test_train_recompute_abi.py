"""Argument checks of the recompute backward (include/sdb200.h: sdb_render_rays_backward_recompute) and the sizes it relies
on.  The checks come before any CUDA call, so they run without a GPU; the pointers handed over are never dereferenced."""
import ctypes

from scenedreamer_b200 import _lib, render

EINVAL, EUNSUPPORTED = -1, -2
D = 0x1000


def _params(n_img, raw5d=False, pack_stride=0, precision=2):
    p = render._RenderParams()
    p.n_img, p.H, p.W, p.M, p.S = n_img, 20, 36, 4, 12
    for f in ('d_voxel_id', 'd_depth2', 'd_raydirs', 'd_cam_ori', 'd_global_enc', 'd_fractions', 'd_label_lut', 'd_mlp_pack',
              'd_sky', 'd_sky_avg', 'd_net_out', 'd_workspace'):
        setattr(p, f, D)
    p.n_lut, p.L, p.log2_T, p.base_res, p.level_S, p.precision = 15, 16, 19, 16, 0.5, precision
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


def test_recompute_backward_refuses_null_arguments():
    bw = _lib.lib().sdb_render_rays_backward_recompute
    p3, vg = _params(3), _view_grads()
    assert bw(None, D, ctypes.byref(vg), None) == EINVAL
    assert bw(ctypes.byref(p3), None, ctypes.byref(vg), None) == EINVAL
    assert bw(ctypes.byref(p3), D, None, None) == EINVAL
    for f in ('d_grad_net_out', 'd_bwd_pack', 'd_table', 'd_grad_table', 'd_grad_global_enc', 'd_grad_w1ext', 'd_grad_wh',
              'd_grad_wsig', 'd_grad_wout', 'd_grad_sky', 'd_grad_sky_avg', 'd_workspace'):
        v = _view_grads()
        setattr(v.g, f, None)
        assert bw(ctypes.byref(p3), D, ctypes.byref(v), None) == EINVAL, f
    for f in ('d_cam_ori', 'd_mlp_pack', 'd_net_out', 'd_sky_avg'):
        p = _params(3)
        setattr(p, f, None)
        assert bw(ctypes.byref(p), D, ctypes.byref(vg), None) == EINVAL, f
    for n in (0, -2):
        assert bw(ctypes.byref(_params(n)), D, ctypes.byref(vg), None) == EINVAL


def test_recompute_backward_refuses_what_the_recording_forward_refuses():
    L = _lib.lib()
    bw, vg = L.sdb_render_rays_backward_recompute, _view_grads()
    for n in (1, 3):
        assert bw(ctypes.byref(_params(n, raw5d=True)), D, ctypes.byref(vg), None) == EUNSUPPORTED
        assert bw(ctypes.byref(_params(n, precision=1)), D, ctypes.byref(vg), None) == EUNSUPPORTED
        # and the recording forward agrees on both
        assert L.sdb_render_rays_train_forward(ctypes.byref(_params(n, raw5d=True)), D, None) == EUNSUPPORTED
        assert L.sdb_render_rays_train_forward(ctypes.byref(_params(n, precision=1)), D, None) == EUNSUPPORTED
    assert bw(ctypes.byref(_params(3, precision=3)), D, ctypes.byref(vg), None) == EUNSUPPORTED


def test_recompute_backward_refuses_bad_strides():
    L = _lib.lib()
    bw = L.sdb_render_rays_backward_recompute
    p3 = _params(3)
    for k, bad in (('w1ext_stride', 256 * 144 - 1), ('wh_stride', -1), ('wsig_stride', 8), ('wout_stride', 64 * 271),
                   ('sky_avg_stride', 63)):
        assert bw(ctypes.byref(p3), D, ctypes.byref(_view_grads(**{k: bad})), None) == EINVAL, k
    v = _view_grads()
    v.g.bwd_pack_stride = -8
    assert bw(ctypes.byref(p3), D, ctypes.byref(v), None) == EINVAL
    v.g.bwd_pack_stride = L.sdb_mlp_backward_pack_bytes() - 256
    assert bw(ctypes.byref(p3), D, ctypes.byref(v), None) == EINVAL
    # the forward pack stride: one pack per view, at least one pack of the forward's precision apart (0 = shared)
    vg = _view_grads()
    assert bw(ctypes.byref(_params(3, pack_stride=-64)), D, ctypes.byref(vg), None) == EINVAL
    assert bw(ctypes.byref(_params(3, pack_stride=L.sdb_mlp_pack_bytes(2) - 256)), D, ctypes.byref(vg), None) == EINVAL
    assert bw(ctypes.byref(_params(3, pack_stride=L.sdb_mlp_pack_bytes(0) - 256, precision=0)), D, ctypes.byref(vg), None) == EINVAL


# sdb_render_train_record_bytes(n, H, W, S) for n = 1, 3, 8 and sdb_render_backward_workspace_bytes(1, H, W, S, 16, 19), as
# the library computed them before the recompute backward existed
SIZES = {(262, 262, 24): ((6935221248, 20805663744, 55481769472), 7141322752),
         (20, 36, 12): ((55632896, 166897664, 445060096), 323565568),
         (570, 990, 24): ((55185075200, 165555225600, 441480600832), 54957506560)}


def test_size_functions_unchanged():
    """The recompute backward takes the one-view record and the one-view workspace the record-mode backward takes, and
    neither size changed."""
    L = _lib.lib()
    for (H, W, S), (records, workspace) in SIZES.items():
        assert tuple(L.sdb_render_train_record_bytes(n, H, W, S) for n in (1, 3, 8)) == records, (H, W, S)
        for n in (1, 3, 8):
            assert L.sdb_render_backward_workspace_bytes(n, H, W, S, 16, 19) == workspace, (H, W, S, n)
    for H, W, S in ((262, 262, 24), (20, 36, 12), (36, 52, 64)):
        out = (ctypes.c_int64 * 20)()
        assert L.sdb_debug_train_layout(1, H, W, S, 16, 19, out) == 0
        assert L.sdb_render_train_record_bytes(1, H, W, S) == out[18]
        for n in (1, 3, 8):
            assert L.sdb_render_backward_workspace_bytes(n, H, W, S, 16, 19) == out[19]
            assert L.sdb_render_train_record_bytes(n, H, W, S) > (n - 1) * out[18]
        # the recomputed net_out of a view lands in the workspace's compositing-gradient array: it must fit there
        assert out[12] - out[11] >= H * W * 64 * 4
    assert L.sdb_render_train_record_bytes(0, 262, 262, 24) == 0 and L.sdb_render_train_record_bytes(1, 262, 262, 65) == 0
