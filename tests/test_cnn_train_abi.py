"""Argument checks of the RenderCNN training entry points (include/sdb200.h, f1 under autograd).  They come before any
CUDA call, so they run without a GPU; the pointers handed over are never dereferenced."""
import ctypes

from scenedreamer_b200 import _lib, rendercnn

EINVAL, EUNSUPPORTED = -1, -2


def test_cnn_train_entry_points_refuse_bad_arguments():
    L = _lib.lib()
    d = ctypes.c_void_p(0x1000)
    assert L.sdb_cnn_train_record_bytes(0, 8) == 0 and L.sdb_cnn_train_record_bytes(8, -1) == 0
    assert L.sdb_cnn_backward_workspace_bytes(0, 8) == 0 and L.sdb_cnn_backward_workspace_bytes(8, 0) == 0
    assert L.sdb_cnn_train_record_bytes(262, 262) > 0 and L.sdb_cnn_backward_workspace_bytes(262, 262) > 0
    assert L.sdb_cnn_backward_pack_bytes() > 0
    # precision 1 (bf16 x3) is a pack of the training path only
    assert L.sdb_cnn_pack_bytes(1) == L.sdb_cnn_pack_bytes(2) and L.sdb_cnn_pack_bytes(3) == 0 and L.sdb_cnn_pack_bytes(-1) == 0
    assert L.sdb_cnn_pack(*([d] * 14), 3, d, None) == EUNSUPPORTED
    assert L.sdb_cnn_pack(*([d] * 13 + [None]), 1, d, None) == EINVAL
    assert L.sdb_cnn_workspace_bytes(8, 8, 1) == 0
    assert L.sdb_cnn_forward(d, 8, 8, d, d, 1, d, None, d, 0, None) == EUNSUPPORTED
    # training forward
    assert L.sdb_cnn_train_forward(None, 8, 8, d, d, d, None, d, None) == EINVAL
    assert L.sdb_cnn_train_forward(d, 8, 8, d, d, d, None, None, None) == EINVAL
    assert L.sdb_cnn_train_forward(d, 0, 8, d, d, d, None, d, None) == EINVAL
    assert L.sdb_cnn_train_forward(d, 8, -2, d, d, d, None, d, None) == EINVAL
    # backward pack and backward
    assert L.sdb_cnn_pack_backward(*([d] * 6 + [None, d]), None) == EINVAL
    assert L.sdb_cnn_pack_backward(*([d] * 7 + [None]), None) == EINVAL
    g = rendercnn._CnnGrads()
    gp = ctypes.byref(g)
    assert L.sdb_cnn_backward(8, 8, None, d, d, d, d, d, gp, d, None) == EINVAL
    assert L.sdb_cnn_backward(8, 8, d, None, None, d, d, d, gp, d, None) == EINVAL      # neither dL/d rgb nor dL/d raw
    assert L.sdb_cnn_backward(8, 8, d, d, None, None, d, d, gp, d, None) == EINVAL
    assert L.sdb_cnn_backward(8, 8, d, d, None, d, d, d, None, d, None) == EINVAL
    assert L.sdb_cnn_backward(8, 8, d, d, None, d, d, d, gp, None, None) == EINVAL
    assert L.sdb_cnn_backward(0, 8, d, d, None, d, d, d, gp, d, None) == EINVAL
    assert L.sdb_cnn_backward(8, -1, d, None, d, d, d, d, gp, d, None) == EINVAL


def test_cnn_record_layout_matches_record_size():
    L = _lib.lib()
    out = (ctypes.c_int64 * 14)()
    assert L.sdb_cnn_debug_record_layout(0, 8, out) == EINVAL and L.sdb_cnn_debug_record_layout(8, 8, None) == EINVAL
    assert L.sdb_cnn_debug_record_layout(262, 262, out) == 0
    Hp, Wp, offs = out[0], out[1], list(out[2:])
    assert (Hp, Wp) == (266, 386)
    pair = Hp * 32 * Wp * 16 * 2
    assert offs[1] >= Hp * 8 * Wp * 16 * 2                               # x: 8-channel pair first
    assert all(b - a == pair for a, b in zip(offs[1:10], offs[2:11]))     # y1 .. y4 back to back, u right before its y
    assert offs[-1] == L.sdb_cnn_train_record_bytes(262, 262) and offs[-1] >= offs[10] + 3 * 262 * 262 * 4
