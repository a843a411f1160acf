"""Argument checks of the mixed-precision recording forward (sdb_render_rays_train_forward with precision 0, include/sdb200.h):
its batch pack stride is held to the fp16 x1 pack's size, and bf16 x3 stays refused.  The checks come before any CUDA call,
so they run without a GPU; the pointers handed over are never dereferenced."""
import ctypes

from scenedreamer_b200 import _lib
from test_train_views_abi import D, EINVAL, EUNSUPPORTED, _params


def _with_precision(n_img, precision, pack_stride=0):
    p = _params(n_img, pack_stride=pack_stride)
    p.precision = precision
    return p


def test_fp16_train_forward_pack_stride_is_the_fp16_pack():
    L = _lib.lib()
    fw = L.sdb_render_rays_train_forward
    one = L.sdb_mlp_pack_bytes(0)
    assert one < L.sdb_mlp_pack_bytes(2)                       # the fp16 x1 pack has no lo part
    assert fw(ctypes.byref(_with_precision(3, 0, one - 256)), D, None) == EINVAL
    assert fw(ctypes.byref(_with_precision(3, 0, -64)), D, None) == EINVAL
    assert fw(ctypes.byref(_with_precision(3, 0)), None, None) == EINVAL


def test_bf16x3_train_forward_stays_unsupported():
    L = _lib.lib()
    fw = L.sdb_render_rays_train_forward
    for n, stride in ((1, 0), (3, 0), (3, L.sdb_mlp_pack_bytes(1))):
        assert fw(ctypes.byref(_with_precision(n, 1, stride)), D, None) == EUNSUPPORTED
    for prec in (-1, 3):
        assert fw(ctypes.byref(_with_precision(1, prec)), D, None) == EUNSUPPORTED
