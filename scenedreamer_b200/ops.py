"""Python mirrors of the reference's native entry points, over libsdb200's C ABI.

Same names, argument meaning and error behaviour as the pybind functions of the reference:
  voxlib.*          imaginaire/model_utils/gancraft/voxlib/voxlib.cpp:25-31
  _gridencoder.*    gridencoder/src/bindings.cpp:5-8
Tensors are torch CUDA tensors; only their data pointers, shapes and the current CUDA stream
cross into the library (PyTorch is the allocator / stream plumbing, not the compute path).
"""
import ctypes
import weakref

import numpy as np
import torch

from . import _lib


def _ptr(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def _stream(t):
    return ctypes.c_void_p(torch.cuda.current_stream(t.device).cuda_stream)


def _check_cuda(t, name):
    if not isinstance(t, torch.Tensor) or not t.is_cuda:
        raise RuntimeError('%s must be a CUDA tensor' % name)


def _check_input(t, name, dtype=None):
    _check_cuda(t, name)
    if not t.is_contiguous():
        raise RuntimeError('%s must be contiguous' % name)
    if dtype is not None and t.dtype != dtype:
        raise RuntimeError('%s must be a %s tensor' % (name, str(dtype).replace('torch.', '')))


def _f3(t):
    a = torch.as_tensor(t).detach().to('cpu', torch.float32).reshape(-1)
    if a.numel() != 3:
        raise RuntimeError('camera vectors must have 3 elements')
    return (ctypes.c_float * 3)(*[float(v) for v in a])


# ------------------------------------------------------------------------------------------------
# voxlib
# ------------------------------------------------------------------------------------------------
HEIGHT_BOUND_BLOCK_LOG2 = 4          # 16 x 16 column blocks; None disables the empty-space bound
_height_bounds = {}      # id(voxel tensor OBJECT) -> (weakref to it, tensor._version, block_log2, int16 bound)


def height_bound(in_voxel, block_log2=None):
    """Highest occupied height per column block of `in_voxel` (sdb_build_height_bound), cached per tensor object and
    tensor version: the reference hands the same `voxel_t` tensor to every frame of a scene (scenedreamer.py:578), an
    in-place edit bumps `_version`, a new scene is a new tensor object.  Edits that bypass torch's version counter
    (`.data`, numpy views) need `invalidate_height_bound(t)`."""
    L = HEIGHT_BOUND_BLOCK_LOG2 if block_log2 is None else block_log2
    key = id(in_voxel)
    ent = _height_bounds.get(key)
    if ent is not None and ent[0]() is in_voxel and ent[1] == in_voxel._version and ent[2] == L:
        return ent[3], L
    dims = (ctypes.c_int64 * 3)(*in_voxel.shape)
    strides = (ctypes.c_int64 * 3)(*in_voxel.stride())
    n = int(_lib.lib().sdb_height_bound_elems(dims, int(L)))
    hb = torch.empty(n, dtype=torch.int16, device=in_voxel.device)
    with torch.cuda.device(in_voxel.device):
        code = _lib.lib().sdb_build_height_bound(_ptr(in_voxel), dims, strides, int(L), _ptr(hb), _stream(in_voxel))
    _lib.check(code, 'sdb_build_height_bound')
    _height_bounds[key] = (weakref.ref(in_voxel, lambda _r, k=key: _height_bounds.pop(k, None)), in_voxel._version, L, hb)
    return hb, L


def invalidate_height_bound(in_voxel):
    _height_bounds.pop(id(in_voxel), None)


def ray_voxel_intersection_perspective(in_voxel, cam_ori, cam_dir, cam_up, cam_f, cam_c, img_dims, max_samples,
                                       empty_space_bound=True, band=None):
    """-> [voxel_id int32 [H,W,M,1], depth2 f32 [2,H,W,M,1], raydirs f32 [H,W,1,3]]  (voxlib.cpp:11).
    empty_space_bound: use the cached height bound of the volume (bit-identical results, see height_bound).
    band = (first_row, band_rows, band_stride): img_dims[0] output rows taken from the frame in bands of band_rows rows that start
    at first_row and lie band_stride frame rows apart (single-frame sharding; cam_c stays the whole frame's principal point)."""
    _check_cuda(in_voxel, 'in_voxel')
    if in_voxel.dtype != torch.int32 or in_voxel.dim() != 3:
        raise RuntimeError('in_voxel must be a 3-D int32 tensor')
    H, W, M = int(img_dims[0]), int(img_dims[1]), int(max_samples)
    dev = in_voxel.device
    hb, L = (None, 0)
    if empty_space_bound and HEIGHT_BOUND_BLOCK_LOG2 is not None and in_voxel.shape[0] <= 32767:
        hb, L = height_bound(in_voxel)
    with torch.cuda.device(dev):
        voxel_id = torch.empty(H, W, M, 1, dtype=torch.int32, device=dev)
        depth2 = torch.empty(2, H, W, M, 1, dtype=torch.float32, device=dev)
        raydirs = torch.empty(H, W, 1, 3, dtype=torch.float32, device=dev)
        dims = (ctypes.c_int64 * 3)(*in_voxel.shape)
        strides = (ctypes.c_int64 * 3)(*in_voxel.stride())
        cc = (ctypes.c_float * 2)(float(cam_c[0]), float(cam_c[1]))
        im = (ctypes.c_int32 * 2)(H, W)
        if band is None:
            code = _lib.lib().sdb_ray_voxel_intersection_perspective_ex(
                _ptr(in_voxel), dims, strides, _f3(cam_ori), _f3(cam_dir), _f3(cam_up), float(cam_f), cc, im, M,
                _ptr(voxel_id), _ptr(depth2), _ptr(raydirs), _ptr(hb), int(L), _stream(in_voxel))
        else:
            bd = (ctypes.c_int32 * 3)(int(band[0]), int(band[1]), int(band[2]))
            code = _lib.lib().sdb_ray_voxel_intersection_perspective_bands(
                _ptr(in_voxel), dims, strides, _f3(cam_ori), _f3(cam_dir), _f3(cam_up), float(cam_f), cc, im, M, bd,
                _ptr(voxel_id), _ptr(depth2), _ptr(raydirs), _ptr(hb), int(L), _stream(in_voxel))
    _lib.check(code, 'ray_voxel_intersection_perspective')
    return [voxel_id, depth2, raydirs]


def _pe_shape(t, dim):
    dim = dim % t.dim()
    pre = int(np.prod(t.shape[:dim])) if dim > 0 else 1
    post = int(np.prod(t.shape[dim:]))
    return dim, pre, post


def positional_encoding(in_feature, ndegrees, dim, incl_orig):
    _check_input(in_feature, 'in_feature', torch.float32)
    dim, pre, post = _pe_shape(in_feature, dim)
    stride = 2 * int(ndegrees) + (1 if incl_orig else 0)
    shape = list(in_feature.shape)
    shape[dim] *= stride
    out = torch.empty(shape, dtype=torch.float32, device=in_feature.device)
    with torch.cuda.device(in_feature.device):
        code = _lib.lib().sdb_positional_encoding(_ptr(in_feature), _ptr(out), pre, post, int(ndegrees),
                                                  int(bool(incl_orig)), _stream(in_feature))
    _lib.check(code, 'positional_encoding')
    return out


def positional_encoding_backward(out_feature_grad, out_feature, ndegrees, dim, incl_orig):
    _check_input(out_feature_grad, 'out_feature_grad', torch.float32)
    _check_input(out_feature, 'out_feature', torch.float32)
    stride = 2 * int(ndegrees) + (1 if incl_orig else 0)
    d = dim % out_feature.dim()
    shape = list(out_feature.shape)
    shape[d] //= stride
    in_grad = torch.empty(shape, dtype=torch.float32, device=out_feature.device)
    _, pre, post = _pe_shape(in_grad, d)
    with torch.cuda.device(out_feature.device):
        code = _lib.lib().sdb_positional_encoding_backward(_ptr(out_feature_grad), _ptr(out_feature), _ptr(in_grad),
                                                           pre, post, int(ndegrees), int(bool(incl_orig)),
                                                           _stream(out_feature))
    _lib.check(code, 'positional_encoding_backward')
    return in_grad


def _sp_args(in_feature, corner_lut_t, in_worldcoord):
    _check_input(in_feature, 'in_feature', torch.float32)           # CHECK_CONTIGUOUS(in_feature) in the reference
    _check_cuda(corner_lut_t, 'in_corner_lut')
    _check_cuda(in_worldcoord, 'in_worldcoord')
    if in_feature.dim() != 2 or corner_lut_t.dim() != 3 or corner_lut_t.dtype != torch.int32:
        raise RuntimeError('sp_trilinear_worldcoord: in_feature must be [M, C] float32 and in_corner_lut a 3-D int32 tensor')
    if in_worldcoord.dtype != torch.float32 or in_worldcoord.shape[-1] != 3 or in_worldcoord.dim() > 8:
        raise RuntimeError('sp_trilinear_worldcoord: in_worldcoord must be float32 [..., 3] with at most 8 dimensions')
    dims = (ctypes.c_int64 * 3)(*corner_lut_t.shape)
    strides = (ctypes.c_int64 * 3)(*corner_lut_t.stride())         # any strides, like the reference (:401-406)
    wc = in_worldcoord.contiguous().reshape(-1, 3)
    return dims, strides, wc


def sp_trilinear_worldcoord(in_feature, corner_lut_t, in_worldcoord, ign_zero, channel_pos):
    """-> out_feature float32 [..., C] (voxlib.cpp:15).  channel_pos: -1 keeps the channels last in memory, e.g. -3 lays
    the result out channel-first ([.., C, H, W] in memory) while the returned view still has C last, like the
    reference's transposed allocation (sp_trilinear_worldcoord_kernel.cu:410-424)."""
    dims, strides, wc = _sp_args(in_feature, corner_lut_t, in_worldcoord)
    E, C = wc.shape[0], in_feature.shape[1]
    out = torch.empty(E, C, dtype=torch.float32, device=in_feature.device)
    with torch.cuda.device(in_feature.device):
        code = _lib.lib().sdb_sp_trilinear_worldcoord(_ptr(in_feature), int(in_feature.shape[0]), int(C), _ptr(corner_lut_t), dims,
                                                      strides, _ptr(wc), int(E), int(bool(ign_zero)), _ptr(out),
                                                      _stream(in_feature))
    _lib.check(code, 'sp_trilinear_worldcoord')
    out = out.reshape(tuple(in_worldcoord.shape[:-1]) + (C,))
    nd = in_worldcoord.dim()
    cp = channel_pos + nd if channel_pos < 0 else channel_pos
    if not 0 <= cp < nd:
        raise RuntimeError('sp_trilinear_worldcoord: channel_pos out of range')
    if cp != nd - 1:
        out = out.movedim(-1, cp).contiguous().movedim(cp, -1)
    return out


def sp_trilinear_worldcoord_backward(out_feature_grad, in_feature, corner_lut_t, in_worldcoord, ign_zero, need_coord_grad):
    """-> [in_feature_grad float32 [M, C]] (voxlib.cpp:17); coordinates get no gradient (the reference asserts
    need_coord_grad == false, sp_trilinear_worldcoord_kernel.cu:454)."""
    if need_coord_grad:
        raise RuntimeError('sp_trilinear_worldcoord_backward: need_coord_grad is not supported (nor by the reference)')
    _check_cuda(out_feature_grad, 'out_feature_grad')
    dims, strides, wc = _sp_args(in_feature, corner_lut_t, in_worldcoord)
    E, C = wc.shape[0], in_feature.shape[1]
    if out_feature_grad.dtype != torch.float32 or tuple(out_feature_grad.shape) != tuple(in_worldcoord.shape[:-1]) + (C,):
        raise RuntimeError('sp_trilinear_worldcoord_backward: out_feature_grad must be float32 [..., C]')
    g = out_feature_grad.contiguous().reshape(E, C)
    grad = torch.empty_like(in_feature)
    with torch.cuda.device(in_feature.device):
        code = _lib.lib().sdb_sp_trilinear_worldcoord_backward(_ptr(g), int(in_feature.shape[0]), int(C), _ptr(corner_lut_t), dims,
                                                               strides, _ptr(wc), int(E), int(bool(ign_zero)), _ptr(grad),
                                                               _stream(in_feature))
    _lib.check(code, 'sp_trilinear_worldcoord_backward')
    return [grad]


# ------------------------------------------------------------------------------------------------
# _gridencoder
# ------------------------------------------------------------------------------------------------
def _check_ge(t, name, floating=True, dtype=torch.float32):
    _check_input(t, name)
    if floating and t.dtype != dtype:
        raise RuntimeError('%s must be a %s tensor (the table\'s dtype decides: float32, or float16 for the reference\'s '
                           'autocast path; coordinates are always float32)' % (name, str(dtype).replace('torch.', '')))
    if not floating and t.dtype != torch.int32:
        raise RuntimeError('%s must be an int tensor' % name)


def _ge_dtype(embeddings, C):
    """The reference dispatches on the table's dtype (gridencoder.cu:442); float64 tables are not built here."""
    if embeddings.dtype == torch.float32:
        return torch.float32, ''
    if embeddings.dtype == torch.float16:
        if int(C) % 2:
            raise RuntimeError('GridEncoding: float16 tables need an even C (gridencoder/grid.py:38 keeps odd C in float32)')
        return torch.float16, '_f16'
    raise RuntimeError('embeddings must be a float32 or float16 tensor')


def grid_encode_forward(inputs, embeddings, offsets, outputs, B, D, C, L, S, H, calc_grad_inputs, dy_dx, gridtype,
                        align_corners):
    """Caller-allocated outputs [L,B,C] / dy_dx in the table's dtype, returns None (gridencoder.h:12)."""
    dt, sfx = _ge_dtype(embeddings, C)
    _check_ge(inputs, 'inputs')
    for t, n in ((embeddings, 'embeddings'), (outputs, 'outputs'), (dy_dx, 'dy_dx')):
        _check_ge(t, n, dtype=dt)
    _check_ge(offsets, 'offsets', floating=False)
    with torch.cuda.device(inputs.device):
        code = getattr(_lib.lib(), 'sdb_grid_encode_forward' + sfx)(
            _ptr(inputs), _ptr(embeddings), _ptr(offsets), _ptr(outputs), int(B), int(D), int(C), int(L), float(S),
            int(H), int(bool(calc_grad_inputs)), _ptr(dy_dx), int(gridtype), int(bool(align_corners)),
            _stream(inputs))
    if code == -2:
        raise RuntimeError('GridEncoding: D must be 2..5 and C must be 1, 2, 4, or 8.')
    _lib.check(code, 'grid_encode_forward')


def grid_encode_backward(grad, inputs, embeddings, offsets, grad_embeddings, B, D, C, L, S, H, calc_grad_inputs,
                         dy_dx, grad_inputs, gridtype, align_corners):
    dt, sfx = _ge_dtype(embeddings, C)
    _check_ge(inputs, 'inputs')
    for t, n in ((grad, 'grad'), (embeddings, 'embeddings'), (grad_embeddings, 'grad_embeddings'),
                 (dy_dx, 'dy_dx'), (grad_inputs, 'grad_inputs')):
        _check_ge(t, n, dtype=dt)
    _check_ge(offsets, 'offsets', floating=False)
    with torch.cuda.device(inputs.device):
        code = getattr(_lib.lib(), 'sdb_grid_encode_backward' + sfx)(
            _ptr(grad), _ptr(inputs), _ptr(embeddings), _ptr(offsets), _ptr(grad_embeddings), int(B), int(D), int(C),
            int(L), float(S), int(H), int(bool(calc_grad_inputs)), _ptr(dy_dx), _ptr(grad_inputs), int(gridtype),
            int(bool(align_corners)), _stream(inputs))
    if code == -2:
        raise RuntimeError('GridEncoding: D must be 2..5 and C must be 1, 2, 4, or 8.')
    _lib.check(code, 'grid_encode_backward')


# ------------------------------------------------------------------------------------------------
# f4: rejection statistics of the camera sampler
# ------------------------------------------------------------------------------------------------
def pose_stats(voxel_id, depth2, n_bins=680, out=None):
    """voxel_id [H,W,M,1] int32, depth2 [2,H,W,M,1] (a raycast result) -> float32 [2] on the device:
    (mean non-NaN first-hit depth, entropy of the first-hit voxel ids) -- scenedreamer.py:127-142, no host round trip."""
    _check_input(voxel_id, 'voxel_id', torch.int32)
    _check_input(depth2, 'depth2', torch.float32)
    H, W, M = voxel_id.shape[:3]
    L = _lib.lib()
    dev = voxel_id.device
    stats = out if out is not None else torch.empty(2, dtype=torch.float32, device=dev)
    ws = torch.empty(int(L.sdb_pose_stats_workspace_bytes(int(n_bins))), dtype=torch.uint8, device=dev)
    with torch.cuda.device(dev):
        code = L.sdb_pose_stats(_ptr(voxel_id), _ptr(depth2), int(H), int(W), int(M), int(n_bins), _ptr(stats), _ptr(ws), _stream(voxel_id))
    _lib.check(code, 'pose_stats')
    return stats


# ------------------------------------------------------------------------------------------------
# diagnostics
# ------------------------------------------------------------------------------------------------
def tc_selftest(a, b, bf16=False, variant=0):
    """C = A @ B^T through the library's wgmma path.  a [128,K], b [N,K] fp32 CUDA."""
    _check_input(a, 'a', torch.float32)
    _check_input(b, 'b', torch.float32)
    N, K = b.shape
    c = torch.empty(128, N, dtype=torch.float32, device=a.device)
    with torch.cuda.device(a.device):
        code = _lib.lib().sdb_tc_selftest(_ptr(a), _ptr(b), _ptr(c), int(N), int(K), int(bool(bf16)), int(variant),
                                          _stream(a))
    _lib.check(code, 'tc_selftest')
    return c
