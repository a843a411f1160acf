"""ctypes loader for libsdb200.so (include/sdb200.h).  Fails loudly: there is no fallback path."""
import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, 'libsdb200.so')
_lib = None

c_void_p, c_int, c_i32, c_u32, c_i64, c_f32 = (ctypes.c_void_p, ctypes.c_int, ctypes.c_int32, ctypes.c_uint32,
                                               ctypes.c_int64, ctypes.c_float)
_F3 = ctypes.POINTER(ctypes.c_float)

# every symbol include/sdb200.h declares: name -> (restype, argtypes)
SIGNATURES = {
    'sdb_version': (c_int, []),
    'sdb_build_info': (ctypes.c_char_p, []),
    'sdb_error_string': (ctypes.c_char_p, [c_int]),
    'sdb_camera_frame': (None, [_F3, _F3, _F3, _F3, _F3]),
    'sdb_ray_voxel_intersection_perspective': (c_int, [
        c_void_p, ctypes.POINTER(c_i64), ctypes.POINTER(c_i64), _F3, _F3, _F3, c_f32, _F3,
        ctypes.POINTER(c_i32), c_i32, c_void_p, c_void_p, c_void_p, c_void_p]),
    'sdb_height_bound_elems': (c_i64, [ctypes.POINTER(c_i64), c_i32]),
    'sdb_build_height_bound': (c_int, [c_void_p, ctypes.POINTER(c_i64), ctypes.POINTER(c_i64), c_i32, c_void_p, c_void_p]),
    'sdb_ray_voxel_intersection_perspective_ex': (c_int, [
        c_void_p, ctypes.POINTER(c_i64), ctypes.POINTER(c_i64), _F3, _F3, _F3, c_f32, _F3,
        ctypes.POINTER(c_i32), c_i32, c_void_p, c_void_p, c_void_p, c_void_p, c_i32, c_void_p]),
    'sdb_ray_voxel_intersection_perspective_bands': (c_int, [
        c_void_p, ctypes.POINTER(c_i64), ctypes.POINTER(c_i64), _F3, _F3, _F3, c_f32, _F3,
        ctypes.POINTER(c_i32), c_i32, ctypes.POINTER(c_i32), c_void_p, c_void_p, c_void_p, c_void_p, c_i32, c_void_p]),
    'sdb_grid_encode_forward': (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_u32, c_u32, c_u32, c_u32, c_f32,
                                        c_u32, c_int, c_void_p, c_u32, c_int, c_void_p]),
    'sdb_grid_encode_backward': (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_u32, c_u32, c_u32,
                                         c_u32, c_f32, c_u32, c_int, c_void_p, c_void_p, c_u32, c_int, c_void_p]),
    'sdb_grid_encode_forward_f16': (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_u32, c_u32, c_u32, c_u32, c_f32,
                                        c_u32, c_int, c_void_p, c_u32, c_int, c_void_p]),
    'sdb_grid_encode_backward_f16': (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_u32, c_u32, c_u32,
                                         c_u32, c_f32, c_u32, c_int, c_void_p, c_void_p, c_u32, c_int, c_void_p]),
    'sdb_positional_encoding': (c_int, [c_void_p, c_void_p, c_i64, c_i64, c_i32, c_int, c_void_p]),
    'sdb_positional_encoding_backward': (c_int, [c_void_p, c_void_p, c_void_p, c_i64, c_i64, c_i32, c_int, c_void_p]),
    'sdb_sp_trilinear_worldcoord': (c_int, [c_void_p, c_i64, c_i32, c_void_p, ctypes.POINTER(c_i64), ctypes.POINTER(c_i64),
                                            c_void_p, c_i64, c_int, c_void_p, c_void_p]),
    'sdb_sp_trilinear_worldcoord_backward': (c_int, [c_void_p, c_i64, c_i32, c_void_p, ctypes.POINTER(c_i64),
                                                     ctypes.POINTER(c_i64), c_void_p, c_i64, c_int, c_void_p, c_void_p]),
    'sdb_render_workspace_bytes': (c_i64, [c_i32, c_i32, c_i32]),
    'sdb_render_rays_forward': (c_int, [c_void_p, c_void_p]),
    'sdb_preblend_table': (c_int, [c_void_p, c_void_p, c_i32, c_i32, c_f32, c_i32, c_void_p, c_void_p]),
    'sdb_mlp_pack_bytes': (c_i64, [c_i32]),
    'sdb_pack_mlp': (c_int, [c_void_p, c_void_p, c_void_p, c_i32, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                             c_void_p, c_i32, c_void_p, c_void_p]),
    'sdb_sky_pack_bytes': (c_i64, [c_i32]),
    'sdb_pack_sky_mlp': (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_i32, c_void_p, c_void_p]),
    'sdb_sky_workspace_bytes': (c_i64, [c_i32, c_i32, c_i32]),
    'sdb_sky_forward': (c_int, [c_void_p, c_i32, c_i32, c_i32, c_void_p, c_i64, c_i32, c_void_p, c_void_p, c_void_p,
                                c_void_p]),
    'sdb_render_train_record_bytes': (c_i64, [c_i32, c_i32, c_i32, c_i32]),
    'sdb_render_rays_train_forward': (c_int, [c_void_p, c_void_p, c_void_p]),
    'sdb_mlp_backward_pack_bytes': (c_i64, []),
    'sdb_pack_mlp_backward': (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    'sdb_render_backward_workspace_bytes': (c_i64, [c_i32, c_i32, c_i32, c_i32, c_i32, c_i32]),
    'sdb_render_rays_backward': (c_int, [c_void_p, c_void_p, c_void_p, c_void_p]),
    'sdb_sky_train_record_bytes': (c_i64, [c_i32, c_i32, c_i32]),
    'sdb_sky_train_forward': (c_int, [c_void_p, c_i32, c_i32, c_i32, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    'sdb_sky_backward_pack_bytes': (c_i64, []),
    'sdb_pack_sky_mlp_backward': (c_int, [c_void_p, c_void_p, c_void_p, c_void_p]),
    'sdb_sky_backward_workspace_bytes': (c_i64, [c_i32, c_i32, c_i32]),
    'sdb_sky_backward': (c_int, [c_i32, c_i32, c_i32, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                 c_void_p]),
    'sdb_render_rays_backward_views': (c_int, [c_void_p, c_void_p, c_void_p, c_void_p]),
    'sdb_render_rays_backward_recompute': (c_int, [c_void_p, c_void_p, c_void_p, c_void_p]),
    'sdb_sky_train_forward_views': (c_int, [c_void_p, c_i32, c_i32, c_i32, c_void_p, c_i64, c_void_p, c_void_p, c_void_p, c_void_p,
                                            c_void_p]),
    'sdb_sky_backward_views': (c_int, [c_i32, c_i32, c_i32, c_void_p, c_void_p, c_void_p, c_i64, c_void_p, c_void_p, c_void_p]),
    'sdb_cnn_pack_bytes': (c_i64, [c_i32]),
    'sdb_cnn_pack': (c_int, [c_void_p] * 14 + [c_i32, c_void_p, c_void_p]),
    'sdb_cnn_workspace_bytes': (c_i64, [c_i32, c_i32, c_i32]),
    'sdb_cnn_forward': (c_int, [c_void_p, c_i32, c_i32, c_void_p, c_void_p, c_i32, c_void_p, c_void_p, c_void_p, c_i32, c_void_p]),
    'sdb_cnn_train_record_bytes': (c_i64, [c_i32, c_i32]),
    'sdb_cnn_train_forward': (c_int, [c_void_p, c_i32, c_i32, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    'sdb_cnn_backward_pack_bytes': (c_i64, []),
    'sdb_cnn_pack_backward': (c_int, [c_void_p] * 9),
    'sdb_cnn_backward_workspace_bytes': (c_i64, [c_i32, c_i32]),
    'sdb_cnn_backward': (c_int, [c_i32, c_i32, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                 c_void_p]),
    'sdb_cnn_pack_bytes_ex': (c_i64, [c_i32]),
    'sdb_cnn_pack_ex': (c_int, [c_void_p] * 14 + [c_i32, c_void_p, c_void_p]),
    'sdb_cnn_train_record_bytes_ex': (c_i64, [c_i32, c_i32, c_i32]),
    'sdb_cnn_train_forward_ex': (c_int, [c_void_p, c_i32, c_i32, c_void_p, c_void_p, c_i32, c_void_p, c_void_p, c_void_p, c_void_p]),
    'sdb_cnn_backward_pack_bytes_ex': (c_i64, [c_i32]),
    'sdb_cnn_pack_backward_ex': (c_int, [c_void_p] * 7 + [c_i32, c_void_p, c_void_p]),
    'sdb_cnn_backward_workspace_bytes_ex': (c_i64, [c_i32, c_i32, c_i32]),
    'sdb_cnn_backward_ex': (c_int, [c_i32, c_i32, c_i32, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                    c_void_p, c_void_p]),
    'sdb_cnn_debug_record_layout_ex': (c_int, [c_i32, c_i32, c_i32, ctypes.POINTER(c_i64)]),
    'sdb_adam_step': (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_i64, ctypes.c_double, ctypes.c_double, ctypes.c_double,
                              ctypes.c_double, c_i64, c_void_p]),
    'sdb_pose_stats_workspace_bytes': (c_i64, [c_i32]),
    'sdb_pose_stats': (c_int, [c_void_p, c_void_p, c_i32, c_i32, c_i32, c_i32, c_void_p, c_void_p, c_void_p]),
    'sdb_world_build': (c_int, [c_void_p, c_void_p, c_i32, c_i32, c_i32, c_void_p, c_i32, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                c_void_p, c_void_p]),
    'sdb_world_truncate': (c_int, [c_void_p, c_i32, c_i32, c_i32, c_i32, c_void_p, c_void_p]),
    'sdb_scene_scatter': (c_int, [c_void_p, c_i64, c_i32, c_i32, c_i32, c_i32, c_i32, c_void_p, c_void_p]),
    'sdb_launch_count': (c_i64, []),
    'sdb_debug_train_layout': (c_int, [c_i32, c_i32, c_i32, c_i32, c_i32, c_i32, ctypes.POINTER(c_i64)]),
    'sdb_cnn_debug_record_layout': (c_int, [c_i32, c_i32, ctypes.POINTER(c_i64)]),
    'sdb_debug_set_progress_buffer': (None, [c_void_p]),
    'sdb_modulate_forward': (c_int, [ctypes.POINTER(c_void_p), c_void_p, c_i32, c_i32, c_i32, c_void_p, c_void_p, c_void_p, c_void_p]),
    'sdb_modulate_backward': (c_int, [ctypes.POINTER(c_void_p), ctypes.POINTER(c_void_p), c_void_p, c_void_p, c_void_p, c_void_p,
                                      c_i32, c_i32, c_i32, c_void_p, c_void_p, c_void_p]),
    'sdb_tc_selftest_mn': (c_int, [c_void_p, c_void_p, c_void_p, c_i32, c_i32, c_void_p]),
    'sdb_tc_selftest': (c_int, [c_void_p, c_void_p, c_void_p, c_i32, c_i32, c_i32, c_i32, c_void_p]),
}


def lib():
    """The loaded library; builds it first if the .so is missing and nvcc is available."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            # one process per GPU: only one of them may run nvcc into the shared _obj/ directory; the others wait on the lock
            # and find the finished library (build() re-checks its stamp under the lock)
            import fcntl
            from . import build as _build
            with open(LIB_PATH + '.lock', 'w') as lk:
                fcntl.flock(lk, fcntl.LOCK_EX)
                try:
                    _build.build()
                finally:
                    fcntl.flock(lk, fcntl.LOCK_UN)
        if not os.path.exists(LIB_PATH):
            raise RuntimeError('scenedreamer_b200: %s is missing and could not be built; '
                               'this package has no CPU or PyTorch fallback' % LIB_PATH)
        L = ctypes.CDLL(LIB_PATH)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(L, name)          # AttributeError here == header/library mismatch: fail loudly
            fn.restype = res
            fn.argtypes = args
        _lib = L
    return _lib


def check(code, what):
    if code != 0:
        msg = lib().sdb_error_string(int(code)).decode()
        raise RuntimeError('%s failed: %s (code %d)' % (what, msg, code))
