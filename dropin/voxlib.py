"""Drop-in for the reference's top-level `voxlib` extension module (GANcraft voxlib).

The reference imports it as `import voxlib` / `from voxlib import ray_voxel_intersection_perspective`
(imaginaire/model_utils/gancraft/voxlib/{__init__,positional_encoding,sp_trilinear}.py) and the
pybind table it expects is imaginaire/model_utils/gancraft/voxlib/voxlib.cpp:25-31.  Put this
directory (dropin/) on PYTHONPATH ahead of any built reference extension and the reference's
Python runs unchanged on the H100-native kernels of libsdb200 (scenedreamer_b200.ops).

Importing this module also arms the fused per-pixel path: `imaginaire.generators.scenedreamer.Generator`
is patched at class level as soon as it exists (scenedreamer_b200.integration; SDB200_FUSED=0 turns that off),
so inference.py / train.py need no edit.
"""
from scenedreamer_b200 import integration as _integration
from scenedreamer_b200 import ops as _ops

_integration.install_import_hook()


def ray_voxel_intersection_perspective(in_voxel, cam_ori, cam_dir, cam_up, cam_f, cam_c, img_dims, max_samples):
    """voxlib.cpp:11 -- exactly the reference's eight positional arguments.  The empty-space bound of the volume is
    built on first use and cached per voxel tensor (scenedreamer_b200.ops.height_bound); results are bit-identical."""
    _integration.ensure_installed()
    return _ops.ray_voxel_intersection_perspective(in_voxel, cam_ori, cam_dir, cam_up, cam_f, cam_c, img_dims, max_samples)


def positional_encoding(in_feature, ndegrees, dim, incl_orig):
    """voxlib.cpp:20."""
    _integration.ensure_installed()
    return _ops.positional_encoding(in_feature, ndegrees, dim, incl_orig)


def positional_encoding_backward(out_feature_grad, out_feature, ndegrees, dim, incl_orig):
    """voxlib.cpp:22."""
    return _ops.positional_encoding_backward(out_feature_grad, out_feature, ndegrees, dim, incl_orig)


def sp_trilinear_worldcoord(in_feature, corner_lut_t, in_worldcoord, ign_zero, channel_pos):
    """voxlib.cpp:15."""
    return _ops.sp_trilinear_worldcoord(in_feature, corner_lut_t, in_worldcoord, ign_zero, channel_pos)


def sp_trilinear_worldcoord_backward(out_feature_grad, in_feature, corner_lut_t, in_worldcoord, ign_zero, need_coord_grad):
    """voxlib.cpp:17."""
    return _ops.sp_trilinear_worldcoord_backward(out_feature_grad, in_feature, corner_lut_t, in_worldcoord, ign_zero,
                                                 need_coord_grad)
