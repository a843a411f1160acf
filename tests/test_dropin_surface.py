"""CPU tests of the drop-in boundary: the C-ABI library loads and exports every symbol of
include/sdb200.h, the Python mirrors exist with the reference's names / signatures, and the
`gridencoder` package builds the same state (no compute calls without a GPU)."""
import ctypes
import inspect
import os
import re
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), '..'))
DROPIN = os.path.join(ROOT, 'dropin')


def test_library_exports_every_declared_symbol():
    from scenedreamer_b200 import _lib
    L = _lib.lib()
    hdr = open(os.path.join(ROOT, 'include', 'sdb200.h')).read()
    hdr = re.sub(r'/\*.*?\*/', '', hdr, flags=re.S)
    declared = set(re.findall(r'\b(sdb_[a-z0-9_]+)\s*\(', hdr)) - {'sdb_render_params'}
    assert len(declared) >= 18
    for name in sorted(declared):
        assert hasattr(L, name), 'libsdb200.so does not export %s' % name
        assert name in _lib.SIGNATURES, 'scenedreamer_b200/_lib.py has no signature for %s' % name
    assert L.sdb_version() >= 100
    assert b'sm_90a' in L.sdb_build_info()
    assert b'invalid' in L.sdb_error_string(-1)
    # host-only entry point: camera frame matches the oracle bit for bit
    import oracle
    f, s, u = (ctypes.c_float * 3)(), (ctypes.c_float * 3)(), (ctypes.c_float * 3)()
    L.sdb_camera_frame((ctypes.c_float * 3)(-45.25, 204.8, -409.6), (ctypes.c_float * 3)(1, 0, 0), f, s, u)
    of, os_, ou = oracle.camera_frame([-45.25, 204.8, -409.6], [1, 0, 0])
    assert list(f) == of.tolist() and list(s) == os_.tolist() and list(u) == ou.tolist()
    assert L.sdb_mlp_pack_bytes(2) > L.sdb_mlp_pack_bytes(0) > 700000
    assert L.sdb_render_workspace_bytes(1, 570, 990) == (72 * 62 + 8 + 570 * 990) * 4      # counters, tile list, camera slot, live-ray queue


def test_render_params_struct_matches_header():
    """ctypes mirror of sdb_render_params vs the C compiler's layout."""
    import subprocess
    import tempfile
    from scenedreamer_b200.render import _RenderParams
    src = '#include "%s"\n#include <stdio.h>\n#include <stddef.h>\nint main(){printf("%%zu", sizeof(sdb_render_params));' % \
          os.path.join(ROOT, 'include', 'sdb200.h')
    for name, _ in _RenderParams._fields_:
        src += 'printf(" %%zu", offsetof(sdb_render_params, %s));' % name
    src += 'return 0;}\n'
    with tempfile.TemporaryDirectory() as d:
        c = os.path.join(d, 't.c')
        open(c, 'w').write(src)
        subprocess.check_call(['gcc', c, '-o', os.path.join(d, 't')])
        vals = [int(v) for v in subprocess.check_output([os.path.join(d, 't')]).split()]
    assert vals[0] == ctypes.sizeof(_RenderParams)
    assert vals[1:] == [getattr(_RenderParams, n).offset for n, _ in _RenderParams._fields_]


@pytest.fixture()
def dropin_path():
    """dropin/ first on the path, then the reference's own Python (staged copy or /root/reference): the `gridencoder`
    package is the REFERENCE's, running on dropin/_gridencoder.py (gridencoder/grid.py:9-12 imports it by name)."""
    from oracle import refgen
    ref = refgen.reference_python_root()
    mods = ('voxlib', '_gridencoder', 'gridencoder', 'gridencoder.grid')
    sys.path.insert(0, DROPIN)
    if ref is not None:
        sys.path.insert(1, ref)
    for m in mods:
        sys.modules.pop(m, None)
    yield ref
    sys.path.remove(DROPIN)
    if ref is not None:
        sys.path.remove(ref)
    for m in mods:
        sys.modules.pop(m, None)


def test_voxlib_and_gridencoder_module_surface(dropin_path):
    import voxlib
    import _gridencoder
    # pybind table of the reference: voxlib/voxlib.cpp:25-31, gridencoder/src/bindings.cpp:5-8
    for name in ('ray_voxel_intersection_perspective', 'sp_trilinear_worldcoord', 'sp_trilinear_worldcoord_backward',
                 'positional_encoding', 'positional_encoding_backward'):
        assert callable(getattr(voxlib, name))
    assert list(inspect.signature(voxlib.ray_voxel_intersection_perspective).parameters) == [
        'in_voxel', 'cam_ori', 'cam_dir', 'cam_up', 'cam_f', 'cam_c', 'img_dims', 'max_samples']
    assert list(inspect.signature(voxlib.positional_encoding).parameters) == ['in_feature', 'ndegrees', 'dim', 'incl_orig']
    assert list(inspect.signature(_gridencoder.grid_encode_forward).parameters) == [
        'inputs', 'embeddings', 'offsets', 'outputs', 'B', 'D', 'C', 'L', 'S', 'H', 'calc_grad_inputs', 'dy_dx', 'gridtype',
        'align_corners']
    assert list(inspect.signature(_gridencoder.grid_encode_backward).parameters) == [
        'grad', 'inputs', 'embeddings', 'offsets', 'grad_embeddings', 'B', 'D', 'C', 'L', 'S', 'H', 'calc_grad_inputs',
        'dy_dx', 'grad_inputs', 'gridtype', 'align_corners']
    # CUDA-only like the reference (CHECK_CUDA): CPU tensors are rejected, nothing silently falls back
    with pytest.raises(RuntimeError):
        voxlib.ray_voxel_intersection_perspective(torch.zeros(4, 4, 4, dtype=torch.int32), [0., 0, 0], [1., 0, 0],
                                                  [0., 1, 0], 1.0, [0.5, 0.5], [2, 2], 2)
    with pytest.raises(RuntimeError):
        voxlib.positional_encoding(torch.zeros(3, 3), 2, -1, True)
    with pytest.raises(RuntimeError):
        voxlib.sp_trilinear_worldcoord(torch.zeros(4, 2), torch.zeros(2, 2, 2, dtype=torch.int32), torch.zeros(3, 3), False, -1)
    # import-time stand-ins of the two StyleGAN2 extensions imaginaire.layers hard-imports
    import bias_act_cuda
    import upfirdn2d_cuda
    with pytest.raises(RuntimeError):
        upfirdn2d_cuda.upfirdn2d(None)
    with pytest.raises(RuntimeError):
        bias_act_cuda.bias_act(None)


def test_gridencoder_module_state(dropin_path, golden_ops):
    if dropin_path is None:
        pytest.skip('reference Python not available (oracle/_ref/py, /root/reference)')
    from gridencoder import GridEncoder
    from gridencoder.grid import VarGridEncoder
    ge = GridEncoder(input_dim=5, num_levels=16, level_dim=8, base_resolution=16, log2_hashmap_size=19,
                     desired_resolution=2048, gridtype='hash', align_corners=False)
    assert torch.equal(ge.offsets, torch.from_numpy(golden_ops['ge5_offsets']))
    assert ge.per_level_scale == float(golden_ops['ge5_per_level_scale'][0])
    assert tuple(ge.embeddings.shape) == (8388608, 8) and ge.output_dim == 128
    assert set(ge.state_dict().keys()) == {'embeddings', 'offsets'}
    assert float(ge.embeddings.abs().max()) <= 1e-4
    ge3 = GridEncoder(input_dim=3, num_levels=8, level_dim=2, base_resolution=4, log2_hashmap_size=12, desired_resolution=64)
    assert torch.equal(ge3.offsets, torch.from_numpy(golden_ops['ge3_offsets']))
    v = VarGridEncoder(input_dim=3, num_levels=4, level_dim=2, base_resolution=4, log2_hashmap_size=10,
                       desired_resolution=32, gridtype='tiled', hash_entries=64)
    assert v.embeddings.shape[0] == v.offset - 64
    with pytest.raises(RuntimeError):
        ge3(torch.zeros(5, 3))          # CPU input: the backend refuses, like the reference's CHECK_CUDA


def test_integration_patch_is_importable():
    from scenedreamer_b200 import integration
    assert callable(integration.patch_generator) and callable(integration.fused_forward_perpix)
    assert list(inspect.signature(integration.fused_forward_perpix).parameters) == [
        'self', 'blk_feats', 'voxel_id', 'depth2', 'raydirs', 'cam_ori_t', 'z', 'global_enc']
