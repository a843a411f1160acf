"""The precision-taking RenderCNN training entry points (include/sdb200.h, f1 under autograd at a chosen precision) and the
generator hook's SDB200_CNN_AMP switch, without a GPU: argument checks come before any CUDA call (the pointers handed over
are never dereferenced), sizes are arithmetic, and the hook runs with the engine replaced by a recorder."""
import ctypes
import types

import pytest
import torch

from scenedreamer_b200 import _lib, integration, rendercnn

EINVAL, EUNSUPPORTED = -1, -2
TRAIN = (0, 1, 3)                     # fp16 x1, bf16 x3, bf16 x1
BAD = (2, -1, 4, 7)


def test_pack_ex_accepts_every_pack_precision():
    L = _lib.lib()
    d = ctypes.c_void_p(0x1000)
    for p in (0, 1, 2):
        assert L.sdb_cnn_pack_bytes_ex(p) == L.sdb_cnn_pack_bytes(p) > 0
    assert L.sdb_cnn_pack_bytes_ex(3) == L.sdb_cnn_pack_bytes_ex(0)          # one 16-bit plane per weight, bf16 or fp16
    assert L.sdb_cnn_pack_bytes_ex(-1) == 0 and L.sdb_cnn_pack_bytes_ex(4) == 0
    for i in range(15):                                                        # every pointer, the pack included
        args = [d] * 15
        args[i] = None
        assert L.sdb_cnn_pack_ex(*args[:14], 3, args[14], None) == EINVAL
    assert L.sdb_cnn_pack_ex(*([d] * 14), 4, d, None) == EUNSUPPORTED
    assert L.sdb_cnn_pack_ex(*([d] * 14), -1, d, None) == EUNSUPPORTED
    # the old entry keeps its range
    assert L.sdb_cnn_pack_bytes(3) == 0 and L.sdb_cnn_pack(*([d] * 14), 3, d, None) == EUNSUPPORTED


def test_train_entries_refuse_bad_arguments():
    L = _lib.lib()
    d = ctypes.c_void_p(0x1000)
    for p in BAD:
        assert L.sdb_cnn_train_record_bytes_ex(8, 8, p) == 0
        assert L.sdb_cnn_backward_pack_bytes_ex(p) == 0
        assert L.sdb_cnn_backward_workspace_bytes_ex(8, 8, p) == 0
        assert L.sdb_cnn_train_forward_ex(d, 8, 8, d, d, p, d, None, d, None) == EUNSUPPORTED
        assert L.sdb_cnn_pack_backward_ex(*([d] * 7), p, d, None) == EUNSUPPORTED
        g = rendercnn._CnnGrads()
        assert L.sdb_cnn_backward_ex(8, 8, p, d, d, None, d, d, d, ctypes.byref(g), d, None) == EUNSUPPORTED
        out = (ctypes.c_int64 * 14)()
        assert L.sdb_cnn_debug_record_layout_ex(8, 8, p, out) == EUNSUPPORTED
    for p in TRAIN:
        assert L.sdb_cnn_train_record_bytes_ex(0, 8, p) == 0 and L.sdb_cnn_train_record_bytes_ex(8, -1, p) == 0
        assert L.sdb_cnn_backward_workspace_bytes_ex(0, 8, p) == 0 and L.sdb_cnn_backward_workspace_bytes_ex(8, 0, p) == 0
        assert L.sdb_cnn_backward_pack_bytes_ex(p) > 0
        # training forward: NULLs (d_rgb_raw may be NULL) and H / W <= 0 come before the precision
        for i in (0, 3, 4, 6, 8):
            args = [d, 8, 8, d, d, p, d, None, d, None]
            args[i] = None
            assert L.sdb_cnn_train_forward_ex(*args) == EINVAL, (p, i)
        assert L.sdb_cnn_train_forward_ex(d, 0, 8, d, d, p, d, None, d, None) == EINVAL
        assert L.sdb_cnn_train_forward_ex(d, 8, -2, d, d, p, d, None, d, None) == EINVAL
        assert L.sdb_cnn_train_forward_ex(None, 8, 8, d, d, 2, d, None, d, None) == EINVAL
        # backward pack
        for i in range(8):
            args = [d] * 8
            args[i] = None
            assert L.sdb_cnn_pack_backward_ex(*args[:7], p, args[7], None) == EINVAL
        # backward
        g = rendercnn._CnnGrads()
        gp = ctypes.byref(g)
        assert L.sdb_cnn_backward_ex(8, 8, p, None, d, d, d, d, d, gp, d, None) == EINVAL
        assert L.sdb_cnn_backward_ex(8, 8, p, d, None, None, d, d, d, gp, d, None) == EINVAL   # neither dL/d rgb nor dL/d raw
        assert L.sdb_cnn_backward_ex(8, 8, p, d, d, None, None, d, d, gp, d, None) == EINVAL
        assert L.sdb_cnn_backward_ex(8, 8, p, d, d, None, d, None, d, gp, d, None) == EINVAL
        assert L.sdb_cnn_backward_ex(8, 8, p, d, d, None, d, d, None, gp, d, None) == EINVAL
        assert L.sdb_cnn_backward_ex(8, 8, p, d, d, None, d, d, d, None, d, None) == EINVAL
        assert L.sdb_cnn_backward_ex(8, 8, p, d, d, None, d, d, d, gp, None, None) == EINVAL
        assert L.sdb_cnn_backward_ex(0, 8, p, d, d, None, d, d, d, gp, d, None) == EINVAL
        assert L.sdb_cnn_backward_ex(8, -1, p, d, None, d, d, d, d, gp, d, None) == EINVAL
        out = (ctypes.c_int64 * 14)()
        assert L.sdb_cnn_debug_record_layout_ex(0, 8, p, out) == EINVAL
        assert L.sdb_cnn_debug_record_layout_ex(8, 8, p, None) == EINVAL


@pytest.mark.parametrize('H,W', [(2, 5), (37, 150), (262, 262), (570, 990)])
def test_sizes_at_each_precision(H, W):
    L = _lib.lib()
    assert L.sdb_cnn_train_record_bytes_ex(H, W, 1) == L.sdb_cnn_train_record_bytes(H, W)
    assert L.sdb_cnn_backward_workspace_bytes_ex(H, W, 1) == L.sdb_cnn_backward_workspace_bytes(H, W)
    assert L.sdb_cnn_backward_pack_bytes_ex(1) == L.sdb_cnn_backward_pack_bytes()
    assert L.sdb_cnn_backward_pack_bytes_ex(0) == L.sdb_cnn_backward_pack_bytes_ex(3) == L.sdb_cnn_backward_pack_bytes() // 2
    Hp, Wp = H + 4, (W + 127) // 128 * 128 + 2
    up = lambda n: (n + 255) // 256 * 256
    plane = Hp * 32 * Wp * 16                                            # one 16-bit plane of 256 channels
    rgb = up(3 * H * W * 4)
    for p in (0, 3):
        # x (one plane of 64 channels), nine 256-channel activations (y1 t1 u2 y2 t2 u3 y3 t3 y4) of one plane, rgb fp32
        assert L.sdb_cnn_train_record_bytes_ex(H, W, p) == up(Hp * 8 * Wp * 16) + 9 * plane + rgb
        assert L.sdb_cnn_backward_workspace_bytes_ex(H, W, p) == 3 * plane
        assert 2 * L.sdb_cnn_train_record_bytes_ex(H, W, p) - rgb == L.sdb_cnn_train_record_bytes(H, W)     # half, but rgb
        assert 2 * L.sdb_cnn_backward_workspace_bytes_ex(H, W, p) == L.sdb_cnn_backward_workspace_bytes(H, W)
    if (H, W) == (262, 262):
        assert L.sdb_cnn_train_record_bytes_ex(H, W, 0) == 487_097_344          # 464.5 MiB, against 928.2 MiB at bf16 x3
        assert L.sdb_cnn_train_record_bytes(H, W) == 973_370_880


@pytest.mark.parametrize('precision', TRAIN)
def test_record_layout_ex_matches_record_size(precision):
    L = _lib.lib()
    out, old = (ctypes.c_int64 * 14)(), (ctypes.c_int64 * 14)()
    assert L.sdb_cnn_debug_record_layout_ex(262, 262, precision, out) == 0
    Hp, Wp, offs = out[0], out[1], list(out[2:])
    assert (Hp, Wp) == (266, 386)
    planes = 2 if precision == 1 else 1
    act = Hp * 32 * Wp * 16 * planes
    assert offs[0] == 0 and offs[1] == Hp * 8 * Wp * 16 * planes           # x first, 8 channels
    assert all(b - a == act for a, b in zip(offs[1:10], offs[2:11]))      # y1 .. y4 back to back, u right before its y
    assert offs[-1] == L.sdb_cnn_train_record_bytes_ex(262, 262, precision) and offs[-1] >= offs[10] + 3 * 262 * 262 * 4
    if precision == 1:
        assert L.sdb_cnn_debug_record_layout(262, 262, old) == 0 and list(old) == list(out)


# ---- the generator hook: SDB200_CNN_AMP parsing and routing, the engine replaced by a recorder ----------------------------
class _Net:
    """Just enough of the per-pixel feature map for the hook's checks."""
    is_cuda, dtype, shape, requires_grad = True, torch.float32, (1, 4, 4, 64), True

    def dim(self):
        return 4


def _fake_generator(calls):
    class Gen:                                               # stands in for imaginaire.generators.scenedreamer.Generator
        def _forward_perpix(self, *a):
            return ('ref',)

        def _forward_perpix_sub(self, *a):
            return ('ref',)

        def _forward_global(self, net_out, z):
            calls.append(('reference',))
            return 'ref'

    integration.install(Gen)
    gen = Gen()
    gen.denoiser = torch.nn.Linear(2, 2)
    st = integration._state(gen)

    class Engine:
        def forward_train(self, net_out, z, P, precision=rendercnn.PRECISION_BF16X3):
            calls.append(('train', precision))
            return 'train'

        def forward(self, net_out, z):
            calls.append(('inference',))
            return 'inf'
    st.get_cnn = lambda g: Engine()
    return gen, st


class _Autocast:
    """CUDA autocast state as torch.autocast('cuda', dtype) sets it, without needing a device."""

    def __init__(self, dtype):
        self.dtype = dtype

    def __enter__(self):
        self.old = (torch.is_autocast_enabled(), torch.get_autocast_dtype('cuda'))
        torch.set_autocast_enabled('cuda', True)
        torch.set_autocast_dtype('cuda', self.dtype)

    def __exit__(self, *a):
        torch.set_autocast_enabled('cuda', self.old[0])
        torch.set_autocast_dtype('cuda', self.old[1])


def test_switch_parsing(monkeypatch):
    monkeypatch.delenv('SDB200_CNN_AMP', raising=False)
    assert not integration.cnn_amp_enabled()
    for v, on in (('1', True), ('yes', True), ('0', False), ('off', False), ('false', False), ('False', False), ('', False)):
        monkeypatch.setenv('SDB200_CNN_AMP', v)
        assert integration.cnn_amp_enabled() == on, v
    with _Autocast(torch.float16):
        assert integration.cnn_amp_precision() == rendercnn.PRECISION_FP16 == 0
    with _Autocast(torch.bfloat16):
        assert integration.cnn_amp_precision() == rendercnn.PRECISION_BF16 == 3


def test_hook_routes_autocast_training_calls(monkeypatch):
    for k in ('SDB200_CNN_AMP', 'SDB200_CNN', 'SDB200_FUSED'):
        monkeypatch.delenv(k, raising=False)
    calls = []
    gen, st = _fake_generator(calls)
    f, net, z = integration.fused_forward_global, _Net(), torch.zeros(1, 256)
    s0 = dict(st.stats)
    delta = lambda: {k: st.stats[k] - s0[k] for k in ('cnn_train_calls', 'cnn_amp_train_calls', 'cnn_reference_calls')}

    assert f(gen, net, z) == 'train' and calls[-1] == ('train', rendercnn.PRECISION_BF16X3)     # no autocast: bf16 x3
    with _Autocast(torch.float16):
        assert f(gen, net, z) == 'ref'                                     # switch off (default): the reference, as before
    assert delta() == {'cnn_train_calls': 1, 'cnn_amp_train_calls': 0, 'cnn_reference_calls': 1}

    monkeypatch.setenv('SDB200_CNN_AMP', '1')
    with _Autocast(torch.float16):
        assert f(gen, net, z) == 'train' and calls[-1] == ('train', rendercnn.PRECISION_FP16)
    with _Autocast(torch.bfloat16):
        assert f(gen, net, z) == 'train' and calls[-1] == ('train', rendercnn.PRECISION_BF16)
    assert delta() == {'cnn_train_calls': 3, 'cnn_amp_train_calls': 2, 'cnn_reference_calls': 1}
    assert f(gen, net, z) == 'train' and calls[-1] == ('train', rendercnn.PRECISION_BF16X3)     # the switch is for autocast only
    assert delta()['cnn_amp_train_calls'] == 2

    # no gradients under autocast: the inference kernel, with or without the switch
    gen.denoiser.requires_grad_(False)
    nograd = _Net()
    nograd.requires_grad = False
    with _Autocast(torch.float16):
        assert f(gen, nograd, z) == 'inf' and calls[-1] == ('inference',)
    gen.denoiser.requires_grad_(True)

    # SDB200_CNN=0 and SDB200_FUSED=0 still win
    for k in ('SDB200_CNN', 'SDB200_FUSED'):
        monkeypatch.setenv(k, '0')
        with _Autocast(torch.bfloat16):
            assert f(gen, net, z) == 'ref' and calls[-1] == ('reference',)
        monkeypatch.delenv(k)
    assert delta() == {'cnn_train_calls': 4, 'cnn_amp_train_calls': 2, 'cnn_reference_calls': 3}


def test_forward_train_refuses_an_unknown_precision():
    eng = types.SimpleNamespace(prefix='denoiser.')
    net = types.SimpleNamespace(is_cuda=True, dtype=torch.float32, shape=(1, 2, 2, 64), dim=lambda: 4)
    for p in (rendercnn.PRECISION_FP16X3, 5):
        with pytest.raises(ValueError, match='training precision'):
            rendercnn.RenderCNNEngine.forward_train(eng, net, None, {}, precision=p)
