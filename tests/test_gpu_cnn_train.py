"""RenderCNN + tanh under autograd on the tensor cores (sdb_cnn_train_forward / sdb_cnn_backward, bf16 x3) against float64
autograd of the oracle's restatement, the reference's own RenderCNN module, and the reference composition through the
Generator hook."""
import os
import sys

import pytest
import torch

import oracle
from scenedreamer_b200 import rendercnn

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]
DEV = 'cuda:0'


def _inputs(H, W, seed=0):
    g = torch.Generator().manual_seed(seed)
    net_out = (torch.rand(1, H, W, 64, generator=g) * 2 - 1).to(DEV)
    z = torch.randn(1, 256, generator=g).to(DEV)
    P = {k: v.to(DEV) for k, v in oracle.make_cnn_params(seed + 1).items()}
    G = (torch.randn(1, 3, H, W, generator=g).to(DEV), torch.randn(1, 3, H, W, generator=g).to(DEV))
    return net_out, z, P, G


def _rel(a, b):
    a, b = a.double(), b.double()
    return float((a - b).norm() / b.norm().clamp_min(1e-300))


def _grads(fn, net_out, z, P, G, which, dtype):
    x = net_out.detach().to(dtype).clone().requires_grad_(True)
    zz = z.detach().to(dtype).clone().requires_grad_(True)
    Q = {k: v.detach().to(dtype).clone().requires_grad_(True) for k, v in P.items()}
    rgb, raw = fn(x, zz, Q)
    loss = 0
    if which in ('rgb', 'both'):
        loss = loss + (rgb * G[0].to(dtype)).sum()
    if which in ('raw', 'both'):
        loss = loss + (raw * G[1].to(dtype)).sum()
    loss.backward()
    return rgb.detach(), {'net_out': x.grad, 'z': zz.grad, **{k: v.grad for k, v in Q.items()}}


def _ours(x, z, Q):
    return rendercnn.RenderCNNEngine(Q).forward_train(x, z, Q)


def _oracle(x, z, Q):
    return oracle.render_cnn(x, z, Q, dtype=torch.float64)


_SIGMA_OUT = (('y1', 3), ('t1', 4), ('y2', 6), ('t2', 7), ('y3', 9), ('t3', 10), ('y4', 11))


def _recorded_signs(rec, H, W):
    """LeakyReLU outputs > 0, as the training forward recorded them (the hi bf16 plane of each sigma output)."""
    import ctypes
    from scenedreamer_b200 import _lib
    lay = (ctypes.c_int64 * 14)()
    assert _lib.lib().sdb_cnn_debug_record_layout(H, W, lay) == 0
    Hp, Wp = lay[0], lay[1]
    n = Hp * 32 * Wp * 16
    out = {}
    for name, i in _SIGMA_OUT:
        hi = rec[lay[i]:lay[i] + n].view(torch.bfloat16).reshape(Hp, 32, Wp, 8)[1:H + 1, :, 1:W + 1, :]
        out[name] = (hi.permute(1, 3, 0, 2).reshape(1, 256, H, W) > 0)
    return out


def _masked_f64(signs):
    """RenderCNN + tanh in float64 whose LeakyReLU slopes are the recorded ones: it separates the arithmetic of the path
    (bf16 x3 products, fp32 sums) from the slopes that flip where a value within the split's ~2^-17 error crosses zero."""
    import torch.nn.functional as F

    def fn(x, z, Q):
        W = lambda n: Q['denoiser.' + n]
        act = lambda t, name: torch.where(signs[name], t, 0.2 * t)
        mod = lambda t, w, b: t * (w[..., None, None] + 1) + b[..., None, None]
        m = torch.chunk(F.linear(z, W('fc_z_cond.weight'), W('fc_z_cond.bias')), 4, dim=-1)
        x = x.permute(0, 3, 1, 2)
        y1 = act(F.conv2d(x, W('conv1.weight'), W('conv1.bias')), 'y1')
        t1 = act(F.conv2d(y1, W('conv2a.weight'), W('conv2a.bias'), padding=1), 't1')
        y2 = act(mod(y1 + F.conv2d(t1, W('conv2b.weight'), None, padding=1), m[0], m[1]), 'y2')
        t2 = act(F.conv2d(y2, W('conv3a.weight'), W('conv3a.bias'), padding=1), 't2')
        y3 = act(mod(y2 + F.conv2d(t2, W('conv3b.weight'), None, padding=1), m[2], m[3]), 'y3')
        t3 = act(F.conv2d(y3, W('conv4a.weight'), W('conv4a.bias')), 't3')
        y4 = act(y3 + F.conv2d(t3, W('conv4b.weight'), W('conv4b.bias')), 'y4')
        raw = F.conv2d(y4, W('conv4.weight'), W('conv4.bias'))
        return torch.tanh(raw), raw
    return fn


# Against float64 autograd the slopes of the path flip where an activation within bf16 x3's error of zero crosses it:
# rel-L2 ~3e-3 on frames of thousands of pixels.  2 x 5 has 10 pixels, where a handful of flips decide the norm, so its bar
# is statistical.  With the recorded slopes the path is held to its arithmetic.
_TOL_F64 = {(37, 150): 1e-2, (8, 128): 1e-2, (2, 5): 5e-2, (262, 262): 1e-2}
_TOL_MASKED = 1e-4


@pytest.mark.parametrize('which', ['rgb', 'raw', 'both'])
@pytest.mark.parametrize('H,W', [(37, 150), (8, 128), (2, 5), (262, 262)])
def test_cnn_gradients_match_float64_autograd(H, W, which):
    net_out, z, P, G = _inputs(H, W)
    captured = {}

    def ours(x, zz, Q):
        rgb, raw = _ours(x, zz, Q)
        captured['signs'] = _recorded_signs(rgb.grad_fn.records[0], H, W)
        return rgb, raw

    rgb, got = _grads(ours, net_out, z, P, G, which, torch.float32)
    ref_rgb, ref = _grads(_oracle, net_out, z, P, G, which, torch.float64)
    _, masked = _grads(_masked_f64(captured['signs']), net_out, z, P, G, which, torch.float64)
    e_fwd = float((rgb.double() - ref_rgb).abs().max())
    errs = {k: _rel(got[k], ref[k]) for k in ref}
    errs_m = {k: _rel(got[k], masked[k]) for k in ref}
    short = lambda d: ' '.join('%s %.1e' % (k.replace('denoiser.', ''), v) for k, v in d.items())
    print('RenderCNN train %dx%d (%s): max|tanh - f64| %.2e\n  rel-L2 vs f64 %s\n  rel-L2 vs f64 with recorded slopes %s' % (
        H, W, which, e_fwd, short(errs), short(errs_m)))
    assert e_fwd <= 1e-4
    for k in ref:
        assert errs_m[k] <= _TOL_MASKED, (k, errs_m[k])
        assert errs[k] <= _TOL_F64[(H, W)], (k, errs[k])


def test_cnn_second_backward_raises_and_frozen_weights_get_no_gradient():
    net_out, z, P, G = _inputs(8, 128)
    Q = {k: v.clone().requires_grad_(k == 'denoiser.fc_z_cond.weight') for k, v in P.items()}
    x = net_out.clone().requires_grad_(True)
    rgb, raw = rendercnn.RenderCNNEngine(Q).forward_train(x, z, Q)
    loss = (rgb * G[0]).sum()
    loss.backward(retain_graph=True)
    assert x.grad is not None and Q['denoiser.fc_z_cond.weight'].grad is not None
    assert Q['denoiser.conv2a.weight'].grad is None
    with pytest.raises(RuntimeError, match='released by its first backward'):
        loss.backward()


def test_cnn_gradients_match_reference_module():
    """The reference's own RenderCNN (fp32, TF32 off) under autograd at 262 x 262: every parameter gradient."""
    from oracle import refgen
    ref_root = refgen.reference_python_root()
    if ref_root is None:
        pytest.skip('reference Python not staged')
    for pth in (ref_root, os.path.join(refgen.ROOT, 'dropin'), refgen.STUBS):
        if pth not in sys.path:
            sys.path.append(pth)
    from imaginaire.generators.gancraft_base import RenderCNN
    net_out, z, P, G = _inputs(262, 262, seed=3)
    mod = RenderCNN(64, style_dim=256).to(DEV)
    mod.load_state_dict({k[len('denoiser.'):]: v for k, v in P.items()})
    old = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    try:
        raw = mod(net_out.permute(0, 3, 1, 2).contiguous(), z)
        (torch.tanh(raw) * G[0]).sum().backward()
    finally:
        torch.backends.cudnn.allow_tf32 = old
    _, ours = _grads(_ours, net_out, z, P, G, 'rgb', torch.float32)
    for k, v in mod.named_parameters():
        e = _rel(ours['denoiser.' + k], v.grad)
        print('reference RenderCNN %s: rel-L2 %.2e' % (k, e))
        assert e <= 1e-2, (k, e)


def test_generator_training_step_runs_the_cnn_backward():
    """Generator.forward under autograd through the hook: the CNN takes the tensor-core training path, and its gradients
    match the same seeded step with SDB200_CNN=0 (the reference's composition, TF32 off)."""
    from test_gpu_generator import _have_reference
    if not _have_reference():
        pytest.skip('reference Python / extensions not staged in oracle/_ref (oracle/build_ref.py)')
    from oracle import refgen
    refgen.setup('dropin')
    gen, _ = refgen.build_generator(1024, DEV)
    refgen.set_world(gen, refgen.synthetic_world(1024), DEV)
    from scenedreamer_b200 import integration, ops
    integration.ensure_installed()
    import imaginaire.model_utils.gancraft.camctl as camctl
    vox = gen.voxel.voxel_t
    pose = camctl.EvalCameraController(gen.voxel, maxstep=8, pattern=0, cam_ang=72)[1]
    H = W = 64 + gen.pad
    vid, dep, rd = ops.ray_voxel_intersection_perspective(vox, pose[0], pose[1], pose[2], pose[3] * (W - 1),
                                                          [(H - 1) / 2, (W - 1) / 2], [H, W], 6)
    data = dict(images=torch.zeros(1, 3, 64, 64, device=DEV), voxel_id=vid.unsqueeze(0), depth2=dep.unsqueeze(0),
                raydirs=rd.unsqueeze(0), cam_ori_t=pose[0].unsqueeze(0).to(DEV))
    names = ('denoiser.conv2a.weight', 'denoiser.fc_z_cond.weight', 'render_net.fc_1.weight', 'hash_encoder.embeddings')
    params = dict(gen.named_parameters())
    qs = [params[n] for n in names] + list(gen.denoiser.parameters())
    gen.coarse_deterministic_sampling = False
    gen.num_samples = 24
    old_tf32 = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False

    def step(cnn):
        os.environ['SDB200_CNN'] = cnn
        for q in qs:
            q.requires_grad_(True)
            q.grad = None
        if hasattr(gen, 'sky_avg'):
            del gen.sky_avg
        torch.manual_seed(5)
        out = gen(data, random_style=True)
        loss = out['fake_images'].square().mean()
        loss.backward(retain_graph=True)
        return loss, {n: params[n].grad.clone() for n in names}

    try:
        _, ref = step('0')
        st = gen._sdb200.stats
        before = (st['cnn_train_calls'], st['cnn_reference_calls'])
        loss, ours = step('1')
        assert st['cnn_train_calls'] == before[0] + 1 and st['cnn_reference_calls'] == before[1]
        for n in names:
            e = _rel(ours[n], ref[n])
            print('generator step %s: rel-L2 vs reference CNN %.2e' % (n, e))
            assert e <= 1e-2, (n, e)
        with pytest.raises(RuntimeError, match='released by its first backward'):
            loss.backward()
    finally:
        os.environ.pop('SDB200_CNN', None)
        torch.backends.cudnn.allow_tf32 = old_tf32
        for q in qs:
            q.requires_grad_(False)
            q.grad = None
