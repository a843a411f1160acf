"""RenderCNN + tanh trained in one 16-bit pass (sdb_cnn_*_ex at precision 0 = fp16 and 3 = bf16), the path the generator hook
takes under torch.autocast with SDB200_CNN_AMP=1:

  * the fp16 training forward computes what the fp16 inference forward computes, bit for bit; the bf16 one is held to the
    reference composition's own distance to float64 under bf16 autocast;
  * its gradients against float64 autograd with the slopes the record holds (the path's arithmetic) and with their own
    slopes, per tensor, against the reference composition's distance under the same autocast;
  * precision 1 of the _ex entries is the bf16 x3 path of the entries without _ex, bit for bit;
  * the real Generator under fp16 autocast with the switch on, and under torch.amp.GradScaler.
Bounds are at most 4x the worst value measured on an NVIDIA H100 80GB HBM3 (power limit 700 W); DESIGN.md section 4."""
import ctypes

import pytest
import torch
import torch.nn.functional as F

import oracle
from scenedreamer_b200 import _lib, integration, rendercnn
from test_gpu_cnn_train import _grads, _inputs, _masked_f64, _oracle, _rel
from test_gpu_train_views import generator  # noqa: F401  (module fixture)

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1800)]
DEV = 'cuda:0'
AMP_DTYPE = {rendercnn.PRECISION_FP16: torch.float16, rendercnn.PRECISION_BF16: torch.bfloat16}
PLANE_DTYPE = AMP_DTYPE
VS_COMPOSITION = 2.0          # our distance to float64 <= this x the reference composition's own under the same autocast, per
                              # tensor (worst measured ratio 1.61, fp16 at 2 x 5; 1.36 at 37 x 150, 1.11 at 262 x 262; the bf16
                              # forward 0.61)
TOL_MASKED = {rendercnn.PRECISION_FP16: 4e-3,     # rel-L2 vs float64 with the recorded slopes (worst measured 1.19e-3)
              rendercnn.PRECISION_BF16: 7e-2}     # (worst measured 1.88e-2)
GEN_GRAD_TOL = 3e-2           # Generator under fp16 autocast, SDB200_CNN_AMP=1 vs SDB200_CNN=0, rel-L2 per parameter (worst
                              # measured 7.7e-3, render_net.fc_1.weight; 7.9e-4 .. 3.0e-3 on the denoiser)
REORDER_TOL = 9e-7            # rel-L2 between two runs of a gradient summed with float atomics (run-to-run order only;
                              # worst measured 2.35e-7, the old entry against itself and _ex(1) against it alike)


def _p(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def _check(rc, what):
    assert rc == 0, (what, rc)


def _mod(P, z):
    return F.linear(z, P['denoiser.fc_z_cond.weight'], P['denoiser.fc_z_cond.bias']).reshape(4, 256).contiguous()


def _pack(L, P, precision, old=False):
    ts = [P['denoiser.' + n].float().contiguous() for n in rendercnn._NAMES]
    pk = torch.zeros(int(L.sdb_cnn_pack_bytes_ex(precision)), dtype=torch.uint8, device=DEV)      # the tail padding too
    fn = L.sdb_cnn_pack if old else L.sdb_cnn_pack_ex
    _check(fn(*[_p(t) for t in ts], precision, _p(pk), None), 'pack')
    return pk


def _amp(precision):
    return torch.autocast('cuda', dtype=AMP_DTYPE[precision])


def _train_node(rgb):
    node = rgb.grad_fn
    while not hasattr(node, 'records'):                      # under autocast: the cast to autocast's dtype comes first
        node = node.next_functions[0][0]
    return node


def _recorded_signs(rec, H, W, precision):
    """LeakyReLU outputs > 0 as the one-pass training forward recorded them (its single plane of each sigma output)."""
    lay = (ctypes.c_int64 * 14)()
    assert _lib.lib().sdb_cnn_debug_record_layout_ex(H, W, precision, lay) == 0
    Hp, Wp = lay[0], lay[1]
    n = Hp * 32 * Wp * 16
    out = {}
    for name, i in (('y1', 3), ('t1', 4), ('y2', 6), ('t2', 7), ('y3', 9), ('t3', 10), ('y4', 11)):
        pl = rec[lay[i]:lay[i] + n].view(PLANE_DTYPE[precision]).reshape(Hp, 32, Wp, 8)[1:H + 1, :, 1:W + 1, :]
        out[name] = (pl.permute(1, 3, 0, 2).reshape(1, 256, H, W) > 0)
    return out


# ---- 1. forward ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('H,W', [(37, 150), (262, 262)])
def test_fp16_train_forward_equals_inference_forward(H, W):
    L = _lib.lib()
    net_out, z, P, _ = _inputs(H, W)
    pk = _pack(L, P, 0)
    m = _mod(P, z)
    x = net_out[0].contiguous()
    rgb_i, raw_i, rgb_t, raw_t = [torch.full((3, H, W), float('nan'), device=DEV) for _ in range(4)]
    ws = torch.empty(int(L.sdb_cnn_workspace_bytes(H, W, 0)), dtype=torch.uint8, device=DEV)
    rec = torch.empty(int(L.sdb_cnn_train_record_bytes_ex(H, W, 0)), dtype=torch.uint8, device=DEV)
    _check(L.sdb_cnn_forward(_p(x), H, W, _p(pk), _p(m), 0, _p(rgb_i), _p(raw_i), _p(ws), 0, None), 'forward')
    _check(L.sdb_cnn_train_forward_ex(_p(x), H, W, _p(pk), _p(m), 0, _p(rgb_t), _p(raw_t), _p(rec), None), 'train_forward_ex')
    torch.cuda.synchronize()
    assert torch.equal(rgb_i, rgb_t) and torch.equal(raw_i, raw_t)


def test_bf16_train_forward_vs_float64():
    H, W = 262, 262
    net_out, z, P, _ = _inputs(H, W)
    with torch.no_grad():
        ref_rgb, ref_raw = oracle.render_cnn(net_out.double(), z.double(), P, dtype=torch.float64)
        with _amp(rendercnn.PRECISION_BF16):
            c_rgb, c_raw = oracle.render_cnn(net_out, z, P, dtype=torch.float32)
    L = _lib.lib()
    pk, m, x = _pack(L, P, 3), _mod(P, z), net_out[0].contiguous()
    rgb, raw = torch.empty(3, H, W, device=DEV), torch.empty(3, H, W, device=DEV)
    rec = torch.empty(int(L.sdb_cnn_train_record_bytes_ex(H, W, 3)), dtype=torch.uint8, device=DEV)
    _check(L.sdb_cnn_train_forward_ex(_p(x), H, W, _p(pk), _p(m), 3, _p(rgb), _p(raw), _p(rec), None), 'train_forward_ex')
    torch.cuda.synchronize()
    for name, ours, comp, ref in (('rgb', rgb, c_rgb[0], ref_rgb[0]), ('raw', raw, c_raw[0], ref_raw[0])):
        e, ec = float((ours.double() - ref).abs().max()), float((comp.double() - ref).abs().max())
        print('bf16 x1 training forward %s: max|. - f64| %.3e, reference composition under bf16 autocast %.3e' % (name, e, ec))
        assert e <= VS_COMPOSITION * ec, (name, e, ec)


# ---- 2. gradients --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('which', ['rgb', 'raw', 'both'])
@pytest.mark.parametrize('H,W', [(37, 150), (8, 128), (2, 5), (262, 262)])
def test_one_pass_gradients_vs_float64(H, W, which):
    net_out, z, P, G = _inputs(H, W)
    _, ref = _grads(_oracle, net_out, z, P, G, which, torch.float64)
    failures = []
    for prec in (rendercnn.PRECISION_FP16, rendercnn.PRECISION_BF16):
        captured = {}

        def ours(x, zz, Q):
            with _amp(prec):
                rgb, raw = rendercnn.RenderCNNEngine(Q).forward_train(x, zz, Q, precision=prec)
            assert rgb.dtype == raw.dtype == AMP_DTYPE[prec]
            captured['signs'] = _recorded_signs(_train_node(rgb).records[0], H, W, prec)
            return rgb.float(), raw.float()

        def composition(x, zz, Q):
            with _amp(prec):
                rgb, raw = oracle.render_cnn(x, zz, Q, dtype=torch.float32)
            return rgb.float(), raw.float()
        _, got = _grads(ours, net_out, z, P, G, which, torch.float32)
        _, masked = _grads(_masked_f64(captured['signs']), net_out, z, P, G, which, torch.float64)
        _, comp = _grads(composition, net_out, z, P, G, which, torch.float32)
        for k in ref:
            e, em, ec = _rel(got[k], ref[k]), _rel(got[k], masked[k]), _rel(comp[k], ref[k])
            print('%s %dx%d (%s) %-26s rel-L2: vs f64 %.3e, vs f64 with recorded slopes %.3e, composition vs f64 %.3e' % (
                AMP_DTYPE[prec], H, W, which, k.replace('denoiser.', ''), e, em, ec))
            if em > TOL_MASKED[prec]:
                failures.append((prec, k, 'masked', em))
            if e > VS_COMPOSITION * ec:
                failures.append((prec, k, 'vs composition', e, ec))
    assert not failures, failures


# ---- 3. precision 1 of the _ex entries is the entries without _ex --------------------------------------------------------
def test_ex_precision_1_is_the_bf16x3_path_bit_for_bit():
    """Packs, record, rgb, raw and dL/d net_out bit for bit.  The bias, dm and weight gradients are sums the kernels finish
    with float atomics, whose order changes from run to run: two runs of the entry without _ex differ in their last bits
    as well, so those are held to that spread."""
    H, W = 37, 150
    L = _lib.lib()
    net_out, z, P, G = _inputs(H, W)
    x, m = net_out[0].contiguous(), _mod(P, z)
    conv_w = [P['denoiser.' + n].float().contiguous() for n in rendercnn._CONV_W]
    runs = []
    for ex in (False, False, True):
        pk = _pack(L, P, 1, old=not ex)
        bp = torch.empty(int(L.sdb_cnn_backward_pack_bytes_ex(1) if ex else L.sdb_cnn_backward_pack_bytes()), dtype=torch.uint8,
                         device=DEV)
        nrec = L.sdb_cnn_train_record_bytes_ex(H, W, 1) if ex else L.sdb_cnn_train_record_bytes(H, W)
        rec = torch.full((int(nrec),), 0xAB, dtype=torch.uint8, device=DEV)
        rgb, raw = torch.empty(3, H, W, device=DEV), torch.empty(3, H, W, device=DEV)
        nws = L.sdb_cnn_backward_workspace_bytes_ex(H, W, 1) if ex else L.sdb_cnn_backward_workspace_bytes(H, W)
        work = torch.empty(int(nws), dtype=torch.uint8, device=DEV)
        gx, gm = torch.empty(H, W, 64, device=DEV), torch.empty(4, 256, device=DEV)
        gp = [torch.empty_like(P['denoiser.' + n]) for n in rendercnn._NAMES]
        grads = rendercnn._CnnGrads(_p(gx), _p(gm), *[_p(t) for t in gp])
        if ex:
            _check(L.sdb_cnn_pack_backward_ex(*[_p(t) for t in conv_w], 1, _p(bp), None), 'pack_backward_ex')
            _check(L.sdb_cnn_train_forward_ex(_p(x), H, W, _p(pk), _p(m), 1, _p(rgb), _p(raw), _p(rec), None), 'train_forward_ex')
            _check(L.sdb_cnn_backward_ex(H, W, 1, _p(rec), _p(G[0][0]), _p(G[1][0]), _p(bp), _p(pk), _p(m), ctypes.byref(grads),
                                         _p(work), None), 'backward_ex')
        else:
            _check(L.sdb_cnn_pack_backward(*[_p(t) for t in conv_w], _p(bp), None), 'pack_backward')
            _check(L.sdb_cnn_train_forward(_p(x), H, W, _p(pk), _p(m), _p(rgb), _p(raw), _p(rec), None), 'train_forward')
            _check(L.sdb_cnn_backward(H, W, _p(rec), _p(G[0][0]), _p(G[1][0]), _p(bp), _p(pk), _p(m), ctypes.byref(grads),
                                      _p(work), None), 'backward')
        torch.cuda.synchronize()
        runs.append([pk, bp, rec, rgb, raw, gx, gm] + gp)
    names = ['pack', 'backward pack', 'record', 'rgb', 'raw', 'net_out grad', 'mod grad'] + list(rendercnn._NAMES)
    for i, (n, a, a2, b) in enumerate(zip(names, *runs)):
        if i < 6:
            assert torch.equal(a, a2) and torch.equal(a, b), n
        else:
            e, e_old = _rel(b, a), _rel(a2, a)
            print('%-14s rel-L2 _ex(1) vs old %.2e, old vs old %.2e' % (n, e, e_old))
            assert e <= REORDER_TOL and e_old <= REORDER_TOL, (n, e, e_old)


# ---- 4. and 5. the generator under autocast with SDB200_CNN_AMP=1 --------------------------------------------------------
GEN_PARAMS = ('render_net.fc_1.weight', 'hash_encoder.embeddings', 'denoiser.fc_z_cond.weight')


@pytest.fixture
def amp_cnn_gen(generator, monkeypatch):  # noqa: F811
    gen = generator
    mods = dict(gen.named_parameters())
    names = list(GEN_PARAMS) + ['denoiser.' + n for n in rendercnn._NAMES]
    params = [mods[k] for k in names]
    saved = [q.detach().clone() for q in params]
    for q in params:
        q.requires_grad_(True)
        q.grad = None
    if hasattr(gen, 'sky_avg'):
        del gen.sky_avg
    gen.coarse_deterministic_sampling = False
    gen.num_samples = 24
    for k in ('SDB200_CNN', 'SDB200_CNN_AMP', 'SDB200_FUSED'):
        monkeypatch.delenv(k, raising=False)
    try:
        yield gen, names, params
    finally:
        with torch.no_grad():
            for q, s in zip(params, saved):
                q.copy_(s)
                q.requires_grad_(False)
                q.grad = None


def _data(gen):
    from test_gpu_amp import _data as data
    return data(gen, 1)


def _cnn_stats(gen):
    st = integration._state(gen).stats
    return {k: st[k] for k in ('cnn_train_calls', 'cnn_amp_train_calls', 'cnn_reference_calls')}


def _fp16_step(gen, names, params, monkeypatch, env):
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    try:
        before = _cnn_stats(gen)
        torch.manual_seed(5)
        with torch.autocast('cuda', dtype=torch.float16):
            out = gen(_data(gen), random_style=True)
            loss = out['fake_images'].float().square().mean()
        loss.backward()
        torch.cuda.synchronize()
        grads = {k: q.grad.clone() for k, q in zip(names, params)}
        for q in params:
            q.grad = None
        after = _cnn_stats(gen)
        return grads, {k: after[k] - before[k] for k in after}, out['fake_images'].dtype
    finally:
        for k in env:
            monkeypatch.delenv(k)


def test_generator_under_fp16_autocast_trains_the_cnn_in_one_pass(amp_cnn_gen, monkeypatch):
    gen, names, params = amp_cnn_gen
    ref, d_ref, dt_ref = _fp16_step(gen, names, params, monkeypatch, {'SDB200_CNN': '0'})
    ours, d, dt = _fp16_step(gen, names, params, monkeypatch, {'SDB200_CNN_AMP': '1'})
    _, d_off, _ = _fp16_step(gen, names, params, monkeypatch, {})
    print('hook stats: SDB200_CNN=0 %s, SDB200_CNN_AMP=1 %s, default %s' % (d_ref, d, d_off))
    assert d_ref == {'cnn_train_calls': 0, 'cnn_amp_train_calls': 0, 'cnn_reference_calls': 1}
    assert d == {'cnn_train_calls': 1, 'cnn_amp_train_calls': 1, 'cnn_reference_calls': 0}
    assert d_off == {'cnn_train_calls': 0, 'cnn_amp_train_calls': 0, 'cnn_reference_calls': 1}     # the switch is off by default
    assert dt == dt_ref == torch.float16
    worst = 0.0
    for k in names:
        assert bool(torch.isfinite(ours[k]).all()) and float(ours[k].abs().max()) > 0, k
        e = _rel(ours[k], ref[k])
        worst = max(worst, e)
        print('generator step under fp16 autocast %-30s rel-L2 SDB200_CNN_AMP=1 vs SDB200_CNN=0: %.3e' % (k, e))
    assert worst <= GEN_GRAD_TOL, worst


def test_gradscaler_steps_and_skips_with_the_switch_on(amp_cnn_gen, monkeypatch):
    gen, names, params = amp_cnn_gen
    monkeypatch.setenv('SDB200_CNN_AMP', '1')
    den = [(k, q) for k, q in zip(names, params) if k.startswith('denoiser.')]
    data = _data(gen)
    opt = torch.optim.Adam(params, lr=1e-4, eps=1e-7, betas=(0.0, 0.999))
    scaler = torch.amp.GradScaler('cuda')
    inject = {'on': False}

    def inf_at_one_pixel(g):
        g = g.clone()
        g[0, 0, g.shape[2] // 2, g.shape[3] // 2] = float('inf')
        return g

    def step():
        opt.zero_grad(set_to_none=True)
        with torch.autocast('cuda', dtype=torch.float16):
            img = gen(data, random_style=True)['fake_images']
            if inject['on']:
                img.register_hook(inf_at_one_pixel)
            loss = img.float().square().mean()
        scaler.scale(loss).backward()
        finite = {k: bool(torch.isfinite(q.grad).all()) for k, q in den}
        scaler.step(opt)
        scaler.update()
        return finite
    before = _cnn_stats(gen)
    start = [q.detach().clone() for _, q in den]
    for _ in range(3):
        assert all(step().values())
    torch.cuda.synchronize()
    d = {k: v - before[k] for k, v in _cnn_stats(gen).items()}
    assert d == {'cnn_train_calls': 3, 'cnn_amp_train_calls': 3, 'cnn_reference_calls': 0}, d
    after3 = [q.detach().clone() for _, q in den]
    for (k, _), a, b in zip(den, start, after3):
        assert bool(torch.isfinite(b).all()) and not torch.equal(a, b), (k, 'did not change over three steps')
    scale = scaler.get_scale()
    inject['on'] = True
    finite = step()
    torch.cuda.synchronize()
    print('inf at one pixel of dL/d rgb: finite denoiser gradients %s; scale %g -> %g' % (
        [k for k, v in finite.items() if v], scale, scaler.get_scale()))
    assert not any(finite.values()), finite                     # the inf reaches every denoiser gradient ...
    assert all(torch.equal(a, q.detach()) for a, (_, q) in zip(after3, den))     # ... so the step is skipped
    assert scaler.get_scale() < scale


# ---- 6. autograd edge cases ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize('precision', [rendercnn.PRECISION_FP16, rendercnn.PRECISION_BF16])
def test_second_backward_raises_and_frozen_weights_get_no_gradient(precision):
    net_out, z, P, G = _inputs(8, 128)
    Q = {k: v.clone().requires_grad_(k == 'denoiser.fc_z_cond.weight') for k, v in P.items()}
    x = net_out.clone().requires_grad_(True)
    with _amp(precision):
        rgb, raw = rendercnn.RenderCNNEngine(Q).forward_train(x, z, Q, precision=precision)
        loss = (rgb.float() * G[0]).sum()
    loss.backward(retain_graph=True)
    assert x.grad is not None and x.grad.dtype == torch.float32
    assert Q['denoiser.fc_z_cond.weight'].grad is not None and Q['denoiser.fc_z_cond.weight'].grad.dtype == torch.float32
    assert Q['denoiser.conv2a.weight'].grad is None
    with pytest.raises(RuntimeError, match='released by its first backward'):
        loss.backward()
