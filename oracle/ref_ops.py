"""Python face of the CPU oracle (TEST INFRASTRUCTURE ONLY -- see oracle/__init__.py).

Native-op restatements live in oracle.c (DDA, hash-grid encode fwd/bwd, positional encoding);
this file wraps them with ctypes and restates the reference's pure-PyTorch stages of the
per-pixel path (sampling, label lookup, MLPs, compositing) in plain torch fp32 on CPU.
Citations are relative to /root/reference/.
"""
import ctypes
import os
import subprocess

import numpy as np
import torch
import torch.nn.functional as F

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None


def build_oracle_lib():
    subprocess.check_call(["make", "-s", "-C", _HERE, "liboracle.so"])


def _lib():
    global _LIB
    if _LIB is None:
        path = os.path.join(_HERE, "liboracle.so")
        if not os.path.exists(path):
            build_oracle_lib()
        _LIB = ctypes.CDLL(path)
    return _LIB


def _p(t, ctype):
    return ctypes.cast(t.data_ptr(), ctypes.POINTER(ctype))


def _f32(x):
    return torch.as_tensor(x, dtype=torch.float32).detach().cpu().contiguous()


def num_threads():
    return int(_lib().sdo_num_threads())


# ----------------------------------------------------------------------------------------------
# a1: ray / voxel intersection.  voxlib/ray_voxel_intersection.cu:52-235, :253-325
# ----------------------------------------------------------------------------------------------
def camera_frame(cam_dir, cam_up):
    d, u = _f32(cam_dir), _f32(cam_up)
    out = torch.empty(3, 3, dtype=torch.float32)
    _lib().sdo_camera_frame(_p(d, ctypes.c_float), _p(u, ctypes.c_float),
                            _p(out[0], ctypes.c_float), _p(out[1], ctypes.c_float), _p(out[2], ctypes.c_float))
    return out[0], out[1], out[2]  # fwd, side, up


def ray_voxel_intersection_perspective(voxel, cam_ori, cam_dir, cam_up, cam_f, cam_c, img_dims, max_samples,
                                       return_steps=False):
    """Same signature/returns as voxlib.ray_voxel_intersection_perspective (voxlib.cpp:11)."""
    assert voxel.dtype == torch.int32 and voxel.dim() == 3
    voxel = voxel.cpu()
    H, W, M = int(img_dims[0]), int(img_dims[1]), int(max_samples)
    vid = torch.empty(H, W, M, 1, dtype=torch.int32)
    dep = torch.empty(2, H, W, M, 1, dtype=torch.float32)
    rd = torch.empty(H, W, 1, 3, dtype=torch.float32)
    steps = torch.zeros(H, W, dtype=torch.int32) if return_steps else None
    dims = (ctypes.c_int64 * 3)(*voxel.shape)
    strides = (ctypes.c_int64 * 3)(*voxel.stride())
    o, d, u = _f32(cam_ori), _f32(cam_dir), _f32(cam_up)
    cc = (ctypes.c_float * 2)(float(cam_c[0]), float(cam_c[1]))
    im = (ctypes.c_int * 2)(H, W)
    _lib().sdo_ray_voxel_intersection_perspective(
        _p(voxel, ctypes.c_int32), dims, strides, _p(o, ctypes.c_float), _p(d, ctypes.c_float),
        _p(u, ctypes.c_float), ctypes.c_float(cam_f), cc, im, ctypes.c_int(M),
        _p(vid, ctypes.c_int32), _p(dep, ctypes.c_float), _p(rd, ctypes.c_float),
        _p(steps, ctypes.c_int32) if return_steps else None)
    if return_steps:
        return [vid, dep, rd], steps
    return [vid, dep, rd]


# ----------------------------------------------------------------------------------------------
# a6/a7/a13: hash-grid encoder.  gridencoder/src/gridencoder.cu:35-343, gridencoder/grid.py
# ----------------------------------------------------------------------------------------------
def grid_offsets(input_dim=5, num_levels=16, per_level_scale=None, base_resolution=16, log2_hashmap_size=19,
                 desired_resolution=2048, align_corners=False):
    """Level offsets exactly as GridEncoder.__init__ computes them (gridencoder/grid.py:97-124)."""
    if desired_resolution is not None:
        per_level_scale = np.exp2(np.log2(desired_resolution / base_resolution) / (num_levels - 1))
    offsets, offset = [], 0
    max_params = 2 ** log2_hashmap_size
    for i in range(num_levels):
        resolution = int(np.ceil(base_resolution * per_level_scale ** i))
        n = min(max_params, (resolution if align_corners else resolution + 1) ** input_dim)
        n = int(np.ceil(n / 8) * 8)
        offsets.append(offset)
        offset += n
    offsets.append(offset)
    return torch.from_numpy(np.array(offsets, dtype=np.int32)), float(per_level_scale)


def level_scales_libm(L, per_level_scale, base_resolution):
    S = np.float32(np.log2(per_level_scale))
    return torch.tensor([np.exp2(np.float32(np.float32(l) * S), dtype=np.float32) * np.float32(base_resolution)
                         - np.float32(1.0) for l in range(L)], dtype=torch.float32)


def _scales_ptr(level_scales):
    if level_scales is None:
        return None, None
    t = _f32(level_scales)
    return t, _p(t, ctypes.c_float)


def grid_encode_forward(inputs, embeddings, offsets, per_level_scale, base_resolution, calc_grad_inputs=False,
                        gridtype=0, align_corners=False, level_scales=None):
    """inputs [B,D] in [0,1] -> (outputs [L,B,C], dy_dx [B,L*D*C] or None); the raw kernel contract."""
    inputs, embeddings = _f32(inputs), _f32(embeddings)
    offsets = offsets.to(torch.int32).cpu().contiguous()
    B, D = inputs.shape
    L, C = offsets.numel() - 1, embeddings.shape[1]
    S = np.log2(per_level_scale)
    out = torch.empty(L, B, C, dtype=torch.float32)
    dy_dx = torch.empty(B, L * D * C, dtype=torch.float32) if calc_grad_inputs else None
    _keep, sp = _scales_ptr(level_scales)
    _lib().sdo_grid_encode_forward(
        _p(inputs, ctypes.c_float), _p(embeddings, ctypes.c_float), _p(offsets, ctypes.c_int32),
        _p(out, ctypes.c_float), ctypes.c_uint32(B), ctypes.c_uint32(D), ctypes.c_uint32(C), ctypes.c_uint32(L),
        ctypes.c_float(S), ctypes.c_uint32(base_resolution), ctypes.c_int(bool(calc_grad_inputs)),
        _p(dy_dx, ctypes.c_float) if calc_grad_inputs else None, ctypes.c_uint32(gridtype),
        ctypes.c_int(bool(align_corners)), sp)
    return out, dy_dx


def grid_encode_backward(grad, inputs, embeddings, offsets, per_level_scale, base_resolution, dy_dx=None,
                         gridtype=0, align_corners=False, level_scales=None):
    """grad [L,B,C] -> (grad_embeddings, grad_inputs or None)."""
    grad, inputs, embeddings = _f32(grad), _f32(inputs), _f32(embeddings)
    offsets = offsets.to(torch.int32).cpu().contiguous()
    B, D = inputs.shape
    L, C = offsets.numel() - 1, embeddings.shape[1]
    S = np.log2(per_level_scale)
    ge = torch.zeros_like(embeddings)
    calc = dy_dx is not None
    gi = torch.zeros(B, D, dtype=torch.float32) if calc else None
    if calc:
        dy_dx = _f32(dy_dx)
    _keep, sp = _scales_ptr(level_scales)
    _lib().sdo_grid_encode_backward(
        _p(grad, ctypes.c_float), _p(inputs, ctypes.c_float), _p(embeddings, ctypes.c_float),
        _p(offsets, ctypes.c_int32), _p(ge, ctypes.c_float), ctypes.c_uint32(B), ctypes.c_uint32(D),
        ctypes.c_uint32(C), ctypes.c_uint32(L), ctypes.c_float(S), ctypes.c_uint32(base_resolution),
        ctypes.c_int(calc), _p(dy_dx, ctypes.c_float) if calc else None,
        _p(gi, ctypes.c_float) if calc else None, ctypes.c_uint32(gridtype), ctypes.c_int(bool(align_corners)), sp)
    return ge, gi


def grid_encoder_module_forward(inputs, embeddings, offsets, per_level_scale, base_resolution=16, bound=1,
                                gridtype=0, align_corners=False, level_scales=None):
    """GridEncoder.forward (gridencoder/grid.py:140-156): [-bound,bound] -> [0,1], encode, [.., L*C]."""
    x = (_f32(inputs) + bound) / (2 * bound)
    prefix = list(x.shape[:-1])
    out, _ = grid_encode_forward(x.reshape(-1, x.shape[-1]), embeddings, offsets, per_level_scale,
                                 base_resolution, False, gridtype, align_corners, level_scales)
    L, B, C = out.shape
    return out.permute(1, 0, 2).reshape(prefix + [L * C])


# ----------------------------------------------------------------------------------------------
# a9: positional encoding.  voxlib/positional_encoding_kernel.cu:40-118, positional_encoding.py:45-54
# ----------------------------------------------------------------------------------------------
def _pe_shapes(x, dim):
    dim = dim % x.dim()
    pre = int(np.prod(x.shape[:dim])) if dim > 0 else 1
    post = int(np.prod(x.shape[dim:]))
    return dim, pre, post


def positional_encoding(x, ndegrees, dim=-1, incl_orig=False):
    x = _f32(x)
    dim, pre, post = _pe_shapes(x, dim)
    stride = 2 * ndegrees + (1 if incl_orig else 0)
    shape = list(x.shape)
    shape[dim] *= stride
    out = torch.empty(shape, dtype=torch.float32)
    _lib().sdo_positional_encoding(_p(x, ctypes.c_float), _p(out, ctypes.c_float), ctypes.c_int64(pre),
                                   ctypes.c_int64(post), ctypes.c_int(ndegrees), ctypes.c_int(bool(incl_orig)))
    return out


def positional_encoding_backward(out_grad, out, ndegrees, dim=-1, incl_orig=False):
    out_grad, out = _f32(out_grad), _f32(out)
    stride = 2 * ndegrees + (1 if incl_orig else 0)
    shape = list(out.shape)
    d = dim % out.dim()
    shape[d] //= stride
    g = torch.empty(shape, dtype=torch.float32)
    _, pre, post = _pe_shapes(g, d)
    _lib().sdo_positional_encoding_backward(
        _p(out_grad, ctypes.c_float), _p(out, ctypes.c_float), _p(g, ctypes.c_float), ctypes.c_int64(pre),
        ctypes.c_int64(post), ctypes.c_int(ndegrees), ctypes.c_int(bool(incl_orig)))
    return g


def positional_encoding_pt(pts, pe_degrees, dim=-1, incl_orig=False):
    """The reference's own pure-PyTorch statement (positional_encoding.py:45-54), restated."""
    parts = []
    for i in range(pe_degrees):
        parts.append(torch.sin(pts * np.pi * 2 ** i))
        parts.append(torch.cos(pts * np.pi * 2 ** i))
    if incl_orig:
        parts.append(pts)
    return torch.cat(parts, dim=dim)


# ----------------------------------------------------------------------------------------------
# a2: depth sampling.  imaginaire/model_utils/gancraft/mc_utils.py:82-151
# (use_box_boundaries=False branch, the only one SceneDreamer configures)
# ----------------------------------------------------------------------------------------------
def _cumsum_seq(x, dim):
    """Sequential float32 prefix sum == torch's CUDA cumsum over a non-innermost dim
    (ATen ScanKernels tensor_kernel_scan_outer_dim: acc = acc + x[i] in the tensor dtype).
    torch's CPU cumsum accumulates in double, so it is NOT used here."""
    outs, acc = [], None
    for i in range(x.shape[dim]):
        xi = x.select(dim, i)
        acc = xi.clone() if acc is None else acc + xi
        outs.append(acc)
    return torch.stack(outs, dim=dim)


def deterministic_fractions(nsamples):
    """mc_utils.py:118-120: torch.linspace(0, 1, nsamples+2)[1:-1] built on the CPU in fp32."""
    return torch.linspace(0, 1, nsamples + 2)[1:-1].clone()


def sample_depth_batched(depth2, nsamples, deterministic=False, sample_depth=3.0, uniforms=None):
    """depth2 [N,2,H,W,M,1] -> rand_depth [N,H,W,S,1], new_dists [N,H,W,S,1], idx (int64) with S=nsamples-1.

    `uniforms` ([N,H,W,nsamples,1], U[0,1)) replaces torch.rand for the stratified branch so that
    the kernel under test can be fed identical randomness."""
    depth2 = _f32(depth2)
    bs, dim0, dim1 = depth2.size(0), depth2.size(2), depth2.size(3)
    dists = depth2[:, 1] - depth2[:, 0]
    dists[torch.isnan(dists)] = 0
    accu_depth = _cumsum_seq(dists, -2)
    total_depth = accu_depth[..., [-1], :]
    total_depth = torch.clamp(total_depth, None, sample_depth)
    rand_shape = [bs, dim0, dim1, nsamples, 1]
    if deterministic:
        rand_samples = torch.empty(rand_shape, dtype=torch.float32)
        rand_samples[..., :, 0] = deterministic_fractions(nsamples)
    else:
        assert uniforms is not None
        rand_samples = _f32(uniforms).clone().reshape(rand_shape)
        rand_samples = rand_samples / nsamples
        rand_samples[..., :, 0] += torch.linspace(0, 1, nsamples + 1)[:-1]
    rand_samples = rand_samples * total_depth
    rand_samples, _ = torch.sort(rand_samples, dim=-2, descending=False)
    midpoints = (rand_samples[..., 1:, :] + rand_samples[..., :-1, :]) / 2
    new_dists = rand_samples[..., 1:, :] - rand_samples[..., :-1, :]
    idx = torch.sum(midpoints.unsqueeze(-3) > accu_depth.unsqueeze(-2), dim=-3)
    depth_deltas = depth2[:, 0, :, :, 1:, :] - depth2[:, 1, :, :, :-1, :]
    depth_deltas = _cumsum_seq(depth_deltas, -2)
    depth_deltas = torch.cat([depth2[:, 0, :, :, [0], :], depth_deltas + depth2[:, 0, :, :, [0], :]], dim=-2)
    heads = torch.gather(depth_deltas, -2, idx)
    rand_depth = heads + midpoints
    return rand_depth, new_dists, idx


# ----------------------------------------------------------------------------------------------
# a10: compositing weights.  mc_utils.py:75-79, :154-161
# ----------------------------------------------------------------------------------------------
def cumsum_exclusive(t, dim):
    c = _cumsum_seq(t, dim)
    c = torch.roll(c, 1, dim)
    c.index_fill_(dim, torch.tensor([0], dtype=torch.long), 0)
    return c


def volum_rendering_relu(sigma, dists, dim=2):
    free_energy = F.relu(sigma) * dists
    a = 1 - torch.exp(-free_energy.float())
    b = torch.exp(-cumsum_exclusive(free_energy, dim=dim))
    return a * b


# ----------------------------------------------------------------------------------------------
# a8/a9: MLPs.  imaginaire/model_utils/layers.py:57-126 (LightningMLP), :184-271 (ModLinear);
# imaginaire/generators/gancraft_base.py:91-126 (StyleMLP), :129-169 (SKYMLP).
# Parameters are passed as a flat dict keyed by the reference's state-dict names.
# ----------------------------------------------------------------------------------------------
def _lrelu(x):
    return F.leaky_relu(x, 0.2)


def mod_linear(x, z, P, name):
    """ModLinear.forward with bias=False, mod_bias=True, output_mode=True (layers.py:241-271).
    x [B, n, I], z [B, Cz]."""
    alpha = torch.addmm(P[name + '.bias_alpha'].unsqueeze(0), z, P[name + '.weight_alpha'].t())   # [B, I]
    w = P[name + '.weight'].unsqueeze(0) * alpha.unsqueeze(1)                                      # [B, O, I]
    beta = torch.addmm(P[name + '.bias_beta'].unsqueeze(0), z, P[name + '.weight_beta'].t())       # [B, O]
    return torch.baddbmm(beta.unsqueeze(1), x, w.transpose(1, 2))


def render_mlp(x, z, labels, P, prefix='render_net'):
    """LightningMLP.forward with use_seg=True, viewdir_dim=0.  x [B, n, 128] features, z [B, 256] style,
    labels [B, n] int64 reduced labels (the one-hot @ fc_m_a.weight^T product is an embedding lookup)."""
    p = prefix + '.'
    f = F.linear(x, P[p + 'fc_1.weight'], P[p + 'fc_1.bias'])
    onehot = F.one_hot(labels, P[p + 'fc_m_a.weight'].shape[1]).to(torch.float32)
    f = f + F.linear(onehot, P[p + 'fc_m_a.weight'])
    f = _lrelu(f)
    f = _lrelu(mod_linear(f, z, P, p + 'fc_2'))
    f = _lrelu(mod_linear(f, z, P, p + 'fc_3'))
    f = _lrelu(mod_linear(f, z, P, p + 'fc_4'))
    sigma = F.linear(f, P[p + 'fc_sigma.weight'], P[p + 'fc_sigma.bias'])
    f = _lrelu(mod_linear(f, z, P, p + 'fc_5'))
    f = _lrelu(mod_linear(f, z, P, p + 'fc_6'))
    c = F.linear(f, P[p + 'fc_out_c.weight'], P[p + 'fc_out_c.bias'])
    return sigma, c


def sky_mlp(x, z, P, prefix='sky_net'):
    """SKYMLP.forward.  x [B, n, 33] PE'd ray dirs, z [B, 256]."""
    p = prefix + '.'
    zz = F.linear(z, P[p + 'fc_z_a.weight']).unsqueeze(1)
    y = _lrelu(F.linear(x, P[p + 'fc1.weight'], P[p + 'fc1.bias']) + zz)
    for k in (2, 3, 4, 5):
        y = _lrelu(F.linear(y, P[p + 'fc%d.weight' % k], P[p + 'fc%d.bias' % k]))
    return F.linear(y, P[p + 'fc_out_c.weight'], P[p + 'fc_out_c.bias'])


def style_mlp(z, P, prefix='style_net', num_layers=5):
    """StyleMLP.forward with normalize_input=True, output_act=True."""
    p = prefix + '.'
    z = F.normalize(z, p=2, dim=-1)
    for i in range(num_layers):
        z = _lrelu(F.linear(z, P[p + 'fc_layers.%d.weight' % i], P[p + 'fc_layers.%d.bias' % i]))
    return _lrelu(F.linear(z, P[p + 'fc_out.weight'], P[p + 'fc_out.bias']))


def make_params(seed=0, stress=False, style_dim=128, interm=256, hidden=256, feat=128, nlabels=12, out_c=64,
                table_entries=16 * (1 << 19), level_dim=8, table_scale=0.1):
    """Synthetic weights with the reference's state-dict names/shapes.

    stress=False: module default init followed by custom_init (kaiming_normal(a=0.2)*0.5, zero bias;
                  scenedreamer.py:66-78).  Every layer halves the activation RMS, so outputs are ~1e-3.
    stress=True : gains chosen so hidden activations stay O(1), sigma spans roughly +-200 and colour
                  features exceed +-1 (exercises clamp, opacity saturation and the style modulation);
                  this is the weight set the 1e-3 parity bar is meaningful on.
    """
    g = torch.Generator().manual_seed(seed)
    P = {}

    def kaiming(o, i, gain):
        std = gain * np.sqrt(2.0 / (1 + 0.2 ** 2)) / np.sqrt(i)
        return torch.randn(o, i, generator=g) * std

    wg = 1.0 if stress else 0.5
    bg = 0.1 if stress else 0.0
    # style_net: Linear(style_dim,256), 4x Linear(256,256), fc_out Linear(256, interm)
    dims = [style_dim] + [256] * 5
    for i in range(5):
        P['style_net.fc_layers.%d.weight' % i] = kaiming(dims[i + 1], dims[i], wg)
        P['style_net.fc_layers.%d.bias' % i] = torch.randn(dims[i + 1], generator=g) * bg
    P['style_net.fc_out.weight'] = kaiming(interm, 256, wg)
    P['style_net.fc_out.bias'] = torch.randn(interm, generator=g) * bg
    # render_net
    r = 'render_net.'
    P[r + 'fc_m_a.weight'] = kaiming(hidden, nlabels, wg) * (0.5 if stress else 1.0)
    P[r + 'fc_1.weight'] = kaiming(hidden, feat, wg * (8.0 if stress else 1.0))
    P[r + 'fc_1.bias'] = torch.randn(hidden, generator=g) * bg
    for k in (2, 3, 4, 5, 6):
        n = r + 'fc_%d' % k
        P[n + '.weight'] = kaiming(hidden, hidden, wg)
        P[n + '.weight_alpha'] = torch.randn(hidden, interm, generator=g) / np.sqrt(interm) * (0.5 if stress else 1.0)
        P[n + '.bias_alpha'] = torch.ones(hidden)
        P[n + '.weight_beta'] = torch.randn(hidden, interm, generator=g) / np.sqrt(interm) * (0.5 if stress else 1.0)
        P[n + '.bias_beta'] = torch.zeros(hidden)
    P[r + 'fc_sigma.weight'] = kaiming(1, hidden, wg * (120.0 if stress else 1.0))
    P[r + 'fc_sigma.bias'] = torch.full((1,), 20.0 if stress else 0.0)
    P[r + 'fc_out_c.weight'] = kaiming(out_c, hidden, wg * (1.5 if stress else 1.0))
    P[r + 'fc_out_c.bias'] = torch.randn(out_c, generator=g) * bg
    # sky_net
    s = 'sky_net.'
    P[s + 'fc_z_a.weight'] = kaiming(hidden, interm, wg)
    P[s + 'fc1.weight'] = kaiming(hidden, 33, wg)
    P[s + 'fc1.bias'] = torch.randn(hidden, generator=g) * bg
    for k in (2, 3, 4, 5):
        P[s + 'fc%d.weight' % k] = kaiming(hidden, hidden, wg)
        P[s + 'fc%d.bias' % k] = torch.randn(hidden, generator=g) * bg
    P[s + 'fc_out_c.weight'] = kaiming(out_c, hidden, wg * (1.5 if stress else 1.0))
    P[s + 'fc_out_c.bias'] = torch.randn(out_c, generator=g) * bg
    # hash table (U(-0.1, 0.1) so the encode numerics are exercised)
    P['hash_encoder.embeddings'] = (torch.rand(table_entries, level_dim, generator=g) * 2 - 1) * table_scale
    return P


# ----------------------------------------------------------------------------------------------
# f1: RenderCNN + tanh.  imaginaire/generators/gancraft_base.py:172-225 (RenderCNN), :588-603 (_forward_global)
# ----------------------------------------------------------------------------------------------
def make_cnn_params(seed=0, in_ch=64, hidden=256, style=256, gain=1.4):
    """Synthetic `denoiser.*` weights with the reference's state-dict names / shapes; gains keep activations O(1)."""
    g = torch.Generator().manual_seed(seed)
    P = {}

    def conv(name, o, i, k, bias=True):
        P['denoiser.%s.weight' % name] = torch.randn(o, i, k, k, generator=g) * (gain / np.sqrt(i * k * k))
        if bias:
            P['denoiser.%s.bias' % name] = torch.randn(o, generator=g) * 0.1
    conv('conv1', hidden, in_ch, 1)
    conv('conv2a', hidden, hidden, 3)
    conv('conv2b', hidden, hidden, 3, bias=False)
    conv('conv3a', hidden, hidden, 3)
    conv('conv3b', hidden, hidden, 3, bias=False)
    conv('conv4a', hidden, hidden, 1)
    conv('conv4b', hidden, hidden, 1)
    conv('conv4', 3, hidden, 1)
    P['denoiser.conv4.weight'] *= 0.2                          # raw image O(1): tanh not saturated
    P['denoiser.fc_z_cond.weight'] = torch.randn(4 * hidden, style, generator=g) * (0.5 / np.sqrt(style))
    P['denoiser.fc_z_cond.bias'] = torch.randn(4 * hidden, generator=g) * 0.1
    return P


def render_cnn(net_out, z, P, prefix='denoiser.', dtype=torch.float32):
    """net_out [N,H,W,C] (as _forward_perpix returns it), z [N,256] -> (tanh image, raw image) [N,3,H,W].
    Restates RenderCNN.forward (gancraft_base.py:201-225) + the permute / tanh of _forward_global (:598-601)."""
    import torch.nn.functional as F
    W = lambda n: P[prefix + n].to(net_out.device, dtype)
    x = net_out.to(dtype).permute(0, 3, 1, 2).contiguous()
    adapt = torch.chunk(F.linear(z.to(net_out.device, dtype), W('fc_z_cond.weight'), W('fc_z_cond.bias')), 4, dim=-1)
    act = lambda t: F.leaky_relu(t, 0.2)
    mod = lambda t, w, b: t * (w[..., None, None] + 1) + b[..., None, None]
    y = act(F.conv2d(x, W('conv1.weight'), W('conv1.bias')))
    y = y + F.conv2d(act(F.conv2d(y, W('conv2a.weight'), W('conv2a.bias'), padding=1)), W('conv2b.weight'), None, padding=1)
    y = act(mod(y, adapt[0], adapt[1]))
    y = y + F.conv2d(act(F.conv2d(y, W('conv3a.weight'), W('conv3a.bias'), padding=1)), W('conv3b.weight'), None, padding=1)
    y = act(mod(y, adapt[2], adapt[3]))
    y = y + F.conv2d(act(F.conv2d(y, W('conv4a.weight'), W('conv4a.bias'))), W('conv4b.weight'), W('conv4b.bias'))
    y = act(y)
    raw = F.conv2d(y, W('conv4.weight'), W('conv4.bias'))
    return torch.tanh(raw), raw


# ----------------------------------------------------------------------------------------------
# voxlib.sp_trilinear_worldcoord (surface parity; never reached by SceneDreamer).
# imaginaire/model_utils/gancraft/voxlib/sp_trilinear_worldcoord_kernel.cu:48-198 (forward), :205-338 (backward)
# ----------------------------------------------------------------------------------------------
def sp_trilinear_corners(corner_lut, worldcoord, ign_zero):
    """-> (idx int64 [E, 8] with -1 = nothing, w float32 [E, 8]); corner j: bit2 = x+1, bit1 = y+1, bit0 = z+1 (:90-105)."""
    wc = _f32(worldcoord).reshape(-1, 3)
    fl = torch.floor(wc)
    loc = wc - fl
    one = torch.tensor(1.0, dtype=torch.float32)
    ws, ids = [], []
    dims = torch.tensor(corner_lut.shape)
    v0 = torch.minimum(torch.maximum(fl.nan_to_num(0.0).to(torch.int64), torch.zeros(3, dtype=torch.int64)), dims - 1)
    v1 = torch.minimum(torch.maximum(fl.nan_to_num(0.0).to(torch.int64) + 1, torch.zeros(3, dtype=torch.int64)), dims - 1)
    for j in range(8):
        b = ((j >> 2) & 1, (j >> 1) & 1, j & 1)
        f = [loc[:, d] if b[d] else one - loc[:, d] for d in range(3)]
        ws.append((f[0] * f[1]) * f[2])                                   # fp32, left to right like the reference
        c = [v1[:, d] if b[d] else v0[:, d] for d in range(3)]
        ids.append(corner_lut[c[0], c[1], c[2]].to(torch.int64))
    idx = torch.stack(ids, 1)
    idx[torch.isnan(wc).any(1)] = -1                                      # "hard boundary check": NaN selects nothing (:108-111)
    if ign_zero:
        idx = idx - 1
    return idx, torch.stack(ws, 1)


def sp_trilinear_worldcoord(in_feature, corner_lut, worldcoord, ign_zero=False):
    """out[e, c] = sum_j fmaf(feature[idx_j][c], w_j, acc), j = 0..7 (:186-191) -- sequential fp32 FMAs."""
    idx, w = sp_trilinear_corners(corner_lut.cpu(), worldcoord.cpu(), ign_zero)
    feat = _f32(in_feature).double()
    E, C = idx.shape[0], feat.shape[1]
    acc = torch.zeros(E, C, dtype=torch.float32)
    for j in range(8):
        ok = idx[:, j] >= 0
        rows = feat[idx[:, j].clamp(min=0)]
        upd = (rows * w[:, j:j + 1].double() + acc.double()).to(torch.float32)      # one rounding per fma
        acc = torch.where(ok[:, None], upd, acc)
    return acc.reshape(tuple(worldcoord.shape[:-1]) + (C,))


def sp_trilinear_worldcoord_backward(out_grad, in_feature, corner_lut, worldcoord, ign_zero=False):
    """feature_grad[idx_j][c] += g[c] * w_j (:323-329), accumulated here in float64."""
    idx, w = sp_trilinear_corners(corner_lut.cpu(), worldcoord.cpu(), ign_zero)
    C = in_feature.shape[1]
    g = _f32(out_grad).reshape(-1, C)
    grad = torch.zeros(in_feature.shape[0], C, dtype=torch.float64)
    for j in range(8):
        ok = idx[:, j] >= 0
        grad.index_add_(0, idx[ok, j], (g[ok] * w[ok, j:j + 1]).double())
    return grad.to(torch.float32)


# ----------------------------------------------------------------------------------------------
# a3-a5, a8-a11: the whole per-pixel stage.  imaginaire/generators/scenedreamer.py:285-428
# ----------------------------------------------------------------------------------------------
def forward_perpix(P, voxel_id, depth2, raydirs, cam_ori_t, z, global_enc, voxel_dims, mc2reduced_lut,
                   offsets, per_level_scale, num_samples=24, sample_depth=3.0, deterministic=True,
                   uniforms=None, dists_scale=0.25, sky_avg=None, ignore_id=0, dirt_id=3,
                   pe_sky=(5, True), base_resolution=16, chunk_rays=16384, level_scales=None):
    """Restates Generator._forward_perpix for the SceneDreamer inference/training configuration
    (clip_feat_map=True, keep_sky_out=True, keep_sky_out_avgpool=True, sky_global_avgpool=True,
    sample_use_box_boundaries=False, raw_noise_std=0, viewdir PE disabled).

    voxel_id [N,H,W,M,1] int32, depth2 [N,2,H,W,M,1], raydirs [N,H,W,1,3], cam_ori_t [N,3],
    z [N,256] (output of style_net), global_enc [N,2].  sky_avg: [N,1,1,1,64] or None (-> batch mean,
    scenedreamer.py:395).  Returns dict with net_out [N,H,W,64], weights, rand_depth, new_idx, ...
    """
    voxel_id = voxel_id.cpu()
    depth2, raydirs, cam_ori_t, z, global_enc = map(_f32, (depth2, raydirs, cam_ori_t, z, global_enc))
    N, H, W, M = voxel_id.shape[:4]
    sky_mask = voxel_id[:, :, :, [-1], :] == 0
    sky_only_mask = voxel_id[:, :, :, [0], :] == 0
    rand_depth, new_dists, new_idx = sample_depth_batched(
        depth2, num_samples + 1, deterministic=deterministic, sample_depth=sample_depth, uniforms=uniforms)
    bad = torch.isnan(rand_depth) | torch.isinf(rand_depth)
    rand_depth[bad] = 0.0
    worldcoord2 = raydirs * rand_depth + cam_ori_t[:, None, None, None, :]
    lut = mc2reduced_lut.to(torch.long)
    reduced = lut[voxel_id.long()]
    reduced[reduced == ignore_id] = dirt_id
    mc_masks = torch.gather(reduced, -2, new_idx).long()                # [N,H,W,S,1]

    delim = torch.tensor([float(v) for v in voxel_dims], dtype=torch.float32)
    normalized = worldcoord2 / delim * 2 - 1
    genc = global_enc[:, None, None, None, :].expand(-1, H, W, normalized.shape[3], -1)
    normalized = torch.cat([normalized, genc], dim=-1)                  # [N,H,W,S,5]

    S = normalized.shape[3]
    sig = torch.empty(N, H * W, S, 1)
    col = torch.empty(N, H * W, S, 64)
    nflat = normalized.reshape(N, H * W, S, 5)
    lflat = mc_masks.reshape(N, H * W, S)
    for n in range(N):
        for r0 in range(0, H * W, chunk_rays):
            r1 = min(H * W, r0 + chunk_rays)
            feat = grid_encoder_module_forward(nflat[n, r0:r1], P['hash_encoder.embeddings'], offsets,
                                               per_level_scale, base_resolution, level_scales=level_scales)
            s_, c_ = render_mlp(feat.reshape(1, -1, feat.shape[-1]), z[n:n + 1],
                                lflat[n, r0:r1].reshape(1, -1), P)
            sig[n, r0:r1] = s_.reshape(r1 - r0, S, 1)
            col[n, r0:r1] = c_.reshape(r1 - r0, S, 64)
    net_out_s = sig.reshape(N, H, W, S, 1)
    net_out_c = col.reshape(N, H, W, S, 64)

    pe = positional_encoding_pt(raydirs, pe_sky[0], -1, pe_sky[1])       # [N,H,W,1,33]
    skynet_out_c = sky_mlp(pe.reshape(N, H * W, -1), z, P).reshape(N, H, W, 1, 64)

    weights = volum_rendering_relu(net_out_s, new_dists * dists_scale, dim=-2)
    weights = weights * torch.logical_not(sky_only_mask).float()
    total_weights = torch.sum(weights, dim=-2, keepdim=True)
    is_gnd = (worldcoord2[..., [0]] <= 1.0).any(dim=-2, keepdim=True)
    nosky_mask = torch.logical_or(torch.logical_not(sky_mask), is_gnd).float()
    sky_weight = 1.0 - total_weights
    if sky_avg is None:
        sky_avg = torch.mean(skynet_out_c, dim=[1, 2], keepdim=True)
    sky_used = skynet_out_c * (1.0 - nosky_mask) + sky_avg * nosky_mask
    rgbs = torch.clamp(net_out_c, -1, 1) + 1
    rgbs_sky = torch.clamp(sky_used, -1, 1) + 1
    net_out = torch.sum(weights * rgbs, dim=-2, keepdim=True) + sky_weight * rgbs_sky
    net_out = net_out.squeeze(-2) - 1
    depth_map = torch.sum(weights * rand_depth, dim=-2)                   # scenedreamer.py:816
    return dict(net_out=net_out, new_dists=new_dists, weights=weights, total_weights=total_weights,
                rand_depth=rand_depth, net_out_s=net_out_s, net_out_c=net_out_c, skynet_out_c=skynet_out_c,
                sky_used=sky_used, nosky_mask=nosky_mask, sky_mask=sky_mask, sky_only_mask=sky_only_mask,
                new_idx=new_idx, labels=mc_masks, worldcoord2=worldcoord2, normalized=normalized,
                depth_map=depth_map, sky_avg=sky_avg)


# ----------------------------------------------------------------------------------------------
# Differentiable restatement (training parity): the per-pixel stage under torch.autograd, with the
# hash-grid forward/backward of oracle.c behind the same autograd.Function the reference uses
# (gridencoder/grid.py:19-87: _grid_encode.forward / .backward).
# ----------------------------------------------------------------------------------------------
class _GridEncodeFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, inputs, embeddings, offsets, per_level_scale, base_resolution, level_scales):
        calc = bool(inputs.requires_grad)
        out, dy_dx = grid_encode_forward(inputs, embeddings, offsets, per_level_scale, base_resolution, calc,
                                         level_scales=level_scales)
        ctx.save_for_backward(inputs.detach(), embeddings.detach(), offsets)
        ctx.dy_dx, ctx.args = dy_dx, (per_level_scale, base_resolution, level_scales)
        L, B, C = out.shape
        return out.permute(1, 0, 2).reshape(B, L * C)                       # grid.py:52

    @staticmethod
    def backward(ctx, grad):
        inputs, embeddings, offsets = ctx.saved_tensors
        pls, base, ls = ctx.args
        L = offsets.numel() - 1
        B = inputs.shape[0]
        C = embeddings.shape[1]
        g = grad.reshape(B, L, C).permute(1, 0, 2).contiguous()             # grid.py:72
        ge, gi = grid_encode_backward(g, inputs, embeddings, offsets, pls, base, dy_dx=ctx.dy_dx, level_scales=ls)
        return gi, ge, None, None, None, None


def forward_perpix_autograd(P, voxel_id, depth2, raydirs, cam_ori_t, z, global_enc, voxel_dims, mc2reduced_lut,
                            offsets, per_level_scale, num_samples=24, sample_depth=3.0, deterministic=True,
                            uniforms=None, dists_scale=0.25, ignore_id=0, dirt_id=3, pe_sky=(5, True),
                            base_resolution=16, level_scales=None):
    """forward_perpix with the autograd graph kept (small frames only): returns net_out [N,H,W,64] that can be
    back-propagated to P[...] (leaf tensors with requires_grad), z and global_enc.  sky_avg is the batch mean as in
    training (scenedreamer.py:395)."""
    voxel_id = voxel_id.cpu()
    depth2, raydirs, cam_ori_t = map(_f32, (depth2, raydirs, cam_ori_t))
    N, H, W, M = voxel_id.shape[:4]
    with torch.no_grad():
        sky_mask = voxel_id[:, :, :, [-1], :] == 0
        sky_only_mask = voxel_id[:, :, :, [0], :] == 0
        rand_depth, new_dists, new_idx = sample_depth_batched(
            depth2, num_samples + 1, deterministic=deterministic, sample_depth=sample_depth, uniforms=uniforms)
        bad = torch.isnan(rand_depth) | torch.isinf(rand_depth)
        rand_depth[bad] = 0.0
        worldcoord2 = raydirs * rand_depth + cam_ori_t[:, None, None, None, :]
        lut = mc2reduced_lut.to(torch.long)
        reduced = lut[voxel_id.long()]
        reduced[reduced == ignore_id] = dirt_id
        mc_masks = torch.gather(reduced, -2, new_idx).long()
        delim = torch.tensor([float(v) for v in voxel_dims], dtype=torch.float32)
        normalized = worldcoord2 / delim * 2 - 1
    S = normalized.shape[3]
    genc = global_enc[:, None, None, None, :].expand(-1, H, W, S, -1)
    x5 = torch.cat([normalized, genc], dim=-1)                              # scenedreamer.py:300-302
    x01 = (x5 + 1) / 2                                                      # grid.py:144
    feats = _GridEncodeFn.apply(x01.reshape(-1, 5), P['hash_encoder.embeddings'], offsets, per_level_scale,
                                base_resolution, level_scales).reshape(N, H * W * S, -1)
    sig, col = render_mlp(feats, z, mc_masks.reshape(N, H * W * S), P)
    net_out_s = sig.reshape(N, H, W, S, 1)
    net_out_c = col.reshape(N, H, W, S, 64)
    pe = positional_encoding_pt(raydirs, pe_sky[0], -1, pe_sky[1])
    skynet_out_c = sky_mlp(pe.reshape(N, H * W, -1), z, P).reshape(N, H, W, 1, 64)
    weights = volum_rendering_relu(net_out_s, new_dists * dists_scale, dim=-2)
    weights = weights * torch.logical_not(sky_only_mask).float()
    total_weights = torch.sum(weights, dim=-2, keepdim=True)
    is_gnd = (worldcoord2[..., [0]] <= 1.0).any(dim=-2, keepdim=True)
    nosky_mask = torch.logical_or(torch.logical_not(sky_mask), is_gnd).float()
    sky_weight = 1.0 - total_weights
    sky_avg = torch.mean(skynet_out_c, dim=[1, 2], keepdim=True)
    sky_used = skynet_out_c * (1.0 - nosky_mask) + sky_avg * nosky_mask
    rgbs = torch.clamp(net_out_c, -1, 1) + 1
    rgbs_sky = torch.clamp(sky_used, -1, 1) + 1
    net_out = torch.sum(weights * rgbs, dim=-2, keepdim=True) + sky_weight * rgbs_sky
    return net_out.squeeze(-2) - 1
