"""Host side of the fused per-pixel renderer (libsdb200: sdb_render_rays_forward & friends).

Mirrors the role of Generator._forward_perpix (imaginaire/generators/scenedreamer.py:313-428) and
of the tile loop in inference_givenstyle (:600-628): given the ray/voxel intersection buffers, the
style code and the scene code it returns the per-pixel feature map `net_out` (+ depth, opacity).
All heavy work happens in the CUDA library; torch is used to allocate tensors, to fold the style
modulation into the weights (tiny [256x256] elementwise products, once per style code).
"""
import ctypes
import os

import numpy as np
import torch
import torch.nn.functional as F

from . import _lib, ops

PRECISION_FP16 = 0      # one fp16 tensor-core pass per product (~1e-3 relative)
PRECISION_BF16X3 = 1    # bf16 hi/lo split, 3 passes (~2e-5 relative), range-safe
PRECISION_FP16X3 = 2    # fp16 hi/lo split, 3 passes (~1e-6 relative, |activations| < 65504): the parity default


class _RenderParams(ctypes.Structure):
    _fields_ = [
        ('n_img', ctypes.c_int32), ('H', ctypes.c_int32), ('W', ctypes.c_int32), ('M', ctypes.c_int32),
        ('S', ctypes.c_int32),
        ('d_voxel_id', ctypes.c_void_p), ('d_depth2', ctypes.c_void_p), ('d_raydirs', ctypes.c_void_p),
        ('d_cam_ori', ctypes.c_void_p),
        ('voxel_dims', ctypes.c_float * 3),
        ('d_global_enc', ctypes.c_void_p),
        ('sample_depth', ctypes.c_float), ('dists_scale', ctypes.c_float),
        ('d_fractions', ctypes.c_void_p), ('d_uniforms', ctypes.c_void_p),
        ('d_label_lut', ctypes.c_void_p), ('n_lut', ctypes.c_int32),
        ('d_table', ctypes.c_void_p), ('d_table3', ctypes.c_void_p),
        ('L', ctypes.c_int32), ('log2_T', ctypes.c_int32), ('level_S', ctypes.c_float), ('base_res', ctypes.c_int32),
        ('d_mlp_pack', ctypes.c_void_p), ('mlp_pack_stride', ctypes.c_int64), ('precision', ctypes.c_int32),
        ('d_sky', ctypes.c_void_p), ('d_sky_avg', ctypes.c_void_p),
        ('d_net_out', ctypes.c_void_p), ('d_depth_out', ctypes.c_void_p), ('d_total_weight', ctypes.c_void_p),
        ('d_weights_out', ctypes.c_void_p), ('d_rand_depth_out', ctypes.c_void_p),
        ('d_workspace', ctypes.c_void_p),
        ('early_stop_transmittance', ctypes.c_float),
        ('cam_ori_value', ctypes.c_float * 3),
    ]


# Default early-termination threshold of the inference path: a ray tile stops once every live ray's transmittance is
# below it.  The samples skipped carry less than this compositing weight, i.e. < 2e-7 on net_out and < 1e-4 on a depth
# of ~1000 voxels -- far inside the 1e-3 parity bar; 0 turns it off (the reference's arithmetic sample for sample).
EARLY_STOP_T = 1e-7


def _ptr(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def _stream(dev):
    return ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)


_MOD_LAYERS = (2, 3, 4, 5, 6)
_MOD_FIELDS = ('weight', 'weight_alpha', 'bias_alpha', 'weight_beta', 'bias_beta')


def _modulated_weights_torch(P, z, prefix='render_net'):
    p = prefix + '.'
    wh, bh = [], []
    for k in _MOD_LAYERS:
        n = p + 'fc_%d' % k
        alpha = torch.addmm(P[n + '.bias_alpha'].unsqueeze(0), z.unsqueeze(0), P[n + '.weight_alpha'].t())   # [1, I]
        beta = torch.addmm(P[n + '.bias_beta'].unsqueeze(0), z.unsqueeze(0), P[n + '.weight_beta'].t())      # [1, O]
        wh.append(P[n + '.weight'].unsqueeze(0) * alpha.unsqueeze(1))                                         # [1, O, I]
        bh.append(beta)
    return torch.cat(wh, 0).contiguous(), torch.cat(bh, 0).contiguous()


def _ptr_array(tensors):
    return (ctypes.c_void_p * len(tensors))(*[t.data_ptr() for t in tensors])


class _ModulateFn(torch.autograd.Function):
    """(wh [5,O,I], bh [5,O]) = fold(z [Cz], the 25 ModLinear tensors) on the device in two launches; backward in three
    (csrc/modulate.cu) instead of autograd's chain of small ATen nodes."""

    @staticmethod
    def forward(ctx, z, *params):
        L = _lib.lib()
        dev = z.device
        O, I = params[0].shape
        Cz = z.numel()
        zc = z.detach().contiguous()
        ps = [t.detach() for t in params]
        with torch.cuda.device(dev):
            alpha = torch.empty(5, I, dtype=torch.float32, device=dev)
            wh = torch.empty(5, O, I, dtype=torch.float32, device=dev)
            bh = torch.empty(5, O, dtype=torch.float32, device=dev)
            _lib.check(L.sdb_modulate_forward(_ptr_array(ps), _ptr(zc), int(O), int(I), int(Cz), _ptr(alpha), _ptr(wh), _ptr(bh),
                                              _stream(dev)), 'sdb_modulate_forward')
        ctx.save_for_backward(zc, alpha, *ps)
        ctx.dims = (int(O), int(I), int(Cz))
        return wh, bh

    @staticmethod
    def backward(ctx, g_wh, g_bh):
        L = _lib.lib()
        zc, alpha, *ps = ctx.saved_tensors
        dev = zc.device
        O, I, Cz = ctx.dims
        with torch.cuda.device(dev):
            g_wh = (g_wh if g_wh is not None else torch.zeros(5, O, I, device=dev)).to(torch.float32).contiguous()
            g_bh = (g_bh if g_bh is not None else torch.zeros(5, O, device=dev)).to(torch.float32).contiguous()
            grads = [torch.empty_like(t) for t in ps]
            dalpha = torch.empty(5, I, dtype=torch.float32, device=dev)
            dz = torch.empty(Cz, dtype=torch.float32, device=dev)
            _lib.check(L.sdb_modulate_backward(_ptr_array(ps), _ptr_array(grads), _ptr(zc), _ptr(alpha), _ptr(g_wh), _ptr(g_bh),
                                               O, I, Cz, _ptr(dalpha), _ptr(dz), _stream(dev)), 'sdb_modulate_backward')
        return (dz,) + tuple(grads)


def modulated_weights(P, z, prefix='render_net'):
    """Fold the style modulation of ModLinear into plain weights for ONE style code z [256]
    (model_utils/layers.py:247-260): W' = W * alpha (per input column), bias = beta.  Differentiable w.r.t. the 25 tensors
    and z; on CUDA float32 contiguous inputs one fused forward / backward (csrc/modulate.cu), otherwise the same algebra in torch
    ops (SDB200_FUSED_MOD=0 forces that)."""
    p = prefix + '.'
    names = [p + 'fc_%d.%s' % (k, f) for f in _MOD_FIELDS for k in _MOD_LAYERS]
    ts = [P[n] for n in names]
    ok = z.is_cuda and z.dim() == 1 and os.environ.get('SDB200_FUSED_MOD', '1') != '0' and \
        all(t.is_cuda and t.dtype == torch.float32 and t.is_contiguous() and t.device == z.device for t in ts + [z])
    if ok:
        O, I = ts[0].shape
        Cz = z.numel()
        ok = all(tuple(ts[l].shape) == (O, I) and tuple(ts[5 + l].shape) == (I, Cz) and tuple(ts[10 + l].shape) == (I,) and
                 tuple(ts[15 + l].shape) == (O, Cz) and tuple(ts[20 + l].shape) == (O,) for l in range(5))
    if not ok:
        return _modulated_weights_torch(P, z, prefix)
    return _ModulateFn.apply(z, *ts)


def pack_mlp(P, z, precision=PRECISION_FP16X3, prefix='render_net'):
    """z [N, 256] (style_net output) -> uint8 tensor [N, pack_bytes] on z's device."""
    L = _lib.lib()
    dev = z.device
    nbytes = int(L.sdb_mlp_pack_bytes(int(precision)))
    N = z.shape[0]
    pack = torch.empty(N, nbytes, dtype=torch.uint8, device=dev)
    p = prefix + '.'
    w1 = P[p + 'fc_1.weight'].contiguous()
    b1 = P[p + 'fc_1.bias'].contiguous()
    emb = P[p + 'fc_m_a.weight'].t().contiguous()            # [labels, 256]
    wsig = P[p + 'fc_sigma.weight'].reshape(-1).contiguous()
    bsig = P[p + 'fc_sigma.bias'].reshape(-1).contiguous()
    wout = P[p + 'fc_out_c.weight'].contiguous()
    bout = P[p + 'fc_out_c.bias'].contiguous()
    with torch.cuda.device(dev):
        for i in range(N):
            wh, bh = modulated_weights(P, z[i], prefix)
            code = L.sdb_pack_mlp(_ptr(w1), _ptr(b1), _ptr(emb), int(emb.shape[0]), _ptr(wh), _ptr(bh), _ptr(wsig),
                                  _ptr(bsig), _ptr(wout), _ptr(bout), int(precision), _ptr(pack[i]), _stream(dev))
            _lib.check(code, 'sdb_pack_mlp')
    return pack


def preblend_table(embeddings, global_enc, log2_T=19, per_level_scale=None, base_res=16, L=16):
    """[L*T, 8] raw 5-D hash table + scene code [2] -> pre-blended 3-D table of the same shape."""
    dev = embeddings.device
    out = torch.empty_like(embeddings)
    genc = global_enc.reshape(-1)[:2].to(dev, torch.float32).contiguous()
    with torch.cuda.device(dev):
        code = _lib.lib().sdb_preblend_table(_ptr(embeddings), _ptr(out), int(L), int(log2_T),
                                             float(np.log2(per_level_scale)), int(base_res), _ptr(genc),
                                             _stream(dev))
    _lib.check(code, 'sdb_preblend_table')
    return out


_fraction_cache = {}


def deterministic_fractions(S, device):
    """torch.linspace(0, 1, S+3)[1:-1] built on the CPU like the reference (mc_utils.py:118-120); one upload per
    (S, device), not one per frame."""
    key = ('det', int(S), str(device))
    t = _fraction_cache.get(key)
    if t is None:
        t = _fraction_cache[key] = torch.linspace(0, 1, S + 3)[1:-1].contiguous().to(device)
    return t


def stratified_offsets(S, device):
    """torch.linspace(0, 1, S+2)[:-1] (mc_utils.py:125)."""
    key = ('str', int(S), str(device))
    t = _fraction_cache.get(key)
    if t is None:
        t = _fraction_cache[key] = torch.linspace(0, 1, S + 2, device=device)[:-1].contiguous()
    return t


def pack_sky_mlp(P, z, precision=PRECISION_FP16X3, prefix='sky_net'):
    """z [N, 256] -> uint8 [N, sky_pack_bytes]: SKYMLP weights with fc_z_a(z) folded into the first bias."""
    L = _lib.lib()
    dev = z.device
    nbytes = int(L.sdb_sky_pack_bytes(int(precision)))
    N = z.shape[0]
    pack = torch.empty(N, nbytes, dtype=torch.uint8, device=dev)
    p = prefix + '.'
    w1 = P[p + 'fc1.weight'].contiguous()
    wh = torch.stack([P[p + 'fc%d.weight' % k] for k in (2, 3, 4, 5)]).contiguous()
    bh = torch.stack([P[p + 'fc%d.bias' % k] for k in (2, 3, 4, 5)]).contiguous()
    wout = P[p + 'fc_out_c.weight'].contiguous()
    bout = P[p + 'fc_out_c.bias'].contiguous()
    zz = F.linear(z, P[p + 'fc_z_a.weight'])                      # [N, 256]  (gancraft_base.py:159)
    with torch.cuda.device(dev):
        for i in range(N):
            b1 = (P[p + 'fc1.bias'] + zz[i]).contiguous()
            code = L.sdb_pack_sky_mlp(_ptr(w1), _ptr(b1), _ptr(wh), _ptr(bh), _ptr(wout), _ptr(bout), int(precision),
                                      _ptr(pack[i]), _stream(dev))
            _lib.check(code, 'sdb_pack_sky_mlp')
    return pack


def sky_forward(raydirs, sky_pack, precision=PRECISION_FP16X3):
    """a9 on the tensor-core engine: raydirs [N,H,W,1,3] -> (sky [N,H,W,64], sky_avg [N,64])."""
    dev = raydirs.device
    N, H, W = raydirs.shape[:3]
    if not raydirs.is_cuda or not raydirs.is_contiguous() or raydirs.dtype != torch.float32:
        raise RuntimeError('raydirs must be a contiguous float32 CUDA tensor')
    L = _lib.lib()
    sky = torch.empty(N, H, W, 64, dtype=torch.float32, device=dev)
    avg = torch.empty(N, 64, dtype=torch.float32, device=dev)
    ws = torch.empty(int(L.sdb_sky_workspace_bytes(N, H, W)), dtype=torch.uint8, device=dev)
    stride = int(sky_pack.stride(0)) if (sky_pack.dim() == 2 and sky_pack.shape[0] > 1) else 0
    with torch.cuda.device(dev):
        code = L.sdb_sky_forward(_ptr(raydirs), N, H, W, _ptr(sky_pack), stride, int(precision), _ptr(sky), _ptr(avg),
                                 _ptr(ws), _stream(dev))
    _lib.check(code, 'sdb_sky_forward')
    return sky, avg


def sky_features(P, raydirs, z, prefix='sky_net', pe=(5, True)):
    """a9 through cuBLAS (kept as an independent cross-check of sky_forward): PE(raydir) -> SKYMLP
    (gancraft_base.py:150-169).  raydirs [N,H,W,1,3], z [N,256] -> [N,H,W,64]."""
    N, H, W = raydirs.shape[:3]
    enc = ops.positional_encoding(raydirs.contiguous(), pe[0], -1, pe[1]).reshape(N, H * W, -1)
    p = prefix + '.'
    zz = F.linear(z, P[p + 'fc_z_a.weight']).unsqueeze(1)
    y = F.leaky_relu(F.linear(enc, P[p + 'fc1.weight'], P[p + 'fc1.bias']) + zz, 0.2)
    for k in (2, 3, 4, 5):
        y = F.leaky_relu(F.linear(y, P[p + 'fc%d.weight' % k], P[p + 'fc%d.bias' % k]), 0.2)
    return F.linear(y, P[p + 'fc_out_c.weight'], P[p + 'fc_out_c.bias']).reshape(N, H, W, -1)


def render_rays_forward(voxel_id, depth2, raydirs, cam_ori, global_enc, voxel_dims, label_lut, mlp_pack, sky, sky_avg,
                        table=None, table3=None, num_samples=24, sample_depth=3.0, dists_scale=0.25, uniforms=None,
                        precision=PRECISION_FP16X3, per_level_scale=None, base_res=16, log2_T=19, L=16,
                        want_depth=True, want_samples=False, early_stop=None):
    """Fused a2-a12.  Shapes follow the reference:
    voxel_id [N,H,W,M,1] int32, depth2 [N,2,H,W,M,1], raydirs [N,H,W,1,3], cam_ori [N,3], global_enc [N,2],
    sky [N,H,W,64], sky_avg [N,64]; label_lut int32 [n] (ignore already mapped to dirt).
    Returns dict(net_out [N,H,W,64], depth [N,H,W], total_weight [N,H,W] and, with want_samples,
    weights / rand_depth [N,H,W,S,1] as _forward_perpix returns them)."""
    dev = voxel_id.device
    N, H, W, M = voxel_id.shape[:4]
    S = int(num_samples)
    for t, n in ((voxel_id, 'voxel_id'), (depth2, 'depth2'), (raydirs, 'raydirs'), (sky, 'sky')):
        if not t.is_cuda or not t.is_contiguous():
            raise RuntimeError('%s must be a contiguous CUDA tensor' % n)
    if voxel_id.dtype != torch.int32:
        raise RuntimeError('voxel_id must be int32')
    net_out = torch.empty(N, H, W, 64, dtype=torch.float32, device=dev)
    depth = torch.empty(N, H, W, dtype=torch.float32, device=dev) if want_depth else None
    tw = torch.empty(N, H, W, dtype=torch.float32, device=dev) if want_depth else None
    wts = torch.empty(N, H, W, S, 1, dtype=torch.float32, device=dev) if want_samples else None
    rdp = torch.empty(N, H, W, S, 1, dtype=torch.float32, device=dev) if want_samples else None
    Lb = _lib.lib()
    ws = torch.empty(int(Lb.sdb_render_workspace_bytes(N, H, W)), dtype=torch.uint8, device=dev)
    genc = global_enc.to(dev, torch.float32).reshape(N, 2).contiguous()
    lut = label_lut.to(dev, torch.int32).contiguous()
    sky = sky.reshape(N, H, W, 64)
    sky_avg = sky_avg.to(dev, torch.float32).reshape(N, 64).contiguous()
    prm, keep = _RenderParams(), []
    _fill_render_params(prm, keep, voxel_id, depth2, raydirs, cam_ori, genc, voxel_dims, lut, mlp_pack, sky, sky_avg,
                        table=table, table3=table3, S=S, sample_depth=sample_depth, dists_scale=dists_scale, uniforms=uniforms,
                        precision=precision, per_level_scale=per_level_scale, base_res=base_res, log2_T=log2_T, L=L,
                        net_out=net_out, depth=depth, tw=tw, wts=wts, rdp=rdp, ws=ws,
                        early_stop=EARLY_STOP_T if early_stop is None else early_stop)
    with torch.cuda.device(dev):
        code = Lb.sdb_render_rays_forward(ctypes.byref(prm), _stream(dev))
    _lib.check(code, 'sdb_render_rays_forward')
    # `workspace`: int32[0] = number of live (non sky-only) 16x8 ray tiles the kernel shaded (diagnostics / bench bookkeeping)
    return dict(net_out=net_out, depth=depth, total_weight=tw, weights=wts, rand_depth=rdp, workspace=ws)


def reduced_label_lut(mc2reduced, ignore_id=0, dirt_id=3):
    """mc id -> reduced label with ignore -> dirt folded in (mc_utils.py:241-246, ign2dirt=True)."""
    lut = torch.as_tensor(mc2reduced).to(torch.int32).clone()
    lut[lut == ignore_id] = dirt_id
    return lut


class FusedPerPixelRenderer:
    """Caches per-style weight packs, the per-scene pre-blended table and runs one frame.

    P: dict of parameters with the reference's state-dict names (render_net.*, sky_net.*,
    hash_encoder.embeddings) on the CUDA device."""

    def __init__(self, P, voxel_dims, label_lut, per_level_scale, precision=PRECISION_FP16X3, preblend=True,
                 base_res=16, log2_T=19, L=16):
        self.P, self.voxel_dims, self.lut = P, [float(v) for v in voxel_dims], label_lut
        self.pls, self.precision, self.preblend = per_level_scale, precision, preblend
        self.base_res, self.log2_T, self.L = base_res, log2_T, L
        self.invalidate()
        self.lut_dev = None
        self.sky_impl = 'native'     # 'native' = sdb_sky_forward (wgmma), 'torch' = cuBLAS cross-check
        self.early_stop = None       # None = module default EARLY_STOP_T, 0 = off

    # Cache keys hold a REFERENCE to the keyed tensor (so its address cannot be recycled for another tensor while the
    # entry lives) and compare identity + torch's version counter.  A fresh style code per call -- what the reference's
    # style_net produces -- is a new object and repacks.  Edits that bypass the version counter (`.data`) need invalidate().
    @staticmethod
    def _same(entry, t, extra):
        return entry is not None and entry[0] is t and entry[1] == t._version and entry[2] == extra

    def invalidate(self):
        self._pack_key = self._pack = self._t3_key = self._t3 = self._sky_key = self._sky_pack = None

    def pack_for(self, z):
        if not self._same(self._pack_key, z, self.precision):
            self._pack, self._pack_key = pack_mlp(self.P, z, self.precision), (z, z._version, self.precision)
        return self._pack

    def sky_pack_for(self, z):
        if not self._same(self._sky_key, z, self.precision):
            self._sky_pack, self._sky_key = pack_sky_mlp(self.P, z, self.precision), (z, z._version, self.precision)
        return self._sky_pack

    def table3_for(self, global_enc):
        """Pre-blended table of this scene code.  Keyed on the scene-code tensor OBJECT (+ version) and on the table's
        storage + version: no device->host read of the code on the frame path."""
        emb = self.P['hash_encoder.embeddings']
        extra = (emb.data_ptr(), emb._version)
        if not self._same(self._t3_key, global_enc, extra):
            self._t3 = preblend_table(emb, global_enc, self.log2_T, self.pls, self.base_res, self.L)
            self._t3_key = (global_enc, global_enc._version, extra)
        return self._t3

    def forward(self, voxel_id, depth2, raydirs, cam_ori, z, global_enc, num_samples=24, sample_depth=3.0,
                dists_scale=0.25, uniforms=None, sky_avg=None, sky=None, want_samples=False):
        N = voxel_id.shape[0]
        if sky is None:
            if self.sky_impl == 'native':
                sky, avg = sky_forward(raydirs, self.sky_pack_for(z), self.precision)
                sky_avg = avg if sky_avg is None else sky_avg
            else:
                sky = sky_features(self.P, raydirs, z)
        if sky_avg is None:
            sky_avg = sky.mean(dim=(1, 2))                       # scenedreamer.py:395 / :597
        pack = self.pack_for(z)
        if self.lut_dev is None or self.lut_dev.device != voxel_id.device:
            self.lut_dev = self.lut.to(voxel_id.device, torch.int32).contiguous()      # once, not one H2D per frame
        kw = {}
        if self.preblend and N == 1:
            kw['table3'] = self.table3_for(global_enc)
        else:
            kw['table'] = self.P['hash_encoder.embeddings']
        out = render_rays_forward(voxel_id, depth2, raydirs, cam_ori, global_enc, self.voxel_dims, self.lut_dev, pack, sky,
                                  sky_avg, num_samples=num_samples, sample_depth=sample_depth, dists_scale=dists_scale,
                                  uniforms=uniforms, precision=self.precision, per_level_scale=self.pls,
                                  base_res=self.base_res, log2_T=self.log2_T, L=self.L, want_samples=want_samples,
                                  early_stop=self.early_stop, **kw)
        out['sky'], out['sky_avg'] = sky, sky_avg
        return out


# ================================================================================================
# Training: fused forward that records the pass + the fused backward (sdb_render_rays_backward)
# ================================================================================================
# The training record and the backward workspace are several GB each (3.9 + 4.0 KB per sample).  Asking torch's caching
# allocator for them every step makes it split and re-grow its multi-GB blocks (a 7.4 GB request right after a 6.9 GB
# one was carved out of the cached 7.4 GB block ends in cudaMalloc) -- measured as 10-40 ms of jitter per step.  They are
# therefore recycled through this small pool: ONE parked buffer per (device, role); a buffer of another size replaces the
# parked one (a crop-size change does not accumulate multi-GB entries), further buffers of a multi-view batch go back to
# torch's allocator.  Reuse is stream-ordered: forward and backward of a step run on the same (current) stream.
_scratch_pool = {}


def _take_scratch(nbytes, dev, role):
    key = (str(dev), role)
    t = _scratch_pool.pop(key, None)
    if t is not None and t.numel() == int(nbytes):
        return t
    del t                                                    # wrong size: release it before asking for the new one
    return torch.empty(int(nbytes), dtype=torch.uint8, device=dev)


def _give_scratch(t, role):
    if t is not None:
        _scratch_pool[(str(t.device), role)] = t             # replaces (and thereby frees) a parked buffer of another size


def clear_scratch():
    """Hand the parked training record / backward workspace (several GB) back to torch's allocator."""
    _scratch_pool.clear()


class _RenderGrads(ctypes.Structure):
    _fields_ = [
        ('d_grad_net_out', ctypes.c_void_p), ('d_bwd_pack', ctypes.c_void_p), ('bwd_pack_stride', ctypes.c_int64),
        ('d_table', ctypes.c_void_p),
        ('d_grad_table', ctypes.c_void_p), ('d_grad_global_enc', ctypes.c_void_p), ('d_grad_w1ext', ctypes.c_void_p),
        ('d_grad_wh', ctypes.c_void_p), ('d_grad_wsig', ctypes.c_void_p), ('d_grad_wout', ctypes.c_void_p),
        ('d_grad_sky', ctypes.c_void_p), ('d_grad_sky_avg', ctypes.c_void_p), ('d_workspace', ctypes.c_void_p),
    ]


class _RenderViewGrads(ctypes.Structure):
    _fields_ = [('g', _RenderGrads), ('w1ext_stride', ctypes.c_int64), ('wh_stride', ctypes.c_int64),
                ('wsig_stride', ctypes.c_int64), ('wout_stride', ctypes.c_int64), ('sky_avg_stride', ctypes.c_int64)]


class _SkyViewGrads(ctypes.Structure):
    _fields_ = [('d_grad_w1ext', ctypes.c_void_p), ('w1ext_stride', ctypes.c_int64), ('d_grad_wh', ctypes.c_void_p),
                ('wh_stride', ctypes.c_int64), ('d_grad_wout', ctypes.c_void_p), ('wout_stride', ctypes.c_int64)]


def _view_sum(g):
    """Gradient of a tensor all views share: the sum of the per-view gradients [N, ...] (the one view itself when N == 1)."""
    return g[0] if g.shape[0] == 1 else g.sum(0)


def _fill_render_params(prm, keep, voxel_id, depth2, raydirs, cam_ori, genc, voxel_dims, lut, mlp_pack, sky, sky_avg, *,
                        table=None, table3=None, S, sample_depth, dists_scale, uniforms, precision, per_level_scale, base_res,
                        log2_T, L, net_out, depth, tw, wts, rdp, ws, early_stop=0.0):
    """Fills an sdb_render_params over the raw `table` or the pre-blended `table3` (the other is None); `keep` collects
    tensors that must outlive the call.  A host-side camera origin of a single view is passed by value (no H2D copy to wait
    for); any other goes to the device.  A 2-D `mlp_pack` of several rows holds one pack per image."""
    dev = voxel_id.device
    N, H, W, M = voxel_id.shape[:4]
    if uniforms is None:
        frac = deterministic_fractions(S, dev)
    else:
        frac = stratified_offsets(S, dev)
        uniforms = uniforms.to(dev, torch.float32).reshape(N * H * W, S + 1).contiguous()
    prm.n_img, prm.H, prm.W, prm.M, prm.S = N, H, W, M, S
    prm.d_voxel_id, prm.d_depth2, prm.d_raydirs = _ptr(voxel_id), _ptr(depth2), _ptr(raydirs)
    if not cam_ori.is_cuda and N == 1:
        prm.d_cam_ori, prm.cam_ori_value = None, (ctypes.c_float * 3)(*[float(v) for v in cam_ori.reshape(3)])
    else:
        cam_ori = cam_ori.to(dev, torch.float32).reshape(N, 3).contiguous()
        prm.d_cam_ori = _ptr(cam_ori)
    keep += [frac, uniforms, cam_ori]
    prm.voxel_dims = (ctypes.c_float * 3)(*[float(v) for v in voxel_dims])
    prm.d_global_enc = _ptr(genc)
    prm.sample_depth, prm.dists_scale = float(sample_depth), float(dists_scale)
    prm.d_fractions, prm.d_uniforms = _ptr(frac), _ptr(uniforms)
    prm.d_label_lut, prm.n_lut = _ptr(lut), int(lut.numel())
    prm.d_table, prm.d_table3 = _ptr(table), _ptr(table3)
    prm.L, prm.log2_T, prm.level_S, prm.base_res = int(L), int(log2_T), float(np.log2(per_level_scale)), int(base_res)
    prm.d_mlp_pack = _ptr(mlp_pack)
    prm.mlp_pack_stride = int(mlp_pack.stride(0)) if (mlp_pack.dim() == 2 and mlp_pack.shape[0] > 1) else 0
    prm.precision = int(precision)
    prm.early_stop_transmittance = float(early_stop)
    prm.d_sky, prm.d_sky_avg = _ptr(sky), _ptr(sky_avg)
    prm.d_net_out, prm.d_depth_out, prm.d_total_weight = _ptr(net_out), _ptr(depth), _ptr(tw)
    prm.d_weights_out, prm.d_rand_depth_out = _ptr(wts), _ptr(rdp)
    prm.d_workspace = _ptr(ws)
    return prm


class _FusedRenderTrainFn(torch.autograd.Function):
    """net_out = fused_render(embeddings, global_enc, effective LightningMLP weights, sky, sky_avg).

    N views of one scene in one recorded pass.  wh [N,5,256,256], bh [N,5,256] are what ModLinear produces for each
    view's style code (W' = W * alpha, beta; layers.py:247-260): the caller computes them with ordinary torch ops so that
    autograd carries dL/dW', dL/dbeta on to the raw parameters and to the style codes.  sky [N,H,W,64], sky_avg [N,64];
    genc holds the one scene code of all views.  The weights every view shares get the sum of the per-view gradients."""

    @staticmethod
    def forward(ctx, cfg, embeddings, genc, w1, b1, fc_m_a, wh, bh, wsig, bsig, wout, bout, sky, sky_avg):
        L = _lib.lib()
        voxel_id, depth2, raydirs = cfg['voxel_id'], cfg['depth2'], cfg['raydirs']
        dev = voxel_id.device
        N, H, W, M = voxel_id.shape[:4]
        if tuple(wh.shape[:2]) != (N, 5) or tuple(bh.shape[:2]) != (N, 5):
            raise RuntimeError('fused training path: wh / bh need one [5, ...] set per view')
        S = int(cfg['num_samples'])
        for t, n in ((voxel_id, 'voxel_id'), (depth2, 'depth2'), (raydirs, 'raydirs')):
            if not t.is_cuda or not t.is_contiguous():
                raise RuntimeError('%s must be a contiguous CUDA tensor' % n)
        f32 = lambda t: t.detach().to(dev, torch.float32).contiguous()
        embeddings_, genc_ = f32(embeddings), f32(genc).reshape(-1)[:2].contiguous()
        w1_, b1_, wh_, bh_ = f32(w1), f32(b1), f32(wh), f32(bh)
        emb_ = f32(fc_m_a).t().contiguous()                         # [labels, 256]
        wsig_, bsig_, wout_, bout_ = f32(wsig).reshape(-1), f32(bsig).reshape(-1), f32(wout), f32(bout)
        sky_, sky_avg_ = f32(sky).reshape(N, H, W, 64), f32(sky_avg).reshape(N, 64)
        cam_ori = cfg['cam_ori'].to(dev, torch.float32).reshape(N, 3).contiguous()
        lut = cfg['lut'].to(dev, torch.int32).contiguous()
        prec = int(cfg['precision'])
        with torch.cuda.device(dev):
            pack = torch.empty(N, int(L.sdb_mlp_pack_bytes(prec)), dtype=torch.uint8, device=dev)      # one pack per view
            for i in range(N):
                _lib.check(L.sdb_pack_mlp(_ptr(w1_), _ptr(b1_), _ptr(emb_), int(emb_.shape[0]), _ptr(wh_[i]), _ptr(bh_[i]),
                                          _ptr(wsig_), _ptr(bsig_), _ptr(wout_), _ptr(bout_), prec, _ptr(pack[i]), _stream(dev)),
                           'sdb_pack_mlp')
            table3 = preblend_table(embeddings_, genc_, cfg['log2_T'], cfg['per_level_scale'], cfg['base_res'], cfg['L'])
            net_out = torch.empty(N, H, W, 64, dtype=torch.float32, device=dev)
            depth = torch.empty(N, H, W, dtype=torch.float32, device=dev)
            tw = torch.empty(N, H, W, dtype=torch.float32, device=dev)
            wts = torch.empty(N, H, W, S, 1, dtype=torch.float32, device=dev)
            rdp = torch.empty(N, H, W, S, 1, dtype=torch.float32, device=dev)
            ws = torch.empty(int(L.sdb_render_workspace_bytes(N, H, W)), dtype=torch.uint8, device=dev)
            recompute = bool(cfg.get('recompute'))
            # recompute: no record now -- the backward rebuilds each view's record just before differentiating it, from what
            # ctx.keep holds alive (rays, uniforms, camera origins, packs, table3, sky, sky_avg).  The inference kernel without
            # early termination computes what the recording kernel computes, bit for bit.
            record = None if recompute else _take_scratch(L.sdb_render_train_record_bytes(N, H, W, S), dev, 'record')
            prm, keep = _RenderParams(), []
            _fill_render_params(prm, keep, voxel_id, depth2, raydirs, cam_ori, genc_, cfg['voxel_dims'], lut, pack, sky_, sky_avg_,
                                table3=table3, S=S, sample_depth=cfg['sample_depth'], dists_scale=cfg['dists_scale'],
                                uniforms=cfg.get('uniforms'), precision=prec, per_level_scale=cfg['per_level_scale'],
                                base_res=cfg['base_res'], log2_T=cfg['log2_T'], L=cfg['L'], net_out=net_out, depth=depth, tw=tw,
                                wts=wts, rdp=rdp, ws=ws)
            if recompute:
                _lib.check(L.sdb_render_rays_forward(ctypes.byref(prm), _stream(dev)), 'sdb_render_rays_forward')
            else:
                _lib.check(L.sdb_render_rays_train_forward(ctypes.byref(prm), _ptr(record), _stream(dev)),
                           'sdb_render_rays_train_forward')
        ctx.cfg, ctx.prm, ctx.keep = cfg, prm, keep + [cam_ori, lut, pack, table3, net_out, depth, tw, wts, rdp, ws, genc_, sky_,
                                                       sky_avg_]
        ctx.record, ctx.recompute, ctx.released = record, recompute, False
        if recompute:
            # the backward reads the caller's rays, uniforms, camera origins and sky features again: saved so that autograd
            # refuses a backward after one of them was modified in place instead of differentiating another pass
            ctx.save_for_backward(voxel_id, depth2, raydirs, sky_, sky_avg_, *[t for t in keep if t is not None])
        ctx.saved = (embeddings_, w1_, wh_, wsig_, wout_)
        ctx.shapes = (tuple(fc_m_a.shape), tuple(wsig.shape), tuple(bsig.shape), tuple(sky.shape), tuple(sky_avg.shape),
                      tuple(genc.shape), tuple(wh.shape), tuple(bh.shape))
        ctx.mark_non_differentiable(depth, tw, wts, rdp)
        return net_out, depth, tw, wts, rdp

    @staticmethod
    def backward(ctx, g_net_out, *_unused):
        L = _lib.lib()
        if ctx.released:
            raise RuntimeError('fused render: the training record of this pass was released by its first backward '
                               '(retain_graph / double backward are not supported on the fused path)')
        if ctx.recompute:
            ctx.saved_tensors      # the version check of the inputs the recompute reads (RuntimeError if one was modified)
        cfg, prm = ctx.cfg, ctx.prm
        embeddings_, w1_, wh_, wsig_, wout_ = ctx.saved
        dev = embeddings_.device
        N, H, W, S = prm.n_img, prm.H, prm.W, prm.S
        g = g_net_out.to(torch.float32).contiguous()
        with torch.cuda.device(dev):
            bpack = torch.empty(N, int(L.sdb_mlp_backward_pack_bytes()), dtype=torch.uint8, device=dev)      # one per view
            for i in range(N):
                _lib.check(L.sdb_pack_mlp_backward(_ptr(w1_), _ptr(wh_[i]), _ptr(wsig_), _ptr(wout_), _ptr(bpack[i]), _stream(dev)),
                           'sdb_pack_mlp_backward')
            g_table = torch.empty_like(embeddings_)
            g_genc = torch.empty(2, dtype=torch.float32, device=dev)
            g_w1ext = torch.empty(N, 256, 144, dtype=torch.float32, device=dev)
            g_wh = torch.empty(N, 5, 256, 272, dtype=torch.float32, device=dev)
            g_wsig = torch.empty(N, 8, 272, dtype=torch.float32, device=dev)
            g_wout = torch.empty(N, 64, 272, dtype=torch.float32, device=dev)
            g_sky = torch.empty(N, H, W, 64, dtype=torch.float32, device=dev)      # every ray's is written (sdb200.h)
            g_sky_avg = torch.empty(N, 64, dtype=torch.float32, device=dev)
            wsb = _take_scratch(L.sdb_render_backward_workspace_bytes(N, H, W, S, int(cfg['L']), int(cfg['log2_T'])), dev, 'bwd')
            vg = _RenderViewGrads()
            gr = vg.g
            gr.d_grad_net_out, gr.d_bwd_pack, gr.bwd_pack_stride = _ptr(g), _ptr(bpack), int(bpack.stride(0))
            gr.d_table = _ptr(embeddings_)
            gr.d_grad_table, gr.d_grad_global_enc, gr.d_grad_w1ext = _ptr(g_table), _ptr(g_genc), _ptr(g_w1ext)
            gr.d_grad_wh, gr.d_grad_wsig, gr.d_grad_wout = _ptr(g_wh), _ptr(g_wsig), _ptr(g_wout)
            gr.d_grad_sky, gr.d_grad_sky_avg, gr.d_workspace = _ptr(g_sky), _ptr(g_sky_avg), _ptr(wsb)
            vg.w1ext_stride, vg.wh_stride, vg.wsig_stride = g_w1ext.stride(0), g_wh.stride(0), g_wsig.stride(0)
            vg.wout_stride, vg.sky_avg_stride = g_wout.stride(0), g_sky_avg.stride(0)
            if ctx.recompute:
                # one view's record, rebuilt for every view in turn
                record = _take_scratch(L.sdb_render_train_record_bytes(1, H, W, S), dev, 'record')
                _lib.check(L.sdb_render_rays_backward_recompute(ctypes.byref(prm), _ptr(record), ctypes.byref(vg), _stream(dev)),
                           'sdb_render_rays_backward_recompute')
            else:
                record = ctx.record
                _lib.check(L.sdb_render_rays_backward_views(ctypes.byref(prm), _ptr(record), ctypes.byref(vg), _stream(dev)),
                           'sdb_render_rays_backward_views')
        # stream-ordered reuse: the next forward / backward run on the same stream after these kernels
        _give_scratch(wsb, 'bwd')
        _give_scratch(record, 'record')
        ctx.record, ctx.released = None, True
        s_fcma, s_wsig, s_bsig, s_sky, s_skyavg, s_genc, s_wh, s_bh = ctx.shapes
        n_lab = s_fcma[1]
        d_genc = torch.zeros(s_genc, dtype=torch.float32, device=dev)
        d_genc.view(-1)[:2] = g_genc
        return (None, g_table, d_genc,
                _view_sum(g_w1ext[:, :, :128]).contiguous(), _view_sum(g_w1ext[:, :, 143]).contiguous(),
                _view_sum(g_w1ext[:, :, 128:128 + n_lab]).contiguous(),
                g_wh[:, :, :, :256].reshape(s_wh), g_wh[:, :, :, 256].reshape(s_bh),
                _view_sum(g_wsig[:, 0, :256]).reshape(s_wsig), _view_sum(g_wsig[:, 0, 256]).reshape(s_bsig),
                _view_sum(g_wout[:, :, :256]).contiguous(), _view_sum(g_wout[:, :, 256]).contiguous(),
                g_sky.reshape(s_sky), g_sky_avg.reshape(s_skyavg))


class _SkyTrainFn(torch.autograd.Function):
    """sky [N,H,W,64] = SKYMLP(PE(raydirs)) on the wgmma engine, differentiable w.r.t. the weights.
    b1 [N,256] is each view's effective layer-0 bias fc1.bias + fc_z_a(z) (gancraft_base.py:159-160), formed by the caller in
    torch; the other weights are shared by the views and get the sum of their gradients."""

    @staticmethod
    def forward(ctx, raydirs, w1, b1, wh, bh, wout, bout):
        L = _lib.lib()
        dev = raydirs.device
        N, H, W = raydirs.shape[:3]
        if b1.numel() != N * 256:
            raise RuntimeError('fused sky training path: b1 needs one [256] bias per view')
        f32 = lambda t: t.detach().to(dev, torch.float32).contiguous()
        w1_, b1_, wh_, bh_, wout_, bout_ = f32(w1), f32(b1).reshape(N, 256), f32(wh), f32(bh), f32(wout), f32(bout)
        rd = raydirs.detach().contiguous()
        with torch.cuda.device(dev):
            pack = torch.empty(N, int(L.sdb_sky_pack_bytes(PRECISION_FP16X3)), dtype=torch.uint8, device=dev)      # one per view
            for i in range(N):
                _lib.check(L.sdb_pack_sky_mlp(_ptr(w1_), _ptr(b1_[i]), _ptr(wh_), _ptr(bh_), _ptr(wout_), _ptr(bout_),
                                              PRECISION_FP16X3, _ptr(pack[i]), _stream(dev)), 'sdb_pack_sky_mlp')
            sky = torch.empty(N, H, W, 64, dtype=torch.float32, device=dev)
            avg = torch.empty(N, 64, dtype=torch.float32, device=dev)
            ws = torch.empty(int(L.sdb_sky_workspace_bytes(N, H, W)), dtype=torch.uint8, device=dev)
            record = _take_scratch(L.sdb_sky_train_record_bytes(N, H, W), dev, 'sky_record')
            _lib.check(L.sdb_sky_train_forward_views(_ptr(rd), N, H, W, _ptr(pack), int(pack.stride(0)), _ptr(sky), _ptr(avg),
                                                     _ptr(ws), _ptr(record), _stream(dev)), 'sdb_sky_train_forward_views')
        ctx.dims, ctx.record, ctx.saved = (N, H, W), record, (wh_, wout_)
        ctx.shapes = (tuple(b1.shape),)
        return sky

    @staticmethod
    def backward(ctx, g_sky):
        L = _lib.lib()
        if ctx.record is None:
            raise RuntimeError('fused sky branch: the training record was released by the first backward')
        N, H, W = ctx.dims
        wh_, wout_ = ctx.saved
        dev = wh_.device
        g = g_sky.to(torch.float32).contiguous()
        with torch.cuda.device(dev):
            bpack = torch.empty(int(L.sdb_sky_backward_pack_bytes()), dtype=torch.uint8, device=dev)
            _lib.check(L.sdb_pack_sky_mlp_backward(_ptr(wh_), _ptr(wout_), _ptr(bpack), _stream(dev)), 'sdb_pack_sky_mlp_backward')
            g_w1ext = torch.empty(N, 256, 48, dtype=torch.float32, device=dev)
            g_wh = torch.empty(N, 4, 256, 272, dtype=torch.float32, device=dev)
            g_wout = torch.empty(N, 64, 272, dtype=torch.float32, device=dev)
            wsb = _take_scratch(L.sdb_sky_backward_workspace_bytes(N, H, W), dev, 'sky_bwd')
            vg = _SkyViewGrads(_ptr(g_w1ext), g_w1ext.stride(0), _ptr(g_wh), g_wh.stride(0), _ptr(g_wout), g_wout.stride(0))
            _lib.check(L.sdb_sky_backward_views(N, H, W, _ptr(ctx.record), _ptr(g), _ptr(bpack), 0, ctypes.byref(vg), _ptr(wsb),
                                                _stream(dev)), 'sdb_sky_backward_views')
        _give_scratch(wsb, 'sky_bwd')
        _give_scratch(ctx.record, 'sky_record')
        ctx.record = None
        return (None, _view_sum(g_w1ext[:, :, :33]).contiguous(), g_w1ext[:, :, 47].reshape(ctx.shapes[0]),
                _view_sum(g_wh[:, :, :, :256]).contiguous(), _view_sum(g_wh[:, :, :, 256]).contiguous(),
                _view_sum(g_wout[:, :, :256]).contiguous(), _view_sum(g_wout[:, :, 256]).contiguous())


def sky_features_train(P, raydirs, z, prefix='sky_net'):
    """Differentiable a9 on the tensor-core engine for N views: gradients reach P['sky_net.*'] and z [N,256]."""
    p = prefix + '.'
    # gancraft_base.py:159-160, [N,256]; view by view, so that a batch forms each bias exactly as a single-view call does
    b1 = P[p + 'fc1.bias'] + torch.cat([F.linear(z[i:i + 1], P[p + 'fc_z_a.weight']) for i in range(z.shape[0])])
    wh = torch.stack([P[p + 'fc%d.weight' % k] for k in (2, 3, 4, 5)])
    bh = torch.stack([P[p + 'fc%d.bias' % k] for k in (2, 3, 4, 5)])
    return _SkyTrainFn.apply(raydirs, P[p + 'fc1.weight'], b1, wh, bh, P[p + 'fc_out_c.weight'], P[p + 'fc_out_c.bias'])


def render_rays_train(P, voxel_id, depth2, raydirs, cam_ori, z, global_enc, voxel_dims, label_lut, per_level_scale,
                      num_samples=24, sample_depth=3.0, dists_scale=0.25, uniforms=None, base_res=16, log2_T=19, L=16,
                      prefix='render_net', sky_prefix='sky_net', sky_impl='native', sky_avg=None, precision=PRECISION_FP16X3,
                      recompute=False):
    """Differentiable fused a2-a12 for N views of ONE scene in one recorded pass (voxel_id [N,H,W,M,1], z [N,256],
    global_enc [1,2] or N equal rows): gradients reach P['hash_encoder.embeddings'], P['render_net.*'], P['sky_net.*'], z
    and global_enc (everything Generator._forward_perpix differentiates under train.py), summed over the views as autograd
    sums them.  sky_avg: None = each view's own frame mean of its sky features (scenedreamer.py:395), else a caller-supplied
    mean [N or 1, 64] used as every view's (scenedreamer.py:391-392; differentiable when it requires grad).
    sky_impl: 'native' = the sky branch on the tensor-core engine too (sky_features_train), 'torch' = torch autograd /
    cuBLAS fp32 on top of the PE kernel (independent cross-check).
    precision: of the recording forward's MLP, PRECISION_FP16X3 (fp32-grade) or PRECISION_FP16 (one fp16 pass, for
    mixed-precision training); the sky branch and the backward are fp32-grade either way.  The torch glue runs in fp32 with
    autocast off, whatever the caller's autocast state and the dtypes of z / global_enc / sky_avg; autograd hands their
    gradients back in their own dtypes.
    recompute: False = the forward keeps a per-sample record of every view until the backward (about 3.9 KB per sample:
    6.9 GB per 262x262 view at 24 spp); True = it keeps none, and the backward rebuilds one view's record at a time just
    before differentiating that view (sdb_render_rays_backward_recompute), so the record no longer grows with the batch.
    The outputs are the same bit for bit and the gradients differ only in the order of fp32 atomics; the cost is one more
    recording forward per view.  The backward reads voxel_id, depth2, raydirs, uniforms, cam_ori and the sky features again:
    modifying one of them in place between forward and backward makes the backward raise, as for any tensor autograd saved.
    In either mode a second backward through the same graph (retain_graph) raises."""
    with torch.autocast('cuda', enabled=False):
        return _render_rays_train(P, voxel_id, depth2, raydirs, cam_ori, z.float(), global_enc.float(), voxel_dims, label_lut,
                                  per_level_scale, num_samples, sample_depth, dists_scale, uniforms, base_res, log2_T, L, prefix,
                                  sky_prefix, sky_impl, None if sky_avg is None else sky_avg.float(), precision, recompute)


def _render_rays_train(P, voxel_id, depth2, raydirs, cam_ori, z, global_enc, voxel_dims, label_lut, per_level_scale, num_samples,
                       sample_depth, dists_scale, uniforms, base_res, log2_T, L, prefix, sky_prefix, sky_impl, sky_avg, precision,
                       recompute):
    p = prefix + '.'
    N = voxel_id.shape[0]
    if z.shape[0] != N:
        raise ValueError('render_rays_train: z needs one style code per view (%d), got %d' % (N, z.shape[0]))
    mods = [modulated_weights(P, z[i], prefix) for i in range(N)]          # differentiable w.r.t. P and z
    wh, bh = torch.stack([m[0] for m in mods]), torch.stack([m[1] for m in mods])
    if sky_impl == 'native':
        sky = sky_features_train(P, raydirs, z, prefix=sky_prefix)         # [N,H,W,64]
    else:
        sky = sky_features(P, raydirs, z, prefix=sky_prefix)
    if sky_avg is None:                                                    # scenedreamer.py:395, view by view: the same reduction
        sky_avg = torch.cat([sky[i:i + 1].mean(dim=(1, 2)) for i in range(N)]) if N > 1 else sky.mean(dim=(1, 2))  # as one view
    else:
        sky_avg = sky_avg.reshape(-1, 64).expand(N, 64)
    cfg = dict(voxel_id=voxel_id, depth2=depth2, raydirs=raydirs, cam_ori=cam_ori, lut=label_lut, voxel_dims=voxel_dims,
               num_samples=num_samples, sample_depth=sample_depth, dists_scale=dists_scale, uniforms=uniforms,
               per_level_scale=per_level_scale, base_res=base_res, log2_T=log2_T, L=L, precision=precision, recompute=recompute)
    net_out, depth, tw, wts, rdp = _FusedRenderTrainFn.apply(
        cfg, P['hash_encoder.embeddings'], global_enc, P[p + 'fc_1.weight'], P[p + 'fc_1.bias'], P[p + 'fc_m_a.weight'],
        wh, bh, P[p + 'fc_sigma.weight'], P[p + 'fc_sigma.bias'], P[p + 'fc_out_c.weight'], P[p + 'fc_out_c.bias'], sky,
        sky_avg)
    return dict(net_out=net_out, depth=depth, total_weight=tw, weights=wts, rand_depth=rdp, sky=sky, sky_avg=sky_avg)
