"""Host side of the tensor-core RenderCNN (libsdb200: sdb_cnn_pack / sdb_cnn_forward, and under autograd
sdb_cnn_train_forward_ex / sdb_cnn_backward_ex).

Mirrors Base3DGenerator._forward_global (imaginaire/generators/gancraft_base.py:588-603): per-pixel feature map
[N,H,W,64] + style code -> (tanh image, raw image) [N,3,H,W], with RenderCNN.forward (:201-225) evaluated once on the
whole frame.  torch allocates; the style modulation vector fc_z_cond(z) (one 256x1024 GEMV) is computed in torch.
"""
import ctypes

import torch
import torch.nn.functional as F

from . import _lib

PRECISION_FP16 = 0      # one fp16 pass per product (the class of the reference's default, cuDNN TF32)
PRECISION_BF16X3 = 1    # bf16 hi/lo split, 3 passes: the training forward and backward (gradients need bf16's range)
PRECISION_FP16X3 = 2    # fp16 hi/lo split, 3 passes: fp32-grade (parity default)
PRECISION_BF16 = 3      # one bf16 pass per product: the training path under bf16 autocast (training only)

TRAIN_PRECISIONS = (PRECISION_FP16, PRECISION_BF16X3, PRECISION_BF16)

_NAMES = ('conv1.weight', 'conv1.bias', 'conv2a.weight', 'conv2a.bias', 'conv2b.weight', 'conv3a.weight', 'conv3a.bias',
          'conv3b.weight', 'conv4a.weight', 'conv4a.bias', 'conv4b.weight', 'conv4b.bias', 'conv4.weight', 'conv4.bias')


def _ptr(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def _stream(dev):
    return ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)


def supported(P, prefix='denoiser.'):
    """The kernel is specialised for SceneDreamer's RenderCNN: 64 -> 256 hidden -> 3."""
    want = {'conv1.weight': (256, 64, 1, 1), 'conv2a.weight': (256, 256, 3, 3), 'conv2b.weight': (256, 256, 3, 3),
            'conv3a.weight': (256, 256, 3, 3), 'conv3b.weight': (256, 256, 3, 3), 'conv4a.weight': (256, 256, 1, 1),
            'conv4b.weight': (256, 256, 1, 1), 'conv4.weight': (3, 256, 1, 1), 'fc_z_cond.weight': (1024, None)}
    for k, shp in want.items():
        t = P.get(prefix + k)
        if t is None or len(t.shape) != len(shp) or any(a is not None and a != b for a, b in zip(shp, t.shape)):
            return False
    return True


_CONV_W = ('conv1.weight', 'conv2a.weight', 'conv2b.weight', 'conv3a.weight', 'conv3b.weight', 'conv4a.weight', 'conv4b.weight')


class _RenderCNNTrainFn(torch.autograd.Function):
    """(precision, net_out [N,H,W,64], mod [N or 1,4,256], the 14 denoiser tensors in _NAMES order) -> (rgb, raw)
    [N,3,H,W] fp32.  The forward packs the weights at `precision` (one of TRAIN_PRECISIONS) and keeps one record per
    view; the backward runs sdb_cnn_backward_ex per view at the same precision and releases the records."""

    @staticmethod
    def forward(ctx, precision, net_out, mod, *params):
        L = _lib.lib()
        dev = net_out.device
        N, H, W = net_out.shape[:3]
        x = net_out.detach().contiguous()
        m = mod.detach().to(torch.float32).contiguous()
        ws = [t.detach().to(torch.float32).contiguous() for t in params]
        ctx.param_dtypes = [t.dtype for t in params]
        rgb = torch.empty(N, 3, H, W, dtype=torch.float32, device=dev)
        raw = torch.empty(N, 3, H, W, dtype=torch.float32, device=dev)
        with torch.cuda.device(dev):
            pack = torch.empty(int(L.sdb_cnn_pack_bytes_ex(precision)), dtype=torch.uint8, device=dev)
            _lib.check(L.sdb_cnn_pack_ex(*[_ptr(t) for t in ws], precision, _ptr(pack), _stream(dev)), 'sdb_cnn_pack_ex')
            records = []
            for i in range(N):
                rec = torch.empty(int(L.sdb_cnn_train_record_bytes_ex(H, W, precision)), dtype=torch.uint8, device=dev)
                _lib.check(L.sdb_cnn_train_forward_ex(_ptr(x[i]), H, W, _ptr(pack), _ptr(m[i if m.shape[0] > 1 else 0]), precision,
                                                      _ptr(rgb[i]), _ptr(raw[i]), _ptr(rec), _stream(dev)), 'sdb_cnn_train_forward_ex')
                records.append(rec)
        ctx.records, ctx.pack, ctx.mod, ctx.ws, ctx.precision, ctx.mod_dtype = records, pack, m, ws, precision, mod.dtype
        return rgb, raw

    @staticmethod
    def backward(ctx, g_rgb, g_raw):
        if ctx.records is None:
            raise RuntimeError('RenderCNN: the training record of this pass was released by its first backward '
                               '(retain_graph / double backward are not supported on the tensor-core path)')
        L = _lib.lib()
        records, pack, m, ws, prec = ctx.records, ctx.pack, ctx.mod, ctx.ws, ctx.precision
        ctx.records = None
        dev = pack.device
        N = len(records)
        H, W = (g_rgb if g_rgb is not None else g_raw).shape[2:]
        need_x, need_m = ctx.needs_input_grad[1], ctx.needs_input_grad[2]
        need_p = ctx.needs_input_grad[3:]
        g_rgb = g_rgb.to(torch.float32).contiguous() if g_rgb is not None else None
        g_raw = g_raw.to(torch.float32).contiguous() if g_raw is not None else None
        g_x = torch.empty(N, H, W, 64, dtype=torch.float32, device=dev) if need_x else None
        g_m = torch.empty(N, 4, 256, dtype=torch.float32, device=dev) if need_m else None
        g_p = [torch.zeros_like(w) if need else None for w, need in zip(ws, need_p)]
        with torch.cuda.device(dev):
            bpack = torch.empty(int(L.sdb_cnn_backward_pack_bytes_ex(prec)), dtype=torch.uint8, device=dev)
            conv_w = [ws[_NAMES.index(n)] for n in _CONV_W]
            _lib.check(L.sdb_cnn_pack_backward_ex(*[_ptr(t) for t in conv_w], prec, _ptr(bpack), _stream(dev)),
                       'sdb_cnn_pack_backward_ex')
            work = torch.empty(int(L.sdb_cnn_backward_workspace_bytes_ex(H, W, prec)), dtype=torch.uint8, device=dev)
            view_p = [torch.empty_like(t) if t is not None else None for t in g_p] if N > 1 else g_p
            for i in range(N):
                grads = _CnnGrads(_ptr(g_x[i]) if need_x else None, _ptr(g_m[i]) if need_m else None,
                                  *[_ptr(t) for t in view_p])
                _lib.check(L.sdb_cnn_backward_ex(H, W, prec, _ptr(records[i]), _ptr(g_rgb[i]) if g_rgb is not None else None,
                                                 _ptr(g_raw[i]) if g_raw is not None else None, _ptr(bpack), _ptr(pack),
                                                 _ptr(m[i if m.shape[0] > 1 else 0]), ctypes.byref(grads), _ptr(work),
                                                 _stream(dev)), 'sdb_cnn_backward_ex')
                if N > 1:
                    for acc, v in zip(g_p, view_p):
                        if acc is not None:
                            acc.add_(v)
        if g_m is not None and m.shape[0] == 1 and N > 1:
            g_m = g_m.sum(0, keepdim=True)
        if g_m is not None:
            g_m = g_m.to(ctx.mod_dtype)                          # fc_z_cond(z) is half / bf16 under autocast
        g_p = [t.to(dt) if t is not None else None for t, dt in zip(g_p, ctx.param_dtypes)]
        return (None, g_x, g_m) + tuple(g_p)


class _CnnGrads(ctypes.Structure):
    """sdb_cnn_grads (include/sdb200.h): dL/dnet_out, dL/dmod, then the 14 parameter gradients in _NAMES order."""
    _fields_ = [('d_grad_net_out', ctypes.c_void_p), ('d_grad_mod', ctypes.c_void_p)] + \
               [('d_grad_' + n.replace('.weight', '_w').replace('.bias', '_b'), ctypes.c_void_p) for n in _NAMES]


class RenderCNNEngine:
    """P: dict with the reference's state-dict names `denoiser.*` (CUDA fp32).  Packs the weights once; keeps one
    workspace per frame size."""

    def __init__(self, P, precision=PRECISION_FP16X3, prefix='denoiser.'):
        if not supported(P, prefix):
            raise RuntimeError('RenderCNNEngine: unexpected denoiser shapes (expects conv1 64->256, 3x3 256->256, conv4 256->3)')
        self.P, self.prefix, self.precision = P, prefix, int(precision)
        self._pack = None
        self._ws = {}

    def invalidate(self):
        self._pack = None

    def pack(self):
        if self._pack is None:
            L = _lib.lib()
            ts = [self.P[self.prefix + n].detach().to(torch.float32).contiguous() for n in _NAMES]
            dev = ts[0].device
            pack = torch.empty(int(L.sdb_cnn_pack_bytes(self.precision)), dtype=torch.uint8, device=dev)
            with torch.cuda.device(dev):
                _lib.check(L.sdb_cnn_pack(*[_ptr(t) for t in ts], self.precision, _ptr(pack), _stream(dev)), 'sdb_cnn_pack')
            self._pack = pack
        return self._pack

    def modulation(self, z):
        """fc_z_cond(z) -> [N, 4, 256]: (w, b) of the two modulated blocks (gancraft_base.py:208-209)."""
        p = self.prefix
        return F.linear(z, self.P[p + 'fc_z_cond.weight'], self.P[p + 'fc_z_cond.bias']).reshape(z.shape[0], 4, 256).contiguous()

    def forward_train(self, net_out, z, P, precision=PRECISION_BF16X3):
        """Differentiable forward for the training step: P maps the same `denoiser.*` names to the LIVE Parameters
        (state_dict() hands out detached aliases, so self.P cannot carry gradients).  The modulation fc_z_cond(z) is
        torch's own F.linear, so z, fc_z_cond.weight and .bias get their gradients from autograd.
        precision: PRECISION_BF16X3 (fp32-grade), or one pass per product in fp16 (PRECISION_FP16) or bf16
        (PRECISION_BF16), the class of autocast's own convolutions.  The kernels compute in fp32 at every precision;
        under autocast rgb and raw are returned in autocast's dtype, as the reference composition returns them there
        (its convolutions and tanh run in that dtype, gancraft_base.py:201-225, :598-601)."""
        if not net_out.is_cuda or net_out.dtype != torch.float32 or net_out.dim() != 4 or net_out.shape[-1] != 64:
            raise RuntimeError('net_out must be a float32 CUDA tensor [N,H,W,64]')
        if precision not in TRAIN_PRECISIONS:
            raise ValueError('RenderCNN training precision must be one of %s, not %r' % (TRAIN_PRECISIONS, precision))
        p = self.prefix
        mod = F.linear(z.to(net_out.device, torch.float32), P[p + 'fc_z_cond.weight'], P[p + 'fc_z_cond.bias'])
        rgb, raw = _RenderCNNTrainFn.apply(int(precision), net_out, mod.reshape(z.shape[0], 4, 256), *[P[p + n] for n in _NAMES])
        if torch.is_autocast_enabled():
            dt = torch.get_autocast_dtype('cuda')
            rgb, raw = rgb.to(dt), raw.to(dt)
        return rgb, raw

    def forward(self, net_out, z, want_raw=True):
        """net_out [N,H,W,64] fp32 CUDA, z [N,256] (or [1,256]) -> (fake_images [N,3,H,W], fake_images_raw or None)."""
        if not net_out.is_cuda or net_out.dtype != torch.float32 or net_out.dim() != 4 or net_out.shape[-1] != 64:
            raise RuntimeError('net_out must be a float32 CUDA tensor [N,H,W,64]')
        L = _lib.lib()
        dev = net_out.device
        N, H, W = net_out.shape[:3]
        x = net_out.contiguous()
        mod = self.modulation(z.detach().to(dev, torch.float32))
        pack = self.pack()
        rgb = torch.empty(N, 3, H, W, dtype=torch.float32, device=dev)
        raw = torch.empty(N, 3, H, W, dtype=torch.float32, device=dev) if want_raw else None
        key = (H, W, self.precision, str(dev))
        ws = self._ws.get(key)
        ready = 1
        if ws is None:
            self._ws.clear()                                     # one frame size at a time (a few hundred MB to ~2 GB)
            ws = self._ws[key] = torch.empty(int(L.sdb_cnn_workspace_bytes(H, W, self.precision)), dtype=torch.uint8, device=dev)
            ready = 0
        with torch.cuda.device(dev):
            for i in range(N):
                m = mod[i if mod.shape[0] > 1 else 0]
                _lib.check(L.sdb_cnn_forward(_ptr(x[i]), H, W, _ptr(pack), _ptr(m), self.precision, _ptr(rgb[i]),
                                             _ptr(raw[i]) if want_raw else None, _ptr(ws), ready, _stream(dev)), 'sdb_cnn_forward')
                ready = 1
        return rgb, raw
