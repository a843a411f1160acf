"""Decoder of the fused training path's record and backward workspace, and float64 references of each backward stage
(test infrastructure).

The record (sdb_render_rays_train_forward) and the workspace (sdb_render_rays_backward[_views]) are byte buffers whose
offsets come from sdb_debug_train_layout.  A "slot" is one (work item, sample step, tile row):
slot = (work * S + s) * 128 + row, where `work` is the tile's position in the live-tile list of the whole batch.  The
workspace holds ONE view (the last one the backward visited): its slot 0 is record slot first * S * 128 of that view.
The bf16 arrays (x0, act, dz, dc16) are MMA-ready tiles (rf_common.cuh: rec_chunk):
[item = slot / 128][chunk = column / 8][row = slot % 128][8 columns].

The references take plain tensors and work on any device; they compute in float64.
"""
import ctypes

import torch

ROWS, TILE_H, TILE_W = 128, 8, 16
HIDDEN, FEAT, OUT_C, X0_COLS, ACT_COLS, N_ACT = 256, 128, 64, 144, 272, 6
LAYOUT_FIELDS = ('hdr', 'tile_list', 'tile_work', 'rayflags', 'x3', 'x0', 'act', 'mask', 'sig', 'nds', 'c',
                 'dc32', 'dc16', 'dsig32', 'dsig16', 'dz', 'dx0', 'dt3', 'record_bytes', 'workspace_bytes')
PRIMES = (1, 2654435761, 805459861)          # rf_common.cuh: corner3 (dims 0..2 of the hash)


def layout(lib, n_img, H, W, S, L=16, log2_T=19):
    """Byte offsets of the record / workspace arrays and their total sizes (sdb_debug_train_layout)."""
    out = (ctypes.c_int64 * len(LAYOUT_FIELDS))()
    code = lib.sdb_debug_train_layout(n_img, H, W, S, L, log2_T, out)
    if code != 0:
        raise RuntimeError('sdb_debug_train_layout failed (code %d)' % code)
    return dict(zip(LAYOUT_FIELDS, [int(v) for v in out]))


def tiles_of(H, W):
    return (W + TILE_W - 1) // TILE_W, (H + TILE_H - 1) // TILE_H


def untile(t, cols):
    """Flat bf16 tile array of `cols` columns -> [slots, cols] row-major."""
    items = t.numel() // (ROWS * cols)
    return t[:items * ROWS * cols].reshape(items, cols // 8, ROWS, 8).permute(0, 2, 1, 3).reshape(items * ROWS, cols)


def sign_bits(words):
    """Sign words [..., 8] int32 -> bool [..., 256]: bit j of word q is (A[:, 32 q + j] > 0)."""
    bits = torch.arange(32, device=words.device, dtype=torch.int32)
    return ((words.unsqueeze(-1) >> bits) & 1).bool().reshape(*words.shape[:-1], 256)


def bf16_bits(x):
    """Round-to-nearest-even bf16 of fp32 values, as int16 bit patterns."""
    return x.to(torch.float32).to(torch.bfloat16).view(torch.int16)


class Record:
    """Views into one record (and optionally one backward workspace); slot-ordered, device-resident."""

    def __init__(self, lay, record, n_img, H, W, S, workspace=None):
        self.lay, self.n_img, self.H, self.W, self.S = lay, n_img, H, W, S
        self.tiles_x, self.tiles_y = tiles_of(H, W)
        self.tpi = self.tiles_x * self.tiles_y
        n_tiles = n_img * self.tpi
        cap, steps = n_tiles * S * ROWS, n_tiles * S

        def rv(name, n, dtype, buf=record):
            off, size = lay[name], n * torch.empty(0, dtype=dtype).element_size()
            return buf[off:off + size].view(dtype)

        hdr = rv('hdr', 1 + 2 * n_img, torch.int32).cpu()
        self.n_live = int(hdr[0])
        self.views = [(int(hdr[1 + 2 * i]), int(hdr[2 + 2 * i])) for i in range(n_img)]     # {first, count} per view
        n = self.n_live * S * ROWS
        self.tile_list = rv('tile_list', n_tiles, torch.int32)[:self.n_live].long()
        self.tile_work = rv('tile_work', n_tiles, torch.int32).long()
        fl = rv('rayflags', n_tiles * ROWS, torch.int32)[:self.n_live * ROWS]
        self.live, self.nosky, self.valid = (fl & 1).bool(), (fl & 2).bool(), (fl & 4).bool()
        self.x3 = rv('x3', cap * 4, torch.float32).reshape(cap, 4)[:n]
        self.x0 = untile(rv('x0', cap * X0_COLS, torch.bfloat16), X0_COLS)[:n]
        acts = rv('act', N_ACT * cap * ACT_COLS, torch.bfloat16).reshape(N_ACT, cap * ACT_COLS)
        self.act = [untile(a, ACT_COLS)[:n] for a in acts]
        mask = rv('mask', steps * N_ACT * ROWS * 8, torch.int32).reshape(steps, N_ACT, ROWS, 8)[:self.n_live * S]
        self.mask = mask.permute(1, 0, 2, 3).reshape(N_ACT, n, 8)                            # [layer, slot, word]
        self.sig = rv('sig', cap, torch.float32)[:n]
        self.nds = rv('nds', cap, torch.float32)[:n]
        self.c = rv('c', cap * OUT_C, torch.float32).reshape(cap, OUT_C)[:n]
        if workspace is not None:
            wcap = self.tpi * S * ROWS
            self.dc32 = rv('dc32', wcap * OUT_C, torch.float32, workspace).reshape(wcap, OUT_C)
            self.dc16 = untile(rv('dc16', wcap * OUT_C, torch.bfloat16, workspace), OUT_C)
            self.dsig32 = rv('dsig32', wcap, torch.float32, workspace)
            self.dsig16 = rv('dsig16', wcap * 8, torch.bfloat16, workspace).reshape(wcap, 8)
            dz = rv('dz', N_ACT * wcap * HIDDEN, torch.bfloat16, workspace).reshape(N_ACT, wcap * HIDDEN)
            self.dz = [untile(d, HIDDEN) for d in dz]
            self.dx0 = rv('dx0', wcap * FEAT, torch.float32, workspace).reshape(wcap, FEAT)
            self.dt3 = workspace[lay['dt3']:lay['workspace_bytes']].view(torch.float32)

    def view_slots(self, i):
        """Record slot range of view i."""
        first, count = self.views[i]
        return slice(first * self.S * ROWS, (first + count) * self.S * ROWS)

    def rays(self, i):
        """For view i's live items: ray index inside the image [count, 128] and the in-image mask, from the tile list."""
        first, count = self.views[i]
        t = self.tile_list[first:first + count] - i * self.tpi
        y = (t // self.tiles_x * TILE_H)[:, None] + torch.arange(ROWS, device=t.device)[None, :] // TILE_W
        x = (t % self.tiles_x * TILE_W)[:, None] + torch.arange(ROWS, device=t.device)[None, :] % TILE_W
        inside = (y < self.H) & (x < self.W)
        return (y * self.W + x).clamp(max=self.H * self.W - 1), inside

    def sky_only_rays(self, i):
        """In-image rays of view i's tiles without a live item (prepass: net_out is the clamped sky) [n] bool over H*W."""
        dead = self.tile_work[i * self.tpi:(i + 1) * self.tpi] < 0
        m = dead.reshape(self.tiles_y, self.tiles_x).repeat_interleave(TILE_H, 0).repeat_interleave(TILE_W, 1)
        return m[:self.H, :self.W].reshape(-1)


def in_clamp(v):
    return (v >= -1) & (v <= 1)


def composite_backward_ref(sig, nds, c, live, g, sky_used):
    """Backward of volum_rendering_relu + clamp + sky blend for R rays of S samples, in float64.
    sig, nds [R, S]; c [R, S, 64]; live [R] bool; g [R, 64] dL/dnet_out; sky_used [R, 64] the sky feature the ray blends.
    Returns (dc [R, S, 64], dsig [R, S], dsky [R, 64] = (1 - sum w) g [sky in clamp]) and a magnitude scale of each:
    the same expression with every compositing weight w_t replaced by the bound Tb_t of its transmittance's fp32 error
    and every term by its absolute value.  fp32 evaluation errs by a small multiple of 2^-24 of that scale (1 - exp(-e)
    cancels for small e, dsig and 1 - sum w cancel by construction), so the scale, not the value, normalises the error.
    Tb_s = T_s (1 + (s + 1) E_s): the fp32 running sum E_s of s + 1 terms errs by up to (s + 1) 2^-24 E_s, which exp(-E)
    turns into that relative error of T."""
    sig, nds, c, g, sky_used = (t.double() for t in (sig, nds, c, g, sky_used))
    e = sig.clamp(min=0) * nds
    E = torch.cumsum(e, 1) - e
    livef = live.double()[:, None]
    T = torch.exp(-E) * livef
    steps = torch.arange(1, e.shape[1] + 1, dtype=torch.float64, device=e.device)
    Tb = T * (1 + steps * E)
    w = (1 - torch.exp(-e)) * T
    W = w.sum(1)
    gsky = (g * (sky_used.clamp(-1, 1) + 1)).sum(-1)
    dw = ((g[:, None, :] * (c.clamp(-1, 1) + 1)).sum(-1) - gsky[:, None]) * live.double()[:, None]
    suffix = lambda v: v.flip(1).cumsum(1).flip(1) - v                                       # sum over t > s
    pos = (sig > 0).double() * nds
    dsig = (dw * T * torch.exp(-e) - suffix(dw * w)) * pos
    dsig_scale = (dw.abs() * Tb * torch.exp(-e) + suffix(dw.abs() * Tb)) * pos
    cm, sm = in_clamp(c).double(), in_clamp(sky_used).double()
    dc = w[..., None] * g[:, None, :] * cm
    dc_scale = Tb[..., None] * g.abs()[:, None, :] * cm
    dsky = (1 - W)[:, None] * g * sm
    dsky_scale = g.abs() * sm
    return (dc, dsig, dsky), (dc_scale, dsig_scale, dsky_scale)


def chain_ref(dc, dsig, bits, w1, wh, wsig, wout):
    """Data-gradient chain of LightningMLP in float64: dc [n, 64], dsig [n], bits[k] [n, 256] sign of A_{k+1},
    w1 [256, 128], wh [5, 256, 256] (W' of fc_2..fc_6), wsig [256], wout [64, 256].  Returns dZ1..dZ6 and dX0, and for
    each the sum of the magnitudes of its products (|input| @ |W|): a bf16x3 product errs by about 2^-16 of it."""
    dc, dsig = dc.double(), dsig.double()
    slope = [b.double() * 0.8 + 0.2 for b in bits]                # LeakyReLU'(z): 1 where A > 0, else 0.2
    dz, mag = [None] * 6, [None] * 6
    dz[5], mag[5] = (dc @ wout.double()) * slope[5], (dc.abs() @ wout.double().abs()) * slope[5]
    for k in (4, 3, 2, 1, 0):
        a, m = dz[k + 1] @ wh[k].double(), dz[k + 1].abs() @ wh[k].double().abs()
        if k == 3:
            a = a + dsig[:, None] * wsig.double()[None, :]
            m = m + dsig.abs()[:, None] * wsig.double().abs()[None, :]
        dz[k], mag[k] = a * slope[k], m * slope[k]
    return dz, dz[0] @ w1.double(), mag, dz[0].abs() @ w1.double().abs()


def wgrad_ref(Z, A):
    """dW = Z^T A over the samples in float64 and the scale sum |Z|^T |A| that bounds fp32 accumulation of exact
    bf16 x bf16 products."""
    Z, A = Z.double(), A.double()
    return Z.t() @ A, Z.abs().t() @ A.abs()


def level_scales(L, level_S, base_res, device):
    """exp2f(l * level_S) * base_res - 1 in fp32, as the kernels form the per-level grid resolution."""
    lv = torch.arange(L, device=device, dtype=torch.float32)
    return torch.exp2(lv * torch.tensor(level_S, dtype=torch.float32, device=device)) * float(base_res) - 1.0


def table_scatter_ref(x3, dx0, scales, log2_T):
    """Gradient of the pre-blended 3-D table [L << log2_T, 8] from the feature gradients dx0 [n, 16 * 8] of the samples at
    grid positions x3 [n, 4] (w > 0: inside), in float64; returns it and the sum of the absolute contributions."""
    inside = x3[:, 3] > 0
    x, g = x3[inside, :3], dx0[inside].double()
    L, T = scales.numel(), 1 << log2_T
    dt3 = torch.zeros(L * T, 8, dtype=torch.float64, device=x3.device)
    mag = torch.zeros_like(dt3)
    for lvl in range(L):
        pos = (x.double() * float(scales[lvl]) + 0.5).float()              # one fp32 rounding: fmaf(x, scale, 0.5f)
        cell = torch.floor(pos)
        f = (pos - cell).double()
        cell = cell.long()
        gl = g[:, 8 * lvl:8 * lvl + 8]
        for i in range(8):
            b = [(i >> d) & 1 for d in range(3)]
            w = torch.ones_like(f[:, 0])
            h = torch.zeros_like(cell[:, 0])
            for d in range(3):
                w = w * (f[:, d] if b[d] else 1 - f[:, d])
                h = h ^ (((cell[:, d] + b[d]) * PRIMES[d]) & 0xFFFFFFFF)
            row = lvl * T + (h & (T - 1))
            dt3.index_add_(0, row, w[:, None] * gl)
            mag.index_add_(0, row, (w[:, None] * gl).abs())
    return dt3, mag


FP32_TINY = 2.0 ** -126       # the smallest normal fp32: the kernels flush what falls below it


def ratio(a, b, scale):
    """max over elements of |a - b| / (scale + 2^-126)."""
    r = (a.double() - b.double()).abs() / (scale.double() + FP32_TINY)
    return float(r.max()) if r.numel() else 0.0


def rel_l2(a, b):
    a, b = a.double(), b.double()
    return float((a - b).norm() / max(float(b.norm()), 1e-300))


def bf16_ulp(b):
    """Spacing of bf16 values at |b| (8 significant bits); 0 at 0."""
    b = b.double()
    _, ex = torch.frexp(b)
    return torch.where(b == 0, 0.0, torch.ldexp(torch.ones_like(b), ex - 8))
