"""The fp32 bias table at the end of the forward packs (render: beta of fc_2..fc_6, then fc_out_c.bias; sky: fc2..fc5 and
fc_out_c biases).  The fused kernels add entry (l - 1) * 256 + n to column n of layer l where the MMA warpgroup writes a
block out, so each entry must be what a bias K slab would have summed on the tensor core: hi + lo of the 16-bit parts the
pack makes of the bias (fp16(b) at precision 0), exact in fp32."""
import pytest
import torch

import oracle
from scenedreamer_b200 import _lib, render

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
PRECISIONS = (render.PRECISION_FP16, render.PRECISION_BF16X3, render.PRECISION_FP16X3)


def packed_value(b, precision):
    """fp32 value of the 16-bit part(s) of b, computed on the CPU."""
    b = b.detach().float().cpu()
    dt = torch.bfloat16 if precision == render.PRECISION_BF16X3 else torch.float16
    hi = b.to(dt).float()
    if precision == render.PRECISION_FP16:
        return hi
    return hi + (b - hi).to(dt).float()


def bias_table(pack, n):
    return pack[0, pack.shape[1] - 4 * n:].cpu().view(torch.float32)


def spread_biases(P, names, seed):
    """biases over eight decades, so that the lo part is also an fp16 subnormal"""
    g = torch.Generator().manual_seed(seed)
    for k in names:
        b = P[k]
        P[k] = (torch.randn(b.shape, generator=g) * torch.pow(10.0, torch.empty(b.shape).uniform_(-5, 3, generator=g))).to(b.device)


@pytest.mark.parametrize('precision', PRECISIONS)
def test_render_pack_bias_table(precision):
    P = oracle.make_params(seed=5, stress=True)
    spread_biases(P, ['render_net.fc_out_c.bias'] + ['render_net.fc_%d.bias_beta' % k for k in (2, 3, 4, 5, 6)], 11)
    P = {k: v.to(DEV) for k, v in P.items()}
    z = torch.randn(1, 256, generator=torch.Generator().manual_seed(3)).to(DEV)
    pack = render.pack_mlp(P, z, precision)
    _, bh = render.modulated_weights(P, z[0])
    torch.cuda.synchronize()
    want = packed_value(torch.cat([bh.reshape(-1), P['render_net.fc_out_c.bias']]), precision)
    assert want.numel() == 5 * 256 + 64
    assert pack.shape[1] == _lib.lib().sdb_mlp_pack_bytes(precision)
    got = bias_table(pack, want.numel())
    assert torch.equal(got, want), int((got != want).sum())


@pytest.mark.parametrize('precision', PRECISIONS)
def test_sky_pack_bias_table(precision):
    P = oracle.make_params(seed=6, stress=True)
    spread_biases(P, ['sky_net.fc%d.bias' % k for k in (2, 3, 4, 5)] + ['sky_net.fc_out_c.bias'], 12)
    P = {k: v.to(DEV) for k, v in P.items()}
    z = torch.randn(1, 256, generator=torch.Generator().manual_seed(4)).to(DEV)
    pack = render.pack_sky_mlp(P, z, precision)
    torch.cuda.synchronize()
    want = packed_value(torch.cat([P['sky_net.fc%d.bias' % k] for k in (2, 3, 4, 5)] + [P['sky_net.fc_out_c.bias']]), precision)
    assert want.numel() == 4 * 256 + 64
    assert pack.shape[1] == _lib.lib().sdb_sky_pack_bytes(precision)
    got = bias_table(pack, want.numel())
    assert torch.equal(got, want), int((got != want).sum())


@pytest.mark.parametrize('precision', PRECISIONS)
def test_sky_forward_zero_weights_returns_colour_bias(precision):
    """With every sky weight zero, each ray's sky features are the colour head's bias-table entries, bit for bit: the
    accumulators of the last layer are zero and the write-out adds the bias once."""
    P = oracle.make_params(seed=7, stress=True)
    for k in list(P):
        if k.startswith('sky_net.') and k.endswith('.weight'):
            P[k] = torch.zeros_like(P[k])
    spread_biases(P, ['sky_net.fc%d.bias' % k for k in (1, 2, 3, 4, 5)] + ['sky_net.fc_out_c.bias'], 13)
    P = {k: v.to(DEV) for k, v in P.items()}
    z = torch.randn(1, 256, generator=torch.Generator().manual_seed(5)).to(DEV)
    g = torch.Generator().manual_seed(6)
    H, W = 20, 37                                         # partial tiles on both edges
    d = torch.randn(1, H, W, 1, 3, generator=g)
    d = (d / d.norm(dim=-1, keepdim=True)).to(DEV).contiguous()
    sky, _ = render.sky_forward(d, render.pack_sky_mlp(P, z, precision), precision)
    torch.cuda.synchronize()
    want = packed_value(P['sky_net.fc_out_c.bias'], precision).expand(1, H, W, 64)
    got = sky.cpu()
    assert torch.equal(got, want), int((got != want).sum())
