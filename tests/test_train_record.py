"""CPU self-tests of tests/_train_record.py: the float64 stage references against torch.autograd on the forward they
differentiate, and the record decoder against tiles built from the layout rf_common.cuh documents."""
import torch
import torch.nn.functional as F

import _train_record as tr

D = torch.float64


def test_composite_reference_equals_autograd():
    g = torch.Generator().manual_seed(0)
    R, S = 40, 37
    sig = torch.randn(R, S, generator=g, dtype=D) * 3
    sig[0] = -1.0                                              # all-negative sigma: a ray without opacity
    sig[1] = 300.0                                             # dense medium: transmittance underflows
    nds = torch.rand(R, S, generator=g, dtype=D) * 0.5
    c = torch.randn(R, S, 64, generator=g, dtype=D) * 1.5               # beyond [-1, 1]: the clamp passes no gradient there
    live = torch.rand(R, generator=g, dtype=D) > 0.2
    gout = torch.randn(R, 64, generator=g, dtype=D)
    sky = torch.randn(R, 64, generator=g, dtype=D) * 1.5
    (dc, dsig, dsky), (sc, ss, sk) = tr.composite_backward_ref(sig, nds, c, live, gout, sky)

    sig_l, c_l, sky_l = sig.clone().requires_grad_(True), c.clone().requires_grad_(True), sky.clone().requires_grad_(True)
    e = F.relu(sig_l) * nds
    w = (1 - torch.exp(-e)) * torch.exp(-(torch.cumsum(e, 1) - e)) * live[:, None]
    out = (w[..., None] * (c_l.clamp(-1, 1) + 1)).sum(1) + (1 - w.sum(1))[:, None] * (sky_l.clamp(-1, 1) + 1) - 1
    (out * gout).sum().backward()
    for a, b, s in ((dc, c_l.grad, sc), (dsig, sig_l.grad, ss), (dsky, sky_l.grad, sk)):
        assert torch.allclose(a, b, rtol=1e-12, atol=1e-14)
        assert bool(((a.abs() <= s * (1 + 1e-12) + 1e-300) | (s > 0)).all()) and bool((s[a != 0] > 0).all())
    assert bool((dsig[0] == 0).all()) and bool((dsig[~live] == 0).all())


def test_chain_reference_equals_autograd():
    g = torch.Generator().manual_seed(1)
    n = 50
    w1 = torch.randn(256, 128, generator=g, dtype=D) / 11
    wh = torch.randn(5, 256, 256, generator=g, dtype=D) / 16
    bh = torch.randn(5, 256, generator=g, dtype=D) * 0.1
    wsig, wout = torch.randn(256, generator=g, dtype=D) / 16, torch.randn(64, 256, generator=g, dtype=D) / 16
    x0 = torch.randn(n, 128, generator=g, dtype=D).requires_grad_(True)
    acts = [F.leaky_relu(x0 @ w1.t(), 0.2)]
    for k in range(5):
        acts.append(F.leaky_relu(acts[-1] @ wh[k].t() + bh[k], 0.2))
    for a in acts:
        a.retain_grad()
    sigma = acts[3] @ wsig
    col = acts[5] @ wout.t()
    dc, dsig = torch.randn(n, 64, generator=g, dtype=D), torch.randn(n, generator=g, dtype=D)
    ((col * dc).sum() + (sigma * dsig).sum()).backward()
    bits = [a.detach() > 0 for a in acts]
    dz, dx0, mag, mag0 = tr.chain_ref(dc, dsig, bits, w1, wh, wsig, wout)
    assert bool((dx0.abs() <= mag0 * (1 + 1e-12)).all())                   # magnitudes bound the values
    assert all(bool((d.abs() <= m * (1 + 1e-12)).all()) for d, m in zip(dz, mag))
    assert torch.allclose(dx0, x0.grad, rtol=1e-12, atol=1e-14)
    for k in range(6):                                         # dZ_k = dL/dA_k * LeakyReLU'(Z_k)
        assert torch.allclose(dz[k], acts[k].grad * (bits[k].double() * 0.8 + 0.2), rtol=1e-12, atol=1e-14)


def _tile_reference(x):
    """Tiles [slots, cols] by the element offset of rec_chunk: ((item * chunks + chunk) * 1024) + row * 8 + col % 8."""
    slots, cols = x.shape
    out = torch.empty(slots * cols, dtype=x.dtype)
    for s in range(slots):
        for col in range(cols):
            out[((s // 128) * (cols // 8) + col // 8) * 1024 + (s % 128) * 8 + col % 8] = x[s, col]
    return out


def test_untile_inverts_the_record_tiling():
    g = torch.Generator().manual_seed(2)
    for cols in (8, 64, 144, 256, 272):
        x = torch.randn(256, cols, generator=g).to(torch.bfloat16)
        assert torch.equal(tr.untile(_tile_reference(x), cols), x)


def test_sign_words_and_bf16_helpers():
    g = torch.Generator().manual_seed(3)
    a = torch.randn(7, 256, generator=g)
    words = torch.zeros(7, 8, dtype=torch.int64)
    for j in range(256):
        words[:, j // 32] |= (a[:, j] > 0).long() << (j % 32)
    words = torch.where(words >= 2 ** 31, words - 2 ** 32, words).to(torch.int32)
    assert torch.equal(tr.sign_bits(words), a > 0)
    v = torch.tensor([1.0, 1.00390625, 1.005859375, -3.0e-5, 0.0], dtype=torch.float32)
    assert torch.equal(tr.bf16_bits(v), v.to(torch.bfloat16).view(torch.int16))
    assert torch.equal(tr.bf16_ulp(torch.tensor([1.0, 1.5, 0.75, -2.0, 0.0], dtype=D)),
                       torch.tensor([2.0 ** -7, 2.0 ** -7, 2.0 ** -8, 2.0 ** -6, 0.0], dtype=D))
