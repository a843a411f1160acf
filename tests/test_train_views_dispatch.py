"""Dispatch of Generator._forward_perpix under autograd with the batched training pass switched on (SDB200_TRAIN_VIEWS=1):
batches of views and a preset sky mean (no GPU: the renderer and the training pass are replaced by recorders).  The default
dispatch is what tests/test_host_logic.py checks."""
import torch

from scenedreamer_b200 import integration
from test_host_logic import _fake_generator


def test_hook_dispatch_rules_batched_views(monkeypatch):
    monkeypatch.setenv('SDB200_TRAIN_VIEWS', '1')
    calls = []
    gen, vid, dep, rd = _fake_generator(1, monkeypatch, calls)
    ori, z, genc = torch.zeros(1, 3), torch.zeros(1, 4), torch.zeros(1, 2)
    f = integration.fused_forward_perpix
    with torch.no_grad():
        out = f(gen, None, vid, dep, rd, ori, z, genc)
    assert calls == ['inference'] and len(out) == 12
    calls.clear()
    out = f(gen, None, vid, dep, rd, ori, z, genc)                 # parameters require grad -> recording forward + fused backward
    assert calls == ['train'] and len(out) == 12
    calls.clear()
    gen2, vid2, dep2, rd2 = _fake_generator(3, monkeypatch, calls)
    f(gen2, None, vid2, dep2, rd2, torch.zeros(3, 3), torch.zeros(3, 4), genc)
    assert calls == ['train']                                        # a batch = ONE recorded pass over its views
    calls.clear()
    monkeypatch.setenv('SDB200_TRAIN_VIEWS', '0')
    out = f(gen2, None, vid2, dep2, rd2, torch.zeros(3, 3), torch.zeros(3, 4), genc)
    assert calls == ['train'] * 3 and out[0].shape[0] == 3           # ... or one per view
    monkeypatch.setenv('SDB200_TRAIN_VIEWS', '1')
    calls.clear()
    st = integration._state(gen)
    n0 = st.stats['train_calls']
    gen.sky_avg = torch.zeros(1, 64)                                 # preset sky mean under autograd: still the fused pass
    f(gen, None, vid, dep, rd, ori, z, genc)
    assert calls == ['train'] and st.stats['train_calls'] == n0 + 1
    calls.clear()
    f(gen, None, vid, dep, rd, ori, z, torch.tensor([[0.0, 0.0]]).expand(1, 2))
    assert calls == ['train']
    calls.clear()
    del gen.sky_avg
    f(gen2, None, vid2, dep2, rd2, torch.zeros(3, 3), torch.zeros(3, 4), torch.tensor([[0.0, 0.0], [0.5, 0.0], [0.0, 0.0]]))
    assert calls == ['reference']                                    # views of different scenes: reference composition
    calls.clear()
    gen.raw_noise_std = 0.5                                          # option outside the fused path
    with torch.no_grad():
        f(gen, None, vid, dep, rd, ori, z, genc)
    assert calls == ['reference']
    calls.clear()
    gen.raw_noise_std = 0.0
    for q in list(gen.render_net.parameters()) + list(gen.hash_encoder.parameters()) + list(gen.sky_net.parameters()):
        q.requires_grad_(False)
    f(gen, None, vid, dep, rd, ori, z, genc)                        # nothing to differentiate: inference kernel even with grad mode on
    assert calls == ['inference']
