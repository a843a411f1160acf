"""One forward + backward of the stand-alone hash-grid encode op (a6/a7 boundary ops, csrc/gridenc.cu) at the size of one reference
tile (158 x 158 rays x 24 samples, D=5, 16 levels x 8 features, 2^19 entries per hashed level): a fixed workload to time or
profile the two kernels on their own."""
import numpy as np
import torch

from scenedreamer_b200 import ops

DEV = 'cuda:0'
B, L, C, D, H = 158 * 158 * 24, 16, 8, 5, 16
pls = float(np.exp2(np.log2(2048 / H) / (L - 1)))
offs, o = [], 0
for lv in range(L):
    n = min(2 ** 19, (int(np.ceil(H * pls ** lv)) + 1) ** D)
    offs.append(o)
    o += int(np.ceil(n / 8) * 8)
offs.append(o)
g = torch.Generator().manual_seed(0)
emb = ((torch.rand(o, C, generator=g) * 2 - 1) * 0.1).to(DEV)
x = torch.rand(B, D, generator=g).to(DEV)
offsets = torch.tensor(offs, dtype=torch.int32, device=DEV)
out = torch.empty(L, B, C, device=DEV)
dydx = torch.empty(B, L * D * C, device=DEV)
grad = torch.randn(L, B, C, generator=g).to(DEV)
ge, gi = torch.zeros_like(emb), torch.zeros_like(x)
for _ in range(2):
    ops.grid_encode_forward(x, emb, offsets, out, B, D, C, L, float(np.log2(pls)), H, True, dydx, 0, False)
    ops.grid_encode_backward(grad, x, emb, offsets, ge, B, D, C, L, float(np.log2(pls)), H, True, dydx, gi, 0, False)
torch.cuda.synchronize()


def ms(fn, reps=10):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


S = float(np.log2(pls))
print('ok', float(out.abs().mean()), float(ge.abs().sum()), 'SDB_GRIDENC_MINB=%s' % __import__('os').environ.get('SDB_GRIDENC_MINB', 'default'),
      'fwd+dy_dx %.3f ms, fwd %.3f ms, bwd(table+input) %.3f ms' % (
          ms(lambda: ops.grid_encode_forward(x, emb, offsets, out, B, D, C, L, S, H, True, dydx, 0, False)),
          ms(lambda: ops.grid_encode_forward(x, emb, offsets, out, B, D, C, L, S, H, False, dydx, 0, False)),
          ms(lambda: ops.grid_encode_backward(grad, x, emb, offsets, ge, B, D, C, L, S, H, True, dydx, gi, 0, False))))
