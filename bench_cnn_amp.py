"""RenderCNN + tanh under autograd and torch.autocast: the one-pass tensor-core training path (fp16 x1, bf16 x1) against the
reference's composition (oracle.render_cnn on cuDNN) under the same autocast, with the bf16 x3 path without autocast as the
anchor to bench_cnn_train.py.  Arms alternate in one process.  Prints one JSON line.

    python bench_cnn_amp.py [--steps 10] [--warmup 3]

Sizes: 262 x 262 (training crop 256 + pad 6) and 570 x 990 (the C2 padded frame).  Times are CUDA-event medians with L2
flushed before each timed call; per arm the forward, the backward of the forward timed just before it, the step (both),
the record size (ours) and the peak memory one step allocates above what was live before it."""
import argparse
import contextlib
import json
import statistics

import torch

import oracle
from scenedreamer_b200 import _lib, rendercnn

FWD_FLOP_PER_PIXEL = 2 * (64 * 256 + 4 * 9 * 256 * 256 + 2 * 256 * 256 + 256 * 3)
# arm -> (ours?, training precision, autocast dtype or None)
ARMS = {
    'ours_fp16': (True, rendercnn.PRECISION_FP16, torch.float16),
    'ref_fp16': (False, None, torch.float16),
    'ours_bf16': (True, rendercnn.PRECISION_BF16, torch.bfloat16),
    'ref_bf16': (False, None, torch.bfloat16),
    'ours_bf16x3': (True, rendercnn.PRECISION_BF16X3, None),
}


def _event_ms(fn, flush):
    flush.zero_()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=10)
    ap.add_argument('--warmup', type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_cnn_amp.py needs a CUDA GPU')
    dev = 'cuda:0'
    flush = torch.empty(64 << 20, dtype=torch.float32, device=dev)          # 256 MB > L2
    P = {k: v.to(dev) for k, v in oracle.make_cnn_params(1).items()}
    res = {'gpu': torch.cuda.get_device_name(0)}
    try:
        import subprocess
        res['power_limit_w'] = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader,nounits', '-i', '0'],
                                              capture_output=True, text=True).stdout.strip()
    except OSError:
        res['power_limit_w'] = None
    L = _lib.lib()
    for H, W in ((262, 262), (570, 990)):
        g = torch.Generator().manual_seed(0)
        x = (torch.rand(1, H, W, 64, generator=g) * 2 - 1).to(dev).requires_grad_(True)
        z = torch.randn(1, 256, generator=g).to(dev)
        G = torch.randn(1, 3, H, W, generator=g).to(dev)
        Q = {k: v.clone().requires_grad_(True) for k, v in P.items()}
        eng = rendercnn.RenderCNNEngine(Q)

        def make(arm):
            ours, prec, dt = ARMS[arm]
            ctx = (lambda: torch.autocast('cuda', dtype=dt)) if dt is not None else contextlib.nullcontext
            state = {}

            def fwd():
                with ctx():
                    if ours:
                        state['out'] = eng.forward_train(x, z, Q, precision=prec)
                    else:
                        state['out'] = oracle.render_cnn(x, z, Q, dtype=torch.float32)

            def bwd():
                rgb = state.pop('out')[0]
                rgb.backward(G.to(rgb.dtype))

            def step():
                fwd()
                bwd()
            return fwd, bwd, step

        r = {}
        for _ in range(2):                                                 # alternate the arms
            for arm in ARMS:
                fwd, bwd, step = make(arm)
                for _ in range(a.warmup):
                    step()
                torch.cuda.synchronize()
                f_ms, b_ms, s_ms = [], [], []
                for _ in range(a.steps):
                    f_ms.append(_event_ms(fwd, flush))
                    b_ms.append(_event_ms(bwd, flush))
                for _ in range(a.steps):
                    s_ms.append(_event_ms(step, flush))
                for q in list(Q.values()) + [x]:
                    q.grad = None
                torch.cuda.synchronize()
                base = torch.cuda.memory_allocated()
                torch.cuda.reset_peak_memory_stats()
                step()
                torch.cuda.synchronize()
                peak = (torch.cuda.max_memory_allocated() - base) / 2**20
                for q in list(Q.values()) + [x]:
                    q.grad = None
                o = r.setdefault(arm, {})
                for k, v in (('fwd_ms', statistics.median(f_ms)), ('bwd_ms', statistics.median(b_ms)),
                             ('step_ms', statistics.median(s_ms)), ('peak_mb', peak)):
                    o.setdefault(k, []).append(v)
        out = {}
        for arm, o in r.items():
            out[arm] = {k: round(min(v), 3 if k != 'peak_mb' else 1) for k, v in o.items()}
            out[arm]['step_ms_runs'] = [round(v, 3) for v in o['step_ms']]
            ours, prec, _ = ARMS[arm]
            if ours:
                out[arm]['record_mb'] = round(L.sdb_cnn_train_record_bytes_ex(H, W, prec) / 2**20, 1)
        out['algorithmic_tflop_per_step'] = round(3 * H * W * FWD_FLOP_PER_PIXEL / 1e12, 3)
        res['%dx%d' % (H, W)] = out
    print(json.dumps(res))


if __name__ == '__main__':
    main()
