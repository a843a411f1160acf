"""RenderCNN + tanh under autograd: the tensor-core training path (bf16 x3 recording forward + backward) against the
reference's composition (oracle.render_cnn on cuDNN, fp32) in the same process, alternating, with TF32 on (the reference
default) and off.  Prints one JSON line.

    python bench_cnn_train.py [--steps 10] [--warmup 3]

Sizes: 262 x 262 (training crop 256 + pad 6) and 570 x 990 (the C2 padded frame).  Times are CUDA-event medians with L2
flushed between steps.  Algorithmic FLOPs: forward 5.02 MFLOP per pixel, backward twice that (data and weight gradients);
the tensor cores do three times that under the bf16 x3 split."""
import argparse
import json
import statistics

import torch

import oracle
from scenedreamer_b200 import rendercnn

FWD_FLOP_PER_PIXEL = 2 * (64 * 256 + 4 * 9 * 256 * 256 + 2 * 256 * 256 + 256 * 3)


def _time(fn, steps, warmup, flush):
    for _ in range(warmup):
        fn()
    ts = []
    for _ in range(steps):
        flush.zero_()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    return statistics.median(ts)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=10)
    ap.add_argument('--warmup', type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_cnn_train.py needs a CUDA GPU')
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
    for H, W in ((262, 262), (570, 990)):
        g = torch.Generator().manual_seed(0)
        x = (torch.rand(1, H, W, 64, generator=g) * 2 - 1).to(dev).requires_grad_(True)
        z = torch.randn(1, 256, generator=g).to(dev)
        G = torch.randn(1, 3, H, W, generator=g).to(dev)
        Q = {k: v.clone().requires_grad_(True) for k, v in P.items()}
        eng = rendercnn.RenderCNNEngine(Q)
        state = {}

        def ours_fwd():
            state['out'] = eng.forward_train(x, z, Q)

        def ours_bwd():
            state['out'][0].backward(G)

        def ours_step():
            ours_fwd()
            ours_bwd()

        def ref_step():
            rgb, _ = oracle.render_cnn(x, z, Q, dtype=torch.float32)
            rgb.backward(G)

        def ours_bwd_timed():
            ours_fwd()
            torch.cuda.synchronize()
            flush.zero_()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            ours_bwd()
            e1.record()
            torch.cuda.synchronize()
            return e0.elapsed_time(e1)

        old = torch.backends.cudnn.allow_tf32
        r = {}
        try:
            for rnd in range(2):                                           # alternate ours / reference
                r.setdefault('ours_fwd_ms', []).append(_time(ours_fwd, a.steps, a.warmup, flush))
                r.setdefault('ours_bwd_ms', []).append(statistics.median([ours_bwd_timed() for _ in range(a.steps)]))
                r.setdefault('ours_step_ms', []).append(_time(ours_step, a.steps, a.warmup, flush))
                for tf32 in (True, False):
                    torch.backends.cudnn.allow_tf32 = tf32
                    r.setdefault('ref_step_ms_tf32' if tf32 else 'ref_step_ms_fp32', []).append(_time(ref_step, a.steps, a.warmup, flush))
        finally:
            torch.backends.cudnn.allow_tf32 = old
        out = {k: round(min(v), 3) for k, v in r.items()}
        fl = H * W * FWD_FLOP_PER_PIXEL
        out['algorithmic_tflop'] = round(3 * fl / 1e12, 3)
        out['tensor_core_tflop_x3'] = round(9 * fl / 1e12, 3)
        out['ours_step_tflops'] = round(3 * fl / (out['ours_step_ms'] * 1e-3) / 1e12, 1)
        rec_bytes = rendercnn._lib.lib().sdb_cnn_train_record_bytes(H, W)
        out['record_mb'] = round(rec_bytes / 2**20, 1)
        # the training forward clears its record (zero borders) on every call: the same bytes cleared on their own
        buf = torch.empty(rec_bytes, dtype=torch.uint8, device=dev)
        out['record_clear_ms'] = round(_time(buf.zero_, a.steps, a.warmup, flush), 3)
        del buf
        res['%dx%d' % (H, W)] = out
    print(json.dumps(res))


if __name__ == '__main__':
    main()
