"""Per-layer timeline of the fused render kernel (CTA 0, a few steady-state sample steps), from the clock stamps the kernel
records when a diagnostics buffer is armed (rf_common.cuh SDB_STAMP).  Workload = bench.py's C2 frame.

    SDB_NVCC_EXTRA=-DSDB_TIMELINE python -m scenedreamer_b200.build --force
    PYTHONPATH=. python tools/render_timeline.py [first_step]
"""
import ctypes
import sys

import numpy as np
import torch

import bench
from scenedreamer_b200 import _lib, render, synth

DEV = 'cuda:0'
first = int(sys.argv[1]) if len(sys.argv) > 1 else 60
world, poses, P, z, genc, lut = bench.build_workload(DEV)
fr = bench.FrameRenderer(world, P, z, genc, lut, DEV, render.PRECISION_FP16X3, bench.SPP)
cam = synth.frame_camera(world, poses[3], bench.OUT_HW, bench.PAD)
for _ in range(2):
    fr.frame(cam)
torch.cuda.synchronize()
buf = torch.zeros(4096, dtype=torch.int32, device=DEV)
buf[60], buf[61] = 0x7131, first
L = _lib.lib()
L.sdb_debug_set_progress_buffer(ctypes.c_void_p(buf.data_ptr()))
fr.frame(cam)
torch.cuda.synchronize()
L.sdb_debug_set_progress_buffer(ctypes.c_void_p(0))
t = buf[64:64 + 6 * 8 * 8].cpu().numpy().astype(np.int64).reshape(6, 8, 8) & 0xffffffff
NL = 7
names = ['fc_1', 'fc_2', 'fc_3', 'fc_4', 'fc_5', 'fc_6', 'out_c']


def d(a, b):
    return int((a - b) & 0xffffffff) if a and b else -1


print('# cycles (SM clock), CTA 0, sample steps %d..%d of its ray slots; per layer:' % (first, first + 5))
print('#  compute = MMA warpgroup: inputs of the layer ready -> its accumulators written')
print('#  hand    = accumulators written -> seen by the epilogue (half 0)')
print('#  epi     = accumulators seen -> last slab handed over (max of the two halves)')
print('#  next    = accumulators written -> inputs of the next layer ready (MMA warpgroup idle)')
print('%-6s %9s %7s %7s %7s %7s' % ('layer', 'compute', 'hand', 'epi', 'next', 'period'))
for s in range(1, 5):
    for l in range(NL):
        r = t[s, l]
        nxt = t[s, l + 1][0] if l + 1 < NL else t[s + 1, 0][0]
        row = [d(r[1], r[0]), d(r[2], r[1]), max(d(r[3], r[2]), d(r[5], r[4])), d(nxt, r[1]), d(nxt, r[0])]
        if s == 2:
            print('%-6s %9d %7d %7d %7d %7d' % (names[l], *row))
print('# gather role preparing step n+1, relative to the MMA warpgroup entering fc_1 of step n (cycles): start (compositing of n-1 seen), slots refilled,')
print('#   features gathered (all loads + interpolation done), operand buffer free (colour-layer MMAs of step n retired)')
for s in range(1, 5):
    g = t[s + 1, 7]
    base = t[s, 0][0]
    print('gather for step %d: %s   | MMA layer starts of step %d: %s' % (first + s + 1, [d(g[k], base) for k in range(4)], first + s,
                                                                              [d(t[s, l][0], base) for l in range(NL)]))
print('step period (MMA warpgroup, fc_1 to fc_1): %s cycles' % [d(t[s + 1, 0][0], t[s, 0][0]) for s in range(0, 5)])
