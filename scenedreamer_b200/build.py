"""Builds scenedreamer_b200/libsdb200.so (the C-ABI library, include/sdb200.h) with nvcc for sm_90a (H100).

    python -m scenedreamer_b200.build [--force] [-v]

Plain nvcc, no torch headers: the library takes raw device pointers + a cudaStream_t, so it
compiles in seconds and cross-compiles on a machine without a GPU.  The .so is built IN-TREE (git-ignored).
"""
import concurrent.futures
import hashlib
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, 'csrc')
OBJ = os.path.join(HERE, 'csrc', '_obj')
LIB = os.path.join(HERE, 'libsdb200.so')
SOURCES = ['api.cu', 'dda.cu', 'gridenc.cu', 'posenc.cu', 'tc_selftest.cu', 'render_fused.cu', 'render_train.cu', 'wgrad.cu', 'sptrilinear.cu', 'rendercnn.cu', 'optim.cu', 'posestats.cu', 'worldgen.cu', 'modulate.cu']
NVCC_FLAGS = ['-gencode', 'arch=compute_90a,code=sm_90a', '-O3', '-lineinfo', '-std=c++17',
              '-Xcompiler', '-fPIC', '-Xcompiler', '-ffp-contract=off', '--expt-relaxed-constexpr'] + \
             os.environ.get('SDB_NVCC_EXTRA', '').split()      # e.g. -DSDB_TIMELINE (diagnostics build)


def _nvcc():
    for c in (os.environ.get('NVCC'), '/usr/local/cuda/bin/nvcc', 'nvcc'):
        if c and (os.path.isabs(c) and os.path.exists(c) or not os.path.isabs(c)):
            return c
    return 'nvcc'


def _digest(paths):
    h = hashlib.sha256(' '.join(NVCC_FLAGS).encode())
    for p in sorted(paths):
        with open(p, 'rb') as f:
            h.update(f.read())
    return h.hexdigest()


def build(force=False, verbose=False):
    srcs = [s for s in SOURCES if os.path.exists(os.path.join(CSRC, s))]
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(('.cu', '.cuh', '.h'))]
    deps.append(os.path.join(HERE, '..', 'include', 'sdb200.h'))
    stamp = os.path.join(OBJ, 'stamp')
    dig = _digest(deps)
    if not force and os.path.exists(LIB) and os.path.exists(stamp) and open(stamp).read() == dig:
        return LIB
    os.makedirs(OBJ, exist_ok=True)
    nvcc = _nvcc()

    def cc(src):
        obj = os.path.join(OBJ, src[:-3] + '.o')
        cmd = [nvcc] + NVCC_FLAGS + ['-c', os.path.join(CSRC, src), '-o', obj]
        if verbose:
            cmd.insert(1, '-Xptxas=-v')
            print(' '.join(cmd), flush=True)
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError('nvcc failed for %s:\n%s\n%s' % (src, r.stdout, r.stderr))
        if verbose:
            print(r.stderr)
        return obj
    with concurrent.futures.ThreadPoolExecutor(max_workers=min(8, len(srcs))) as ex:
        objs = list(ex.map(cc, srcs))
    # no library dependency besides the CUDA runtime: every kernel on the path, the weight-gradient GEMMs included, is ours
    tmp = LIB + '.tmp.%d' % os.getpid()                       # link aside, then rename: nobody dlopens a half-written file
    cmd = [nvcc, '-shared', '-o', tmp] + objs + ['-gencode', 'arch=compute_90a,code=sm_90a', '-lcudart']
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError('link failed:\n%s\n%s' % (r.stdout, r.stderr))
    os.replace(tmp, LIB)
    with open(stamp, 'w') as f:
        f.write(dig)
    return LIB


if __name__ == '__main__':
    print(build(force='--force' in sys.argv, verbose='-v' in sys.argv))
