"""Host side of the PCG scene cache (worldgen.fused_sample_world, f5) without a GPU: the argument checks of sdb_scene_scatter,
the .npy reader, the slice normalisation of gnd / sky, the coordinate validation, and the read-ahead's use of `random`."""
import concurrent.futures
import ctypes
import os
import random

import numpy as np
import pytest
import torch

from scenedreamer_b200 import _lib, worldgen

EINVAL = -1


def _cpu_alloc(n):
    return torch.empty(n, dtype=torch.uint8)


def write_world(d, SH, X, seed, nnz=40, bad=None, sparse_dtype=np.int16):
    """A world in the layout scripts/pcg_cache.py writes: voxel_sparse int16 [4, nnz], height_map float32 [1,1,X,X],
    semantic_map float32 [1,11,X,X], hmap_mc int64 [X,X]."""
    rng = np.random.default_rng(seed)
    os.makedirs(d, exist_ok=True)
    sp = np.stack([rng.integers(0, SH, nnz), rng.integers(0, X, nnz), rng.integers(0, X, nnz), rng.integers(1, 680, nnz)])
    if bad is not None:
        sp[bad[0], 0] = bad[1]
    np.save(os.path.join(d, 'voxel_sparse.npy'), sp.astype(sparse_dtype))
    np.save(os.path.join(d, 'height_map.npy'), rng.random((1, 1, X, X), dtype=np.float32))
    np.save(os.path.join(d, 'semantic_map.npy'), rng.random((1, 11, X, X), dtype=np.float32))
    np.save(os.path.join(d, 'hmap_mc.npy'), rng.integers(2, SH - 2, (X, X)).astype(np.int64))
    return d


class _Cache:
    """Stand-in for pcg_gen.PCGCache: the same attributes, and a sample_world that draws like the reference (pcg_gen.py:27)."""

    def __init__(self, root, SH=16, X=8):
        self.sample_size, self.sample_height = X, SH
        self.pcg_world_path = [os.path.join(root, p) for p in sorted(os.listdir(root))]
        self.n = len(self.pcg_world_path)
        self.reference_calls = []

    def sample_world(self, device):
        idx = random.randint(0, self.n - 1)
        self.reference_calls.append(idx)


worldgen.install(_Cache)


def test_scene_scatter_refuses_bad_arguments():
    L = _lib.lib()
    d = ctypes.c_void_p(0x1000)
    assert L.sdb_scene_scatter(None, 10, 256, 64, 64, 0, 10, d, None) == EINVAL
    assert L.sdb_scene_scatter(d, 10, 256, 64, 64, 0, 10, None, None) == EINVAL
    assert L.sdb_scene_scatter(d, -1, 256, 64, 64, 0, 10, d, None) == EINVAL
    for SH, X, Z in ((0, 64, 64), (256, 0, 64), (256, 64, -1)):
        assert L.sdb_scene_scatter(d, 10, SH, X, Z, 0, 1, d, None) == EINVAL
    for gnd, sky in ((-1, 10), (10, 10), (11, 10), (0, 257), (256, 257)):
        assert L.sdb_scene_scatter(d, 10, 256, 64, 64, gnd, sky, d, None) == EINVAL


@pytest.mark.parametrize('arr', [
    np.arange(-40, 40, dtype=np.int16).reshape(4, 20),
    np.linspace(0, 1, 2 * 11 * 3 * 5, dtype=np.float32).reshape(2, 11, 3, 5),
    np.arange(35, dtype=np.int64).reshape(5, 7) - 9,
    np.zeros((4, 0), np.int16),
    np.array(3.5, np.float32),
], ids=['int16', 'float32', 'int64', 'empty', 'scalar'])
@pytest.mark.parametrize('order', ['C', 'F'])
def test_read_npy_equals_np_load(tmp_path, arr, order):
    p = str(tmp_path / 'a.npy')
    np.save(p, np.asarray(arr, order=order))
    got, t = worldgen.read_npy(p, _cpu_alloc)
    ref = np.load(p)
    assert got.dtype == ref.dtype and got.shape == ref.shape and np.array_equal(got, ref)
    assert got.flags['C_CONTIGUOUS'] and tuple(t.shape) == ref.shape and np.array_equal(t.numpy(), ref)


def test_read_npy_reads_into_the_given_buffer(tmp_path):
    p = str(tmp_path / 'a.npy')
    np.save(p, np.arange(12, dtype=np.int64).reshape(3, 4))
    buf = torch.zeros(200, dtype=torch.uint8)
    got, t = worldgen.read_npy(p, lambda n: buf)
    assert t.data_ptr() == buf.data_ptr() and got.ctypes.data == buf.data_ptr()


def test_read_npy_refuses_a_truncated_file(tmp_path):
    p = str(tmp_path / 'a.npy')
    np.save(p, np.arange(100, dtype=np.int16))
    with open(p, 'r+b') as f:
        f.truncate(os.path.getsize(p) - 10)
    with pytest.raises(ValueError, match='a.npy'):
        worldgen.read_npy(p, _cpu_alloc)


@pytest.mark.parametrize('gnd,sky', [(0, 256), (5, 100), (0, 1), (255, 256), (100, 300), (256, 300), (300, 400), (-3, 10),
                                     (-3, -1), (-300, 5), (7, 7), (9, 2), (0, 0)])
def test_slice_bounds_follow_python_slicing(gnd, sky):
    SH = 256
    start, stop = worldgen.slice_bounds(np.int64(gnd), np.int64(sky), SH)
    assert range(start, stop) == range(SH)[gnd:sky] and stop >= start
    assert torch.zeros(SH)[np.int64(gnd):np.int64(sky)].shape[0] == stop - start      # what voxel_t[gnd:sky] keeps


@pytest.mark.parametrize('row,value', [(0, 16), (0, -1), (1, 8), (2, -5), (2, 8)])
def test_validation_names_the_file_and_the_range(tmp_path, row, value):
    d = write_world(str(tmp_path / 'w0'), 16, 8, seed=1, bad=(row, value))
    hset = worldgen._HostSet(pin=False)
    with pytest.raises(RuntimeError) as e:
        worldgen.read_world(d, hset, 0, 0, (16, 8, 8))
    msg = str(e.value)
    assert os.path.join(d, 'voxel_sparse.npy') in msg and ('row %d' % row) in msg and str(value) in msg
    with pytest.raises(RuntimeError, match='expected \\[4, nnz\\]'):
        worldgen.validate_sparse(np.zeros((3, 5), np.int16), (16, 8, 8), 'x.npy')


def test_read_world_routes_non_int16_sparse_to_the_reference(tmp_path):
    d = write_world(str(tmp_path / 'w0'), 16, 8, seed=2, sparse_dtype=np.int32)
    w = worldgen.read_world(d, worldgen._HostSet(pin=False), 0, 3, (16, 8, 8))
    assert w.reference and w.idx == 3
    d = write_world(str(tmp_path / 'w1'), 16, 8, seed=2)
    w = worldgen.read_world(d, worldgen._HostSet(pin=False), 1, 4, (16, 8, 8))
    hm = np.load(os.path.join(d, 'hmap_mc.npy'))
    assert not w.reference and w.gnd == hm.min() and type(w.gnd) is type(hm.min())
    assert (w.start, w.stop) == (hm.min(), hm.max() + 1)
    assert np.array_equal(w.sparse_t.numpy(), np.load(os.path.join(d, 'voxel_sparse.npy')))


@pytest.fixture
def stubbed_upload(monkeypatch):
    """The device half replaced by a recorder: (world index, path) of every fused load."""
    loads = []
    monkeypatch.setattr(worldgen, '_upload_world', lambda cache, st, w, dev: loads.append((w.idx, w.path)))
    monkeypatch.delenv('SDB200_SCENECACHE', raising=False)
    return loads


def _reference_draws(seed, n, calls, between=None):
    random.seed(seed)
    out = []
    for k in range(calls):
        out.append(random.randint(0, n - 1))
        if between is not None and k == between:
            random.random()
    return out, random.getstate()


def test_read_ahead_draws_like_the_reference(tmp_path, stubbed_upload):
    for k in range(4):
        write_world(str(tmp_path / ('w%d' % k)), 16, 8, seed=k)
    cache = _Cache(str(tmp_path))
    want, state = _reference_draws(11, cache.n, 8)
    before = dict(worldgen.stats)
    random.seed(11)
    for _ in range(8):
        cache.sample_world('cuda')
    assert random.getstate() == state
    assert [i for i, _ in stubbed_upload] == want and [p for _, p in stubbed_upload] == [cache.pcg_world_path[i] for i in want]
    d = {k: worldgen.stats[k] - before[k] for k in before}
    assert d == {'loads': 8, 'prefetch_hits': 7, 'prefetch_misses': 1, 'reference_loads': 0}
    assert cache.reference_calls == []


def test_a_draw_between_calls_misses_and_loads_the_drawn_world(tmp_path, stubbed_upload):
    for k in range(5):
        write_world(str(tmp_path / ('w%d' % k)), 16, 8, seed=k)
    cache = _Cache(str(tmp_path))
    want, state = _reference_draws(3, cache.n, 6, between=2)
    before = dict(worldgen.stats)
    random.seed(3)
    for k in range(6):
        cache.sample_world('cuda')
        if k == 2:
            random.random()                          # e.g. a camera controller drawing from `random`
    assert random.getstate() == state and [i for i, _ in stubbed_upload] == want
    d = {k: worldgen.stats[k] - before[k] for k in before}
    assert d['loads'] == 6 and d['prefetch_misses'] >= 2 and d['prefetch_hits'] + d['prefetch_misses'] == 6


def test_non_int16_sparse_and_switch_run_the_reference_body(tmp_path, stubbed_upload, monkeypatch):
    write_world(str(tmp_path / 'w0'), 16, 8, seed=0, sparse_dtype=np.int32)
    cache = _Cache(str(tmp_path))
    before = dict(worldgen.stats)
    random.seed(5)
    cache.sample_world('cuda')
    state = random.getstate()
    random.seed(5)
    random.randint(0, 0)
    assert random.getstate() == state and cache.reference_calls == [0] and stubbed_upload == []
    cache.sample_world('cpu')                                         # not a CUDA device
    monkeypatch.setenv('SDB200_SCENECACHE', '0')
    cache.sample_world('cuda')
    assert cache.reference_calls == [0, 0, 0] and stubbed_upload == []
    assert worldgen.stats['reference_loads'] - before['reference_loads'] == 3


def test_failed_read_ahead_is_retried_then_raised(tmp_path, stubbed_upload):
    d = write_world(str(tmp_path / 'w0'), 16, 8, seed=0)
    cache = _Cache(str(tmp_path))
    random.seed(0)
    cache.sample_world('cuda')                                        # one world: the read-ahead holds world 0 again
    st = worldgen._states[cache]

    def failed(msg):
        fut = concurrent.futures.Future()
        fut.set_exception(RuntimeError(msg))
        st.pending = (st.pending[0], st.pending[1], fut)
    st.pending[2].exception()                                          # the read-ahead has finished
    failed('background read failed')
    cache.sample_world('cuda')                                        # retried synchronously: loads
    assert [i for i, _ in stubbed_upload] == [0, 0]
    st.pending[2].exception()
    write_world(d, 16, 8, seed=0, bad=(1, 9))
    failed('background read failed again')
    with pytest.raises(RuntimeError, match='failed again') as e:     # both failed: the background error, from the retry's
        cache.sample_world('cuda')
    assert 'voxel_sparse.npy' in str(e.value.__cause__) and len(stubbed_upload) == 2
