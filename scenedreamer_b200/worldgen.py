"""Host side of the on-device scene builder (libsdb200: sdb_world_build / sdb_world_truncate, sdb_scene_scatter).

Mirrors PCGVoxelGenerator.next_world (imaginaire/model_utils/pcg_gen.py:83-174): bird's-eye-view maps (height, semantic,
tree) + voxel tree models -> the voxel volume `voxel_t[height, x, z]`, the height map used by the camera controllers, the
world-to-local offset and the two conditioning maps.  What stays on the host is O(X*Z) bookkeeping that must consume the
host RNG exactly like the reference (the quantisation of the height map in numpy, the list of tree instances with
`random.choice` per accepted tree); the O(256*X*Z) volume only ever exists in HBM.

Also the training-side counterpart, PCGCache.sample_world (pcg_gen.py:26-46, once per iteration with `pcg_cache: True`):
the cached world's sparse voxel list is scattered on the device straight into the truncated volume (sdb_scene_scatter),
uploaded from pinned memory on a copy stream, and the next iteration's world is read from disk while this one trains.
"""
import concurrent.futures
import ctypes
import math
import os
import random
import weakref

import numpy as np
import torch
import torch.nn.functional as F

from . import _lib

SAMPLE_HEIGHT = 256
PAD_NUM = 16
BOUNDARY = 50
BIOME2MC = [28, 9, 8, 1, 9, 8, 9, 8, 30, 26]                                  # pcg_gen.py:118
BIOME_TREES = [[], [5], [1, 7], [], [1, 2], [1, 2, 3], [4], [0, 3], [5, 6, 7], []]   # pcg_gen.py:105-116, in dict order


def _ptr(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def tree_instances(height_q, tree_map, tree_models, rng=random):
    """The reference's double loop over biomes and tree cells (pcg_gen.py:132-146) without the pasting: returns int32
    [n, 4] = (h + 16, x, z, model id) in iteration order; `rng.choice` is called exactly when the reference calls it."""
    X, Z = height_q.shape
    h16 = height_q.astype(np.int64) + PAD_NUM
    inst = []
    for biome_id in range(len(BIOME2MC)):
        selected = BIOME_TREES[biome_id]
        if len(selected) == 0:
            continue
        xs, zs = np.nonzero(tree_map == biome_id)                              # row-major, like the boolean mask indexing
        for x, z in zip(xs.tolist(), zs.tolist()):
            h = int(h16[x, z])
            if x < BOUNDARY or x > X - BOUNDARY or z < BOUNDARY or z > Z - BOUNDARY or h > SAMPLE_HEIGHT - BOUNDARY:
                continue
            inst.append((h, x, z, rng.choice(selected)))
    return np.asarray(inst, dtype=np.int32).reshape(-1, 4)


def build_world(height_map, semantic_map, tree_map, tree_models, device, rng=random):
    """height_map float [X, Z] (values < 0 are water), semantic_map uint8 [X, Z] in 0..9, tree_map uint8 [X, Z] (255 = none),
    tree_models: sequence of int32 [dh, dx, dz] voxel models (ckpt['assets']).
    -> dict(voxel_t int32 [sky-gnd, X, Z] on `device`, heightmap int64 [X, Z] (CPU, like the reference), gnd_level,
            current_height_map [1,1,X,Z], current_semantic_map [1,C,X,Z] on `device`, total_size)."""
    L = _lib.lib()
    dev = torch.device(device)
    hm = np.array(height_map, copy=True)
    hm[hm < 0] = 0                                                                                   # pcg_gen.py:94
    hq = ((hm - hm.min()) / (1 - hm.min()) * (SAMPLE_HEIGHT - 1)).astype(np.int16)                   # :95
    X, Z = hq.shape
    sem = np.asarray(semantic_map)
    trees = np.asarray(tree_map)
    inst = tree_instances(hq, trees, tree_models, rng)
    models = [np.ascontiguousarray(np.asarray(m.cpu() if torch.is_tensor(m) else m, dtype=np.int32)) for m in tree_models]
    mdim = np.asarray([m.shape for m in models], dtype=np.int32).reshape(-1, 3)
    moff = np.cumsum([0] + [m.size for m in models[:-1]]).astype(np.int64) if models else np.zeros(0, np.int64)
    flat = np.concatenate([m.reshape(-1) for m in models]) if models else np.zeros(1, np.int32)
    label = np.asarray(BIOME2MC, dtype=np.int32)[sem.astype(np.int64)]
    with torch.cuda.device(dev):
        st = ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
        # C-contiguous uploads: the maps may arrive Fortran-ordered (np.load keeps the order of the saved array), and a torch
        # tensor made from such an array keeps transposed strides all the way to the device
        d_hq = torch.from_numpy(np.ascontiguousarray(hq, dtype=np.int32)).to(dev)
        d_label = torch.from_numpy(np.ascontiguousarray(label, dtype=np.int32)).to(dev)
        d_inst = torch.from_numpy(np.ascontiguousarray(inst)).to(dev) if len(inst) else None
        d_models, d_mdim, d_moff = torch.from_numpy(flat).to(dev), torch.from_numpy(mdim).to(dev), torch.from_numpy(moff).to(dev)
        world = torch.empty(SAMPLE_HEIGHT, X, Z, dtype=torch.int32, device=dev)                       # scratch: 1 GB at 1024^2, 4.3 GB at 2048^2
        heightmap = torch.empty(X, Z, dtype=torch.int64, device=dev)
        minmax = torch.empty(2, dtype=torch.int32, device=dev)
        _lib.check(L.sdb_world_build(_ptr(d_hq), _ptr(d_label), X, Z, SAMPLE_HEIGHT, _ptr(d_inst), int(len(inst)), _ptr(d_models),
                                     _ptr(d_mdim), _ptr(d_moff), _ptr(world), _ptr(heightmap), _ptr(minmax), st), 'sdb_world_build')
        gnd, top = [int(v) for v in minmax.cpu()]                                                     # the output shape is data-dependent
        sky = top + 1
        voxel_t = torch.empty(sky - gnd, X, Z, dtype=torch.int32, device=dev)
        _lib.check(L.sdb_world_truncate(_ptr(world), X, Z, gnd, sky, _ptr(voxel_t), st), 'sdb_world_truncate')
        del world
        # O(X*Z) host arithmetic, uploaded: torch's CPU int64 / int division is what the reference's value is bit for bit
        h16 = torch.from_numpy(np.ascontiguousarray(hq, dtype=np.int64)) + PAD_NUM
        current_height_map = (h16 / (SAMPLE_HEIGHT - 1))[None, None].to(dev)                          # :167
        org_sem = torch.from_numpy(np.ascontiguousarray(sem)).to(dev)
        org_sem[torch.from_numpy(np.ascontiguousarray(trees != 255)).to(dev)] = 10                                          # :100-101
        current_semantic_map = F.one_hot(org_sem.to(torch.int64)).to(torch.float).permute(2, 0, 1)[None]   # :168
    return dict(voxel_t=voxel_t, heightmap=heightmap.cpu(), gnd_level=gnd, sky_level=sky, current_height_map=current_height_map,
                current_semantic_map=current_semantic_map, total_size=(X, Z))


def fused_next_world(self, device, world_dir, pcg_asset):
    """Replacement body of PCGVoxelGenerator.next_world (same arguments, same attributes set)."""
    import cv2
    if torch.device(device).type != 'cuda':
        return type(self)._sdb200_reference_next_world(self, device, world_dir, pcg_asset)
    height_map = np.load(os.path.join(world_dir, 'heightmap.npy'))                                    # :87-92
    semantic_map = cv2.imread(os.path.join(world_dir, 'semanticmap.png'), 0)
    tree_map = cv2.imread(os.path.join(world_dir, 'treemap.png'), 0)
    w = build_world(height_map, semantic_map, tree_map, pcg_asset['assets'], device)
    self.total_size = w['total_size']
    self.trans_mat = torch.eye(4)
    self.current_height_map = w['current_height_map']
    self.current_semantic_map = w['current_semantic_map']
    self.heightmap = w['heightmap']
    self.voxel_t = w['voxel_t']
    self.trans_mat[0, 3] += w['gnd_level']


# ------------------------------------------------------------------------------------------------
# PCGCache.sample_world (pcg_gen.py:26-46): one cached scene per training iteration (libsdb200: sdb_scene_scatter)
# ------------------------------------------------------------------------------------------------
stats = {'loads': 0, 'prefetch_hits': 0, 'prefetch_misses': 0, 'reference_loads': 0}
_states = weakref.WeakKeyDictionary()           # PCGCache instance -> _SceneCacheState (kept off the module: deepcopy-safe)


def scene_cache_enabled():
    return os.environ.get('SDB200_SCENECACHE', '1') not in ('0', 'false', 'False', 'off')


def slice_bounds(gnd, sky, n):
    """(start, stop) with range(start, stop) == range(n)[gnd:sky]: what voxel_t[gnd:sky] keeps of a volume of height n."""
    start, stop, _ = slice(int(gnd), int(sky)).indices(n)
    return start, max(start, stop)


def _npy_header(f):
    """(shape, fortran_order, dtype) of an .npy file positioned at its start, or None for a format version this reader leaves
    to np.load."""
    version = np.lib.format.read_magic(f)
    if version == (1, 0):
        return np.lib.format.read_array_header_1_0(f)
    if version == (2, 0):
        return np.lib.format.read_array_header_2_0(f)
    return None


def read_npy(path, alloc):
    """np.load(path) into host memory the caller owns: alloc(nbytes) -> uint8 CPU tensor of at least nbytes (a pinned buffer
    for the upload).  A C-order payload is read with readinto straight into it -- no second host copy; a Fortran-order (or
    otherwise unusual) file goes through np.load + ascontiguousarray and is copied in.
    -> (numpy array equal to np.load(path), torch tensor of the same dtype and shape on the same memory)."""
    with open(path, 'rb') as f:
        hdr = _npy_header(f)
        if hdr is not None:
            shape, fortran, dtype = hdr
            if not fortran and dtype.isnative and not dtype.hasobject and dtype.fields is None:
                n = math.prod(shape) * dtype.itemsize
                buf = alloc(n)
                mv = memoryview(buf.numpy())[:n]
                got = 0
                while got < n:
                    k = f.readinto(mv[got:])
                    if not k:
                        raise ValueError('%s: the file ends after %d of %d payload bytes' % (path, got, n))
                    got += k
                return _typed(buf, n, dtype, shape)
    arr = np.ascontiguousarray(np.load(path))
    buf = alloc(arr.nbytes)
    buf.numpy()[:arr.nbytes] = arr.reshape(-1).view(np.uint8)
    return _typed(buf, arr.nbytes, arr.dtype, arr.shape)


def _typed(buf, n, dtype, shape):
    tdt = torch.from_numpy(np.empty(0, dtype)).dtype
    return buf.numpy()[:n].view(dtype).reshape(shape), buf[:n].view(tdt).reshape(shape)


def validate_sparse(sparse, dims, path):
    """RuntimeError naming the file unless `sparse` is [4, nnz] with rows x, y, z inside dims = (SH, X, Z).  The reference would
    wrap a negative index (index_put) or stop on a device-side assert for one past the end; here the load is refused before
    anything is launched, and the previous scene stays in place."""
    if sparse.ndim != 2 or sparse.shape[0] != 4:
        raise RuntimeError('%s: voxel_sparse has shape %s, expected [4, nnz]' % (path, tuple(sparse.shape)))
    if sparse.shape[1] == 0:
        return
    for row, (name, n) in enumerate(zip(('x (height)', 'y', 'z'), dims)):
        lo, hi = int(sparse[row].min()), int(sparse[row].max())
        if lo < 0 or hi >= n:
            raise RuntimeError('%s: voxel_sparse row %d, %s, spans [%d, %d], outside [0, %d)' % (path, row, name, lo, hi, n))


class _HostSet:
    """One set of host buffers (one per file of a world), pinned for the asynchronous upload.  `event` marks the end of the
    copy that last read the set: whoever fills it next waits on it first."""

    def __init__(self, pin):
        self.pin, self.bufs, self.event = pin, {}, None

    def alloc(self, name):
        def get(n):
            b = self.bufs.get(name)
            if b is None or b.numel() < n:
                b = self.bufs[name] = torch.empty(max(n, 1), dtype=torch.uint8, pin_memory=self.pin)
            return b
        return get

    def wait(self):
        ev, self.event = self.event, None
        if ev is not None:
            ev.synchronize()


class _World:
    """One cache world read into a host set: arrays (numpy) / tensors (torch) on the set's memory, gnd = hmap_mc.min() (the
    numpy scalar the reference adds to trans_mat), [start, stop) the normalised voxel_t[gnd:sky] slice.  reference = True:
    voxel_sparse is not int16, the reference's body loads this world."""

    def __init__(self, idx, set_id, reference=False):
        self.idx, self.set_id, self.reference = idx, set_id, reference


def read_world(path, hset, set_id, idx, dims):
    """The four files of a cache world into `hset`, checked and reduced to what the upload needs (runs on the worker thread
    for a prefetched world, on the caller's thread otherwise)."""
    hset.wait()
    sparse, sparse_t = read_npy(os.path.join(path, 'voxel_sparse.npy'), hset.alloc('voxel_sparse'))
    if sparse.dtype != np.int16:
        return _World(idx, set_id, reference=True)
    w = _World(idx, set_id)
    w.path, w.sparse_t = path, sparse_t
    _, w.height_t = read_npy(os.path.join(path, 'height_map.npy'), hset.alloc('height_map'))
    _, w.semantic_t = read_npy(os.path.join(path, 'semantic_map.npy'), hset.alloc('semantic_map'))
    hmap, _ = read_npy(os.path.join(path, 'hmap_mc.npy'), hset.alloc('hmap_mc'))
    validate_sparse(sparse, dims, os.path.join(path, 'voxel_sparse.npy'))
    w.hmap = np.array(hmap, copy=True)                    # becomes self.heightmap: must outlive the reuse of the host set
    w.gnd = w.hmap.min()                                  # pcg_gen.py:43-44
    w.start, w.stop = slice_bounds(w.gnd, w.hmap.max() + 1, dims[0])
    return w


class _SceneCacheState:
    """Per PCGCache instance: two host sets, the background read in flight, one worker thread and one copy stream per device."""

    def __init__(self, pin):
        self.sets = (_HostSet(pin), _HostSet(pin))
        self.cur = 1                     # set of the world in use; the next read goes to the other one
        self.pending = None              # (world path, set_id, future) of the background read
        self.pool = None
        self.streams = {}

    def executor(self):
        if self.pool is None:
            self.pool = concurrent.futures.ThreadPoolExecutor(max_workers=1, thread_name_prefix='sdb200-scene-cache')
        return self.pool

    def copy_stream(self, dev):
        s = self.streams.get(dev.index)
        if s is None:
            s = self.streams[dev.index] = torch.cuda.Stream(dev)
        return s


def _state(cache):
    st = _states.get(cache)
    if st is None:
        st = _states[cache] = _SceneCacheState(torch.cuda.is_available())
        weakref.finalize(cache, _shutdown, st)
    return st


def _shutdown(st):
    if st.pool is not None:
        st.pool.shutdown(wait=True, cancel_futures=True)


def _dims(cache):
    return (cache.sample_height, cache.sample_size, cache.sample_size)


def _take(cache, st, idx):
    """World `idx`: the background read's when it holds that world's path (waited for if still running), else read now.  A
    failed background read is retried here; its error is raised only if this read fails as well."""
    path = cache.pcg_world_path[idx]
    pend, st.pending = st.pending, None
    set_id, bg_err = 1 - st.cur, None
    if pend is not None:
        ppath, set_id, fut = pend
        try:
            w = fut.result()             # a miss waits too: the read it holds is filling the set this one needs
        except Exception as e:
            w, bg_err = None, (e if ppath == path else None)
        if ppath == path and w is not None:
            stats['prefetch_hits'] += 1
            w.idx = idx
            return w
    stats['prefetch_misses'] += 1
    try:
        return read_world(path, st.sets[set_id], set_id, idx, _dims(cache))
    except Exception as e:
        if bg_err is not None:
            raise bg_err from e
        raise


def _upload_world(cache, st, w, dev):
    """Pinned host set -> device on the copy stream (it overlaps the tail of the previous iteration on the current stream, which
    waits on its event), then the scatter into the truncated volume on the current stream.  Nothing here waits for the device."""
    L = _lib.lib()
    SH, X, Z = _dims(cache)
    if dev.index is None:
        dev = torch.device('cuda', torch.cuda.current_device())
    with torch.cuda.device(dev):
        main = torch.cuda.current_stream(dev)
        cs = st.copy_stream(dev)
        with torch.cuda.stream(cs):                       # allocated in the copy stream's pool, the only stream writing them
            staged = [torch.empty(t.shape, dtype=t.dtype, device=dev) for t in (w.sparse_t, w.height_t, w.semantic_t)]
            for d, h in zip(staged, (w.sparse_t, w.height_t, w.semantic_t)):
                d.copy_(h, non_blocking=True)
            ev = torch.cuda.Event()
            ev.record(cs)
        st.sets[w.set_id].event = ev
        main.wait_event(ev)
        for d in staged:
            d.record_stream(main)                         # read on the current stream: not reused before that work is done
        d_sparse, height, semantic = staged
        voxel_t = torch.empty(w.stop - w.start, X, Z, dtype=torch.int32, device=dev)
        if voxel_t.numel():
            _lib.check(L.sdb_scene_scatter(_ptr(d_sparse), int(d_sparse.shape[1]), SH, X, Z, w.start, w.stop, _ptr(voxel_t),
                                           ctypes.c_void_p(main.cuda_stream)), 'sdb_scene_scatter')
    cache.voxel_t = voxel_t
    cache.current_height_map = height
    cache.current_semantic_map = semantic
    cache.heightmap = torch.from_numpy(w.hmap)
    cache.trans_mat = torch.eye(4)
    cache.trans_mat[0, 3] += w.gnd


def _prefetch_next(cache, st):
    """Read the world the NEXT call will draw, on the worker: the draw is peeked on a copy of the module RNG (the worker never
    touches `random`).  Any other draw from `random` before that call makes the peek miss, which costs a synchronous read."""
    peek = random.Random()
    peek.setstate(random.getstate())
    nxt = peek.randint(0, cache.n - 1)
    sid, path = 1 - st.cur, cache.pcg_world_path[nxt]
    st.pending = (path, sid, st.executor().submit(read_world, path, st.sets[sid], sid, nxt, _dims(cache)))


def fused_sample_world(self, device):
    """Replacement body of PCGCache.sample_world (same argument, same attributes with the same dtypes and values): one
    `random.randint` draw as the reference makes it, the world's files read ahead on a worker thread (pinned buffers), uploaded
    on a copy stream and scattered straight into the truncated volume."""
    reference = type(self)._sdb200_reference_sample_world
    dev = torch.device(device)
    if dev.type != 'cuda' or not scene_cache_enabled():
        stats['reference_loads'] += 1
        return reference(self, device)
    st = _state(self)
    rng = random.getstate()
    idx = random.randint(0, self.n - 1)                                   # pcg_gen.py:27
    w = _take(self, st, idx)
    st.cur = w.set_id
    if w.reference:                                                      # a voxel_sparse that is not int16: the reference's
        stats['reference_loads'] += 1                                    # body, drawing the same idx from the same state
        random.setstate(rng)
        reference(self, device)
    else:
        _upload_world(self, st, w, dev)
        stats['loads'] += 1
    _prefetch_next(self, st)


def install(pcg_cls):
    """Patch PCGVoxelGenerator.next_world and / or PCGCache.sample_world, whichever the class defines (idempotent)."""
    if '_sdb200_reference_next_world' not in pcg_cls.__dict__ and 'next_world' in pcg_cls.__dict__:
        pcg_cls._sdb200_reference_next_world = pcg_cls.next_world
        pcg_cls.next_world = fused_next_world
    if '_sdb200_reference_sample_world' not in pcg_cls.__dict__ and 'sample_world' in pcg_cls.__dict__:
        pcg_cls._sdb200_reference_sample_world = pcg_cls.sample_world
        pcg_cls.sample_world = fused_sample_world
    return pcg_cls
