"""f5: PCGCache.sample_world through the hook (read-ahead on a worker thread, pinned upload on a copy stream, sdb_scene_scatter
into the truncated volume) against the reference's own body (`_sdb200_reference_sample_world`) of the real PCGCache, staged
by oracle/build_ref.py, on cache worlds of the size PCGCache fixes (1024^2 x 256) written by synth.write_cache_world."""
import os
import random

import numpy as np
import pytest
import torch

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1500)]
DEV = torch.device('cuda', 0)
ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), '..'))


@pytest.fixture(scope='module')
def pcg():
    from oracle import refgen
    if refgen.reference_python_root() is None or \
            not os.path.exists(os.path.join(ROOT, 'oracle', '_ref', 'ref_voxlib', 'ref_voxlib.so')):
        pytest.skip('reference Python / extensions not staged in oracle/_ref (oracle/build_ref.py)')
    refgen.setup('dropin')
    import imaginaire.generators.scenedreamer  # noqa: F401  (imports pcg_gen)
    import imaginaire.model_utils.pcg_gen as pcg
    from scenedreamer_b200 import integration
    integration.ensure_installed()
    assert '_sdb200_reference_sample_world' in pcg.PCGCache.__dict__          # armed together with the generator hook
    return pcg


@pytest.fixture(scope='module')
def cache_root(tmp_path_factory):
    """Three worlds: w0 realistic (9-voxel shell + trees, voxels below gnd), w1 with a column up to the top layer
    (sky == 256), w2 a thinner shell on other terrain."""
    from scenedreamer_b200 import synth
    root = tmp_path_factory.mktemp('pcg_cache')
    synth.write_cache_world(str(root / 'w0'), seed=1)
    synth.write_cache_world(str(root / 'w1'), seed=2, peak=True)
    synth.write_cache_world(str(root / 'w2'), seed=3, shell=4)
    return str(root)


def _same_state(ours, ref):
    assert ours.voxel_t.is_cuda and ours.voxel_t.dtype == ref.voxel_t.dtype == torch.int32
    assert ours.voxel_t.shape == ref.voxel_t.shape and torch.equal(ours.voxel_t, ref.voxel_t)
    for name in ('current_height_map', 'current_semantic_map'):
        a, b = getattr(ours, name), getattr(ref, name)
        assert a.device == b.device and a.dtype == b.dtype and a.shape == b.shape and torch.equal(a, b), name
    assert ours.heightmap.device.type == 'cpu' and ours.heightmap.dtype == ref.heightmap.dtype == torch.int64
    assert torch.equal(ours.heightmap, ref.heightmap)
    assert ours.trans_mat.dtype == ref.trans_mat.dtype and torch.equal(ours.trans_mat, ref.trans_mat)


def _run_both(pcg, root, seed, calls, between=()):
    """`calls` consecutive loads on two instances, each with its own `random` stream from the same seed: the reference's body
    and the hook, compared after every call.  -> (world indices drawn, stats delta)."""
    from scenedreamer_b200 import worldgen
    ref, ours = pcg.PCGCache(root), pcg.PCGCache(root)
    random.seed(seed)
    rs_ref = rs_ours = random.getstate()
    before = dict(worldgen.stats)
    drawn = []
    for k in range(calls):
        peek = random.Random()
        peek.setstate(rs_ref)
        drawn.append(peek.randint(0, ref.n - 1))
        random.setstate(rs_ref)
        pcg.PCGCache._sdb200_reference_sample_world(ref, DEV)
        if k in between:
            random.random()
        rs_ref = random.getstate()
        random.setstate(rs_ours)
        ours.sample_world(DEV)
        if k in between:
            random.random()                                  # another consumer of `random` between iterations
        rs_ours = random.getstate()
        _same_state(ours, ref)
    assert rs_ours == rs_ref                                 # `random` consumed exactly as the reference consumes it
    torch.cuda.synchronize()
    return drawn, {k: worldgen.stats[k] - before[k] for k in before}, ours, ref


def _seed_covering(n, calls, want):
    for s in range(1000):
        random.seed(s)
        d = [random.randint(0, n - 1) for _ in range(calls)]
        if want(d):
            return s


def test_six_loads_equal_the_reference(pcg, cache_root):
    seed = _seed_covering(3, 6, lambda d: set(d) == {0, 1, 2} and any(a == b for a, b in zip(d, d[1:])))
    drawn, st, ours, _ = _run_both(pcg, cache_root, seed, 6)
    print('worlds drawn', drawn, 'stats', st)
    assert set(drawn) == {0, 1, 2}
    assert st == {'loads': 6, 'prefetch_hits': 5, 'prefetch_misses': 1, 'reference_loads': 0}


def test_world_edges_voxels_below_ground_and_top_layer(pcg, cache_root):
    sp = np.load(os.path.join(cache_root, 'w0', 'voxel_sparse.npy'))
    hm = np.load(os.path.join(cache_root, 'w0', 'hmap_mc.npy'))
    assert sp.shape[1] > 9 * 1024 * 1024 and int((sp[0] < hm.min()).sum()) > 0          # realistic nnz, voxels below gnd
    assert int(np.load(os.path.join(cache_root, 'w1', 'hmap_mc.npy')).max()) + 1 == 256
    # one world at a time: each instance sees only that world
    for name in ('w0', 'w1'):
        ref, ours = pcg.PCGCache(cache_root), pcg.PCGCache(cache_root)
        for c in (ref, ours):
            c.pcg_world_path, c.n = [os.path.join(cache_root, name)], 1
        random.seed(0)
        pcg.PCGCache._sdb200_reference_sample_world(ref, DEV)
        random.seed(0)
        ours.sample_world(DEV)
        _same_state(ours, ref)
        h = np.load(os.path.join(cache_root, name, 'hmap_mc.npy'))
        assert ours.voxel_t.shape[0] == h.max() + 1 - h.min()
        if name == 'w1':
            assert int(ours.trans_mat[0, 3]) + ours.voxel_t.shape[0] == 256 and int((ours.voxel_t[-1] != 0).sum()) >= 1


def test_forced_miss_still_loads_the_drawn_world(pcg, cache_root):
    seed = _seed_covering(3, 5, lambda d: len(set(d)) >= 2)
    drawn, st, _, _ = _run_both(pcg, cache_root, seed, 5, between=(1, 2))
    print('worlds drawn', drawn, 'stats', st)
    assert st['loads'] == 5 and st['reference_loads'] == 0 and st['prefetch_misses'] >= 1
    assert st['prefetch_hits'] + st['prefetch_misses'] == 5


def _raycast(vox):
    from scenedreamer_b200 import ops
    H = W = 262
    ori = torch.tensor([float(vox.shape[0]) + 8.0, 200.0, 230.0])
    d = torch.tensor([-0.45, 1.0, 0.8])
    up = torch.tensor([1.0, 0.0, 0.0])
    return ops.ray_voxel_intersection_perspective(vox, ori, d / d.norm(), up, 220.0, [(H - 1) / 2, (W - 1) / 2], [H, W], 6)


def _equal_rays(a, b):
    assert torch.equal(a[0], b[0]) and torch.equal(a[2], b[2])
    assert torch.equal(torch.nan_to_num(a[1], nan=-1.0), torch.nan_to_num(b[1], nan=-1.0))


def test_raycast_after_a_scene_switch(pcg, cache_root):
    """The DDA's height bound is keyed on the volume tensor: after a switch the raycast on the new volume equals the one on
    the reference's volume bit for bit (a stale bound would skip the new scene's geometry)."""
    ref, ours = pcg.PCGCache(cache_root), pcg.PCGCache(cache_root)
    for name in ('w2', 'w0', 'w1'):
        for c in (ref, ours):
            c.pcg_world_path, c.n = [os.path.join(cache_root, name)], 1
        random.seed(1)
        pcg.PCGCache._sdb200_reference_sample_world(ref, DEV)
        random.seed(1)
        ours.sample_world(DEV)
        a, b = _raycast(ours.voxel_t), _raycast(ref.voxel_t)
        _equal_rays(a, b)
        assert float((a[0][..., 0, 0] != 0).float().mean()) > 0.2                         # the rays hit this scene


def test_malformed_world_is_refused_and_the_previous_one_stays(pcg, cache_root, tmp_path):
    from scenedreamer_b200 import synth
    bad_xz = synth.write_cache_world(str(tmp_path / 'bad_xz'), seed=4, shell=2, bad=(1, 1024))
    bad_h = synth.write_cache_world(str(tmp_path / 'bad_h'), seed=4, shell=2, bad=(0, 256))
    ours = pcg.PCGCache(cache_root)
    ours.pcg_world_path, ours.n = [os.path.join(cache_root, 'w0')], 1
    ours.sample_world(DEV)
    vox = ours.voxel_t
    before = _raycast(vox)
    for bad, what in ((bad_xz, 'row 1'), (bad_h, 'row 0')):
        ours.pcg_world_path = [bad]
        with pytest.raises(RuntimeError, match=what) as e:
            ours.sample_world(DEV)
        assert os.path.join(bad, 'voxel_sparse.npy') in str(e.value)
        assert ours.voxel_t is vox
        _equal_rays(_raycast(ours.voxel_t), before)
    ours.pcg_world_path = [os.path.join(cache_root, 'w0')]
    ours.sample_world(DEV)
    _equal_rays(_raycast(ours.voxel_t), before)


def test_get_batch_with_a_pcg_cache(pcg, cache_root, monkeypatch):
    """Generator._get_batch (hooked sampler) over a PCGCache: the same batch and the same torch / numpy / `random` states as
    the reference's _get_batch with the reference's sample_world."""
    from oracle import refgen
    gen, _ = refgen.build_generator(1024, DEV)
    gen.voxel = pcg.PCGCache(cache_root)
    gen.cam_res, gen.crop_size, gen.pad = [360, 640], [256, 256], 6          # configs/scenedreamer_train.yaml
    cls = type(gen)
    outs, rngs = [], []
    for arm in ('reference', 'fused', 'fused'):
        if arm == 'reference':
            monkeypatch.setenv('SDB200_SCENECACHE', '0')
        else:
            monkeypatch.delenv('SDB200_SCENECACHE', raising=False)
        torch.manual_seed(77)
        np.random.seed(77)
        random.seed(77)
        fn = cls._sdb200_reference_get_batch if arm == 'reference' else cls._get_batch
        o = fn(gen, 2, DEV)
        outs.append((o, gen.voxel.voxel_t.clone(), gen.voxel.trans_mat.clone()))
        rngs.append((torch.get_rng_state().clone(), np.random.get_state()[1].copy(), random.getstate()))
    (ref, rvox, rmat) = outs[0]
    for (o, vox, mat), rng in zip(outs[1:], rngs[1:]):
        assert torch.equal(vox, rvox) and torch.equal(mat, rmat)
        assert torch.equal(ref[0], o[0]) and torch.equal(ref[2], o[2]) and torch.equal(ref[3], o[3])
        assert torch.equal(torch.nan_to_num(ref[1], nan=-1.0), torch.nan_to_num(o[1], nan=-1.0))
        assert torch.equal(rngs[0][0], rng[0]) and np.array_equal(rngs[0][1], rng[1]) and rngs[0][2] == rng[2]
