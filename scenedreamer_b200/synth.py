"""Synthetic scenes and evaluation cameras.

No checkpoint, terrain library or dataset is available offline, so benchmarks and tests render a
seeded procedural scene.  The voxelisation restates what the reference's PCGVoxelGenerator does
to BEV maps (imaginaire/model_utils/pcg_gen.py:94-178) so that the hot path sees the same input
layout: an int32 volume ``voxel_t[height, x, z]`` holding Minecraft-style block ids, a 17-voxel
surface shell, pasted "trees", truncated to [gnd_level, sky_level).  Camera poses restate
EvalCameraController patterns 0 and 4 (imaginaire/model_utils/gancraft/camctl.py:9-60,148-178,
296-325).  Everything here is host-side numpy/torch on the CPU and O(scene) or O(frames).
"""
import numpy as np
import torch

BIOME2MC = np.array([28, 9, 8, 1, 9, 8, 9, 8, 30, 26], dtype=np.int32)   # pcg_gen.py:118
SAMPLE_HEIGHT = 256


def _smooth_noise(rs, size, cells):
    """Bilinear upsample of a (cells+1)^2 random lattice to size^2."""
    g = rs.rand(cells + 1, cells + 1).astype(np.float32)
    x = np.linspace(0, cells, size, endpoint=False, dtype=np.float32)
    i = np.floor(x).astype(np.int64)
    f = x - i
    top = g[i][:, i] * (1 - f)[None, :] + g[i][:, i + 1] * f[None, :]
    bot = g[i + 1][:, i] * (1 - f)[None, :] + g[i + 1][:, i + 1] * f[None, :]
    return top * (1 - f)[:, None] + bot * f[:, None]


def make_bev(size=1024, seed=3407):
    """Seeded BEV maps: height in [-0.1, 1), semantic in {0..9} (9 = water), tree_map (255 = none)."""
    rs = np.random.RandomState(seed)
    h = 0.6 * _smooth_noise(rs, size, 16) + 0.3 * _smooth_noise(rs, size, 64) + 0.1 * _smooth_noise(rs, size, 256)
    h = (h - h.min()) / (h.max() - h.min())
    h = (h * 0.42 - 0.04).astype(np.float32)              # up to ~0.38 -> ~100 voxels of relief; <0 = water
    sem = np.floor(_smooth_noise(rs, size, 24) * 8.999).astype(np.uint8)
    sem = np.clip(sem, 0, 8)
    sem[h < 0.0] = 9
    tree = np.full((size, size), 255, dtype=np.uint8)
    m = (rs.rand(size, size) < 0.01) & (sem != 9)
    tree[m] = sem[m]
    return h, sem, tree


def make_tree_models(seed=1):
    """Stand-ins for ckpt['assets']: small trunk(17)+canopy(18) voxel models, int32 [h, x, z]."""
    rs = np.random.RandomState(seed)
    models = []
    for k in range(8):
        th = 5 + k % 4
        m = np.zeros((th + 4, 5, 5), dtype=np.int32)
        m[:th, 2, 2] = 17
        canopy = rs.rand(4, 5, 5) < 0.8
        m[th:th + 4][canopy] = 18
        models.append(m)
    return models


class SyntheticVoxelWorld:
    """Duck-types the attributes of PCGVoxelGenerator the render path and camera controller read:
    voxel_t, heightmap, trans_mat, current_height_map, current_semantic_map, world2local()."""

    def __init__(self, size=1024, seed=3407, device='cpu'):
        self.sample_size = size
        self.sample_height = SAMPLE_HEIGHT
        h, sem, tree = make_bev(size, seed)
        self._build(h, sem, tree, make_tree_models(), seed, device)

    def _build(self, height_map, semantic_map, tree_map, tree_models, seed, device):
        SH = self.sample_height
        height_map = height_map.copy()
        height_map[height_map < 0] = 0
        hi = ((height_map - height_map.min()) / (1 - height_map.min()) * (SH - 1)).astype(np.int16).astype(np.int64)
        X, Z = hi.shape
        world = np.zeros((SH, X, Z), dtype=np.int32)
        lab = BIOME2MC[semantic_map.astype(np.int64)]
        xi, zi = np.meshgrid(np.arange(X), np.arange(Z), indexing='ij')
        world[hi, xi, zi] = lab
        for k in range(16):
            world[np.clip(hi + k + 1, 0, SH - 1), xi, zi] = lab
        hi16 = hi + 16
        rs = np.random.RandomState(seed + 17)
        border = 50
        txs, tzs = np.nonzero(tree_map != 255)
        for x, z in zip(txs, tzs):
            hh = hi16[x, z]
            if x < border or x > X - border or z < border or z > Z - border or hh > SH - border:
                continue
            tm = tree_models[rs.randint(len(tree_models))]
            sl = world[hh:hh + tm.shape[0], x:x + tm.shape[1], z:z + tm.shape[2]]
            mask = sl == 0
            sl[mask] = tm[:sl.shape[0], :sl.shape[1], :sl.shape[2]][mask]
        nz = world != 0
        any_nz = nz.any(axis=0)
        top = SH - 1 - np.argmax(nz[::-1], axis=0)
        top[~any_nz] = 0
        gnd, sky = int(top.min()), int(top.max()) + 1
        self.heightmap = torch.from_numpy(top.astype(np.int64))
        self.gnd_level = gnd
        self.trans_mat = torch.eye(4)
        self.trans_mat[0, 3] += gnd
        self.voxel_t = torch.from_numpy(np.ascontiguousarray(world[gnd:sky])).to(device)
        self.current_height_map = torch.from_numpy((hi16 / (SH - 1)).astype(np.float32))[None, None].to(device)
        sem2 = semantic_map.astype(np.int64).copy()
        sem2[tree_map != 255] = 10
        oh = np.zeros((11, X, Z), dtype=np.float32)
        oh[sem2, xi, zi] = 1.0
        self.current_semantic_map = torch.from_numpy(oh)[None].to(device)

    def world2local(self, v, is_vec=False):
        v = torch.as_tensor(v, dtype=torch.float32)
        if is_vec:
            return v.clone()
        out = v.clone()
        out[0] = out[0] - self.trans_mat[0, 3]
        return out


def _get_height(heightmap, loc0, loc1, minheight):
    loc0, loc1 = int(loc0), int(loc1)
    height = float(minheight)
    for dx in range(-3, 4):
        for dy in range(-3, 4):
            x, y = loc0 + dx, loc1 + dy
            if 0 <= x < heightmap.shape[0] and 0 <= y < heightmap.shape[1]:
                height = max(height, float(heightmap[x, y]) + 2)
    return height


def _filtfilt(hist, decay):
    n = len(hist)
    out, prev = [], hist[0]
    for i in range(n):
        prev = max(prev - decay, hist[i])
        out.append(prev)
    prev = hist[-1]
    for i in range(n - 1, -1, -1):
        prev = max(prev - decay, hist[i])
        out[i] = max(prev, out[i])
    return out


def eval_camera_poses(world, maxstep=40, pattern=0, cam_ang=72.0, smooth_decay_multiplier=None):
    """List of (cam_ori[3], cam_dir[3], cam_up[3], cam_f) float32 CPU tensors / python float."""
    if smooth_decay_multiplier is None:
        smooth_decay_multiplier = 150.0 / maxstep
    vx, vz = world.voxel_t.size(1), world.voxel_t.size(2)
    circle = torch.linspace(0, 2 * np.pi, steps=maxstep)
    size = min(vx, vz) / 2
    shift, size = size * 0.2, size * 0.8
    if pattern == 0:
        move = torch.ones(maxstep)
        far_h, near_scale = 70.0, 0.5
    elif pattern == 4:
        move = torch.linspace(1.0, 0.5, steps=maxstep)
        far_h, near_scale = 90.0, 0.3
    else:
        raise NotImplementedError('only camera patterns 0 and 4 are restated')
    fars = []
    for i in range(maxstep):
        fars.append((torch.sin(circle[i]) * size * move[i] + vx / 2 + shift,
                     torch.cos(circle[i]) * size * move[i] + vz / 2 + shift))
    hist = [_get_height(world.heightmap, fx, fz, far_h) for fx, fz in fars]
    hist = _filtfilt(hist, 0.2 * smooth_decay_multiplier)
    poses = []
    cam_f = 0.5 / np.tan(np.deg2rad(cam_ang / 2))
    for i in range(maxstep):
        far = torch.tensor([hist[i], float(fars[i][0]), float(fars[i][1])], dtype=torch.float32)
        near = torch.tensor([60.0,
                             float(torch.sin(circle[i] + 0.5 * np.pi) * size * near_scale * move[i] + vx / 2 + shift),
                             float(torch.cos(circle[i] + 0.5 * np.pi) * size * near_scale * move[i] + vz / 2 + shift)],
                            dtype=torch.float32)
        poses.append((world.world2local(far), world.world2local(near - far, is_vec=True),
                      world.world2local(torch.tensor([1.0, 0, 0]), is_vec=True), float(cam_f)))
    return poses


def frame_camera(world, pose, resolution_hw=(540, 960), pad=30):
    """Kernel parameters for one frame exactly as inference_givenstyle derives them
    (imaginaire/generators/scenedreamer.py:575-580)."""
    cam_ori, cam_dir, cam_up, cam_f = pose
    cam_res = [resolution_hw[0] + pad, resolution_hw[1] + pad]
    f = cam_f * (resolution_hw[1] - 1)
    c = [(cam_res[0] - 1) / 2, (cam_res[1] - 1) / 2]
    return cam_ori, cam_dir, cam_up, float(f), c, cam_res
