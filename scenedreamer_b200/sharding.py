"""Multi-GPU sharding of the render path.

Rays are independent given replicated read-only state (voxel volume, hash table, MLP weights), so
frames shard across ranks with NO data-path collective; the single collective of the path is one
all-gather of the finished per-frame maps.  One process per GPU (torch.distributed, NCCL on GPUs,
gloo in the CPU tests).
"""
import torch
import torch.distributed as dist


def frames_for_rank(n_frames, rank, world_size):
    """Frame f is rendered by rank f mod world_size (round-robin keeps camera-path neighbours apart,
    which balances sky-heavy and ground-heavy frames)."""
    return list(range(rank, n_frames, world_size))


def frame_owner(frame, world_size):
    return frame % world_size


def gather_frames(local, group=None):
    """local: [n_local, ...] finished maps of this rank's frames (same n_local on every rank; pad the
    last round with a repeat if n_frames % world_size != 0).  Returns [world_size * n_local, ...]
    ordered by global frame index f = i * world_size + rank."""
    world = dist.get_world_size(group) if dist.is_initialized() else 1
    if world == 1:
        return local
    n_local = local.shape[0]
    out = torch.empty((world * n_local,) + tuple(local.shape[1:]), dtype=local.dtype, device=local.device)
    dist.all_gather_into_tensor(out, local.contiguous(), group=group)      # rank-major concatenation along dim 0
    out = out.view((world, n_local) + tuple(local.shape[1:]))
    # out[r, i] is frame i * world + r  ->  interleave ranks
    return out.transpose(0, 1).reshape((world * n_local,) + tuple(local.shape[1:]))


def cyclic_bands(H, rank, world_size, band_tiles=2, tile_h=8):
    """Single-frame sharding, balanced without knowing the cost profile: the frame is cut into thin bands of `band_tiles`
    tile rows and band b goes to rank b mod world_size.  (The cost of a row is neither flat nor monotonic -- sky at the top
    is free, near ground at the bottom terminates within a few samples, the horizon in the middle is the expensive part -- so
    one contiguous band per rank, or a band paired with its mirror, leave some ranks idle.  The band height of 2 tile rows was
    chosen on an 8-GPU box of the previous GPU generation and is carried over untested on H100.)
    Returns the rank's bands as (y0, y1) in frame order; every rank gets the same NUMBER of slots, trailing ones may be empty."""
    bh = band_tiles * tile_h if world_size > 1 else H          # one GPU: the frame is one band
    n_bands = (H + bh - 1) // bh
    per_rank = (n_bands + world_size - 1) // world_size
    out = []
    for j in range(per_rank):
        b = j * world_size + rank
        y0 = min(H, b * bh)
        out.append((y0, min(H, y0 + bh)))
    return out



def band_spec(bands):
    """(first_row, band_rows, band_stride, total_rows) of a rank's non-empty bands for the banded raycast
    (ops.ray_voxel_intersection_perspective(..., band=...)): equally spaced bands of equal height, only the last may be shorter."""
    bands = [b for b in bands if b[1] > b[0]]
    if not bands:
        raise ValueError('no rows for this rank')
    bh = bands[0][1] - bands[0][0]
    stride = (bands[1][0] - bands[0][0]) if len(bands) > 1 else bh
    if any(b[0] != bands[0][0] + k * stride for k, b in enumerate(bands)) or any(b[1] - b[0] != bh for b in bands[:-1]) or \
            bands[-1][1] - bands[-1][0] > bh or stride < bh:
        raise ValueError('bands are not equally spaced / equally high: %r' % (bands,))
    return bands[0][0], bh, stride, sum(b[1] - b[0] for b in bands)


def assemble_bands(gathered, world_size, n_slots, band_rows):
    """Inverse of cyclic_bands after the all-gather: `gathered` [world_size, C, n_slots * band_rows, W] holds, for every rank, its band
    slots one after the other (slot j of rank r = band j * world_size + r, short / missing bands zero-padded to band_rows);
    returns [C, n_slots * world_size * band_rows, W] in frame order (rows beyond the frame height are the padding)."""
    C, W = gathered.shape[1], gathered.shape[-1]
    a = gathered.reshape(world_size, C, n_slots, band_rows, W)
    return a.permute(1, 2, 0, 3, 4).reshape(C, n_slots * world_size * band_rows, W)


def global_mean(band_means, group=None):
    """Frame-global mean of a per-ray quantity from per-band means: `band_means` = [(mean [C] or [1, C], number of rays)] of THIS
    rank's bands; one all-gather of C + 1 floats per rank (the band sums and the ray count), combined in rank order on every rank.
    Single-frame sharding needs it for the sky features: the reference averages them over the WHOLE frame (scenedreamer.py:592-598).
    Returns [1, C]."""
    first = band_means[0][0]
    C = first.numel()
    part = torch.zeros(C + 1, dtype=torch.float32, device=first.device)
    for mean_band, n_band in band_means:
        part[:C] += mean_band.reshape(C).to(torch.float32) * float(n_band)
        part[C] += float(n_band)
    world = dist.get_world_size(group) if dist.is_available() and dist.is_initialized() else 1
    if world == 1:
        return (part[:C] / part[C]).reshape(1, C)
    allp = torch.empty(world, C + 1, dtype=torch.float32, device=first.device)
    dist.all_gather_into_tensor(allp, part.reshape(1, C + 1), group=group)
    return (allp[:, :C].sum(0) / allp[:, C].sum()).reshape(1, C)
