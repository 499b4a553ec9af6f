"""Scene sharding across ranks for the two hot paths (SURVEY.md §8e).

Scenes are independent units (noise -> DDIM -> occupancy grid -> render): rank r takes scenes r, r+W, r+2W, ... exactly like the
reference's `DistributedSampler(shuffle=False)` (lib/datasets/samplers/distributed_sampler.py:53-59, `indices[rank::world]`).
There is no collective on the data path; `gather_scene_outputs` is the eval-side exchange (the reference all-gathers Inception
features inside mmgen's FID.feed; we gather whatever per-scene tensor the caller produced) and works with NCCL or gloo."""
import math
import random

import numpy as np
import torch
import torch.distributed as dist


def scene_indices(num_scenes, rank=None, world_size=None, samples_per_gpu=None):
    """indices of the scenes this rank processes (strided; ragged tails allowed).

    With `samples_per_gpu`, the test loader's order under a distributed launch: mmgen's `DistributedSampler(shuffle=False)`
    [mmgen-memory] gives every rank `ceil(N / W / samples_per_gpu) * samples_per_gpu` indices of the list 0..N-1 padded by repeating
    its head, `indices[rank::W]`, so every rank runs the same number of full batches."""
    if rank is None:
        rank = dist.get_rank() if dist.is_available() and dist.is_initialized() else 0
    if world_size is None:
        world_size = dist.get_world_size() if dist.is_available() and dist.is_initialized() else 1
    if samples_per_gpu is None:
        return list(range(rank, num_scenes, world_size))
    total = int(math.ceil(num_scenes * 1.0 / world_size / samples_per_gpu)) * samples_per_gpu * world_size
    indices = list(range(num_scenes))
    indices += indices[:total - num_scenes]
    if len(indices) != total:        # the padding repeats the head once: the sampler's own assertion
        raise ValueError(f'{num_scenes} scenes cannot fill {world_size} ranks x {total // world_size} samples')
    return indices[rank::world_size]


def train_indices(num_scenes, epoch=0, seed=0, rank=0, world_size=1, samples_per_gpu=1, split_data=False, skip_iter=0):
    """The scene order one rank trains on in epoch `epoch` under a distributed launch: the reference's `DistributedSampler`
    (lib/datasets/samplers/distributed_sampler.py) with `shuffle=True`.  Without `split_data` (or on one rank) the whole list is
    permuted by a `torch.Generator` seeded `seed + epoch`, padded by repeating its head to `ceil(N / W / spg) * spg * W` and strided
    `[rank::W]`.  With `split_data` each rank permutes its own contiguous range `round(linspace(0, N, W + 1))` -- the scenes whose
    latents `SceneCache` keeps on that rank -- padded to the longest range's batches.  The first `skip_iter` indices are dropped (a
    resumed run's position in the epoch)."""
    if split_data and world_size > 1:
        points = np.round(np.linspace(0, num_scenes, num=world_size + 1)).astype(np.int64)
        ranges = [torch.arange(start=int(points[r]), end=int(points[r + 1])) for r in range(world_size)]
        num_samples = int(np.max([np.ceil(len(r) * 1.0 / samples_per_gpu) for r in ranges])) * samples_per_gpu
        g = torch.Generator()
        g.manual_seed(seed + epoch)
        inds = ranges[rank]
        indices = inds[torch.randperm(len(inds), generator=g)].tolist()
        indices += indices[:(num_samples - len(indices))]
    else:
        num_samples = int(math.ceil(num_scenes * 1.0 / world_size / samples_per_gpu)) * samples_per_gpu
        total = num_samples * world_size
        g = torch.Generator()
        g.manual_seed(seed + epoch)
        indices = torch.randperm(num_scenes, generator=g).tolist()
        indices += indices[:(total - len(indices))]
        if len(indices) != total:
            raise ValueError(f'{num_scenes} scenes cannot fill {world_size} ranks x {num_samples} samples')
        indices = indices[rank:total:world_size]
    return indices[skip_iter:]


def disjoint_first_batch(indices, samples_per_gpu, last_batch, rng=random):
    """The reference's `check_batch_disjoint` (lib/datasets/samplers/distributed_sampler.py:71-81) on one epoch's order, so that no
    scene is read in the first batch of an epoch while its latent from the previous epoch's last batch may still be being written:
    raises when the epoch's last two batches share a scene; when its first batch shares a scene with `last_batch` (the previous
    epoch's last batch), the first batch is redrawn by `rng.choices` (python's global generator, as the reference) from the scenes
    past the first two batches that are not in `last_batch`.  Returns (the order, the set of this epoch's last batch)."""
    spg = samples_per_gpu
    indices = list(indices)
    if not set(indices[-2 * spg:-spg]).isdisjoint(indices[-spg:]):
        raise RuntimeError('Batch Disjoint Check Failed! Dataset is too small.')
    if not set(indices[:spg]).isdisjoint(last_batch):
        pool = set(indices[2 * spg:]).difference(last_batch)
        if len(pool) < spg:
            raise RuntimeError('Batch Disjoint Check Failed! Dataset is too small.')
        indices[:spg] = rng.choices(list(pool), k=spg)
    return indices, set(indices[-spg:])


def gather_scene_outputs(local, num_scenes, group=None):
    """local: tensor [n_local, ...] for `scene_indices(num_scenes)` in order -> [num_scenes, ...] on every rank (scene order)."""
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size(group) == 1:
        return local
    world, rank = dist.get_world_size(group), dist.get_rank(group)
    n_max = (num_scenes + world - 1) // world
    pad = local.new_zeros((n_max,) + tuple(local.shape[1:]))
    pad[:local.shape[0]] = local
    bufs = [torch.empty_like(pad) for _ in range(world)]
    dist.all_gather(bufs, pad.contiguous(), group=group)
    out = local.new_zeros((num_scenes,) + tuple(local.shape[1:]))
    for r in range(world):
        idx = scene_indices(num_scenes, r, world)
        out[idx] = bufs[r][:len(idx)]
    return out


# ---------------------------------------------------------------------------------------------------------------------
# view sharding (SURVEY.md §8e, secondary mode): few scenes, many views -- broadcast the scene, shard the views
# ---------------------------------------------------------------------------------------------------------------------
def view_range(num_views, rank=None, world_size=None):
    """contiguous [lo, hi) range of views rendered by this rank (sizes differ by at most one)"""
    if rank is None:
        rank = dist.get_rank() if dist.is_available() and dist.is_initialized() else 0
    if world_size is None:
        world_size = dist.get_world_size() if dist.is_available() and dist.is_initialized() else 1
    return (num_views * rank) // world_size, (num_views * (rank + 1)) // world_size


def max_views_per_rank(num_views, world_size):
    return max(view_range(num_views, r, world_size)[1] - view_range(num_views, r, world_size)[0] for r in range(world_size))


def broadcast_scene(code, density_bitfield, src=0, group=None):
    """rank `src` owns the scene(s): code [B,3,C,H,W] fp32 (1.2 - 6.3 MB per scene) and the occupancy bitfield (32 KB) go to every rank"""
    if dist.is_available() and dist.is_initialized() and dist.get_world_size(group) > 1:
        dist.broadcast(code, src, group=group)
        dist.broadcast(density_bitfield, src, group=group)
    return code, density_bitfield


def gather_views(local_images, num_views, group=None, out=None, padded=None):
    """local_images [v_local, ...] (this rank's `view_range`) -> [num_views, ...] on every rank, view order preserved.
    `padded` / `out`: optional preallocated [v_max, ...] / [world * v_max, ...] buffers (NCCL all_gather_into_tensor needs equal sizes)."""
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size(group) == 1:
        return local_images
    world = dist.get_world_size(group)
    v_max = max_views_per_rank(num_views, world)
    if padded is None:
        padded = local_images.new_zeros((v_max,) + tuple(local_images.shape[1:]))
    padded[:local_images.shape[0]].copy_(local_images)
    if out is None:
        out = local_images.new_empty((world * v_max,) + tuple(local_images.shape[1:]))
    dist.all_gather_into_tensor(out, padded, group=group)
    if num_views == world * v_max:
        return out
    return torch.cat([out[r * v_max: r * v_max + (view_range(num_views, r, world)[1] - view_range(num_views, r, world)[0])] for r in range(world)])
