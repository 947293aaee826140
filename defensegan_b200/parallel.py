"""Multi-GPU projection: shard the IMAGE axis across ranks, one all-gather at the end.

Every latent row is independent inside the loop and only the final arg-min couples the R rows
of one image (reference models/gan.py:438-449), so rank g takes images
[bounds[g], bounds[g+1]) together with all of their restarts (rows stay contiguous: image-major
layout, models/gan.py:355-359) and the arg-min is rank-local.  There is no per-step
communication; the only collective is one all-gather of the [B/G, H, W, C] reconstructions
(SURVEY section 8e).  The select kernel writes each rank's result directly into its slot of the
gather buffer, so the collective needs no staging copy.  With use_bn=True the batch statistics
couple all rows (SURVEY F2) and sharding would change results: refused.
"""
from __future__ import annotations

from typing import Callable, List, Optional, Tuple

import torch
import torch.distributed as dist


def shard_bounds(n_images: int, world_size: int) -> List[int]:
    """Contiguous, balanced split: the first (n % world) ranks get one extra image."""
    base, extra = divmod(int(n_images), int(world_size))
    bounds = [0]
    for r in range(world_size):
        bounds.append(bounds[-1] + base + (1 if r < extra else 0))
    return bounds


def sharded_apply(local_fn: Callable, images: torch.Tensor, rec_rr: int, z_init_val: Optional[torch.Tensor] = None,
                  group=None, pixel_weights: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Run `local_fn(images_shard, z0_shard, out_view, first_image)` on this rank's shard and all-gather.

    `local_fn` must write its [b_local, ...] result into `out_view` (a view of the gather
    buffer).  `images` (and `z_init_val` [B*rec_rr, latent]) hold the FULL batch on every rank.
    With `pixel_weights` (anything that broadcasts to the images' shape) the shard's weights are sliced with its images
    and passed as `local_fn(..., pixel_weights=weights_shard)`.
    Returns the full [B, ...] result on every rank.
    """
    world = dist.get_world_size(group) if dist.is_initialized() else 1
    rank = dist.get_rank(group) if dist.is_initialized() else 0
    n = images.shape[0]
    bounds = shard_bounds(n, world)
    lo, hi = bounds[rank], bounds[rank + 1]
    per = max(bounds[i + 1] - bounds[i] for i in range(world))      # slot size (ragged tail padded)
    row = images[0].numel()
    gather = torch.empty((world, per) + tuple(images.shape[1:]), dtype=images.dtype, device=images.device)
    if hi <= lo and hasattr(local_fn, "skip"):
        local_fn.skip()
    if hi > lo:
        z0 = None
        if z_init_val is not None:
            z0 = z_init_val.reshape(n * rec_rr, -1)[lo * rec_rr:hi * rec_rr]
        if pixel_weights is None:
            local_fn(images[lo:hi], z0, gather[rank, :hi - lo], lo)
        else:
            pw = torch.broadcast_to(torch.as_tensor(pixel_weights, device=images.device), images.shape)
            local_fn(images[lo:hi], z0, gather[rank, :hi - lo], lo, pixel_weights=pw[lo:hi])
    if hi - lo < per:
        gather[rank, hi - lo:].zero_()
    if world > 1:
        # in place: this rank's slot of `gather` is the send buffer
        dist.all_gather_into_tensor(gather.view(world * per, row), gather[rank].reshape(per, row), group=group)
    out = torch.cat([gather[r, :bounds[r + 1] - bounds[r]] for r in range(world)], dim=0) if per * world != n \
        else gather.reshape((n,) + tuple(images.shape[1:]))
    return out


def reconstruct_sharded(gan, images: torch.Tensor, z_init_val: Optional[torch.Tensor] = None, group=None,
                        pixel_weights: Optional[torch.Tensor] = None) -> torch.Tensor:
    """gan.reconstruct over all ranks of `group` (NCCL): identical to the single-GPU result
    row for row (no BatchNorm), with `z_init_val` given or drawn (the shards index one common z0 stream).
    `pixel_weights` (see DefenseGANBase.reconstruct) are sliced with the images.
    Ranks with an empty shard still advance the call counter so that later calls stay in step."""
    if bool(gan.use_bn):
        raise RuntimeError("use_bn=True couples all latent rows through batch statistics (SURVEY F2); "
                           "sharding the batch would change the result - run replicas instead")
    if getattr(gan, "rec_sparse_dev", None) is not None:
        raise RuntimeError("rec_sparse_dev is set: the projection with sparse deviations runs on one GPU only; call "
                           "gan.reconstruct per device, or set rec_sparse_dev = None to shard")

    # every rank advances the model's call counter identically, so all shards draw from ONE Philox stream; the shard's
    # first row in that stream is (first image) * rec_rr: row for row the single-GPU draw
    if pixel_weights is not None:       # checked on the full batch, so every rank raises before any collective
        pixel_weights = gan._pixel_weights(pixel_weights, images)

    def local_fn(x, z0, out_view, first_image, **kw):
        gan.reconstruct(x, z_init_val=z0, out=out_view, z_row_offset=first_image * int(gan.rec_rr), **kw)

    local_fn.skip = gan._next_seed      # a rank without images must still consume this call's seed
    return sharded_apply(local_fn, images, int(gan.rec_rr), z_init_val=z_init_val, group=group, pixel_weights=pixel_weights)
