"""Tile sharding of the map across the GPUs of one box (SURVEY.md §8e) — host-side helpers.

`tile_owner` mirrors csrc/lsd_common.cuh::tile_owner bit for bit (tests check it against the device
through the map statistics).  `connect` performs the handle exchange of include/lsdreg.h
"Tile-sharded LIO" over a torch.distributed process group (nccl or gloo).
"""
from __future__ import annotations

import numpy as np

TILE_CELLS = 32   # 16 m tiles at 0.5 m voxels: ~40 tiles per 120 x 80 m block, 13 % halo at reach 1
REACH = {0: 1, 6: 1, 18: 1, 26: 1, 74: 2}   # iVox stencil -> halo (voxels) its search needs; the exact search: exact_reach
STENCIL_EXACT = 1000


def exact_reach(res: float = 0.5, max_sq: float = 5.0) -> int:
    """Halo (voxels) the exact search needs: its last shell, ceil(sqrt(max_sq) / res) + 1, in the device's fp32 (6 at 0.5 m)."""
    inv = np.float32(1.0 / np.float64(np.float32(res)))
    return int(np.ceil(np.sqrt(np.float32(max_sq)) * inv)) + 1


def reach_for(stencil: int, res: float = 0.5) -> int:
    """reach_cells to export for a handle searching with `stencil` (STENCIL_EXACT for knn_mode_exact = 1)."""
    return exact_reach(res) if stencil == STENCIL_EXACT else REACH[stencil]


def cell_of(xyz: np.ndarray, res: float = 0.5) -> np.ndarray:
    """Pos2Grid (ivox3d.h:258-261): round-half-away-from-zero of p * inv_res in fp32."""
    inv = np.float32(1.0 / res)
    v = xyz.astype(np.float32) * inv
    return (np.sign(v) * np.floor(np.abs(v) + np.float32(0.5))).astype(np.int32)


def tile_owner(cx: np.ndarray, cy: np.ndarray, tile: int, world: int) -> np.ndarray:
    tx = np.floor_divide(cx.astype(np.int64), tile).astype(np.uint32)
    ty = np.floor_divide(cy.astype(np.int64), tile).astype(np.uint32)
    with np.errstate(over="ignore"):
        h = (tx * np.uint32(73856093)) ^ (ty * np.uint32(19349663))
        h ^= h >> np.uint32(15)
        h = h * np.uint32(0x2c1b3c6d)
        h ^= h >> np.uint32(12)
    return (h % np.uint32(world)).astype(np.int32)


def owns(cells: np.ndarray, rank: int, world: int, tile: int = TILE_CELLS) -> np.ndarray:
    return tile_owner(cells[:, 0], cells[:, 1], tile, world) == rank


def relevant(cells: np.ndarray, rank: int, world: int, tile: int = TILE_CELLS, reach: int = 1) -> np.ndarray:
    r = np.zeros(cells.shape[0], bool)
    for dx in (-reach, reach):
        for dy in (-reach, reach):
            r |= tile_owner(cells[:, 0] + dx, cells[:, 1] + dy, tile, world) == rank
    return r


def connect(lio, rank: int, world: int, group=None, tile_cells: int = TILE_CELLS, reach_cells: int = 1):
    """Exchange the shard blobs over torch.distributed and connect `lio` to its peers.

    reach_cells must cover the handle's search: `reach_for(ivox_nearby)` — 1 for NEARBY6/18/26, 2 for NEARBY74 — or
    `exact_reach(ivox_resolution)` with knn_mode_exact = 1, and tile_cells must exceed 2 * reach_cells.  The export refuses
    a narrower halo (LsdError), as does a later set_nearby to a wider stencil."""
    import torch
    import torch.distributed as dist
    blob = lio.shard_export(rank, world, tile_cells, reach_cells)
    if world == 1:
        lio.shard_connect(blob[None])
        return
    backend = dist.get_backend(group)
    t = torch.from_numpy(blob)
    if backend == "nccl":
        t = t.cuda()
    out = [torch.empty_like(t) for _ in range(world)]
    dist.all_gather(out, t, group=group)
    lio.shard_connect(np.stack([o.cpu().numpy() for o in out]))
