"""CPU (gloo, world_size 2): host-side logic of the tile-sharded path — ownership partition, halo
sufficiency, and the all-reduce of per-rank normal equations — exercised with the oracle standing in
for the device.  (The device path itself is tests/test_gpu_shard.py.)"""
import os

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from lsdreg import shard, synth
from oracle import eskf
from oracle import oracle as O
from oracle.lio import OracleLio


def test_ownership_is_a_partition_and_halo_covers_the_stencil():
    rng = np.random.default_rng(0)
    cells = rng.integers(-5000, 5000, size=(20000, 3)).astype(np.int32)
    for world in (1, 2, 4, 8):
        own = np.stack([shard.owns(cells, r, world) for r in range(world)])
        assert (own.sum(0) == 1).all()
        for r in range(world):
            rel = shard.relevant(cells, r, world, reach=1)
            assert (rel | ~own[r]).all()                      # owner is always relevant
            # any voxel in the NEARBY18/26 stencil of an owned voxel is relevant to the owner
            for d in ((1, 1), (-1, 0), (0, -1), (1, -1)):
                nb = cells[own[r]].copy(); nb[:, 0] += d[0]; nb[:, 1] += d[1]
                assert shard.relevant(nb, r, world, reach=1).all()
        balance = own.sum(1) / cells.shape[0]
        assert balance.max() < 2.0 / world + 0.05


def _tile_owner_scalar(cx, cy, tile, world):
    """csrc/lsd_common.cuh::tile_owner in Python integers: floor division, 32-bit unsigned hash arithmetic."""
    m = 0xFFFFFFFF
    tx, ty = (cx // tile) & m, (cy // tile) & m
    h = ((tx * 73856093) & m) ^ ((ty * 19349663) & m)
    h ^= h >> 15
    h = (h * 0x2C1B3C6D) & m
    h ^= h >> 12
    return h % world


@pytest.mark.parametrize("reach", [1, 2, 6])
def test_host_mirror_against_brute_force(reach):
    """shard.tile_owner / owns / relevant against their definitions, cell by cell over [-3 tile, 3 tile]^2 (around 0, where
    floor division and truncation differ): relevant(c, r) <=> some voxel within Chebyshev distance `reach` of c in x-y is
    owned by r.  The four-corner test of shard_relevant is only right for tile >= 2 reach + 1 (a tile then spans the whole
    window, so the window's tiles are those of its corners); this is its check at the bound and above it."""
    for tile in (2 * reach + 1, 2 * reach + 2, 3 * reach + 4):
        span = np.arange(-3 * tile, 3 * tile + 1)
        cx, cy = np.meshgrid(span, span, indexing="ij")
        cells = np.stack([cx.ravel(), cy.ravel(), np.zeros(cx.size, np.int64)], 1).astype(np.int32)
        pad = np.arange(-3 * tile - reach, 3 * tile + reach + 1)
        for world in (2, 3, 5):
            own_tab = np.array([[_tile_owner_scalar(int(x), int(y), tile, world) for y in pad] for x in pad])
            got = shard.tile_owner(np.repeat(pad, pad.size), np.tile(pad, pad.size), tile, world).reshape(pad.size, pad.size)
            assert np.array_equal(got, own_tab), (tile, world)
            o = reach                                        # index of span[0] in pad is reach
            for r in range(world):
                mine = own_tab == r
                # brute force: any owned cell in the (2 reach + 1)^2 window
                win = np.zeros((span.size, span.size), bool)
                for dx in range(-reach, reach + 1):
                    for dy in range(-reach, reach + 1):
                        win |= mine[o + dx:o + dx + span.size, o + dy:o + dy + span.size]
                rel = shard.relevant(cells, r, world, tile, reach).reshape(span.size, span.size)
                assert np.array_equal(rel, win), (tile, world, r, np.argwhere(rel != win)[:4])
                assert np.array_equal(shard.owns(cells, r, world, tile).reshape(span.size, span.size), mine[o:-o, o:-o])
            # every cell owned by exactly one rank; negative tiles differ from the positive ones they would truncate to
            assert (sum((own_tab == r).astype(int) for r in range(world)) == 1).all()
        assert any(_tile_owner_scalar(-1, 0, tile, w) != _tile_owner_scalar(0, 0, tile, w) for w in (2, 3, 5))


def test_exact_search_reach():
    """The halo the exact search needs: its last shell ceil(sqrt(max_sq) / res) + 1 (csrc/knn.cuh::knn_exact_warp)."""
    assert shard.exact_reach(0.5) == 6 and shard.exact_reach(1.0) == 4 and shard.exact_reach(0.25) == 10
    assert shard.reach_for(shard.STENCIL_EXACT, 0.5) == 6
    assert [shard.reach_for(s) for s in (0, 6, 18, 26, 74)] == [1, 1, 1, 1, 2]


def _worker(rank, world, port, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    m = synth.block_map(1, 1, 1, 0.5)
    Rgt = synth.rot_from_rpy(0.01, -0.02, 0.3)
    tgt = synth.block_center(0, 0) + np.array([1.0, -2.0, 0.0])
    scan = synth.scan64(2, 120, Rgt, tgt)
    body = O.voxelgrid(scan, 0.5)
    st = eskf.State(); st.rot = eskf.R_to_quat(Rgt); st.pos = tgt + np.array([0.05, -0.03, 0.01])
    # this rank's shard: the relevant map points, the owned queries
    mcells = shard.cell_of(m[:, :3])
    keep = shard.relevant(mcells, rank, world)
    lio = OracleLio(18, expected_cells=1 << 16)
    lio.map.add(np.ascontiguousarray(m[keep, :3]), 0)
    ids = np.nonzero(keep)[0].astype(np.int32)          # keep the global ids
    R = eskf.quat_to_R(st.rot)
    w = (body[:, :3].astype(np.float64) @ R.T + st.pos).astype(np.float32)
    mine = shard.owns(shard.cell_of(w), rank, world)
    n = int(mine.sum())
    lio.near_xyz = np.zeros((n, 5, 3), np.float32); lio.near_ids = np.full((n, 5), -1, np.int32)
    lio.near_cnt = np.zeros(n, np.int32); lio.selected = np.ones(n, np.uint8)
    lio.world = np.zeros((n, 4), np.float32); lio.plane = np.zeros((n, 4), np.float32)
    lio.degenerate_detect = False
    lio._hmodel(np.ascontiguousarray(body[mine]), st, True)
    part = torch.from_numpy(np.concatenate([lio.last["HTH6"].ravel(), lio.last["HTh6"], [lio.last["res_sum"], lio.last["n_eff"]]]))
    dist.all_reduce(part)                                  # the collective of SURVEY.md §8e
    if rank == 0:
        full = OracleLio(18, expected_cells=1 << 16)
        full.map.add(np.ascontiguousarray(m[:, :3]), 0)
        nb = body.shape[0]
        full.near_xyz = np.zeros((nb, 5, 3), np.float32); full.near_ids = np.full((nb, 5), -1, np.int32)
        full.near_cnt = np.zeros(nb, np.int32); full.selected = np.ones(nb, np.uint8)
        full.world = np.zeros((nb, 4), np.float32); full.plane = np.zeros((nb, 4), np.float32)
        full.degenerate_detect = False
        full._hmodel(body, st, True)
        ref = np.concatenate([full.last["HTH6"].ravel(), full.last["HTh6"], [full.last["res_sum"], full.last["n_eff"]]])
        q.put((part.numpy(), ref))
    dist.barrier()
    dist.destroy_process_group()


def test_sharded_normal_equations_allreduce_gloo():
    world = 2
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 29600 + os.getpid() % 300
    procs = [ctx.Process(target=_worker, args=(r, world, port, q)) for r in range(world)]
    [p.start() for p in procs]
    got, ref = q.get(timeout=240)
    [p.join(timeout=60) for p in procs]
    assert all(p.exitcode == 0 for p in procs)
    assert got[-1] == ref[-1] and got[-1] > 500              # same number of effective points
    np.testing.assert_allclose(got, ref, rtol=1e-10, atol=1e-9)
