"""lsdreg — H100-native registration hot path for LSD (lidar-slam-detection).

Import as ``import lsdreg`` (alias module at the repo root; the directory name carries a hyphen).
The compute path is liblsdreg.so (hand-written sm_90a CUDA behind a C ABI, include/lsdreg.h);
this package is its thin host-side mirror.  See DESIGN.md / INTEGRATION.md.
"""
from . import shard, synth  # noqa: F401
from .capi import (  # noqa: F401
    ERR_CAPACITY, ERR_CUDA, ERR_GRID_OVERFLOW, ERR_INVALID, ERR_NO_DEVICE, MAP_SEEDED, NO_EFFECTIVE_POINTS, OK,
    SCAN_TOO_SMALL, MAP_SATURATED, STENCIL_CENTER, STENCIL_EXACT, STENCIL_NEARBY6, STENCIL_NEARBY18, STENCIL_NEARBY26,
    STENCIL_NEARBY74, HashVoxelMap, Matcher, Voxelizer, eskf_update_table, LioFrontend, LsdError, VoxelGrid, init, init_cov, lib, make_state,
    state_boxminus, state_boxplus, ImuProcess, eskf_predict, IMU_INITIALIZING, keyframe_filter, LocalMap, LOCALMAP_NONE, keyframe_save, keyframe_load, ERR_IO, ScanContext, FastLio,
    LoopDetector, find_loop_candidates, loop_information_matrix, LOOP_SKIPPED, LOOP_NO_CANDIDATES, LOOP_COARSE_REJECT,
    LOOP_GICP_DIVERGED, LOOP_GICP_REJECT, LOOP_FOUND, GlobalAligner, galign_merge_candidates,
    OverlapDetector, overlap_find_candidates, overlap_guess, overlap_finetune_guess, OVERLAP_NO_CANDIDATES, OVERLAP_NO_MATCH,
    OVERLAP_GICP_DIVERGED, OVERLAP_GICP_REJECT, OVERLAP_FOUND,
    FloorDetector, ransac_replay, FLOOR_MAPPING, FLOOR_GROUND, FLOOR_RENDER, FLOOR_FOUND, FLOOR_EMPTY, FLOOR_FEW_CANDIDATES,
    FLOOR_NO_MODEL, FLOOR_FEW_INLIERS, FLOOR_NOT_VERTICAL)
from . import capi  # noqa: F401
