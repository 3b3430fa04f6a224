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
    state_boxminus, state_boxplus, ImuProcess, eskf_predict, IMU_INITIALIZING, keyframe_filter, LocalMap, LOCALMAP_NONE, keyframe_save, keyframe_load, ERR_IO, ScanContext, FastLio)
from . import capi  # noqa: F401
