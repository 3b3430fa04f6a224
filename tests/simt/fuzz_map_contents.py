# The hash-voxel map's contents voxel by voxel (lsd_map_dump) against the restatement of IVox::AddPoints (and the compiled
# iVox when it is built), under the SIMT emulator: plain insert, box delete, and every map-level LRU path — re-creation of
# evicted voxels with more than 8 survivors, capacity 1, max_distance 0, table rebuilds, eviction of a voxel with tombstones.
import test_gpu_map_contents as T

T.test_crowded_voxel_negative_coordinates_and_half_boundaries()
T.test_box_delete_contents()
T.test_lru_out_and_back()
T.test_lru_recreated_voxel_keeps_all_its_points()
T.test_lru_voxel_evicted_and_recreated_repeatedly()
for cap, dist in ((1, 0.0), (1, 2.5), (40, 0.0)):
    T.test_lru_small_capacity_and_zero_distance(cap, dist)
T.test_lru_across_table_rebuilds()
T.test_lru_evicts_a_voxel_with_tombstones()
T.test_overfull_voxel_drops_exactly_the_excess()
T.test_points_outside_the_key_range_are_dropped()
print("FUZZ_MAP_CONTENTS_OK")
