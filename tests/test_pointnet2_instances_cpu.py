"""The PointNet++ GPU tests' case lists reach every FPS instance and cluster width, and every tile, capacity and
channel-split edge of ball query, grouping and interpolation.

tests/pointnet2_instances.py restates the launchers' rules; this maps the case lists of test_pointnet2_edges_gpu.py
through them.  Adding an FPS instance or moving a threshold in csrc/pointnet2_kernels.cu without a GPU case that runs it
fails here, without a GPU."""
import numpy as np

import pointnet2_instances as pi
import test_pointnet2_edges_gpu as edges


def test_restated_rules_on_known_shapes():
    assert pi.fps_instances() == (1, 2, 3, 4, 5, 6, 8, 10, 12, 16)
    assert pi.fps_path(20000) == (5, 8)              # the pre-encoder's 20 000 points
    assert pi.fps_path(40000) == (10, 8)             # the ScanNet shape
    assert pi.fps_path(2048) == (4, 1)               # the query sampling
    assert pi.fps_path(6144, 1) == (12, 1) and pi.fps_path(6145, 1) == (16, 1)
    assert pi.fps_path(65536) == (16, 8) and pi.fps_path(65537) == "generic"
    assert pi.fps_path(8193, 1) == (3, 8)            # forced width 1 widened
    assert pi.fps_path(37, 8) == (1, 8)              # block size 32: 64 positions on an 8-CTA cluster
    assert pi.bq_max_nsample() == 5632
    assert pi.bq_tiles(2048) == 1 and pi.bq_tiles(2049) == 2
    assert pi.c_per_block(259, 700, 2) == 2 and pi.ragged_last_slice(259, 700, 2)
    assert pi.c_per_block(256, 1024 * 32, 8) == 128 and not pi.ragged_last_slice(256, 1024 * 32, 8)


def test_fps_cases_reach_every_cell():
    paths = [(c, pi.fps_path(c[1], c[3])) for c in edges.FPS_CASES]
    grid = {(inst, w) for inst in pi.fps_instances() for w in pi.FPS_WIDTHS}
    reached = {p for _, p in paths}
    assert grid <= reached, f"cells no GPU case runs: {sorted(grid - reached)}"
    assert "generic" in reached
    auto = {c[1]: p for c, p in paths if c[3] == 0}
    assert auto.get(4096) == (8, 1) and auto.get(4097) == (2, 8)           # the automatic width switch
    assert auto.get(65536) == (16, 8) and auto.get(65537) == "generic"     # the generic kernel's boundary
    for forced in (1, 2):                                                   # a forced width widened to 8
        assert any(c[3] == forced and p != "generic" and p[1] == 8 for c, p in paths)
    cluster = [c for c, p in paths if p != "generic" and p[1] > 1]
    assert {1, 2, 3, 4} <= {c[2] for c in cluster}                          # rounds around the barrier re-arm
    assert any(c[2] > c[1] for c in cluster)                                # m > n on a cluster
    assert any(c[2] > c[1] for c, p in paths if p != "generic" and p[1] == 1)


def test_threshold_points_straddle_the_skip():
    below, above = edges.threshold_points()
    for lo, hi in zip(below, above):
        assert edges.fps_square_norm(*lo) == edges.MAG_BELOW and float(edges.MAG_BELOW) <= 1e-3
        assert edges.fps_square_norm(*hi) == edges.MAG_ABOVE and float(edges.MAG_ABOVE) > 1e-3
        # one ulp of y apart, and the fp32 value of 1e-3 itself is kept: only an fp64 comparison gets both right
        assert lo[0] == hi[0] and lo[2] == hi[2] and np.nextafter(lo[1], np.float32(1)) == hi[1]
        assert edges.MAG_ABOVE == np.float32(1e-3)


def test_ball_query_cases_reach_every_edge():
    cases = edges.BQ_CASES
    tiles = {pi.bq_tiles(c[1]) for c in cases}
    assert {1, 2} <= tiles and max(tiles) > 2
    assert {2047, 2048, 2049, 4097} <= {c[1] for c in cases}                # either side of the tile boundaries
    assert {1, 31, 33, pi.bq_max_nsample()} <= {c[4] for c in cases}
    assert any(c[4] > 32 * 4 for c in cases)                                # several output passes per lane
    assert any(c[2] % pi.BQ_WARPS for c in cases)                           # idle warps in the last CTA
    assert any(c[5] >= 1000.0 for c in cases)                               # far from the origin


def test_group_and_interpolate_cases_reach_a_ragged_channel_slice():
    group = edges.GROUP_CASES
    for c in (1, 3, 5, 259):
        assert any(g[1] == c for g in group)
    ragged = {g[1] for g in group if pi.ragged_last_slice(g[1], g[3] * g[4], g[0])}
    assert {3, 5, 259} <= ragged
    assert any(g[3] * g[4] % 256 for g in group)                            # a partial last CTA of elements
    assert (8, 256, 2048, 1024, 32, "ball") in group                        # the masked encoder's grouping
    assert {"ball", "one"} <= {g[5] for g in group}
    interp = edges.INTERP_CASES
    assert {3, 5, 259} <= {i[1] for i in interp if pi.ragged_last_slice(i[1], i[2], i[0])}
    assert any(i[2] % 256 for i in interp)


def test_three_nn_cases_reach_every_known_set_edge():
    assert {0, 1, 2, 3, 1023, 1024, 1025, 2049} <= {c[2] for c in edges.NN_CASES}
    assert any(c[1] % 256 for c in edges.NN_CASES)                          # idle threads in the last CTA
