"""CPU side of the device data layer: the numpy restatement (oracle/data_ref.py) is pinned to the REFERENCE's own
RandomCuboid (utils/random_cuboid.py) fed the same random draws, and its sampler is checked for the properties
np.random.choice guarantees (distinct rows, inside the crop, uniform)."""
from pathlib import Path

import numpy as np
import pytest

import data_ref
from coda_neurips2023_b200 import synthetic

GOLDEN = Path(__file__).resolve().parent / "golden" / "random_cuboid_ref.npz"
CASES = [(0, 1500), (1, 3000), (2, 5900), (3, 100)]


def scene(seed, n=6000, g=7):
    rng = np.random.default_rng(seed)
    pts = synthetic.point_clouds(1, n, seed=seed)[0].astype(np.float32)
    boxes = np.zeros((g, 8), np.float32)
    boxes[:, 0:3] = rng.uniform(synthetic.ROOM_MIN + 0.5, synthetic.ROOM_MAX - 0.5, size=(g, 3))
    boxes[:, 3:6] = rng.uniform(0.2, 1.0, size=(g, 3))
    boxes[:, 6] = rng.uniform(-3, 3, size=g)
    boxes[:, 7] = rng.integers(0, 10, size=g)
    return pts, boxes


def replay_table(seed, ncand=100):
    """the candidate crops both sides draw from: crop ranges and centre draws of `ncand` attempts"""
    rng = np.random.default_rng(100 + seed)
    crop_range = 0.5 + rng.random((ncand, 3)) * 0.5
    center_u = rng.random(ncand).astype(np.float32)
    return crop_range, center_u


@pytest.mark.parametrize("seed,min_points", CASES)
def test_random_cuboid_restatement_equals_reference_with_replayed_draws(seed, min_points):
    """utils/random_cuboid.py draws np.random.rand(3) per attempt and np.random.choice(n) when the aspect test
    passes; replaying a table through both gives the same crop, the same kept points and the same kept boxes.  The
    reference's side of the comparison is stored in tests/golden/random_cuboid_ref.npz
    (tests/golden/make_random_cuboid_golden.py)."""
    golden = np.load(GOLDEN)
    ref_pts, ref_boxes = golden[f"pts_{seed}_{min_points}"], golden[f"boxes_{seed}_{min_points}"]
    pts, boxes = scene(seed)
    crop_range, center_u = replay_table(seed)
    chosen, crop, keep = data_ref.random_cuboid(pts, boxes, crop_range, center_u, min_points, aspect=0.8)
    inside = np.all(pts[:, :3].astype(np.float64) <= crop[3:], axis=1) & np.all(pts[:, :3].astype(np.float64) >= crop[:3], axis=1)
    assert np.array_equal(pts[inside], ref_pts)
    assert np.array_equal(boxes[keep], ref_boxes)
    if min_points >= 5900:
        assert chosen == -1 and len(ref_pts) == len(pts)        # no crop keeps that many points: fallback
    else:
        assert chosen >= 0 and 0 < len(ref_pts) < len(pts)


def test_feistel_sampler_draws_distinct_rows_uniformly():
    pts, _ = scene(5, n=5000)
    crop = np.array([-2.0, 0.8, -1.1, 2.5, 5.0, 1.2])
    inside = np.all(pts[:, :3] <= crop[3:], axis=1) & np.all(pts[:, :3] >= crop[:3], axis=1)
    m = int(inside.sum())
    assert m > 1500
    out, choice, count, dims = data_ref.sample_points(pts, crop, seed=1234, nsample=1000)
    assert count == m and len(np.unique(choice)) == 1000 and inside[choice].all()
    assert np.array_equal(out, pts[choice]) and np.array_equal(dims[:3], out[:, :3].min(0))
    # every row of the crop is equally likely: pool many seeds, compare hit counts with the binomial spread
    hits = np.zeros(len(pts))
    for seed in range(300):
        hits[data_ref.sample_points(pts, crop, seed=seed * 7919 + 1, nsample=1000)[1]] += 1
    p = 1000 / m
    z = (hits[inside] - 300 * p) / np.sqrt(300 * p * (1 - p))
    assert abs(z.mean()) < 0.1 and 0.85 < z.std() < 1.15 and np.abs(z).max() < 6
    # fewer points than samples: draws with replacement cover the crop
    out2, choice2, count2, _ = data_ref.sample_points(pts, crop, seed=9, nsample=4 * m)
    assert count2 == m and inside[choice2].all() and len(np.unique(choice2)) > 0.95 * m


def test_scene_transform_is_the_reference_formula_in_float32():
    pts, _ = scene(7, n=2000)
    ang = 0.3
    rot = np.array([[np.cos(ang), -np.sin(ang), 0], [np.sin(ang), np.cos(ang), 0], [0, 0, 1.0]])
    got = data_ref.scene_transform(pts, -1.0, rot, 1.1)
    ref = pts.astype(np.float64).copy()
    ref[:, 0] *= -1
    ref[:, 0:3] = np.dot(ref[:, 0:3], rot.T) * 1.1               # datasets/...:663-700
    assert np.abs(got[:, :3] - ref[:, :3]).max() < 2e-6
