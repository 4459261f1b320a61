"""ScanNet runs without a GPU: OUR model + criterion (CUDA ops replaced by the CPU restatement, ScanNet camera from
tests/scannet_ref.py) against the reference's goldens of the ScanNet cases, the class prompts against the reference's
own list, the ScanNet camera of the synthetic batches, and the shape check of ops.boxes_in_image."""
import json
import shutil

import numpy as np
import pytest
import torch

import model_parity_common as mpc
import scannet_parity_common as spc
import scannet_ref
from coda_neurips2023_b200 import ops, synthetic
from coda_neurips2023_b200.models import model_3detr

GOLDEN = mpc.GOLDEN


@pytest.mark.parametrize("name", list(spc.CASES))
def test_scannet_model_and_criterion_match_reference_on_cpu(name):
    """Same bars as test_model_cpu.py: 2e-4 relative forward / loss, gradients 10 x that (1e-2 at full size)."""
    torch.manual_seed(0)
    with scannet_ref.installed():
        model, out, loss, loss_dict, golden = spc.run(name, "cpu")
        errs = mpc.compare(model, out, loss, loss_dict, golden, rtol=2e-4, atol=1e-5,
                           grad_rtol=1e-2 if name in spc.FULL_SIZE else None)
    assert "pseudo.count" not in golden.files or int(golden["pseudo.count"].sum()) > 0
    worst = max(errs, key=errs.get)
    print(f"{name}: worst {worst} = {errs[worst]:.2e}")


@pytest.fixture
def coda_checkout(tmp_path, monkeypatch):
    """A working directory laid out like a CoDA checkout: datasets/ holds the two ScanNet class files."""
    (tmp_path / "datasets").mkdir()
    for f in (model_3detr.SCANNET_CLASS_NAMES_PATH, model_3detr.SCANNET_CLASS_IDS_PATH):
        shutil.copyfile(GOLDEN / f.split("/")[-1], tmp_path / f)
    monkeypatch.chdir(tmp_path)
    return tmp_path


@pytest.mark.parametrize("flags", ["stage1", "stage2", "seen_only"])
def test_scannet_prompts_equal_the_reference_list(coda_checkout, flags):
    golden = json.loads((GOLDEN / "scannet_prompts.json").read_text())
    args = synthetic.make_args(**golden["flags"][flags])
    assert model_3detr._class_prompts(args) == golden[flags]


def test_scannet_prompts_follow_the_range_lists(coda_checkout):
    args = synthetic.make_args(dataset_name="scannet_anonymous_aligned_image", train_range_list=[4, 2],
                               test_range_list=[2, 1191, 5, 6], reset_scannet_num=2, if_clip_more_prompts=True)
    assert model_3detr._class_prompts(args) == [f"a photo of a {c} in the scene" for c in
                                                ("chair", "table", "door", "mattress")]
    args.if_clip_more_prompts = False
    assert model_3detr._class_prompts(args) == ["a photo of a table in the scene", "a photo of a chair in the scene"]


def test_scannet_class_rows_cover_every_scripted_id():
    names = np.load(GOLDEN / "scannet_200_classname_no_wall_floor.npy")
    rows = model_3detr.scannet_class_rows(names, np.load(GOLDEN / "scannet_200_class2id.npy", allow_pickle=True).item())
    assert len(rows) == len(names) and sorted(rows.values()) == list(range(len(names)))
    assert set(synthetic.SCANNET_TEST_RANGE_LIST) <= set(rows) and set(synthetic.SCANNET_TRAIN_RANGE_LIST) <= set(rows)
    assert 1 not in rows and 3 not in rows            # wall and floor have no row


def test_scannet_prompts_absent_without_class_files(tmp_path, monkeypatch):
    monkeypatch.chdir(tmp_path)
    assert model_3detr._class_prompts(synthetic.make_args(dataset_name="scannet_anonymous_aligned_image")) is None


def test_scannet_batch_camera():
    d = synthetic.make_batch(3, 500, seed=2, image_hw=(968, 1296), camera="scannet")
    assert d["K"].shape == (3, 4, 4) and d["Rtilt"].shape == (3, 4, 4) and d["K"].dtype == np.float64
    assert np.allclose(d["K"][:, 0, 0], synthetic.SCANNET_COLOR_FOCAL)
    half = synthetic.make_batch(1, 500, seed=2, image_hw=(484, 648), camera="scannet")["K"][0]
    assert np.allclose(half[:3, :3], np.diag([0.5, 0.5, 1.0]) @ d["K"][0, :3, :3])
    R = d["Rtilt"][:, :3, :3]
    assert np.allclose(R @ R.transpose(0, 2, 1), np.eye(3), atol=1e-5)
    assert np.allclose(d["Rtilt"][:, 2, 3], synthetic.ROOM_MIN[2] + 1.5, atol=0.1)      # 1.5 m above the floor
    assert np.all(np.abs(d["rot_angle"]) <= np.pi / 6)
    assert set(np.unique(d["zx_flip_array"])) <= {-1.0, 1.0}
    for t, r in zip(d["rot_angle"], d["rot_array"]):
        assert np.allclose(r, np.linalg.inv(synthetic.rotz(t).T))
    with pytest.raises(ValueError):
        synthetic.make_batch(1, 100, camera="kinect")


@pytest.mark.parametrize("name", list(spc.CASES))
def test_scannet_golden_cases_cover_every_validity_branch(name):
    """The reference's last-layer boxes of each ScanNet golden case, projected with the case's camera: some lie
    inside the image, some are clipped at an image edge, some are behind the camera."""
    h, w = spc.IMAGE_HW
    golden = np.load(GOLDEN / f"model_{name}.npz")
    inputs = synthetic.to_device(spc.batch_np(name), "cpu")
    corners = torch.from_numpy(golden["last.box_corners_xyz"])
    u, v, depth = scannet_ref.scannet_uv(scannet_ref.undo_point_augmentation(corners, inputs), inputs)
    front = depth.amin(-1) > 0
    inside = (u >= 0).all(-1) & (u <= w - 1).all(-1) & (v >= 0).all(-1) & (v <= h - 1).all(-1)
    counts = (int((front & inside).sum()), int((front & ~inside).sum()), int((~front).sum()))
    print(f"{name}: inside {counts[0]}, clipped {counts[1]}, behind {counts[2]}")
    assert min(counts) > 0, counts


def test_boxes_in_image_rejects_a_camera_mismatch():
    d = synthetic.to_device(synthetic.make_batch(2, 200, seed=0), "cpu")
    corners, size = torch.zeros(2, 4, 8, 3), torch.ones(2, 4, 3)
    with pytest.raises(ValueError, match=r"K \(2, 3, 3\) and Rtilt \(2, 3, 3\)"):
        ops.boxes_in_image(corners, size, d, camera="scannet")
    s = synthetic.to_device(synthetic.make_batch(2, 200, seed=0, camera="scannet"), "cpu")
    with pytest.raises(ValueError, match=r"K \(2, 4, 4\) and Rtilt \(2, 4, 4\)"):
        ops.boxes_in_image(corners, size, s)
    with pytest.raises(ValueError, match="unknown camera"):
        ops.boxes_in_image(corners, size, s, camera="kinect")


def test_cpu_restatement_scannet_camera_matches_a_pinhole_projection():
    """The restated chain on a hand-made scene: identity augmentation, camera 1 m behind the origin looking along +y."""
    d = synthetic.make_batch(1, 100, seed=0, camera="scannet", image_hw=(968, 1296))
    pose = np.array([[1.0, 0, 0, 0], [0, 0, 1, -1], [0, -1, 0, 0], [0, 0, 0, 1]])
    d.update(Rtilt=pose[None], rot_array=np.eye(3)[None], flip_array=np.ones((1, 1)), zx_flip_array=np.ones((1, 1)),
             scale_array=np.ones((1, 1, 3)), image_flip_array=np.ones((1, 1)))
    inputs = synthetic.to_device(d, "cpu")
    p = torch.tensor([[[[0.5, 1.0, 0.25]] * 8]], dtype=torch.float32)     # 2 m in front of the camera
    u, v, depth = scannet_ref.scannet_uv(scannet_ref.undo_point_augmentation(p, inputs), inputs)
    K = d["K"][0]
    assert torch.allclose(depth, torch.tensor(2.0, dtype=torch.double))
    assert torch.allclose(u, torch.tensor(K[0, 0] * 0.25 + K[0, 2], dtype=torch.double))
    assert torch.allclose(v, torch.tensor(-K[1, 1] * 0.125 + K[1, 2], dtype=torch.double))
