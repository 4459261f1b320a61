"""The 3DETR + CLIP baseline head (`--model_name 3detrmulticlasshead --if_with_clip --test_only`) against the
reference's own Model3DETRMultiClassHead (tests/golden/make_baseline_eval_golden.py), on CPU: prompt lists, state-dict
keys, trainable parameters, and the test-time classification with the CUDA ops replaced by the CPU stand-ins of
oracle/cpu_step.py (coda_clip_classify by an fp64 restatement); and the host reader of ScanNet calibration files."""
import numpy as np
import pytest
import torch

import baseline_eval_common as bec
import cpu_step as cpu_shims
from coda_neurips2023_b200 import ops
from coda_neurips2023_b200.models import model_3detr

def clip_classify_f64(feats, text, scale, row_map, shape):
    f = feats.double()
    f = f / f.norm(dim=1, keepdim=True)
    prob = torch.softmax(float(scale) * f @ text.double().t(), dim=-1) if f.shape[0] else f.new_zeros((0, text.shape[0]))
    rows = torch.zeros((row_map.numel(), text.shape[0]), dtype=torch.float64)
    keep = row_map >= 0
    rows[keep] = prob[row_map[keep].long()]
    rows = rows.float().reshape(*shape, -1)
    return rows, torch.zeros_like(rows)


DATASETS = ["sunrgbd_image", "scannet50_image"]


@pytest.mark.parametrize("dataset_name", DATASETS)
def test_prompts_equal_the_reference(dataset_name):
    golden = np.load(bec.golden_path(dataset_name))
    with bec.class_lists():
        ours = model_3detr._class_prompts(bec.args_for(dataset_name), evaluated=True)
    assert ours == list(golden["prompts"])


@pytest.mark.parametrize("dataset_name", DATASETS)
def test_state_dict_keys_and_trainable_parameters_equal_the_reference(dataset_name):
    model, golden = bec.build_ours("cpu", dataset_name)
    keys = sorted(k for k in model.state_dict() if not k.startswith("clip_model."))
    assert keys == list(golden["state_dict_keys"])
    assert sorted(k for k, p in model.named_parameters() if p.requires_grad) == list(golden["trainable"])
    assert not any(k.startswith(("test_clip_model.", "res_encoder.")) or k == "logit_scale"
                   for k in model.state_dict())


@pytest.mark.parametrize("dataset_name", DATASETS)
def test_classification_matches_the_reference_on_cpu(dataset_name, monkeypatch):
    monkeypatch.setattr(ops, "clip_classify", clip_classify_f64)
    torch.manual_seed(0)
    extents = []
    with cpu_shims.installed():
        sunrgbd_projection = ops.boxes_in_image

        def projection(corners_xyz, size_unnorm, inputs, camera="sunrgbd", extent=False):
            if camera == "scannet":
                boxes, usable, ext = bec.scannet_extent_cpu(corners_xyz, size_unnorm, inputs)
                extents.append(ext)
                return boxes, usable
            return sunrgbd_projection(corners_xyz, size_unnorm, inputs)

        ops.boxes_in_image = projection
        try:
            model, out, golden = bec.run_ours("cpu", dataset_name)
        finally:
            ops.boxes_in_image = sunrgbd_projection
    usable = out["clip_usable_mask"].numpy()
    assert np.array_equal(usable, golden["usable"])
    assert not usable[bec.NO_VIEW_SCENE].any() and usable.sum() > 0
    assert not usable[:, list(bec.ZERO_QUERIES)].any() and (golden["boxes"][:, list(bec.ZERO_QUERIES)] == -1).all()
    boxes = out["clip_boxes_2d"].numpy()
    differ = (boxes != golden["boxes"]).any(-1) & usable
    if extents:       # equal wherever the fp64 extent is not within 1e-3 px of an integer
        ext = extents[-1].numpy()
        near = (np.abs(ext - np.round(ext)) <= 1e-3).any(-1)
        print(f"{dataset_name}: {int((near & usable).sum())} usable boxes at an integer boundary")
        assert not (differ & ~near).any()
    else:
        assert not differ.any()
    print(f"{dataset_name}: integer boxes differing from the reference: {int(differ.sum())} of {int(usable.sum())}")
    prob = out["sem_cls_prob"].numpy()
    assert prob.shape[-1] == len(golden["prompts"])
    assert (prob[~usable] == 0).all() and (out["sem_cls_logits"].numpy() == 0).all()
    assert np.abs(prob - golden["sem_cls_prob"]).max() <= 1e-4
    assert np.abs(out["objectness_prob"].numpy() - golden["objectness_prob"]).max() <= 1e-4
    scale = np.abs(golden["box_corners"]).max()
    assert np.abs(out["box_corners"].numpy() - golden["box_corners"]).max() <= 1e-4 * scale


def test_scannet_calibration_reader_reads_what_the_reference_reads(tmp_path):
    golden = np.load(bec.golden_path("scannet50_image"))
    names = bec.scannet_names()
    K, pose = model_3detr.ScanNetCalibration()(names["calib_name"], names["squence_name"])
    assert np.array_equal(K, golden["calib_K"]) and np.array_equal(pose, golden["calib_pose"])
    read = model_3detr.ScanNetCalibration()
    with pytest.raises(FileNotFoundError, match="pose/1.txt"):
        read(names["calib_name"][:1], ["1"])
    with pytest.raises(FileNotFoundError, match="intrinsic_color.txt"):
        read([str(tmp_path)], ["0"])


def test_unsupported_baseline_options_raise():
    from coda_neurips2023_b200 import synthetic

    for flag in ("if_use_gt_box", "if_expand_box", "if_only_novel_prompt"):
        args = bec.args_for("sunrgbd_image")
        setattr(args, flag, True)
        with pytest.raises(NotImplementedError, match=flag):
            model_3detr.build_3detr_multiclasshead(args, synthetic.SyntheticDatasetConfig(args))
