"""The 3DETR + CLIP baseline head's comparison-class evaluation (`forward(if_cmp_class=True)`, the OV-3DET paper's
classes) against the reference's own head (tests/golden/make_baseline_cmp_golden.py), on CPU: the prompts, the
comparison text, the state-dict keys, and the classification with the CUDA ops replaced by the CPU stand-ins of
oracle/cpu_step.py (coda_clip_classify by an fp64 restatement); and what happens without the comparison list."""
import numpy as np
import pytest
import torch

import baseline_cmp_common as bcc
import baseline_eval_common as bec
import cpu_step as cpu_shims
from coda_neurips2023_b200 import ops, synthetic
from coda_neurips2023_b200.models import model_3detr
from test_baseline_eval_cpu import clip_classify_f64

BPE = bec.GOLDEN / "clip_bpe_merges_48894.txt.gz"


@pytest.mark.parametrize("dataset_name", bcc.DATASETS)
def test_cmp_prompts_equal_the_reference(dataset_name):
    golden = np.load(bcc.golden_path(dataset_name))
    with bcc.class_lists():
        ours = model_3detr.cmp_prompts(bec.args_for(dataset_name))
    assert ours == list(golden["cmp_prompts"])
    assert len(ours) == (19 if "scannet" in dataset_name else 20)


@pytest.mark.parametrize("dataset_name", bcc.DATASETS)
def test_cmp_text_equals_the_reference(dataset_name, monkeypatch):
    """Built where the class lists and the tokenizer's vocabulary are, the head encodes the comparison prompts with
    its CLIP (here the golden's small one) as the reference does."""
    monkeypatch.setenv("CODA_CLIP_BPE", str(BPE))
    golden = np.load(bcc.golden_path(dataset_name))
    with bcc.class_lists(), cpu_shims.installed():
        model, _ = bec.build_ours("cpu", dataset_name)
        assert not model.text_features_synthetic
        model.build_cmp_text(bec.args_for(dataset_name))
    assert model.all_cmp_classes_keys == list(golden["cmp_prompts"])
    want = golden["cmp_text_features_fg_norm"]
    got = model.cmp_text_features_fg_norm
    assert got.dtype == torch.float32 and got.shape == want.shape
    assert np.abs(got.numpy() - want).max() <= 1e-5
    assert torch.allclose(model.cmp_text_features_fg / model.cmp_text_features_fg.norm(dim=1, keepdim=True), got)


@pytest.mark.parametrize("dataset_name", bcc.DATASETS)
def test_cmp_text_adds_no_state_dict_key(dataset_name):
    model, _ = bcc.build_ours("cpu", dataset_name)
    keys = sorted(k for k in model.state_dict() if not k.startswith("clip_model."))
    assert keys == list(np.load(bec.golden_path(dataset_name))["state_dict_keys"])
    assert not any("cmp" in k for k in model.state_dict())
    model.load_state_dict(model.state_dict(), strict=True)


def _projection(extents):
    """ops.boxes_in_image of the CPU stand-ins, with the ScanNet camera restated by bec.scannet_extent_cpu."""
    sunrgbd_projection = ops.boxes_in_image

    def projection(corners_xyz, size_unnorm, inputs, camera="sunrgbd", extent=False):
        if camera == "scannet":
            boxes, usable, ext = bec.scannet_extent_cpu(corners_xyz, size_unnorm, inputs)
            extents.append(ext)
            return boxes, usable
        return sunrgbd_projection(corners_xyz, size_unnorm, inputs)

    return projection


@pytest.mark.parametrize("dataset_name", bcc.DATASETS)
def test_cmp_classification_matches_the_reference_on_cpu(dataset_name, monkeypatch):
    monkeypatch.setattr(ops, "clip_classify", clip_classify_f64)
    torch.manual_seed(0)
    extents = []
    with cpu_shims.installed():
        sunrgbd_projection = ops.boxes_in_image
        ops.boxes_in_image = _projection(extents)
        try:
            model, golden = bcc.build_ours("cpu", dataset_name)
            with torch.no_grad():
                out = model(bec.test_batch("cpu", dataset_name), if_cmp_class=True)["outputs"]
        finally:
            ops.boxes_in_image = sunrgbd_projection
    usable = out["clip_usable_mask"].numpy()
    assert np.array_equal(usable, golden["usable"])
    assert not usable[bec.NO_VIEW_SCENE].any() and usable.sum() > 0
    boxes = out["clip_boxes_2d"].numpy()
    differ = (boxes != golden["boxes"]).any(-1) & usable
    if extents:       # equal wherever the fp64 extent is not within 1e-3 px of an integer
        ext = extents[-1].numpy()
        differ &= ~(np.abs(ext - np.round(ext)) <= 1e-3).any(-1)
    assert not differ.any()
    prob = out["sem_cls_prob"].numpy()
    assert prob.shape == golden["sem_cls_prob"].shape == (bec.BATCH, 128, len(golden["cmp_prompts"]))
    assert out["sem_cls_logits"].shape == prob.shape and (out["sem_cls_logits"].numpy() == 0).all()
    assert (prob[~usable] == 0).all()
    assert np.abs(prob - golden["sem_cls_prob"]).max() <= 1e-4
    assert np.abs(out["objectness_prob"].numpy() - golden["objectness_prob"]).max() <= 1e-4
    assert "text_features_clip" not in out


@pytest.mark.parametrize("dataset_name", bcc.DATASETS)
def test_missing_cmp_list_raises_at_the_forward(dataset_name, monkeypatch):
    """Class lists and vocabulary reachable, the comparison list not: the head builds (every other evaluation works
    without the list), and the first if_cmp_class forward raises, naming the list."""
    monkeypatch.setenv("CODA_CLIP_BPE", str(BPE))
    missing = "ov_3detr_scannet.npy" if "scannet" in dataset_name else "ov_3detr.npy"
    with bcc.class_lists([n for n in bcc.CLASS_LISTS if n != missing]), cpu_shims.installed():
        model, _ = bec.build_ours("cpu", dataset_name)
        assert not model.text_features_synthetic and model.cmp_text_features_fg_norm is None
        with pytest.raises(FileNotFoundError, match="datasets/" + missing):
            model_3detr.cmp_prompts(bec.args_for(dataset_name))
    with cpu_shims.installed(), torch.no_grad():
        with pytest.raises(FileNotFoundError, match="datasets/" + missing):
            model(bec.test_batch("cpu", dataset_name), if_cmp_class=True)


@pytest.mark.parametrize("dataset_name", bcc.DATASETS)
def test_synthetic_cmp_text_is_seeded_and_warned_about(dataset_name):
    args = bec.args_for(dataset_name)
    with pytest.warns(UserWarning, match="class prompts unavailable"):
        model, _ = model_3detr.build_3detr_multiclasshead(args, synthetic.SyntheticDatasetConfig(args))
    n = 19 if "scannet" in dataset_name else 20
    d = model.clip_model.visual.output_dim
    raw = torch.randn(n, d, generator=torch.Generator().manual_seed(model.CMP_SYNTHETIC_SEED))
    assert model.all_cmp_classes_keys is None
    assert torch.equal(model.cmp_text_features_fg, raw)
    assert torch.equal(model.cmp_text_features_fg_norm, raw / raw.norm(dim=1, keepdim=True))
