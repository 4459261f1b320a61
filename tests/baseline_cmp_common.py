"""Shared by the golden generator (tests/golden/make_baseline_cmp_golden.py) and the CPU / GPU tests of the 3DETR +
CLIP baseline head's comparison-class evaluation (forward(if_cmp_class=True), the OV-3DET paper's 20 SUN RGB-D / 19
ScanNet classes): the golden's path, the class lists of a CoDA checkout with the comparison lists, OUR model with the
golden's text, and the batch and dataset config the golden's AP metrics were computed on.  The case itself (arguments,
weights, batch) is the real-test case of baseline_eval_common."""
import os
import tempfile
from contextlib import contextmanager
from pathlib import Path

import numpy as np
import torch

import baseline_eval_common as bec
from coda_neurips2023_b200 import synthetic

DATASETS = list(bec.DATASET_ARGS)
CLASS_LISTS = ("all_classes_trainval_v1.npy", "scannet_200_classname_no_wall_floor.npy", "scannet_200_class2id.npy",
               "ov_3detr.npy", "ov_3detr_scannet.npy")
GT_KEYS = ("gt_box_corners", "gt_box_sem_cls_label", "gt_box_present")
AP_IOU = (0.25, 0.5)


def golden_path(dataset_name):
    short = "scannet" if "scannet" in dataset_name else "sunrgbd"
    return bec.GOLDEN / f"model_baseline_clip_cmp_{short}.npz"


@contextmanager
def class_lists(names=CLASS_LISTS):
    """Runs with the working directory where datasets/ holds `names` (from tests/golden/), as a CoDA checkout has
    them."""
    cwd = os.getcwd()
    with tempfile.TemporaryDirectory() as tmp:
        os.mkdir(Path(tmp) / "datasets")
        for name in names:
            os.symlink(bec.GOLDEN / name, Path(tmp) / "datasets" / name)
        os.chdir(tmp)
        try:
            yield
        finally:
            os.chdir(cwd)


def build_ours(device, dataset_name):
    """OUR baseline head of the real-test golden (bec.build_ours) with the comparison golden's text matrix."""
    model, _ = bec.build_ours(device, dataset_name)
    golden = np.load(golden_path(dataset_name))
    model.cmp_text_features_fg_norm = torch.from_numpy(golden["cmp_text_features_fg_norm"]).to(device)
    return model, golden


def eval_batch(device, dataset_name, golden) -> dict:
    """The golden's batch (bec.test_batch) with the ground truth its AP metrics were computed against."""
    inputs = bec.test_batch(device, dataset_name)
    inputs.update({k: torch.from_numpy(golden[k]).to(device) for k in GT_KEYS})
    return inputs


def dataset_config(args, golden):
    """A dataset config with the comparison classes' count and names, as the comparison split's config has them."""
    cfg = synthetic.SyntheticDatasetConfig(args, num_semcls=len(golden["cmp_class_names"]))
    cfg.class2type = {i: str(n) for i, n in enumerate(golden["cmp_class_names"])}
    return cfg
