"""Generates tests/golden/scannet_prompts.json: the class prompts the REFERENCE model builds for ScanNet runs
(models/model_3detr.py:197-279, `self.all_classes_keys`), for the flags of scripts/coda_scannet_stage1.sh and
scripts/coda_scannet_stage2.sh, and for the seen-only list (without --if_clip_more_prompts).  The reference model
is constructed in this container through tests/golden/_reference_harness.py (no forward pass is needed).

    python tests/golden/make_scannet_prompts_golden.py            (writes into tests/golden/)
"""
import json
import sys
from pathlib import Path

import torch

HERE = Path(__file__).resolve().parent
ROOT = HERE.parents[1]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))
sys.path.insert(0, str(HERE))

import _reference_harness as H  # noqa: E402
import make_model_golden as mmg  # noqa: E402
from coda_neurips2023_b200 import synthetic  # noqa: E402
from param_fill import fill_by_name  # noqa: E402

# the prompt-related flags of the two ScanNet scripts (train / test range lists and reset_scannet_num are
# synthetic.make_args' defaults, taken from the stage-1 script; the stage-2 script passes the same values)
FLAGS = {
    "stage1": dict(dataset_name="scannet_anonymous_aligned_image", if_clip_more_prompts=True, train_range_max=10,
                   test_range_max=60),
    "stage2": dict(dataset_name="scannet_anonymous_aligned_image_with_novel_cate_confi", if_clip_more_prompts=True,
                   train_range_max=10, test_range_max=60, if_clip_weak_labels=True),
    "seen_only": dict(dataset_name="scannet_anonymous_aligned_image", if_clip_more_prompts=False, train_range_max=10,
                      test_range_max=60),
}


def reference_prompts(over):
    args = mmg.reference_args(dict(mmg.mpc._SMALL, **over))
    m3 = H.load("models.model_3detr")
    clip_pkg = H.load("CLIP.clip.clip")
    clip_model_mod = H.load("CLIP.clip.model")

    def fake_clip_load(path, device="cpu", download_root=None, if_transform_tensor=True, **kw):
        torch.manual_seed(0)
        model = clip_model_mod.CLIP(**mmg.TINY_CLIP).float().eval()
        fill_by_name(model, seed=11)
        return model, clip_pkg._transform_for_tensor(model.visual.input_resolution)

    clip_pkg.load = fake_clip_load
    sys.modules["CLIP.clip"].clip.load = fake_clip_load
    model, _ = m3.build_3detr_predictedbox_distillation_head(args, synthetic.SyntheticDatasetConfig(args))
    return list(model.all_classes_keys)


def main():
    out = {name: reference_prompts(over) for name, over in FLAGS.items()}
    out["flags"] = {name: dict(over, train_range_list=list(synthetic.SCANNET_TRAIN_RANGE_LIST),
                               test_range_list=list(synthetic.SCANNET_TEST_RANGE_LIST), reset_scannet_num=50)
                    for name, over in FLAGS.items()}
    (HERE / "scannet_prompts.json").write_text(json.dumps(out, indent=1) + "\n")
    print({k: len(v) for k, v in out.items() if k != "flags"})


if __name__ == "__main__":
    main()
