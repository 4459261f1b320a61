"""Generates tests/golden/model_eval_{small,full}.npz: the REFERENCE's own model in eval mode, run on CPU in this
container the same way make_model_golden.py runs it (tests/golden/_reference_harness.py), on the path
`main.py --test_only` takes: weights filled by name (fill_by_name), BatchNorm running statistics filled by name
(fill_running_stats_by_name), model.eval(), forward(inputs, if_real_test=True) under no_grad.

    python tests/golden/make_model_eval_golden.py [eval_small] [eval_full]     (writes into tests/golden/)
"""
import sys
from pathlib import Path

import numpy as np
import torch

HERE = Path(__file__).resolve().parent
ROOT = HERE.parents[1]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))
sys.path.insert(0, str(HERE))

import make_model_golden as mmg  # noqa: E402  (reference arguments, tiny CLIP, harness)
import model_eval_common as mec  # noqa: E402
import model_parity_common as mpc  # noqa: E402
from coda_neurips2023_b200 import synthetic  # noqa: E402
from param_fill import fill_by_name  # noqa: E402
from running_stats_fill import fill_running_stats_by_name  # noqa: E402

H = mmg.H


def run_reference_eval(name):
    batch, npoints, over, extra = mpc.case(mec.EVAL_CASES[name])
    args = mmg.reference_args(over)
    m3 = H.load("models.model_3detr")
    box_util = H.load("utils.box_util")
    clip_pkg = H.load("CLIP.clip.clip")
    clip_model_mod = H.load("CLIP.clip.model")

    class Cfg(synthetic.SyntheticDatasetConfig):  # corner builders of the REFERENCE
        def box_parametrization_to_corners(self, c, s, a):
            return box_util.get_3d_box_batch_tensor(s, a, box_util.flip_axis_to_camera_tensor(c))

        def box_parametrization_to_corners_xyz(self, c, s, a):
            return box_util.get_3d_box_batch_tensor_xyz(s, a, c)

    cfg = Cfg(args)

    def fake_clip_load(path, device="cpu", download_root=None, if_transform_tensor=True, **kw):
        torch.manual_seed(0)
        model = clip_model_mod.CLIP(**mpc.TINY_CLIP).float().eval()
        fill_by_name(model, seed=11)
        return model, clip_pkg._transform_for_tensor(model.visual.input_resolution)

    clip_pkg.load = fake_clip_load
    sys.modules["CLIP.clip"].clip.load = fake_clip_load
    torch.manual_seed(0)
    model, _ = m3.build_3detr_predictedbox_distillation_head(args, cfg)
    fill_by_name(model, seed=3)
    fill_running_stats_by_name(model, seed=mec.STATS_SEED)
    with torch.no_grad():
        model.text_features_fg = model.clip_model.encode_text(model.text).to(torch.float32)
        model.text_features_fg_norm = model.text_features_fg / model.text_features_fg.norm(dim=1, keepdim=True)
    model.eval()
    inputs = {k: torch.from_numpy(v) for k, v in
              synthetic.make_batch(batch, npoints, seed=5, image_hw=extra.get("image_hw", (531, 730))).items()}
    np.random.seed(123)
    with torch.no_grad():
        out = model(inputs, if_real_test=True)
    return model, out


def main():
    only = sys.argv[1:]
    for name in mec.EVAL_CASES:
        if only and name not in only:
            continue
        model, out = run_reference_eval(name)
        blob = mec.blob(out)
        blob["text_features_fg_norm"] = model.text_features_fg_norm.numpy()
        np.savez_compressed(mec.golden_path(name), **blob)
        print("wrote", name, {k: v.shape for k, v in blob.items() if k.startswith("last.")}, flush=True)


if __name__ == "__main__":
    main()
