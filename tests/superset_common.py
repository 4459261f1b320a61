"""Stage 2 with --if_clip_superset (scripts/coda_sunrgbd_stage2.sh, scripts/coda_scannet_stage2.sh) pinned to the
REFERENCE: the case table shared by tests/golden/make_superset_golden.py and the superset tests, a working directory
laid out like a CoDA checkout (class lists and the LVIS list from tests/golden/), and OUR model / criterion built for
a case the way model_parity_common / scannet_parity_common build theirs -- except that the class and superset text
features are computed by the model itself from its own prompts and tokenizer, with the small CLIP of the goldens."""
import os
import tempfile
import warnings
from contextlib import contextmanager
from pathlib import Path

import numpy as np
import torch

import model_parity_common as mpc
import scannet_parity_common as spc
from coda_neurips2023_b200 import clip as clip_mod
from coda_neurips2023_b200 import synthetic
from coda_neurips2023_b200.criterion import build_criterion
from coda_neurips2023_b200.models import build_model, model_3detr
from param_fill import fill_by_name

GOLDEN = mpc.GOLDEN
BPE = GOLDEN / "clip_bpe_merges_48894.txt.gz"
LISTS = ("all_classes_trainval_v1.npy", "scannet_200_classname_no_wall_floor.npy", "scannet_200_class2id.npy",
         "lvis_1204.npy")

# the prompt-related flags of the two stage-2 scripts (ScanNet range lists: synthetic.make_args' defaults, which are
# the scripts' values)
FLAGS = {
    "sunrgbd": dict(dataset_name="sunrgbd_anonymous_aligned_image_with_novel_cate_confi", if_clip_more_prompts=True,
                    train_range_max=10, test_range_max=46, if_clip_superset=True, if_use_v1=True),
    "scannet": dict(dataset_name="scannet_anonymous_aligned_image_with_novel_cate_confi", if_clip_more_prompts=True,
                    train_range_max=10, test_range_max=60, if_clip_superset=True, reset_scannet_num=50),
}



def _merged(*dicts):
    out = {}
    for d in dicts:
        out.update(d)
    return out


_DISCOVERY = dict(online_nms_update_save_novel_label_clip_driven_with_cate_confidence=True, save_objectness=0.3)
# name -> (dataset, batch, npoints, args overrides, extras).  Weak labels and discovery on; the CLIP-driven keep is
# lowered from the scripts' 0.3 so that random-init predictions over ~1200 classes still yield pseudo-label rows
CASES = {
    "stage2_superset": ("sunrgbd", 2, 2500,
                        _merged(mpc._SMALL, mpc._STAGE2, _DISCOVERY, FLAGS["sunrgbd"],
                                dict(clip_driven_keep_thres=0.0012, online_nms_update_save_epoch=10)),
                        dict(pseudo=True)),
    "scannet_stage2_superset": ("scannet", 2, 2500,
                                _merged(spc._SMALL, spc._SCANNET, spc._STAGE2, FLAGS["scannet"],
                                        dict(clip_driven_keep_thres=0.0012)),
                                dict(pseudo=True)),
}


@contextmanager
def coda_checkout(lvis: bool = True):
    """Runs in a working directory whose datasets/ holds the class lists (and, with `lvis`, the LVIS list), as a
    CoDA checkout has them, with the CLIP BPE vocabulary of tests/golden/."""
    cwd, env = os.getcwd(), os.environ.get("CODA_CLIP_BPE")
    with tempfile.TemporaryDirectory() as tmp:
        os.mkdir(Path(tmp) / "datasets")
        for name in LISTS:
            if lvis or name != "lvis_1204.npy":
                os.symlink(GOLDEN / name, Path(tmp) / "datasets" / name)
        os.chdir(tmp)
        os.environ["CODA_CLIP_BPE"] = str(BPE)
        try:
            yield Path(tmp)
        finally:
            os.chdir(cwd)
            if env is None:
                os.environ.pop("CODA_CLIP_BPE", None)
            else:
                os.environ["CODA_CLIP_BPE"] = env


def tiny_clip(path=None, device="cpu", **kwargs):
    """stands in for clip.load: the small CLIP the goldens use (filled by name with the model)"""
    tiny = clip_mod.CLIP(**mpc.TINY_CLIP).float().eval()
    for p in tiny.parameters():
        p.requires_grad = False
    return tiny.to(device)


def batch_np(name):
    dataset, batch, npoints, _, _ = CASES[name]
    if dataset == "scannet":
        return synthetic.make_batch(batch, npoints, seed=5, image_hw=spc.IMAGE_HW, camera="scannet")
    return synthetic.make_batch(batch, npoints, seed=5, image_hw=(531, 730))


def build(name: str, device: str, criterion_args: dict | None = None):
    """-> (args, model, criterion, inputs, golden).  The text features are computed on `device` from the filled small
    CLIP.  `criterion_args` overrides arguments of the criterion only."""
    dataset, batch, npoints, over, extra = CASES[name]
    golden = np.load(GOLDEN / f"model_{name}.npz")
    args = synthetic.make_args(**over)
    cfg = synthetic.SyntheticDatasetConfig(args)
    load = model_3detr.clip_mod.load
    model_3detr.clip_mod.load = tiny_clip
    try:
        with coda_checkout(), warnings.catch_warnings():
            warnings.simplefilter("ignore")
            model, _ = build_model(args, cfg)
            model.to_device("cpu")
            model.clip_resolution = 224
            fill_by_name(model, seed=3)
            model.to_device(device)
            model.text_features_fg_norm = model.encode_prompts(model.all_classes_keys)
            model.text_features_fg = model.text_features_fg_norm
            model.superset_text_features_fg_norm = model.encode_prompts(model.superset_all_classes_keys)
            model.test_text_features_fg_norm = model.superset_text_features_fg_norm
    finally:
        model_3detr.clip_mod.load = load
    cargs = synthetic.make_args(**dict(over, **(criterion_args or {})))
    criterion = build_criterion(cargs, cfg).to(device)
    model.train()
    model.clip_model.eval()
    inputs = synthetic.to_device(batch_np(name), device)
    if extra.get("pseudo"):
        tmp = tempfile.mkdtemp(prefix="coda_pseudo_")
        inputs["pseudo_box_path"] = [f"{tmp}/scene{i}.npy" for i in range(batch)]
    return args, model, criterion, inputs, golden


def run(name: str, device: str, criterion_args: dict | None = None):
    args, model, criterion, inputs, golden = build(name, device, criterion_args)
    np.random.seed(123)
    out = model(inputs, curr_epoch=0)
    loss, loss_dict = criterion(out, inputs)
    loss.backward()
    return model, out, loss, loss_dict, golden


def check_text_features(model, golden, rtol):
    """the model's class and superset text features against the reference's (max error over max |ref|)"""
    for key, got in (("text_features_fg_norm", model.text_features_fg_norm),
                     ("superset_text_features_fg_norm", model.superset_text_features_fg_norm)):
        exp = golden[key]
        g = got.detach().float().cpu().numpy()
        if g.shape != exp.shape:
            g = g[::4, ::4]       # the golden keeps every 4th row and column of the superset features
        assert g.shape == exp.shape, (key, g.shape, exp.shape)
        err = float(np.abs(g - exp).max() / np.abs(exp).max())
        assert err <= rtol, f"{key}: {err:.2e}"


def check_weak_labels(out, golden):
    last = out["outputs"]
    assert np.array_equal(last["weak_box_cate_label"].cpu().numpy(), golden["last.weak_box_cate_label"])
