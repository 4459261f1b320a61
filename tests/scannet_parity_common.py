"""ScanNet runs of the step (scripts/coda_scannet_stage1.sh / stage2.sh) pinned to the REFERENCE: the case table shared
by tests/golden/make_scannet_golden.py and the ScanNet parity tests, and OUR model / criterion built for a case the
way model_parity_common.build does it for the SUN RGB-D cases -- here with ScanNet batches (4 x 4 colour intrinsics,
camera-to-world pose, ScanNet augmentation bookkeeping) and the ScanNet camera in the crop projection."""
import tempfile
import warnings

import numpy as np
import torch

import model_parity_common as mpc
from coda_neurips2023_b200 import clip as clip_mod
from coda_neurips2023_b200 import synthetic
from coda_neurips2023_b200.criterion import build_criterion
from coda_neurips2023_b200.models import build_model
from param_fill import fill_by_name

GOLDEN = mpc.GOLDEN
IMAGE_HW = (968, 1296)

# dataset name, matcher / loss weights, 10 seen classes and 60 evaluated prompts, 1296 x 968 images (stage-1 script)
_SCANNET = dict(dataset_name="scannet_anonymous_aligned_image", matcher_giou_cost=2.0, matcher_center_cost=0.0,
                matcher_objectness_cost=0.0, loss_no_object_weight=0.25, base_lr=1.4142e-4, train_range_max=10,
                test_range_max=60, image_size_width=1296, image_size_height=968)
_SMALL = dict(mpc._SMALL)
_NODROP = dict(enc_dropout=0.0, dec_dropout=0.0, mlp_dropout=0.0)
_STAGE2 = dict(if_clip_weak_labels=True, loss_feat_seen_softmax_weakly_loss_with_novel_cate_confi_weight=1.0,
               dataset_name="scannet_anonymous_aligned_image_with_novel_cate_confi", confidence_type="non-confidence",
               online_nms_update_save_novel_label_clip_driven_with_cate_confidence=True, save_objectness=0.3,
               online_nms_update_save_epoch=50,
               # 60 text rows: the CLIP-driven keep is lowered from the script's 0.3 so that pseudo-label rows appear
               clip_driven_keep_thres=0.015)

# name -> (batch, npoints, args overrides, extras); extras: pseudo (stage-2 discovery writes pseudo-label rows)
CASES = {
    "scannet_stage1_small": (2, 3000, dict(_SMALL, **_SCANNET), {}),
    "scannet_stage2_discovery": (2, 2500, dict(dict(_SMALL, **_SCANNET), **_STAGE2), dict(pseudo=True)),
    # the stage-1 script's configuration: 40 000 points, 1296 x 968 images, 128 queries, 10 seen / 60 prompts
    "scannet_full": (2, 40000, dict(_NODROP, **_SCANNET, nqueries=128), {}),
}
FULL_SIZE = ("scannet_full",)


def batch_np(name):
    batch, npoints, _, _ = CASES[name]
    return synthetic.make_batch(batch, npoints, seed=5, image_hw=IMAGE_HW, camera="scannet")


def build(name: str, device: str):
    batch, npoints, over, extra = CASES[name]
    golden = np.load(GOLDEN / f"model_{name}.npz")
    args = synthetic.make_args(**over)
    cfg = synthetic.SyntheticDatasetConfig(args)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        model, _ = build_model(args, cfg)
    # the golden generator fills the whole reference model by name, CLIP included: install the small CLIP first
    tiny = clip_mod.CLIP(**mpc.TINY_CLIP).float().eval()
    for p in tiny.parameters():
        p.requires_grad = False
    model.clip_model = tiny
    model.test_clip_model = tiny
    model.res_encoder = tiny.visual
    model.logit_scale = tiny.logit_scale
    model.clip_resolution = 224
    fill_by_name(model, seed=3)
    model.device = device
    model = model.to(device)
    model.text_features_fg_norm = torch.from_numpy(golden["text_features_fg_norm"]).to(device)
    model.text_features_fg = model.text_features_fg_norm
    criterion = build_criterion(args, cfg).to(device)
    model.train()
    model.clip_model.eval()
    inputs = synthetic.to_device(batch_np(name), device)
    if extra.get("pseudo"):
        tmp = tempfile.mkdtemp(prefix="coda_pseudo_")
        inputs["pseudo_box_path"] = [f"{tmp}/scene{i}.npy" for i in range(batch)]
    return args, model, criterion, inputs, golden


def run(name: str, device: str):
    args, model, criterion, inputs, golden = build(name, device)
    np.random.seed(123)
    out = model(inputs, curr_epoch=0)
    loss, loss_dict = criterion(out, inputs)
    loss.backward()
    return model, out, loss, loss_dict, golden
