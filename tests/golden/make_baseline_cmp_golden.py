"""Generates tests/golden/model_baseline_clip_cmp_{sunrgbd,scannet}.npz: the REFERENCE's 3DETR + CLIP baseline head
run on CPU with forward(inputs, if_cmp_class=True) -- the comparison-class evaluation main.py runs on the
`real_cmp_test` split -- on the case of make_baseline_eval_golden.py: the same harness, weights, small CLIP and batch
(whose third scene has no usable box, with zero-size queries and boxes behind the camera).  The reference builds its
comparison text once at construction; it is re-derived here from the filled CLIP, as the generator of the real-test
golden re-derives the evaluated classes' text.

Stored: the usable mask, integer boxes, sem_cls_prob / sem_cls_logits and objectness of the run (what does not depend
on the text, such as the crop features, the tests read from the real-test golden); the comparison prompts and class
names; the normalised comparison text features; and the reference APCalculator's metrics on the run's outputs, with
their ground truth.  That ground truth is made from the reference's own predicted
boxes, so that the metrics are not all zero: in each scene with usable boxes, the six most object-like usable ones,
four labelled with their CLIP class and two with the class after it; in the scene without a usable box, two boxes.
The dataset config has the comparison classes' count and names.

    python tests/golden/make_baseline_cmp_golden.py [sunrgbd_image] [scannet50_image]    (writes into tests/golden/)
"""
import sys
from pathlib import Path
from types import SimpleNamespace

import numpy as np
import torch

HERE = Path(__file__).resolve().parent
ROOT = HERE.parents[1]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))
sys.path.insert(0, str(HERE))

import baseline_cmp_common as bcc  # noqa: E402
import baseline_eval_common as bec  # noqa: E402
import make_baseline_eval_golden as mbeg  # noqa: E402

H = mbeg.H
GT_PER_SCENE = 8


def cmp_reference_model(args):
    """The reference baseline head of make_baseline_eval_golden.py, whose forward(if_real_test=True) runs
    forward(if_cmp_class=True) with the comparison text of the filled CLIP (reference :2092-2095)."""
    m3, model = REFERENCE_MODEL(args)
    forward = model.forward

    def cmp_forward(inputs, if_real_test=False, **kw):
        assert if_real_test
        with torch.no_grad():
            model.cmp_text_features_fg = model.clip_model.encode_text(model.cmp_text)
        return forward(inputs, if_cmp_class=True, **kw)

    model.forward = cmp_forward
    MODELS.append((m3, model))
    return m3, model


REFERENCE_MODEL, MODELS = mbeg.reference_model, []
mbeg.reference_model = cmp_reference_model


def ground_truth(blob):
    """(B, G, 8, 3) corners, (B, G) labels, (B, G) present, from the reference's predicted boxes."""
    prob, obj, corners = blob["sem_cls_prob"], blob["objectness_prob"], blob["box_corners"]
    bsz, _, ncls = prob.shape
    gt_corners = np.zeros((bsz, GT_PER_SCENE, 8, 3), np.float32)
    labels = np.zeros((bsz, GT_PER_SCENE), np.int64)
    present = np.zeros((bsz, GT_PER_SCENE), np.float32)
    for b in range(bsz):
        usable = np.nonzero(blob["usable"][b])[0]
        if usable.size:
            pick = usable[np.argsort(-obj[b, usable], kind="stable")[:6]]
            cls = prob[b, pick].argmax(-1)
            cls[4:] = (cls[4:] + 1) % ncls
        else:
            pick, cls = np.array([5, 9]), np.array([3, ncls - 1])
        n = pick.size
        gt_corners[b, :n], labels[b, :n], present[b, :n] = corners[b, pick], cls, 1
    return gt_corners, labels, present


def ap_metrics(dataset_name, blob, class_names):
    """The reference APCalculator's metrics.  Its empty-box test hands every box to qhull, which fails on the
    single-point hull of a zero-size box away from the origin (ZERO_QUERIES): such a box holds no point, as the device
    point-in-box count finds."""
    from scipy.spatial import QhullError

    apm = H.load("utils.ap_calculator")
    extract = apm.extract_pc_in_box3d

    def extract_or_empty(pc, box3d):
        try:
            return extract(pc, box3d)
        except QhullError:
            assert np.ptp(box3d, axis=0).max() == 0, "qhull failed on a box with extent"
            return pc[:0], np.zeros(len(pc), bool)

    apm.extract_pc_in_box3d = extract_or_empty
    cfg_ds = SimpleNamespace(num_semcls=len(class_names))
    calc = apm.APCalculator(cfg_ds, ap_iou_thresh=list(bcc.AP_IOU),
                            class2type_map={i: str(n) for i, n in enumerate(class_names)}, exact_eval=True,
                            args=SimpleNamespace(dataset_name=dataset_name))
    t = lambda k: torch.from_numpy(blob[k])  # noqa: E731
    calc.step_meter({"outputs": {"box_corners": t("box_corners"), "sem_cls_prob": t("sem_cls_prob"),
                                 "objectness_prob": t("objectness_prob")}},
                    {"point_clouds": torch.from_numpy(bec.make_inputs(dataset_name)["point_clouds"]),
                     **{k: t(k) for k in bcc.GT_KEYS}})
    out = {}
    for thr, rd in calc.compute_metrics().items():
        keys = list(rd.keys())
        out[f"ap.{thr}.keys"] = np.array(keys)
        out[f"ap.{thr}.values"] = np.array([float(rd[k]) for k in keys], np.float64)
        print(dataset_name, f"IoU {thr}: mAP {float(rd['mAP']):.4f} AR {float(rd['AR']):.4f}", flush=True)
    return out


def run_reference(dataset_name):
    blob = mbeg.run_reference(dataset_name)
    m3, model = MODELS[-1]
    fg = model.cmp_text_features_fg
    path = m3.ALL_CMP_CLASS_PATH_SCANNET if "scannet" in dataset_name else m3.ALL_CMP_CLASS_PATH
    class_names = [str(n) for n in np.load(path, allow_pickle=True)]
    blob.update(cmp_prompts=np.array(model.all_cmp_classes_keys), cmp_class_names=np.array(class_names),
                cmp_text_features_fg_norm=(fg / fg.norm(dim=1, keepdim=True)).to(torch.float32).numpy())
    assert blob["sem_cls_prob"].shape[-1] == len(class_names)
    blob.update(zip(bcc.GT_KEYS, ground_truth(blob)))
    blob.update(ap_metrics(dataset_name, blob, class_names))
    # the same in the real-test golden, which the tests read them from
    for k in ("crop_features", "box_corners", "text_features_fg_norm", "prompts", "state_dict_keys", "trainable",
              "calib_K", "calib_pose"):
        blob.pop(k, None)
    return blob


def main():
    only = sys.argv[1:]
    for name in bcc.DATASETS:
        if only and name not in only:
            continue
        blob = run_reference(name)
        np.savez_compressed(bcc.golden_path(name), **blob)
        print("wrote", bcc.golden_path(name).name, "usable per scene", blob["usable"].sum(1), "classes",
              len(blob["cmp_prompts"]), flush=True)


if __name__ == "__main__":
    main()
