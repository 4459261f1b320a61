"""Generates tests/golden/model_baseline_clip_eval_{sunrgbd,scannet}.npz: the REFERENCE's 3DETR + CLIP baseline head
(Model3DETRMultiClassHead) run on CPU in this container the way make_model_eval_golden.py runs the CoDA head
(tests/golden/_reference_harness.py): weights filled by name, BatchNorm running statistics filled by name, the small
random-init CLIP, model.eval(), forward(inputs, if_real_test=True) under no_grad -- the path of
`main.py --model_name 3detrmulticlasshead --if_with_clip --test_only`.

SUN RGB-D (`sunrgbd_image`): SUNRGBD_Calibration is backed by the batch's K / Rtilt (the dataset reads both from the
same calibration file).  ScanNet (`scannet50_image`): the synthetic camera is written as intrinsic/intrinsic_color.txt
and pose/<squence_name>.txt files under tests/golden/baseline_eval_scannet/, the batch carries no K / Rtilt, and the
reference's own SCANNET_Calibration reads those files.  In both, the third scene's camera looks away from the room,
so it has no usable box; the others have boxes inside the image, boxes clipped at an edge, boxes behind the camera
and (through a hook on the size prediction) zero-size boxes.  Besides the outputs it stores what the reference
computes per box on the way: the integer 2-D box, whether the box was classified, the CLIP features of the crops, the
prompt list, the state-dict keys and trainable parameters, and for ScanNet the matrices read from the files.

    python tests/golden/make_baseline_eval_golden.py [sunrgbd_image] [scannet50_image]    (writes into tests/golden/)
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

import baseline_eval_common as bec  # noqa: E402
import make_model_golden as mmg  # noqa: E402
import model_parity_common as mpc  # noqa: E402
from coda_neurips2023_b200 import synthetic  # noqa: E402
from param_fill import fill_by_name  # noqa: E402
from running_stats_fill import fill_running_stats_by_name  # noqa: E402

H = mmg.H


def reference_model(args):
    m3 = H.load("models.model_3detr")
    box_util = H.load("utils.box_util")
    clip_pkg = H.load("CLIP.clip.clip")
    clip_model_mod = H.load("CLIP.clip.model")

    class Cfg(synthetic.SyntheticDatasetConfig):  # corner builders of the REFERENCE
        def box_parametrization_to_corners(self, c, s, a):
            return box_util.get_3d_box_batch_tensor(s, a, box_util.flip_axis_to_camera_tensor(c))

        def box_parametrization_to_corners_xyz(self, c, s, a):
            return box_util.get_3d_box_batch_tensor_xyz(s, a, c)

    def fake_clip_load(path, device="cpu", download_root=None, if_transform_tensor=True, **kw):
        torch.manual_seed(0)
        model = clip_model_mod.CLIP(**mpc.TINY_CLIP).float().eval()
        fill_by_name(model, seed=11)
        return model, clip_pkg._transform_for_tensor(model.visual.input_resolution)

    clip_pkg.load = fake_clip_load
    sys.modules["CLIP.clip"].clip.load = fake_clip_load
    torch.manual_seed(0)
    model, _ = m3.build_3detr_multiclasshead(args, Cfg(args))
    return m3, model


def _write_matrix(path, m):
    path.parent.mkdir(parents=True, exist_ok=True)
    path.write_text("".join(" ".join(repr(float(x)) for x in row) + "\n" for row in m))


def write_scannet_calibration(batch):
    """The synthetic ScanNet camera of each scene as the files a ScanNet checkout holds:
    <calib>/intrinsic/intrinsic_color.txt and <calib>/pose/<squence_name>.txt."""
    for b in range(bec.BATCH):
        calib = bec.scannet_calib_dir(b)
        _write_matrix(calib / "intrinsic" / "intrinsic_color.txt", batch["K"][b])
        _write_matrix(calib / "pose" / f"{bec.squence_name(b)}.txt", batch["Rtilt"][b])


def run_reference(dataset_name):
    args = bec.reference_args(dataset_name)
    m3, model = reference_model(args)
    fill_by_name(model, seed=3)
    fill_running_stats_by_name(model, seed=bec.STATS_SEED)
    with torch.no_grad():    # re-derive the text features from the filled CLIP, as the constructor does (:2088-2090)
        model.text_features_fg = model.clip_model.encode_text(model.text)
        model.text_features_fg_norm = (model.text_features_fg / model.text_features_fg.norm(dim=1, keepdim=True)
                                       ).to(torch.float32)
    model.eval()
    bec.zero_sizes(model.box_processor)
    scannet = "scannet" in dataset_name
    batch = bec.make_inputs(dataset_name)
    inputs = {k: torch.from_numpy(v) for k, v in batch.items()}
    inputs["im_name"] = [f"scene{b}.jpg" for b in range(bec.BATCH)]
    inputs["trans_mtx"] = torch.eye(2, dtype=torch.float64).repeat(bec.BATCH, 1, 1)
    calibs = []
    if scannet:
        write_scannet_calibration(batch)
        inputs.update(bec.scannet_names())
        for k in ("K", "Rtilt"):          # a ScanNet test batch has neither: the calibration comes from the files
            del inputs[k]
        util = m3.scannet_utils

        class RecordingCalibration(util.SCANNET_Calibration):
            def __init__(self, *a, **kw):
                super().__init__(*a, **kw)
                calibs.append((self.K.copy(), self.Rtilt.copy()))

        util.SCANNET_Calibration = RecordingCalibration
    else:
        inputs["calib_name"] = [f"scene{b}" for b in range(bec.BATCH)]
        util = m3.sunrgbd_utils

        class BatchCalibration(util.SUNRGBD_Calibration):
            def __init__(self, calib_name, if_tensor=True):
                b = int(calib_name[len("scene"):])
                self.Rtilt, self.K = inputs["Rtilt"][b].numpy(), inputs["K"][b].numpy()
                self.Rtilt_tensor = torch.from_numpy(self.Rtilt).to(torch.float32)
                self.K_tensor = torch.from_numpy(self.K).to(torch.float32)
                self.f_u, self.f_v, self.c_u, self.c_v = self.K[0, 0], self.K[1, 1], self.K[0, 2], self.K[1, 2]

        util.SUNRGBD_Calibration = BatchCalibration
    projected, feats = [], []
    project = util.compute_box_3d_offset_tensor

    def recording_project(*a):
        r = project(*a)
        projected.append((r[0].clone(), r[2].clone()))
        return r

    util.compute_box_3d_offset_tensor = recording_project
    encode = model.clip_model.encode_image

    def recording_encode(x):
        f = encode(x)
        feats.append((f[0] if isinstance(f, tuple) else f).to(torch.float32).clone())
        return f

    model.clip_model.encode_image = recording_encode
    with torch.no_grad():
        out = model(inputs, if_real_test=True)
    last = out["outputs"]
    bsz, nq = last["sem_cls_prob"].shape[:2]
    sizes = last["size_unnormalized"]
    # the integer boxes and the usability test of reference :2926-2985, from the projected corners; a box whose
    # size is below 1e-16 is skipped before it is projected (its box stays -1)
    boxes = np.full((bsz, nq, 4), -1, np.int32)
    usable = np.zeros((bsz, nq), bool)
    calls = iter(projected)
    for b in range(bsz):
        for q in range(nq):
            if torch.max(sizes[b, q]) < 1e-16:
                continue
            uv, d = next(calls)
            xo, yo = inputs["x_offset"][b], inputs["y_offset"][b]
            w, h = inputs["ori_width"][b], inputs["ori_height"][b]
            xmin = int(min(max(torch.min(uv[:, 0]), yo), w + yo))
            ymin = int(min(max(torch.min(uv[:, 1]), xo), h + xo))
            xmax = int(min(max(torch.max(uv[:, 0]), yo), w + yo))
            ymax = int(min(max(torch.max(uv[:, 1]), xo), h + xo))
            boxes[b, q] = (xmin, ymin, xmax, ymax)
            usable[b, q] = not (torch.min(d) < 0) and xmax - xmin > 0 and ymax - ymin > 0
    assert next(calls, None) is None
    prob = last["sem_cls_prob"].numpy()
    assert np.array_equal(usable, prob.sum(-1) > 0), "the reference classified other boxes than its tests pass"
    blob = {
        "usable": usable, "boxes": boxes,
        "crop_features": torch.cat(feats).numpy() if feats else np.zeros((0, 512), np.float32),
        "sem_cls_prob": prob,
        "sem_cls_logits": last["sem_cls_logits"].numpy(),
        "objectness_prob": last["objectness_prob"].numpy(),
        "box_corners": last["box_corners"].numpy(),
        "text_features_fg_norm": model.text_features_fg_norm.numpy(),
        "logit_scale": np.float32(model.logit_scale),
        "state_dict_keys": np.array(sorted(k for k in model.state_dict() if not k.startswith("clip_model."))),
        "trainable": np.array(sorted(k for k, p in model.named_parameters() if p.requires_grad)),
        "prompts": np.array(model.all_classes_keys),
    }
    if scannet:     # the matrices the reference's SCANNET_Calibration read from the files, one per scene
        blob["calib_K"] = np.stack([k for k, _ in calibs])
        blob["calib_pose"] = np.stack([p for _, p in calibs])
    return blob


def main():
    only = sys.argv[1:]
    for name in bec.DATASET_ARGS:
        if only and name not in only:
            continue
        blob = run_reference(name)
        np.savez_compressed(bec.golden_path(name), **blob)
        print("wrote", bec.golden_path(name).name, "usable per scene", blob["usable"].sum(1), "prompts",
              len(blob["prompts"]), flush=True)


if __name__ == "__main__":
    main()
