"""Generates tests/golden/model_scannet_*.npz from the REFERENCE's own Python model and criterion on CPU, for the
ScanNet cases of tests/scannet_parity_common.py: the same procedure and stored keys as make_model_golden.py (reference
imported through _reference_harness.py, small random-init CLIP, weights filled by name), with ScanNet batches from
coda_neurips2023_b200.synthetic (camera="scannet").  The reference picks scannet_utils for the projection from the
dataset name (models/model_3detr.py:461-466).  Every case, the full-size one included, stores the small key set
(last layer, aux class / centre heads, five gradients) to keep the file small.  For the full-size case it also
writes model_<case>_cpu_noise.json, as make_cpu_noise.py does for the SUN RGB-D cases: how far OUR model run through
the CPU restatement sits from the golden, per key (the GPU parity test widens a gradient's bar to 4 x this).

    python tests/golden/make_scannet_golden.py [case ...]          (writes into tests/golden/)
"""
import os
import sys
import tempfile
from pathlib import Path

import numpy as np
import torch

HERE = Path(__file__).resolve().parent
ROOT = HERE.parents[1]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))
sys.path.insert(0, str(HERE))

import _reference_harness as H  # noqa: E402
import make_model_golden as mmg  # noqa: E402
import scannet_parity_common as spc  # noqa: E402
from coda_neurips2023_b200 import synthetic  # noqa: E402
from param_fill import fill_by_name  # noqa: E402


def run_reference(name):
    batch, npoints, over, extra = spc.CASES[name]
    args = mmg.reference_args(over)
    m3 = H.load("models.model_3detr")
    crit_mod = H.load("criterion")
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
        model = clip_model_mod.CLIP(**mmg.TINY_CLIP).float().eval()
        fill_by_name(model, seed=11)
        return model, clip_pkg._transform_for_tensor(model.visual.input_resolution)

    clip_pkg.load = fake_clip_load
    sys.modules["CLIP.clip"].clip.load = fake_clip_load
    torch.manual_seed(0)
    model, _ = m3.build_3detr_predictedbox_distillation_head(args, cfg)
    fill_by_name(model, seed=3)
    with torch.no_grad():   # text features of the reference's own ScanNet prompts, from the filled CLIP
        model.text_features_fg = model.clip_model.encode_text(model.text).to(torch.float32)
        model.text_features_fg_norm = model.text_features_fg / model.text_features_fg.norm(dim=1, keepdim=True)
    criterion = crit_mod.build_criterion(args, cfg)
    model.train()
    model.clip_model.eval()
    inputs = {k: torch.from_numpy(v) for k, v in spc.batch_np(name).items()}
    paths = None
    if extra.get("pseudo"):
        tmp = tempfile.mkdtemp(prefix="coda_pseudo_ref_")
        paths = inputs["pseudo_box_path"] = [f"{tmp}/scene{i}.npy" for i in range(batch)]
    np.random.seed(123)  # box selection draws (model_3detr.py:991)
    out = model(inputs, curr_epoch=0)
    loss, loss_dict = criterion(out, inputs)
    loss.backward()
    return args, model, out, loss, loss_dict, paths


def main():
    only = sys.argv[1:]
    for name in spc.CASES:
        if only and name not in only:
            continue
        args, model, out, loss, loss_dict, paths = run_reference(name)
        last = out["outputs"]
        blob = {f"last.{k}": last[k].detach().numpy() for k in mmg.KEEP}
        blob["last.text_correlation_embedding"] = last["text_correlation_embedding"].detach().numpy()[:, ::4, ::8]
        blob["last.gt_text_correlation_embedding"] = last["gt_text_correlation_embedding"].numpy()[:, :, ::8]
        blob["last.gt_text_correlation_embedding_mask"] = last["gt_text_correlation_embedding_mask"].numpy()
        blob["last.weak_box_cate_label"] = last["weak_box_cate_label"].numpy()
        blob["last.weak_confidence_weight"] = last["weak_confidence_weight"].numpy()
        blob["text_features_fg_norm"] = model.text_features_fg_norm.numpy()
        for i, aux in enumerate(out["aux_outputs"]):
            blob[f"aux{i}.sem_cls_logits"] = aux["sem_cls_logits"].detach().numpy()
            blob[f"aux{i}.center_normalized"] = aux["center_normalized"].detach().numpy()
        if paths:
            arrs = [np.load(p) if os.path.exists(p) else np.zeros((0, 10), np.float32) for p in paths]
            blob["pseudo.count"] = np.array([len(a) for a in arrs], np.int64)
            blob["pseudo.rows"] = np.concatenate(arrs, axis=0).astype(np.float32).reshape(-1, 10)
            print("pseudo labels per scene:", blob["pseudo.count"], flush=True)
        blob["loss"] = np.float32(loss.item())
        for k, v in loss_dict.items():
            blob[f"loss_dict.{k}"] = np.float32(float(v))
        blob["state_dict_keys"] = np.array(sorted(k for k in model.state_dict().keys() if "clip_model" not in k))
        g = dict(model.named_parameters())
        for pname in (mmg.GRADS[0], mmg.GRADS[2], mmg.GRADS[7], mmg.GRADS[10], mmg.GRADS[13]):
            pname = pname.format(last=args.dec_nlayers - 1)
            blob[f"grad.{pname}"] = mmg.thin(g[pname].grad.numpy())
        np.savez_compressed(HERE / f"model_{name}.npz", **blob)
        print("wrote", name, "loss", float(loss), flush=True)
        if name in spc.FULL_SIZE:
            write_cpu_noise(name)


def write_cpu_noise(name):
    import json
    import subprocess

    # in a fresh interpreter: this one has the reference's modules and stubs installed
    code = f"""
import json, sys, torch
sys.path[:0] = [{str(ROOT)!r}, {str(ROOT / "tests")!r}, {str(ROOT / "oracle")!r}]
import model_parity_common as mpc, scannet_parity_common as spc, scannet_ref
torch.manual_seed(0)
with scannet_ref.installed():
    model, out, loss, ld, golden = spc.run({name!r}, "cpu")
    errs = mpc.compare(model, out, loss, ld, golden, rtol=1.0, atol=1e-5, grad_rtol=1.0)
print(json.dumps({{k: float(f"{{v:.3e}}") for k, v in sorted(errs.items())}}))
"""
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, check=True)
    errs = json.loads(r.stdout.strip().splitlines()[-1])
    (HERE / f"model_{name}_cpu_noise.json").write_text(json.dumps(errs, indent=0))
    print(name, "cpu noise: worst", max(errs, key=errs.get), max(errs.values()), flush=True)


if __name__ == "__main__":
    main()
