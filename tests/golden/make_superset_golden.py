"""Generates the goldens of --if_clip_superset from the REFERENCE's own Python code on CPU
(tests/golden/_reference_harness.py, small random-init CLIP of the reference's class, weights filled by name):

  superset_prompts.json           `superset_all_classes_keys` of the reference model (models/model_3detr.py:282-323)
                                  for the prompt flags of scripts/coda_sunrgbd_stage2.sh and coda_scannet_stage2.sh
  superset_tokens.npz             the reference tokenizer's rows (CLIP/clip/clip.py tokenize) of every such prompt
  model_stage2_superset.npz,      the reference model + criterion run of the cases of tests/superset_common.py, with
  model_scannet_stage2_superset.npz   the keys of make_model_golden.py plus the superset text features

lvis_1204.npy is the reference's datasets/lvis_1204.npy, copied as a data fixture.

    python tests/golden/make_superset_golden.py [prompts] [case ...]          (writes into tests/golden/)
"""
import json
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
import superset_common as ssc  # noqa: E402
from coda_neurips2023_b200 import synthetic  # noqa: E402
from param_fill import fill_by_name  # noqa: E402


def reference_model(over, cfg_cls=synthetic.SyntheticDatasetConfig):
    args = mmg.reference_args(over)
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
    torch.manual_seed(0)
    model, _ = m3.build_3detr_predictedbox_distillation_head(args, cfg_cls(args))
    return args, model


def prompts():
    clip_pkg = H.load("CLIP.clip.clip")
    out, flags, tokens = {}, {}, {}
    for name, over in ssc.FLAGS.items():
        _, model = reference_model(dict(mmg.mpc._SMALL, **over))
        out[name] = list(model.superset_all_classes_keys)
        flags[name] = over
        tokens[name] = clip_pkg.tokenize(out[name]).numpy().astype(np.int32)
    out["flags"] = flags
    (HERE / "superset_prompts.json").write_text(json.dumps(out, indent=1) + "\n")
    np.savez_compressed(HERE / "superset_tokens.npz", **tokens)
    print({k: len(v) for k, v in out.items() if k != "flags"})


def run_reference(name):
    dataset, batch, npoints, over, extra = ssc.CASES[name]
    box_util = H.load("utils.box_util")
    crit_mod = H.load("criterion")

    class Cfg(synthetic.SyntheticDatasetConfig):  # corner builders of the REFERENCE
        def box_parametrization_to_corners(self, c, s, a):
            return box_util.get_3d_box_batch_tensor(s, a, box_util.flip_axis_to_camera_tensor(c))

        def box_parametrization_to_corners_xyz(self, c, s, a):
            return box_util.get_3d_box_batch_tensor_xyz(s, a, c)

    args, model = reference_model(over, Cfg)
    cfg = Cfg(args)
    fill_by_name(model, seed=3)
    with torch.no_grad():   # text features of the reference's own prompts, from the filled CLIP (its :356-360)
        def enc(tokens):
            f = model.clip_model.encode_text(tokens).to(torch.float32)
            return (f / f.norm(dim=1, keepdim=True)).to(torch.float32)

        model.text_features_fg_norm = enc(model.text)
        model.text_features_fg = model.text_features_fg_norm
        model.superset_text_features_fg_norm = enc(model.superset_text)
        model.test_text_features_fg_norm = model.superset_text_features_fg_norm
    criterion = crit_mod.build_criterion(args, cfg)
    model.train()
    model.clip_model.eval()
    inputs = {k: torch.from_numpy(v) for k, v in ssc.batch_np(name).items()}
    tmp = tempfile.mkdtemp(prefix="coda_pseudo_ref_")
    paths = inputs["pseudo_box_path"] = [f"{tmp}/scene{i}.npy" for i in range(batch)]
    np.random.seed(123)  # box selection draws (model_3detr.py:991)
    out = model(inputs, curr_epoch=0)
    loss, loss_dict = criterion(out, inputs)
    loss.backward()
    return args, model, out, loss, loss_dict, paths


def case(name):
    args, model, out, loss, loss_dict, paths = run_reference(name)
    last = out["outputs"]
    blob = {f"last.{k}": last[k].detach().numpy() for k in mmg.KEEP}
    blob["last.text_correlation_embedding"] = last["text_correlation_embedding"].detach().numpy()[:, ::4, ::8]
    blob["last.gt_text_correlation_embedding"] = last["gt_text_correlation_embedding"].numpy()[:, :, ::8]
    blob["last.gt_text_correlation_embedding_mask"] = last["gt_text_correlation_embedding_mask"].numpy()
    blob["last.weak_box_cate_label"] = last["weak_box_cate_label"].numpy()
    blob["last.weak_confidence_weight"] = last["weak_confidence_weight"].numpy()
    blob["text_features_fg_norm"] = model.text_features_fg_norm.numpy()
    # every 4th row and column of the (C, 512) superset features (make_model_golden.thin)
    blob["superset_text_features_fg_norm"] = mmg.thin(model.superset_text_features_fg_norm.numpy())
    for i, aux in enumerate(out["aux_outputs"]):
        blob[f"aux{i}.sem_cls_logits"] = aux["sem_cls_logits"].detach().numpy()
        blob[f"aux{i}.center_normalized"] = aux["center_normalized"].detach().numpy()
    arrs = [np.load(p) if os.path.exists(p) else np.zeros((0, 10), np.float32) for p in paths]
    blob["pseudo.count"] = np.array([len(a) for a in arrs], np.int64)
    blob["pseudo.rows"] = np.concatenate(arrs, axis=0).astype(np.float32).reshape(-1, 10)
    print("pseudo labels per scene:", blob["pseudo.count"], flush=True)
    blob["loss"] = np.float32(loss.item())
    for k, v in loss_dict.items():
        blob[f"loss_dict.{k}"] = np.float32(float(v))
    blob["state_dict_keys"] = np.array(sorted(k for k in model.state_dict().keys() if "clip_model" not in k))
    g = dict(model.named_parameters())
    for pname in (mmg.GRADS[0], mmg.GRADS[2], mmg.GRADS[7], mmg.GRADS[10], mmg.GRADS[11], mmg.GRADS[13]):
        pname = pname.format(last=args.dec_nlayers - 1)
        blob[f"grad.{pname}"] = mmg.thin(g[pname].grad.numpy())
    np.savez_compressed(HERE / f"model_{name}.npz", **blob)
    print("wrote", name, "loss", float(loss), flush=True)


def main():
    only = sys.argv[1:]
    if not only or "prompts" in only:
        prompts()
    for name in ssc.CASES:
        if not only or name in only:
            case(name)


if __name__ == "__main__":
    main()
