"""Eval-mode inference cases (`main.py --test_only`: model.eval(), no_grad, forward(if_real_test=True)) shared by the
golden generator (tests/golden/make_model_eval_golden.py), the CPU plumbing test and the GPU parity test.  Weights
are filled by name (fill_by_name, seed 3, as the training goldens) and the BatchNorm running statistics by name
(running_stats_fill.fill_running_stats_by_name, seed 7), so that eval-mode BatchNorm normalises with non-trivial statistics."""
import numpy as np
import torch

import model_parity_common as mpc
from running_stats_fill import fill_running_stats_by_name

STATS_SEED = 7
# eval case -> training case whose shape, arguments and inputs it reuses
EVAL_CASES = {"eval_small": "stage1_small", "eval_full": "baseline_full"}

LAST_KEYS = ("sem_cls_prob", "objectness_prob", "sem_cls_logits", "center_normalized", "center_unnormalized",
             "size_normalized", "size_unnormalized", "angle_logits", "angle_residual", "angle_continuous",
             "box_corners", "box_corners_xyz")
AUX_KEYS = ("sem_cls_logits", "center_normalized")


def golden_path(name):
    return mpc.GOLDEN / f"model_{name}.npz"


def run(name: str, device: str):
    """OUR model in eval mode on `device` -> (outputs, golden)."""
    base = EVAL_CASES[name]
    args, model, _, inputs, _ = mpc.build(base, device)
    golden = np.load(golden_path(name))
    model.text_features_fg_norm = torch.from_numpy(golden["text_features_fg_norm"]).to(device)
    model.text_features_fg = model.text_features_fg_norm
    fill_running_stats_by_name(model, seed=STATS_SEED)
    model.eval()
    with torch.no_grad():
        out = model(inputs, if_real_test=True)
    return out, golden


def blob(out) -> dict:
    """The stored subset of an eval forward's outputs."""
    last = out["outputs"]
    b = {f"last.{k}": last[k].detach().float().cpu().numpy() for k in LAST_KEYS}
    for i, aux in enumerate(out["aux_outputs"]):
        for k in AUX_KEYS:
            b[f"aux{i}.{k}"] = aux[k].detach().float().cpu().numpy()
    return b


def compare(out, golden, rtol: float, atol: float) -> dict:
    """key -> max |ours - golden| / max |golden| over every stored key; raises when one exceeds rtol + atol / scale
    (the bar of model_parity_common.compare)."""
    ours = blob(out)
    assert set(ours) == {k for k in golden.files if k.startswith(("last.", "aux"))}, \
        sorted(set(ours) ^ {k for k in golden.files if k.startswith(("last.", "aux"))})
    errs = {}
    for k in sorted(ours):
        exp, got = golden[k], ours[k]
        assert got.shape == exp.shape, (k, got.shape, exp.shape)
        scale = max(float(np.abs(exp).max()), 1e-6)
        errs[k] = float(np.abs(got - exp).max()) / scale
        assert errs[k] <= rtol + atol / scale, f"{k}: max err {errs[k]:.3e} (scale {scale:.3e})"
    return errs
