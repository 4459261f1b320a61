"""Generates tests/golden/trainable_grad_params.json: for each training configuration below, the names of the
REFERENCE model's parameters that require a gradient and the names of those that receive one in a training step
(forward, criterion, backward), run on CPU in this container through tests/golden/_reference_harness.py as
make_model_golden.py / make_scannet_golden.py run it.

`main.py` wraps the model in DistributedDataParallel(find_unused_parameters=False) whenever it runs on more than one
GPU.  That only works if every trainable parameter receives a gradient at every step; tests/test_grad_params_cpu.py
holds the package's model to the same sets.

    python tests/golden/make_grad_params_golden.py            (writes into tests/golden/)
"""
import json
import sys
from pathlib import Path

import numpy as np
import torch

HERE = Path(__file__).resolve().parent
ROOT = HERE.parents[1]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))
sys.path.insert(0, str(HERE))

import make_baseline_eval_golden as mbg  # noqa: E402
import make_model_golden as mmg  # noqa: E402
import make_scannet_golden as msg  # noqa: E402
import model_parity_common as mpc  # noqa: E402
from coda_neurips2023_b200 import synthetic  # noqa: E402
from param_fill import fill_by_name  # noqa: E402

H = mmg.H

# the configurations of tests/test_sync_bn_modules_gpu.py
CODA_CASES = ("stage1_small", "stage2_discovery", "masked_small")
SCANNET_CASES = ("scannet_stage1_small",)
BASELINE = "baseline_stage1_small"
# scripts/coda_baseline_sunrgbd.sh: the baseline trains on the box and class losses alone
BASELINE_ARGS = dict(mpc._SMALL, model_name="3detrmulticlasshead", loss_predicted_region_embed_l1_weight=0.0)


def grad_sets(model) -> dict:
    trainable = sorted(n for n, p in model.named_parameters() if p.requires_grad)
    with_grad = sorted(n for n, p in model.named_parameters() if p.requires_grad and p.grad is not None)
    return {"trainable": trainable, "with_grad": with_grad}


def run_baseline():
    """The baseline head (`--model_name 3detrmulticlasshead`) in a training step on the stage1_small batch."""
    args = mmg.reference_args(BASELINE_ARGS)
    args.if_only_novel_prompt = False
    crit_mod = H.load("criterion")
    _, model = mbg.reference_model(args)
    fill_by_name(model, seed=3)
    criterion = crit_mod.build_criterion(args, synthetic.SyntheticDatasetConfig(args))
    model.train()
    if hasattr(model, "clip_model"):
        model.clip_model.eval()
    inputs = {k: torch.from_numpy(v) for k, v in synthetic.make_batch(2, 3000, seed=5).items()}
    np.random.seed(123)
    out = model(inputs, curr_epoch=0)
    loss, _ = criterion(out, inputs)
    loss.backward()
    return model


def main():
    out = {}
    for name in CODA_CASES:
        _, model, _, _, _ = mmg.run_reference(name)
        out[name] = grad_sets(model)
        print(name, len(out[name]["trainable"]), "trainable,", len(out[name]["with_grad"]), "with a gradient", flush=True)
    for name in SCANNET_CASES:
        _, model, _, _, _, _ = msg.run_reference(name)
        out[name] = grad_sets(model)
        print(name, len(out[name]["trainable"]), "trainable,", len(out[name]["with_grad"]), "with a gradient", flush=True)
    out[BASELINE] = grad_sets(run_baseline())
    print(BASELINE, len(out[BASELINE]["trainable"]), "trainable,", len(out[BASELINE]["with_grad"]), "with a gradient")
    (HERE / "trainable_grad_params.json").write_text(json.dumps(out, indent=1) + "\n")


if __name__ == "__main__":
    main()
