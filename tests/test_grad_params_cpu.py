"""Every trainable parameter receives a gradient in a training step, as in the reference (no GPU needed).

`main.py` wraps the model in DistributedDataParallel(find_unused_parameters=False) whenever it runs on more than one
GPU, and DDP then raises at the next step if a trainable parameter got no gradient.  tests/golden/
trainable_grad_params.json records, for each configuration, the reference model's trainable parameters and those that
receive a gradient (tests/golden/make_grad_params_golden.py); OUR model, run through the CPU stand-ins of
oracle/cpu_step.py, must give the same two sets."""
import json
import warnings

import numpy as np
import pytest
import torch

import cpu_step as cpu_shims
import model_parity_common as mpc
import scannet_parity_common as spc
import scannet_ref

GOLDEN = json.loads((mpc.GOLDEN / "trainable_grad_params.json").read_text())
BASELINE_ARGS = dict(mpc._SMALL, model_name="3detrmulticlasshead", loss_predicted_region_embed_l1_weight=0.0)


def _grad_sets(model):
    trainable = sorted(n for n, p in model.named_parameters() if p.requires_grad)
    with_grad = sorted(n for n, p in model.named_parameters() if p.requires_grad and p.grad is not None)
    return {"trainable": trainable, "with_grad": with_grad}


def _run_baseline():
    from coda_neurips2023_b200 import synthetic
    from coda_neurips2023_b200.criterion import build_criterion
    from coda_neurips2023_b200.models import build_model

    args = synthetic.make_args(**BASELINE_ARGS)
    cfg = synthetic.SyntheticDatasetConfig(args)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        model, _ = build_model(args, cfg)
    model.device = "cpu"
    criterion = build_criterion(args, cfg)
    model.train()
    if hasattr(model, "clip_model"):
        model.clip_model.eval()
    inputs = synthetic.to_device(synthetic.make_batch(2, 3000, seed=5), "cpu")
    np.random.seed(123)
    out = model(inputs, curr_epoch=0)
    loss, _ = criterion(out, inputs)
    loss.backward()
    return model


@pytest.mark.parametrize("name", list(GOLDEN))
def test_every_trainable_parameter_gets_a_gradient_as_in_the_reference(name):
    torch.manual_seed(0)
    if name in spc.CASES:
        with scannet_ref.installed():          # the CPU stand-ins with the ScanNet camera
            model = spc.run(name, "cpu")[0]
    else:
        with cpu_shims.installed():
            model = mpc.run(name, "cpu")[0] if name in mpc.CASES else _run_baseline()
    got, exp = _grad_sets(model), GOLDEN[name]
    assert got["trainable"] == exp["trainable"], (sorted(set(got["trainable"]) ^ set(exp["trainable"])))
    assert got["with_grad"] == exp["with_grad"], (sorted(set(got["with_grad"]) ^ set(exp["with_grad"])))
    assert got["with_grad"] == got["trainable"], "a trainable parameter gets no gradient: DDP would raise"
