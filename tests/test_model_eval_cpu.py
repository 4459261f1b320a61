"""CPU (no GPU) plumbing parity of eval-mode inference: OUR model's Python, with the CUDA ops replaced by the CPU
stand-ins of oracle/cpu_step.py, in eval mode (running-statistics BatchNorm) under no_grad with
forward(if_real_test=True), against the REFERENCE model run the same way on CPU
(tests/golden/make_model_eval_golden.py).  Pins the eval wiring and the goldens the GPU parity test uses."""
import pytest
import torch

import cpu_step as cpu_shims
import model_eval_common as mec


@pytest.mark.parametrize("name", list(mec.EVAL_CASES))
def test_eval_forward_matches_reference_on_cpu(name):
    torch.manual_seed(0)
    with cpu_shims.installed():
        out, golden = mec.run(name, "cpu")
    errs = mec.compare(out, golden, rtol=2e-4, atol=1e-5)
    worst = max(errs, key=errs.get)
    print(f"{name}: worst {worst} = {errs[worst]:.2e}")
