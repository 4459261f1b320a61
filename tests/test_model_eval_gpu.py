"""GPU parity of eval-mode inference (`main.py --test_only`: model.eval(), no_grad, forward(if_real_test=True)): OUR
model on the H100 against the REFERENCE run the same way on CPU (tests/golden/make_model_eval_golden.py), the
pre-encoder's inference kernel against the module path it replaces at 48 scenes, and engine.evaluate end to end."""
import warnings

import pytest
import torch

import model_eval_common as mec
from coda_neurips2023_b200 import sa_mlp, synthetic
from param_fill import fill_by_name
from running_stats_fill import fill_running_stats_by_name

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module", autouse=True)
def _lib(built_lib):
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False


@pytest.fixture
def kernel_calls(monkeypatch):
    """counts the calls of the pre-encoder's inference kernel"""
    calls = []
    real = sa_mlp.shared_mlp_max_infer
    monkeypatch.setattr(sa_mlp, "shared_mlp_max_infer", lambda *a: calls.append(1) or real(*a))
    return calls


@pytest.mark.parametrize("name", list(mec.EVAL_CASES))
def test_eval_forward_matches_reference_golden(name, kernel_calls):
    torch.manual_seed(0)
    out, golden = mec.run(name, "cuda")
    assert len(kernel_calls) == 1, "the eval forward must take the pre-encoder's inference kernel"
    errs = mec.compare(out, golden, rtol=1e-4, atol=1e-5)
    worst = max(errs, key=errs.get)
    print(f"PARITY {name}: worst {worst} = {errs[worst]:.2e} (bar 1e-4 relative)")


BATCH = 48


@pytest.fixture(scope="module")
def batch48():
    """the released-model evaluation shape: 48 scenes of 20 000 points, 2048 seeds, 128 queries"""
    args = synthetic.make_args(nqueries=128)
    cfg = synthetic.SyntheticDatasetConfig(args)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        from coda_neurips2023_b200.models import build_model

        model, _ = build_model(args, cfg)
    fill_by_name(model, seed=3)
    fill_running_stats_by_name(model, seed=mec.STATS_SEED)
    model = model.cuda().eval()
    batches = [synthetic.to_device(synthetic.make_batch(BATCH, 20000, seed=s), "cuda") for s in (0, 1)]
    return args, cfg, model, batches


def test_batch48_eval_matches_the_module_path(batch48, kernel_calls, monkeypatch):
    _, _, model, batches = batch48
    with torch.no_grad():
        fused = model(batches[0], if_real_test=True)
        assert len(kernel_calls) == 1
        monkeypatch.setattr(sa_mlp, "infer_applicable", lambda *a: False)
        plain = model(batches[0], if_real_test=True)
        assert len(kernel_calls) == 1
    worst = 0.0
    for k in mec.LAST_KEYS:
        a, b = fused["outputs"][k].float(), plain["outputs"][k].float()
        err = (a - b).abs().max().item() / max(b.abs().max().item(), 1e-6)
        worst = max(worst, err)
        assert err <= 1e-4, f"{k}: {err:.2e}"
    for i, (fa, pa) in enumerate(zip(fused["aux_outputs"], plain["aux_outputs"])):
        for k in mec.AUX_KEYS:
            err = (fa[k] - pa[k]).abs().max().item() / max(pa[k].abs().max().item(), 1e-6)
            worst = max(worst, err)
            assert err <= 1e-4, f"aux{i}.{k}: {err:.2e}"
    print(f"PARITY eval batch {BATCH}: kernel vs module path, worst {worst:.2e} (bar 1e-4)")


def test_engine_evaluate_runs_two_batches_of_48(batch48, kernel_calls):
    from coda_neurips2023_b200 import engine

    args, cfg, model, batches = batch48
    calc = engine.evaluate(args, 0, model, None, cfg, batches, if_real_test=True)
    assert len(kernel_calls) == 2
    assert len(calc._scores) == 2 and calc._scores[0].shape[0] == BATCH
    ret = calc.compute_metrics()
    assert "mAP" in ret[0.25] and "mAP" in ret[0.5]
