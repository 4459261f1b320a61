"""The eval forward of a model converted by torch.nn.SyncBatchNorm.convert_sync_batchnorm (what the reference's main.py
does before it tests on more than one GPU, main.py:992-996) against the same model unconverted, on one GPU.

    python tools/bench_eval_sync_bn.py [--reps N]

Both arms run model.eval(), no_grad, forward(if_real_test=True) on 48 scenes of 20 000 points with 128 queries (the
test_release_models.sh batch), with the same weights and running statistics.  The two alternate, each going first
in every other round.  Prints JSON lines: the card (name, power limit, max SM clock), then per arm the median ms per
batch, peak allocated memory, the number of fused pre-encoder kernel calls per forward, and whether the two arms'
outputs are bit-identical."""
import argparse
import json
import sys
import warnings
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))
sys.path.insert(0, str(ROOT / "tools"))
from bench_eval import SCENES, card, event_ms, median  # noqa: E402
from coda_neurips2023_b200 import ops, sa_mlp, synthetic  # noqa: E402
from param_fill import fill_by_name  # noqa: E402
from running_stats_fill import fill_running_stats_by_name  # noqa: E402


def build():
    from coda_neurips2023_b200.models import build_model

    args = synthetic.make_args(nqueries=128)
    cfg = synthetic.SyntheticDatasetConfig(args)
    torch.manual_seed(0)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        model, _ = build_model(args, cfg)
    fill_by_name(model, seed=3)
    fill_running_stats_by_name(model, seed=7)
    return model.cuda().eval()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_eval_sync_bn.py needs a CUDA device")
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    print(json.dumps(card()), flush=True)
    models = {"plain": build(), "converted": torch.nn.SyncBatchNorm.convert_sync_batchnorm(build()).eval()}
    nsync = sum(isinstance(m, torch.nn.SyncBatchNorm) for m in models["converted"].modules())
    batch = synthetic.to_device(synthetic.make_batch(SCENES, 20000, seed=0), "cuda")
    calls = {"n": 0}
    real = sa_mlp.shared_mlp_max_infer

    def counted(*args, **kw):
        calls["n"] += 1
        return real(*args, **kw)

    sa_mlp.shared_mlp_max_infer = counted

    def run(tag):
        with torch.no_grad():
            out = models[tag](batch, if_real_test=True)["outputs"]
        ops._ACT_CACHE.clear()
        return out

    res = {}
    outs = {}
    for tag in models:                 # warm-up, then peak memory and kernel calls of one forward each
        run(tag)
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        calls["n"] = 0
        outs[tag] = run(tag)
        torch.cuda.synchronize()
        res[tag] = {"peak_gb": round(torch.cuda.max_memory_allocated() / 1e9, 2), "fused_calls": calls["n"], "ms": []}
    same = all(torch.equal(v, outs["converted"][k]) for k, v in outs["plain"].items() if isinstance(v, torch.Tensor))
    del outs
    for i in range(a.reps):
        order = ("plain", "converted") if i % 2 == 0 else ("converted", "plain")
        for tag in order:
            res[tag]["ms"].append(event_ms(lambda: run(tag)))
    print(json.dumps({"what": f"eval forward, {SCENES} scenes x 20000 points, 128 queries", "reps": a.reps,
                      "sync_batchnorm_modules": nsync, "outputs_bit_identical": same,
                      **{f"{tag}_ms_median": round(median(r["ms"]), 2) for tag, r in res.items()},
                      **{f"{tag}_ms_all": [round(x, 2) for x in r["ms"]] for tag, r in res.items()},
                      **{f"{tag}_peak_gb": r["peak_gb"] for tag, r in res.items()},
                      **{f"{tag}_fused_calls": r["fused_calls"] for tag, r in res.items()}}), flush=True)


if __name__ == "__main__":
    main()
