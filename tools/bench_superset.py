"""Cost of the --if_clip_superset contrastive loss on the GPU, in one command:

  1. the loss alone, forward + backward, at R = 8192 embedding rows (8 scenes x 128 queries x 8 decoder layers) and
     C = 1201 superset rows: the shared-text path (ops.text_contrastive_ce: wgmma GEMM + coda_text_ce_fwd / _bwd)
     against the ATen path (normalise, fp32 bmm against the per-layer, per-scene repeated text, scale, cross-entropy),
     alternated, CUDA events; then each of its four kernels alone (GEMM forward, row forward, row backward, GEMM
     backward) with achieved FLOP/s and bytes/s;
  2. the graph-replayed stage-2 superset step at the script's shape (8 scenes x 20 000 points, 128 queries,
     distillation_box_num 32, random-init ViT-B/16, weak labels and discovery on, a non-discovery epoch): the same
     model with the criterion built with and without if_clip_superset, alternated rounds in one process.

    python tools/bench_superset.py --out DIR"""
import argparse
import copy
import json
import os
import subprocess
import sys
import tempfile
import warnings
from pathlib import Path

import numpy as np
import torch
import torch.nn.functional as F

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
from coda_neurips2023_b200 import ops, synthetic  # noqa: E402
from coda_neurips2023_b200._lib import check, lib  # noqa: E402
from coda_neurips2023_b200.criterion import build_criterion  # noqa: E402
from coda_neurips2023_b200.engine import TrainStep  # noqa: E402
from coda_neurips2023_b200.models import build_model  # noqa: E402

ROWS, C, D = 8192, 1201, 512
LAYERS, SCENES = 8, 8


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def timed(fn, n):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def stats(xs):
    xs = sorted(xs)
    return {"median_ms": xs[len(xs) // 2], "min_ms": xs[0], "max_ms": xs[-1]}


def loss_alone(rounds, iters):
    g = torch.Generator().manual_seed(0)
    t = torch.randn(C, D, generator=g)
    t = (t / t.norm(dim=1, keepdim=True)).cuda()
    e0 = torch.randn(ROWS, D, generator=g).cuda()
    label = torch.randint(0, C, (ROWS,), generator=g).cuda()
    w = (torch.rand(ROWS, generator=g) > 0.3).float().cuda()
    scale = torch.tensor([100.0], device="cuda")
    e = e0.clone().requires_grad_(True)

    def new():
        e.grad = None
        ops.text_contrastive_ce(e, t, label, w, scale).sum().backward()

    def aten():
        e.grad = None
        text = t.unsqueeze(0).expand(SCENES, -1, -1).repeat(LAYERS, 1, 1)          # model repeat + criterion repeat
        en = e / (e.norm(dim=-1, keepdim=True) + 1e-32)
        corr = torch.bmm(en.view(LAYERS * SCENES, -1, D), text.permute(0, 2, 1)) * scale
        (F.cross_entropy(corr.transpose(2, 1), label.view(LAYERS * SCENES, -1), reduction="none")
         * w.view(LAYERS * SCENES, -1)).sum().backward()

    for fn in (new, aten):
        timed(fn, 3)
    res = {"new": [], "aten": []}
    for _ in range(rounds):
        res["new"].append(timed(new, iters))
        res["aten"].append(timed(aten, iters))

    # the four kernels of the new path, each alone
    tp = ops._rows_padded4(t)
    ld = tp.shape[0]
    planes = ops._packed_weight(tp, False, ops.DEFAULT_NSPLIT)
    s = torch.empty(ROWS, ld, device="cuda")
    loss, lse, inv = (torch.empty(ROWS, device="cuda") for _ in range(3))
    gout = torch.ones(ROWS, device="cuda")
    ds, dn = torch.empty_like(s), torch.empty_like(e0)
    from coda_neurips2023_b200.ops import _i, _ll, ptr, stream_of

    def gemm_fwd():
        ops.gemm_a32(e0, planes, ld, out=s)

    def row_fwd():
        check(lib().coda_text_ce_fwd(_ll(ROWS), _i(C), _i(ld), _i(D), ptr(s), ptr(e0), ptr(label), ptr(w), ptr(scale),
                                     ptr(loss), ptr(lse), ptr(inv), stream_of(s)), "text_ce_fwd")

    def row_bwd():
        check(lib().coda_text_ce_bwd(_ll(ROWS), _i(C), _i(ld), _i(D), ptr(s), ptr(e0), ptr(label), ptr(w), ptr(scale),
                                     ptr(lse), ptr(inv), ptr(gout), ptr(ds), ptr(dn), stream_of(s)), "text_ce_bwd")

    def gemm_bwd():
        ops.gemm_a32(ds, planes, D, b_mn=True, nsplit=ops.BACKWARD_NSPLIT)

    flop = 2.0 * ROWS * C * D
    sbytes, ebytes = 4.0 * ROWS * ld, 4.0 * ROWS * D
    parts = {}
    for name, fn, kind, amount in (("gemm_fwd", gemm_fwd, "flop", flop), ("row_fwd", row_fwd, "bytes", sbytes + ebytes),
                                   ("row_bwd", row_bwd, "bytes", 2 * sbytes + 2 * ebytes),
                                   ("gemm_bwd", gemm_bwd, "flop", flop)):
        timed(fn, 3)
        ms = sorted(timed(fn, iters) for _ in range(rounds))[rounds // 2]
        rate = amount / (ms * 1e-3)
        parts[name] = {"median_ms": ms, kind: amount,
                       ("TFLOP_per_s" if kind == "flop" else "TB_per_s"): rate / 1e12}
    return {"new": stats(res["new"]), "aten": stats(res["aten"]), "kernels": parts,
            "shape": {"rows": ROWS, "C": C, "D": D, "ld": ld}}


def step_times(rounds, iters):
    args = synthetic.make_args(
        dataset_name="sunrgbd_anonymous_aligned_image_with_novel_cate_confi", nqueries=128, train_range_max=10,
        test_range_max=46, if_clip_superset=True, if_clip_weak_labels=True,
        loss_feat_seen_softmax_weakly_loss_with_novel_cate_confi_weight=1.0, confidence_type="non-confidence",
        online_nms_update_save_novel_label_clip_driven_with_cate_confidence=True, save_objectness=0.3,
        clip_driven_keep_thres=0.3, online_nms_update_save_epoch=50, distillation_box_num=32, clip_arch="ViT-B/16")
    cfg = synthetic.SyntheticDatasetConfig(args)
    aten_args = copy.copy(args)
    aten_args.if_clip_superset = False            # the criterion only: the model still hands out the superset
    tmp = tempfile.mkdtemp(prefix="coda_superset_bench_")
    batch = synthetic.to_device(synthetic.make_batch(SCENES, 20000, seed=40), "cuda")
    batch["pseudo_box_path"] = [f"{tmp}/scene{i}.npy" for i in range(SCENES)]
    steps = {}
    for arm, cargs in (("new", args), ("aten", aten_args)):
        torch.manual_seed(0)
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            model, _ = build_model(args, cfg)
        step = TrainStep(args, model.cuda().train(), build_criterion(cargs, cfg).cuda(), torch.device("cuda", 0))
        np.random.seed(11)
        step.capture(batch, warmup=2, curr_epoch=1.0)       # epoch 1: no discovery, no host copy in the step
        steps[arm] = step
    losses = {arm: float(steps[arm](batch, 1.0)[0]) for arm in steps}
    res = {"new": [], "aten": []}
    for _ in range(rounds):
        for arm in ("new", "aten"):
            res[arm].append(timed(lambda: steps[arm](batch, 1.0), iters))
    return {"new": stats(res["new"]), "aten": stats(res["aten"]), "first_loss": losses,
            "launches_per_step": {arm: steps[arm].launches_per_step for arm in steps},
            "shape": {"scenes": SCENES, "points": 20000, "nqueries": 128, "distillation_box_num": 32,
                      "clip_arch": "ViT-B/16", "superset_rows": C, "epoch": 1}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True, help="output directory")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--loss-iters", type=int, default=50)
    ap.add_argument("--step-iters", type=int, default=10)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_superset needs a CUDA device")
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    out = {"card": card(), "loss": loss_alone(a.rounds, a.loss_iters), "step": step_times(a.rounds, a.step_iters)}
    os.makedirs(a.out, exist_ok=True)
    Path(a.out, "bench_superset.json").write_text(json.dumps(out, indent=1))
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
