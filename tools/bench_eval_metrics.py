"""APCalculator.compute_metrics at the SUN RGB-D test shape: the per-class host loop it used to run (a mask-select, an
argsort and two device-to-host copies per class, then cumulative sums, precision envelope and VOC AP in numpy one
class and one threshold at a time) against the record kernels (coda_eval_records, two stable sorts, coda_eval_ap).

    python tools/bench_eval_metrics.py [--reps N]

The calculator's accumulation is filled directly with what 106 steps of 48 scenes would leave (5050 scenes,
K = 128 boxes, C = 46 classes, IoU thresholds 0.25 and 0.5, per-class proposals: every live box scores every class),
seeded.  The two paths are alternated in one process; each timing ends with the result on the host.  Prints JSON
lines: the card (name, power limit, max SM clock), the record count, the median and all times of each path, and the
largest difference of their per-class AP / precision / recall."""
import argparse
import json
import subprocess
import sys
import time
from pathlib import Path
from types import SimpleNamespace

import numpy as np
import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
from coda_neurips2023_b200.utils import ap_calculator as apc  # noqa: E402

SCENES, K, C, BATCH = 5050, 128, 46, 48
THRESH = [0.25, 0.5]


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    name, power, clock = [s.strip() for s in q[torch.cuda.current_device()].split(",")]
    return {"card": name, "power_limit": power, "max_sm_clock": clock}


def filled_calculator(seed=0, live=0.25):
    """an APCalculator holding what step() would have stored for SCENES scenes"""
    g = torch.Generator(device="cuda").manual_seed(seed)
    ds = SimpleNamespace(num_semcls=C)
    calc = apc.APCalculator(ds, ap_iou_thresh=THRESH, args=SimpleNamespace(dataset_name="sunrgbd"))
    big = torch.iinfo(torch.int64).max
    first_pred = torch.full((C,), big, dtype=torch.int64, device="cuda")
    for lo in range(0, SCENES, BATCH):
        b = min(BATCH, SCENES - lo)
        probs = torch.rand((b, K, C), generator=g, device="cuda")
        probs = probs / probs.sum(-1, keepdim=True)
        obj = torch.rand((b, K), generator=g, device="cuda")
        mask = torch.rand((b, K), generator=g, device="cuda") < live
        tp25 = (torch.rand((b, C, K), generator=g, device="cuda") < 0.05) & mask.unsqueeze(1)
        tp50 = tp25 & (torch.rand((b, C, K), generator=g, device="cuda") < 0.6)
        calc._scores.append(probs * obj.unsqueeze(-1))
        calc._live.append(mask)
        calc._tp.append(torch.stack([tp25, tp50]))
        calc._scene_base.append(lo)
        cnt = torch.randint(0, 3, (C,), generator=g, device="cuda") * b
        calc._gt_count = cnt if calc._gt_count is None else calc._gt_count + cnt
        pos = ((lo + torch.arange(b, device="cuda")).view(b, 1, 1) * C + torch.arange(C, device="cuda").view(1, 1, C)) * K \
            + torch.arange(K, device="cuda").view(1, K, 1)
        first_pred = torch.minimum(first_pred, torch.where(mask.unsqueeze(-1), pos, big).amin(dim=(0, 1)))
    calc._first_pred, calc._first_gt = first_pred, torch.zeros(C, dtype=torch.int64, device="cuda")
    calc.scan_cnt = SCENES
    return calc


def host_loop(calc):
    """the per-class host loop compute_metrics ran before the record kernels -> {thresh: {class: (ap, prec, rec)}}"""
    scores = torch.cat([s.reshape(-1, s.shape[-1]) for s in calc._scores])
    live = torch.cat([m.reshape(-1) for m in calc._live])
    tps = torch.cat([t.permute(0, 1, 3, 2).reshape(t.shape[0], -1, t.shape[2]) for t in calc._tp], dim=1)
    is_det = live.unsqueeze(-1) & torch.isfinite(scores)
    npos = calc._gt_count.cpu().numpy()
    per_class = {}
    has_det = is_det.any(dim=0).cpu().numpy()
    for c in range(scores.shape[1]):
        if not has_det[c] and npos[c] == 0:
            continue
        sel = is_det[:, c]
        s = scores[sel, c]
        order = torch.argsort(-s, stable=True)
        per_class[c] = (s[order].cpu().numpy().astype(np.float64),
                        tps[:, sel, c][:, order].cpu().numpy().astype(np.float64))
    out = {}
    for ti, thresh in enumerate(THRESH):
        out[thresh] = {}
        for c, (_, tp_all) in per_class.items():
            tp = np.cumsum(tp_all[ti])
            fp = np.cumsum(1.0 - tp_all[ti])
            rec = np.zeros_like(tp) if npos[c] == 0 else tp / float(npos[c])
            prec = tp / np.maximum(tp + fp, np.finfo(np.float64).eps)
            out[thresh][c] = (apc.voc_ap(rec, prec), prec[-1] if len(prec) else 0, rec[-1] if len(rec) else 0)
    return out


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    r = fn()
    torch.cuda.synchronize()
    return r, (time.perf_counter() - t0) * 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_eval_metrics needs a CUDA device")
    print(json.dumps(card()), flush=True)
    calc = filled_calculator()
    nrec = len(calc.rank_state().records)
    print(json.dumps({"scenes": SCENES, "K": K, "C": C, "thresholds": THRESH, "records": nrec}), flush=True)
    old, new = timed(lambda: host_loop(calc))[0], timed(calc.compute_metrics)[0]     # warm-up
    t_old, t_new = [], []
    for _ in range(a.reps):
        old, t = timed(lambda: host_loop(calc))
        t_old.append(t)
        new, t = timed(calc.compute_metrics)
        t_new.append(t)
    worst = 0.0
    for thresh in THRESH:
        for c, (eap, eprec, erec) in old[thresh].items():
            r = new[thresh]
            worst = max(worst, abs(r[f"{c} Average Precision"] - eap), abs(r[f"{c} Prec"] - eprec),
                        abs(r[f"{c} Recall"] - erec))
    print(json.dumps({"host_loop_ms_median": float(np.median(t_old)), "host_loop_ms": [round(t, 2) for t in t_old],
                      "record_kernels_ms_median": float(np.median(t_new)),
                      "record_kernels_ms": [round(t, 2) for t in t_new],
                      "max_abs_metric_difference": worst}), flush=True)


if __name__ == "__main__":
    main()
