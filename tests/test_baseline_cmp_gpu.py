"""The 3DETR + CLIP baseline head's comparison-class evaluation (`forward(if_cmp_class=True)`) on the GPU: the model
against the reference golden (tests/golden/make_baseline_cmp_golden.py), the comparison pass against the real-test
pass on one batch, coda_clip_classify at the comparison class counts, the AP metrics of engine.evaluate against the
reference APCalculator's, and a full-size ViT-B/16 batch through engine.evaluate(if_cmp_class=True)."""
import warnings

import numpy as np
import pytest
import torch

import baseline_cmp_common as bcc
import baseline_eval_common as bec
from coda_neurips2023_b200 import engine, ops, synthetic
from coda_neurips2023_b200.models import build_model
from coda_neurips2023_b200.utils.ap_calculator import APCalculator, merge_rank_states
from test_baseline_eval_gpu import TOWER_BAR
from test_baseline_eval_gpu import test_clip_classify_against_fp64 as clip_classify_against_fp64

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("dataset_name", bcc.DATASETS)
def test_cmp_head_matches_the_reference_golden(dataset_name):
    """The bars of test_baseline_head_matches_the_reference_golden: usable mask equal, logits within the tower's
    error, argmax equal where the reference's top two logits are further apart than twice the logits' largest
    difference, |d prob| <= 1e-3."""
    model, golden = bcc.build_ours("cuda", dataset_name)
    with torch.no_grad():
        out = model(bec.test_batch("cuda", dataset_name), if_cmp_class=True)["outputs"]
    usable = out["clip_usable_mask"].cpu().numpy()
    assert np.array_equal(usable, golden["usable"])
    assert not usable[bec.NO_VIEW_SCENE].any() and usable.sum() > 0
    prob = out["sem_cls_prob"].cpu().numpy()
    assert prob.shape == golden["sem_cls_prob"].shape == (bec.BATCH, 128, len(golden["cmp_prompts"]))
    assert (out["sem_cls_logits"] == 0).all()
    real_golden = np.load(bec.golden_path(dataset_name))        # the crop features do not depend on the text
    scale = float(real_golden["logit_scale"])
    text = golden["cmp_text_features_fg_norm"].astype(np.float64)
    unit = lambda f: f / np.linalg.norm(f, axis=1, keepdims=True)   # noqa: E731
    z_ours = scale * unit(out["clip_crop_features"].cpu().numpy().astype(np.float64)) @ text.T
    z_ref = scale * unit(real_golden["crop_features"].astype(np.float64)) @ text.T
    zerr = np.abs(z_ours - z_ref).max()
    assert zerr <= scale * TOWER_BAR
    top2 = np.sort(z_ref, axis=1)[:, -2:]
    clear = top2[:, 1] - top2[:, 0] > 2 * zerr
    print(f"{dataset_name}: logits max-abs {zerr:.2e}; {int(clear.sum())} of {int(usable.sum())} usable boxes with a "
          f"clear class; max |d prob| {np.abs(prob - golden['sem_cls_prob']).max():.2e}")
    assert clear.sum() > usable.sum() // 2
    assert np.array_equal(prob[usable].argmax(1)[clear], golden["sem_cls_prob"][usable].argmax(1)[clear])
    assert (prob[~usable] == 0).all()
    assert np.abs(prob - golden["sem_cls_prob"]).max() <= 1e-3


@pytest.mark.parametrize("dataset_name", bcc.DATASETS)
def test_cmp_pass_differs_from_the_real_test_pass_only_in_the_class_axis(dataset_name):
    """Same projection, crops and tower on one batch: every output but the class scores is the same bits, and the
    class scores are coda_clip_classify of the same crop features with the comparison text."""
    model, _ = bcc.build_ours("cuda", dataset_name)
    batch = bec.test_batch("cuda", dataset_name)
    with torch.no_grad():
        real = model(batch, if_real_test=True)["outputs"]
        cmp = model(batch, if_cmp_class=True)["outputs"]
    assert set(real) == set(cmp)
    for k in ("clip_usable_mask", "clip_boxes_2d", "clip_crop_features"):
        assert torch.equal(real[k], cmp[k]), k
    same = [k for k in real if k not in ("sem_cls_prob", "sem_cls_logits") and isinstance(real[k], torch.Tensor)]
    assert [k for k in same if not torch.equal(real[k], cmp[k])] == []
    bsz, nq = real["clip_usable_mask"].shape
    assert real["sem_cls_prob"].shape == (bsz, nq, model.text_features_fg_norm.shape[0])
    ncls = len(np.load(bcc.golden_path(dataset_name))["cmp_prompts"])
    assert cmp["sem_cls_prob"].shape == cmp["sem_cls_logits"].shape == (bsz, nq, ncls)
    flat = cmp["clip_usable_mask"].reshape(-1)
    row_map = torch.where(flat, flat.to(torch.int32).cumsum(0, dtype=torch.int32) - 1, -1).to(torch.int32)
    prob, _ = ops.clip_classify(cmp["clip_crop_features"], model.cmp_text_features_fg_norm, model.logit_scale,
                                row_map, (bsz, nq))
    assert torch.equal(prob, cmp["sem_cls_prob"])


@pytest.mark.parametrize("c", [19, 20])
@pytest.mark.parametrize("pattern", ["all", "none", "mixed"])
def test_clip_classify_at_the_comparison_class_counts(c, pattern):
    """coda_clip_classify at 48 x 128 rows against the fp64 restatement, in sentinel-padded buffers, run twice."""
    clip_classify_against_fp64(c, pattern)


def _metrics_close(ret, golden, tol):
    worst, bad = 0.0, []
    for thr in bcc.AP_IOU:
        keys, vals = list(golden[f"ap.{thr}.keys"]), golden[f"ap.{thr}.values"]
        assert list(ret[thr].keys()) == keys
        for k, v in zip(keys, vals):
            got = float(ret[thr][k])
            if np.isnan(v) and np.isnan(got):
                continue
            worst = max(worst, abs(got - float(v)))
            if not abs(got - float(v)) <= tol:
                bad.append((thr, str(k), got, float(v)))
    return worst, bad


@pytest.mark.parametrize("dataset_name", bcc.DATASETS)
def test_evaluate_cmp_metrics_match_the_reference(dataset_name):
    """engine.evaluate(if_cmp_class=True) with the comparison classes' dataset config: every entry of the reference
    APCalculator's result dict, at IoU 0.25 and 0.5, in its order; then the same metrics from rank-local calculators,
    one scene per rank, merged."""
    model, golden = bcc.build_ours("cuda", dataset_name)
    args = bec.args_for(dataset_name)
    cfg = bcc.dataset_config(args, golden)
    batch = bcc.eval_batch("cuda", dataset_name, golden)
    outs = []
    hook = model.register_forward_hook(lambda m, i, o: outs.append(o))
    try:
        ret = engine.evaluate(args, 0, model, None, cfg, [batch], if_cmp_class=True).compute_metrics()
    finally:
        hook.remove()
    worst, bad = _metrics_close(ret, golden, 1e-5)
    print(f"{dataset_name}: max |metric - reference| = {worst:.1e}")
    assert not bad, bad
    out = outs[0]["outputs"]
    w = bec.BATCH
    ranks = [APCalculator(cfg, ap_iou_thresh=list(bcc.AP_IOU), class2type_map=cfg.class2type, exact_eval=True,
                          args=args, rank=r, world_size=w) for r in range(w)]
    for r, calc in enumerate(ranks):
        sl = slice(r, r + 1)
        calc.step_meter({k: out[k][sl] for k in ("box_corners", "sem_cls_prob", "objectness_prob")},
                        {k: batch[k][sl] for k in ("point_clouds",) + bcc.GT_KEYS})
    merged = ranks[0].metrics_from_state(merge_rank_states([c.rank_state() for c in ranks]))
    for thr in bcc.AP_IOU:
        assert list(merged[thr].keys()) == list(ret[thr].keys())
        assert np.allclose([float(v) for v in merged[thr].values()], [float(v) for v in ret[thr].values()],
                           rtol=0, atol=1e-12, equal_nan=True)


@pytest.mark.parametrize("dataset_name", bcc.DATASETS)
def test_full_size_vit_b16_batch_through_evaluate_cmp(dataset_name):
    """48 scenes x 20 000 points, 128 queries, a random-init ViT-B/16, the comparison classes of a synthetic run."""
    over = dict(dataset_name=dataset_name, test_range_max=46)
    camera, hw = "sunrgbd", (531, 730)
    if "scannet" in dataset_name:
        over.update(test_range_max=60, reset_scannet_num=50, image_size_width=1296, image_size_height=968)
        camera, hw = "scannet", (968, 1296)
    args = synthetic.make_args(model_name="3detrmulticlasshead", nqueries=128, clip_arch="ViT-B/16", **over)
    ncls = 19 if "scannet" in dataset_name else 20
    cfg = synthetic.SyntheticDatasetConfig(args, num_semcls=ncls)
    torch.manual_seed(0)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        model, _ = build_model(args, cfg)
    model.to_device("cuda")
    batch = synthetic.to_device(synthetic.make_batch(48, 20000, seed=3, image_hw=hw, camera=camera), "cuda")
    outs = []
    hook = model.register_forward_hook(lambda m, i, o: outs.append(o))
    try:
        metrics = engine.evaluate(args, 0, model, None, cfg, [batch], if_cmp_class=True).compute_metrics()
    finally:
        hook.remove()
    out = outs[0]["outputs"]
    prob, usable = out["sem_cls_prob"], out["clip_usable_mask"]
    assert prob.shape == (48, 128, ncls) and usable.shape == (48, 128)
    assert torch.isfinite(prob).all()
    print(f"{dataset_name}: 48 x 128 ViT-B/16 comparison pass, {int(usable.sum())} usable boxes")
    assert usable.any()
    assert torch.allclose(prob[usable].sum(-1), torch.ones((), device="cuda"), rtol=0, atol=1e-5)
    assert (prob[~usable] == 0).all()
    assert metrics and all(isinstance(v, dict) for v in metrics.values())
