"""The 3DETR + CLIP baseline head's test-time classification on the GPU: coda_clip_classify against an fp64
restatement, the model against the reference golden (tests/golden/make_baseline_eval_golden.py), and a full-size
ViT-B/16 batch through engine.evaluate(if_real_test=True)."""
import warnings

import numpy as np
import pytest
import torch

import baseline_eval_common as bec
from coda_neurips2023_b200 import _lib, ops

pytestmark = pytest.mark.gpu

D = 512
TOWER_BAR = 4e-3            # the CLIP tower's max-rel bar of tests/test_clip_gpu.py


def restate(feats, text, scale, row_map, c):
    f = feats.double()
    f = f / f.norm(dim=1, keepdim=True)
    want = torch.zeros((row_map.numel(), c), dtype=torch.float64, device=feats.device)
    keep = row_map >= 0
    if keep.any():
        z = scale * (f[row_map[keep].long()] @ text.double().t())
        want[keep] = torch.softmax(z, dim=-1)
    return want


@pytest.mark.parametrize("c", [1, 46, 60, 232, 1201])
@pytest.mark.parametrize("pattern", ["all", "none", "mixed"])
def test_clip_classify_against_fp64(c, pattern):
    g = torch.Generator(device="cuda").manual_seed(c)
    b, q = 48, 128
    rows = b * q
    usable = {"all": torch.ones(rows, dtype=torch.bool, device="cuda"),
              "none": torch.zeros(rows, dtype=torch.bool, device="cuda"),
              "mixed": torch.rand(rows, generator=g, device="cuda") < 0.6}[pattern]
    if pattern == "mixed":
        usable[: q] = False                                  # one scene without a usable box
    n = int(usable.sum())
    row_map = torch.full((rows,), -1, dtype=torch.int32, device="cuda")
    row_map[usable] = torch.randperm(n, generator=g, device="cuda").to(torch.int32)
    feats = torch.randn((n, D), generator=g, device="cuda") * 3
    text = torch.randn((c, D), generator=g, device="cuda")
    text = text / text.norm(dim=1, keepdim=True)
    scale = torch.tensor([100.0], device="cuda")
    # outputs inside sentinel-filled buffers: nothing may be written around them
    pad = 4096
    pbuf = torch.full((rows * c + 2 * pad,), 7.0, device="cuda")
    lbuf = torch.full_like(pbuf, 7.0)
    prob, logits = pbuf[pad: pad + rows * c].view(b, q, c), lbuf[pad: pad + rows * c].view(b, q, c)
    for _ in range(2):
        with torch.cuda.device(0):
            st = _lib.lib().coda_clip_classify(ops._ll(rows), ops._i(n), ops._i(c), ops._i(D), _lib.ptr(feats),
                                               _lib.ptr(text), _lib.ptr(scale), _lib.ptr(row_map), _lib.ptr(prob),
                                               _lib.ptr(logits), _lib.stream_of(text))
        _lib.check(st, "clip_classify")
        torch.cuda.synchronize()
        if _ == 0:
            first = prob.clone()
    assert torch.equal(first, prob), "run-to-run bits differ"
    assert (pbuf[:pad] == 7).all() and (pbuf[-pad:] == 7).all() and (lbuf[:pad] == 7).all() and (lbuf[-pad:] == 7).all()
    assert (logits == 0).all()
    want = restate(feats, text, 100.0, row_map, c).view(b, q, c)
    normal = want > 1e-30                                     # fp32 holds smaller values as denormals or zero
    diff = (prob.double() - want).abs()
    err = (diff[normal] / want[normal]).max().item() if normal.any() else 0.0
    assert (diff[~normal] <= 1e-36).all()
    assert (prob.view(rows, c)[~usable] == 0).all()
    assert err <= 1e-6, err
    # the wrapper gives the same bits
    p2, l2 = ops.clip_classify(feats, text, scale, row_map, (b, q))
    assert torch.equal(p2, prob) and (l2 == 0).all()


def test_clip_classify_refuses_other_widths():
    x = torch.zeros((2, 256), device="cuda")
    with pytest.raises(_lib.CodaError):
        ops.clip_classify(x, x, torch.ones(1, device="cuda"), torch.zeros(2, dtype=torch.int32, device="cuda"), (2,))


@pytest.mark.parametrize("dataset_name", ["sunrgbd_image", "scannet50_image"])
def test_baseline_head_matches_the_reference_golden(dataset_name):
    """SUN RGB-D with the batch's K / Rtilt; ScanNet with a batch that has neither, so the head reads the
    calibration files the reference read."""
    model, out, golden = bec.run_ours("cuda", dataset_name)
    usable = out["clip_usable_mask"].cpu().numpy()
    assert np.array_equal(usable, golden["usable"])
    assert not usable[:, list(bec.ZERO_QUERIES)].any() and not usable[bec.NO_VIEW_SCENE].any()
    # integer boxes: equal wherever the fp64 extent is not within 1e-3 px of an integer
    _, _, ext = model.project_boxes(bec.test_batch("cuda", dataset_name), out, extent=True)
    ext = ext.cpu().numpy()
    near = (np.abs(ext - np.round(ext)) <= 1e-3).any(-1)
    boxes = out["clip_boxes_2d"].cpu().numpy()
    differ = (boxes != golden["boxes"]).any(-1) & usable
    print(f"{dataset_name}: usable boxes at an integer boundary: {int((near & usable).sum())}; "
          f"differing: {int(differ.sum())} of {int(usable.sum())}")
    assert not (differ & ~near).any()
    feats = out["clip_crop_features"].cpu().numpy()
    gf = golden["crop_features"]
    assert feats.shape == gf.shape
    ferr = np.abs(feats - gf).max() / np.abs(gf).max()
    scale = float(golden["logit_scale"])
    text = golden["text_features_fg_norm"].astype(np.float64)
    unit = lambda f: f / np.linalg.norm(f, axis=1, keepdims=True)   # noqa: E731
    z_ours, z_ref = scale * unit(feats.astype(np.float64)) @ text.T, scale * unit(gf.astype(np.float64)) @ text.T
    zerr = np.abs(z_ours - z_ref).max()
    print(f"{dataset_name}: crop features max-rel {ferr:.2e}, logits max-abs {zerr:.2e} (scale {scale:.2f})")
    assert ferr <= TOWER_BAR
    assert zerr <= scale * TOWER_BAR
    top2 = np.sort(z_ref, axis=1)[:, -2:]
    clear = top2[:, 1] - top2[:, 0] > 2 * scale * TOWER_BAR
    prob = out["sem_cls_prob"].cpu().numpy()
    assert prob.shape[-1] == len(golden["prompts"])
    assert np.array_equal(prob[usable].argmax(1)[clear], golden["sem_cls_prob"][usable].argmax(1)[clear])
    assert (prob[~usable] == 0).all()
    assert np.abs(prob - golden["sem_cls_prob"]).max() <= 1e-3


def test_clip_classify_refuses_operands_on_another_device():
    text = torch.zeros((4, D), device="cuda")
    feats = torch.zeros((2, D), device="cuda")
    rm = torch.zeros(2, dtype=torch.int32, device="cuda")
    with pytest.raises(ValueError, match="scale"):
        ops.clip_classify(feats, text, torch.ones(1), rm, (2,))
    with pytest.raises(ValueError, match="feats"):
        ops.clip_classify(feats.cpu(), text, torch.ones(1, device="cuda"), rm, (2,))


def test_coda_head_eval_outputs_are_the_bits_of_before():
    """The CoDA head shares its class with the baseline head: its eval outputs on one seeded batch are the bits the
    commit before that change computed (tests/golden/make_coda_eval_bits_golden.py)."""
    import model_eval_common as mec

    want = np.load(bec.GOLDEN / "model_eval_small_gpu_bits.npz")
    out, _ = mec.run("eval_small", "cuda")
    got = mec.blob(out)
    assert set(got) == set(want.files)
    differ = [k for k in sorted(got) if not np.array_equal(got[k], want[k])]
    assert not differ, differ


def test_full_size_vit_b16_batch_through_evaluate():
    from coda_neurips2023_b200 import engine, synthetic
    from coda_neurips2023_b200.models import build_model

    args = synthetic.make_args(model_name="3detrmulticlasshead", dataset_name="sunrgbd_image", nqueries=128,
                               clip_arch="ViT-B/16", test_range_max=46)
    cfg = synthetic.SyntheticDatasetConfig(args)
    torch.manual_seed(0)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        model, _ = build_model(args, cfg)
    model.to_device("cuda")
    batch = synthetic.to_device(synthetic.make_batch(48, 20000, seed=3), "cuda")
    torch.cuda.reset_peak_memory_stats()
    calc = engine.evaluate(args, 0, model, None, cfg, [batch], if_real_test=True)
    metrics = calc.compute_metrics()
    peak = torch.cuda.max_memory_allocated() / 2 ** 30
    print(f"48 x 128 ViT-B/16 baseline eval: peak allocated {peak:.2f} GiB")
    assert metrics and all(isinstance(v, dict) for v in metrics.values())
