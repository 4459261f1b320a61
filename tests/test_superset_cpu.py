"""--if_clip_superset without a GPU: the superset prompt lists and their token rows against the reference's own
(tests/golden/superset_prompts.json, superset_tokens.npz from tests/golden/make_superset_golden.py), the missing-LVIS
error, the seeded random superset of synthetic runs, and OUR model + criterion on the two stage-2 superset cases (CUDA
ops replaced by the CPU restatement) against the reference's run of them."""
import json
import warnings

import numpy as np
import pytest
import torch

import model_parity_common as mpc
import scannet_ref
import superset_common as ssc
from coda_neurips2023_b200 import synthetic
from coda_neurips2023_b200.clip.tokenizer import tokenize
from coda_neurips2023_b200.models import build_model, model_3detr

GOLDEN = mpc.GOLDEN
PROMPTS = json.loads((GOLDEN / "superset_prompts.json").read_text())


@pytest.mark.parametrize("dataset, rows", [("sunrgbd", 1201), ("scannet", 1203)])
def test_superset_prompts_equal_the_reference_list(dataset, rows):
    with ssc.coda_checkout():
        got = model_3detr.superset_prompts(synthetic.make_args(**PROMPTS["flags"][dataset]))
    assert got == PROMPTS[dataset]
    assert len(got) == rows


@pytest.mark.parametrize("dataset", ["sunrgbd", "scannet"])
def test_superset_token_rows_equal_the_reference_tokenizer(dataset):
    prompts = PROMPTS[dataset]
    # names the BPE treats specially: hyphens, and an LVIS name that carries a trailing space
    assert "a photo of a flip-flop  in the scene" in prompts
    assert any("-" in p for p in prompts if p != "a photo of a flip-flop  in the scene")
    exp = np.load(GOLDEN / "superset_tokens.npz")[dataset]
    got = tokenize(prompts, vocab_path=str(ssc.BPE)).numpy()
    assert got.shape == exp.shape
    bad = [prompts[i] for i in np.nonzero((got != exp).any(axis=1))[0]]
    assert not bad, bad[:5]


def test_missing_lvis_list_is_an_error_naming_the_path():
    with ssc.coda_checkout(lvis=False):
        args = synthetic.make_args(**PROMPTS["flags"]["sunrgbd"])
        with pytest.raises(FileNotFoundError, match=model_3detr.ALL_SUPERCLASS_PATH):
            model_3detr.superset_prompts(args)
        load = model_3detr.clip_mod.load
        model_3detr.clip_mod.load = ssc.tiny_clip
        try:
            with pytest.raises(FileNotFoundError, match=model_3detr.ALL_SUPERCLASS_PATH), warnings.catch_warnings():
                warnings.simplefilter("ignore")
                build_model(args, synthetic.SyntheticDatasetConfig(args))
        finally:
            model_3detr.clip_mod.load = load


def test_without_class_lists_the_superset_is_the_seeded_random_rows(tmp_path, monkeypatch):
    monkeypatch.chdir(tmp_path)
    monkeypatch.setattr(model_3detr.clip_mod, "load", ssc.tiny_clip)
    args = synthetic.make_args(if_clip_superset=True, test_range_max=46, if_clip_more_prompts=True)
    assert model_3detr.superset_prompts(args) is None
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        model, _ = build_model(args, synthetic.SyntheticDatasetConfig(args))
    feats = torch.randn(46, 512, generator=torch.Generator().manual_seed(1234))
    sup = torch.randn(1201, 512, generator=torch.Generator().manual_seed(4321))
    sup[:10] = feats[:10]
    assert model.superset_all_classes_keys is None
    assert torch.equal(model.superset_text_features_fg_norm.cpu(), sup / sup.norm(dim=1, keepdim=True))


@pytest.mark.parametrize("name", list(ssc.CASES))
def test_superset_model_and_criterion_match_reference_on_cpu(name):
    """Same bars as test_model_cpu.py: 2e-4 relative forward / loss, gradients 10 x that."""
    torch.manual_seed(0)
    with scannet_ref.installed():
        model, out, loss, loss_dict, golden = ssc.run(name, "cpu")
        ssc.check_text_features(model, golden, rtol=1e-5)
        ssc.check_weak_labels(out, golden)
        errs = mpc.compare(model, out, loss, loss_dict, golden, rtol=2e-4, atol=1e-5)
    assert int(golden["pseudo.count"].sum()) > 0
    assert "loss_dict.loss_feat_seen_softmax_weakly_loss_with_novel_cate_confi" in golden.files
    worst = max(errs, key=errs.get)
    print(f"{name}: worst {worst} = {errs[worst]:.2e}")
