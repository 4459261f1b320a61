"""The benchmarked CLIP image tower -- ViT-B/32, 12 layers, fp16 weights, fp16 wgmma GEMMs + the single-tile
fused attention + the fp16 LayerNorm kernel -- against the REFERENCE's own VisionTransformer
(CLIP/clip/model.py:593-659) on the same name-keyed fp16-rounded weights and the same 32 crops
(tests/golden/clip_vit_b32.npz, made by tests/golden/make_clip_vit_golden.py from /root/reference).

The golden holds the reference evaluated in fp32 arithmetic on those fp16 weights (`cls32`, the exact answer) and
in fp16 arithmetic on CPU (`cls16`, what the reference's own half-precision run gives: 1.4e-3 max-rel, cosine
0.9999993 from exact).  Bar for ours, written here: max-rel error vs exact <= 2 x the reference-fp16 run's own
error (and <= 4e-3 absolute bound), cosine similarity >= 0.99999 on every crop."""
from pathlib import Path

import numpy as np
import pytest
import torch

from param_fill import fill_by_name

pytestmark = pytest.mark.gpu
GOLDEN = Path(__file__).resolve().parent / "golden" / "clip_vit_b32.npz"


def _crops(n=32):
    g = torch.Generator().manual_seed(77)     # tests/golden/make_clip_vit_golden.py:crops
    x = torch.randn(n, 3, 224, 224, generator=g)
    x[:, :, :40, :] = 1.9
    return x.half()


def test_vit_b32_fp16_tower_matches_reference_golden(built_lib):
    from coda_neurips2023_b200 import _lib
    from coda_neurips2023_b200.clip import model as cm

    gold = np.load(GOLDEN)
    vit = cm.VisionTransformer(input_resolution=224, patch_size=32, width=768, layers=12, heads=12, output_dim=512)
    fill_by_name(vit, seed=21)
    cm.convert_weights(vit)
    vit = vit.cuda().eval()
    n0 = _lib.LAUNCHES
    with torch.no_grad():
        cls, tok = vit(_crops().cuda())
    assert _lib.LAUNCHES - n0 >= 12 * 6, "the tower did not run on the package's own kernels"
    assert cls.dtype == torch.float16
    cls = cls.float().cpu().numpy()
    tok = tok.float().cpu().numpy()[:, ::7, ::8]
    exact, ref16 = gold["cls32"], gold["cls16"]
    scale = np.abs(exact).max()
    ref_err = np.abs(ref16 - exact).max() / scale
    our_err = np.abs(cls - exact).max() / scale
    cos = (cls * exact).sum(1) / (np.linalg.norm(cls, axis=1) * np.linalg.norm(exact, axis=1))
    tok_err = np.abs(tok - gold["tok32"]).max() / np.abs(gold["tok32"]).max()
    print(f"PARITY clip_vit_b32: ours max-rel {our_err:.2e} (reference fp16 run {ref_err:.2e}), min cosine "
          f"{cos.min():.7f}, tokens max-rel {tok_err:.2e}")
    assert our_err <= min(2.0 * ref_err, 4e-3)
    assert cos.min() >= 0.99999
    assert tok_err <= 4e-3
