"""The ViT-B/16 CLIP tower without a GPU.

  * OUR VisionTransformer in fp32 at B/16 geometry (patch 16, 197 tokens), with the CPU stand-ins of
    oracle/cpu_step.py for the kernels, against `cls32` / `tok32` of the reference's own tower
    (tests/golden/clip_vit_b16.npz): parameter names, geometry and the 197-token math.
  * Which kernel coda_attention_fwd_half runs for a sequence length and how many key tiles it walks, restated in
    plain Python (csrc/attention_sm90.cu), and checked against the lengths the GPU tests run."""
from pathlib import Path

import numpy as np
import torch

import cpu_step as cpu_shims
from param_fill import fill_by_name
from test_attention_edges_gpu import HALF_CASES
from test_clip_b16_gpu import KERNEL_CASES, KERNEL_L

GOLDEN = Path(__file__).resolve().parent / "golden" / "clip_vit_b16.npz"
KT = 64                 # keys per tile (attention_common.cuh: attn::KT)
NT, NWG = 4, 2          # ResCfg: resident tiles (l <= 256) and warpgroups (attention_sm90.cu)


def test_vit_b16_fp32_on_cpu_matches_reference_golden():
    from coda_neurips2023_b200.clip import model as cm

    gold = np.load(GOLDEN)
    n = 8
    g = torch.Generator().manual_seed(77)     # tests/golden/make_clip_vit_golden.py:crops
    x = torch.randn(32, 3, 224, 224, generator=g)
    x[:, :, :40, :] = 1.9
    x = x.half()[:n].float()
    with cpu_shims.installed():
        vit = cm.VisionTransformer(input_resolution=224, patch_size=16, width=768, layers=12, heads=12, output_dim=512)
        fill_by_name(vit, seed=21)
        cm.convert_weights(vit)              # fp16-rounded weights, evaluated in fp32 (as `cls32` was)
        vit = vit.float().eval()
        with torch.no_grad():
            cls, tok = vit(x)
    assert tok.shape == (n, 197, 512)
    cls_err = np.abs(cls.numpy() - gold["cls32"][:n]).max() / np.abs(gold["cls32"][:n]).max()
    tok_err = np.abs(tok.numpy()[:, ::7, ::8] - gold["tok32"][:n]).max() / np.abs(gold["tok32"][:n]).max()
    print(f"B/16 fp32 on CPU vs reference: cls max-rel {cls_err:.2e}, tokens max-rel {tok_err:.2e}")
    assert cls_err < 1e-4 and tok_err < 1e-4


def half_kernel(l: int, hd: int = 64):
    """coda_attention_fwd_half: l <= 64 -> the pack pass + attn_fwd_kernel<64, 1, 1, true>; 64 < l <= 256 -> the
    resident kernel; anything else -> CODA_EINVAL (None)"""
    if hd != 64 or l <= 0 or l > NT * KT:
        return None
    return "pack" if l <= KT else "resident"


def walk(l: int) -> dict:
    """tiles of the resident kernel: every CTA loads all ceil(l / 64) K / V tiles; warpgroup w takes query tiles
    w, w + NWG, ... and walks every key tile; the last tile is partial when 64 does not divide l"""
    nt = -(-l // KT)
    return dict(key_tiles=nt, tail=l % KT != 0, per_wg=[len(range(w, nt, NWG)) for w in range(NWG)])


def test_kernel_choice_by_length():
    assert [half_kernel(l) for l in (1, 50, 64)] == ["pack"] * 3
    assert [half_kernel(l) for l in (65, 197, 256)] == ["resident"] * 3
    assert half_kernel(257) is None and half_kernel(197, hd=128) is None
    assert walk(197) == dict(key_tiles=4, tail=True, per_wg=[2, 2])
    assert walk(129) == dict(key_tiles=3, tail=True, per_wg=[2, 1])


def test_gpu_lengths_cover_every_tile_count_tail_and_boundary():
    assert all(half_kernel(l) == "resident" for l in KERNEL_L)
    assert all(half_kernel(l) == "pack" for l in HALF_CASES)
    seen = {(walk(l)["key_tiles"], walk(l)["tail"]) for l in KERNEL_L} | {(1, l % KT != 0) for l in HALF_CASES}
    assert seen >= {(n, t) for n in (1, 2, 3, 4) for t in (False, True)}, seen
    # both sides of the 64 / 256 boundaries, and a warpgroup with one query tile next to one with two
    assert {64} <= set(HALF_CASES) and {65, 256} <= set(KERNEL_L)
    assert any(walk(l)["per_wg"] == [2, 1] for l in KERNEL_L)
    # the step's shape: 256 crops x 12 heads at 197 tokens
    assert (197, 256, 12) in KERNEL_CASES
