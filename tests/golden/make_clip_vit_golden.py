"""Golden for the CLIP image tower as the step runs it (SURVEY 8a row a12): the REFERENCE's own
`VisionTransformer` (CLIP/clip/model.py:593-659), ViT-B/32 geometry (12 layers, width 768, 12 heads,
patch 32, 50 tokens), name-keyed random weights rounded to fp16 exactly as `convert_weights` does
(model.py:1146-1166), run on CPU

  * in fp32 arithmetic on those fp16 weights  -> `cls32` / `tok32`: the infinitely-precise answer,
  * in fp16 arithmetic (what the reference executes on a GPU)  -> `cls16`: how far the reference's own
    fp16 run sits from that answer; the parity test holds our fp16 wgmma tower to the same distance.

Weights are not stored (tests/param_fill.py regenerates them by name), the 32 input crops are (seeded,
fp16-rounded CLIP-normalised pixels).

    python tests/golden/make_clip_vit_golden.py        (writes tests/golden/clip_vit_b32.npz)
"""
import sys
from pathlib import Path

import numpy as np
import torch

HERE = Path(__file__).resolve().parent
ROOT = HERE.parents[1]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))
sys.path.insert(0, str(HERE))

import _reference_harness as H  # noqa: E402
from param_fill import fill_by_name  # noqa: E402

GEOM = dict(input_resolution=224, patch_size=32, width=768, layers=12, heads=12, output_dim=512)
NCROPS, SEED = 32, 21


def crops(n=NCROPS):
    g = torch.Generator().manual_seed(77)
    # CLIP-normalised pixel statistics: roughly unit variance, a few saturated (white padding) regions
    x = torch.randn(n, 3, 224, 224, generator=g)
    x[:, :, :40, :] = 1.9          # white bars, as the square padding of a crop leaves them
    return x.half()


def main():
    M = H.load("CLIP.clip.model")
    torch.manual_seed(0)
    vit = M.VisionTransformer(**GEOM).eval()
    fill_by_name(vit, seed=SEED)
    M.convert_weights(vit)              # Linear / conv / in_proj / proj -> fp16 (LayerNorm stays fp32)
    x16 = crops()
    with torch.no_grad():
        ideal = vit.float()
        # .float() keeps the fp16-ROUNDED values: fp32 arithmetic on the weights the GPU run uses
        cls32, tok32 = ideal(x16.float())
        blob = {"cls32": cls32.numpy(), "tok32": tok32[:, ::7, ::8].numpy().copy()}
        try:
            fill_by_name(vit, seed=SEED)
            M.convert_weights(vit)
            vit16 = vit
            for m in vit16.modules():          # LayerNorm parameters stay fp32 (reference LayerNorm upcasts)
                pass
            cls16, _ = vit16(x16)
            blob["cls16"] = cls16.float().numpy()
            d = (cls16.float() - cls32)
            print("reference fp16-on-CPU vs fp32: max rel", float(d.abs().max() / cls32.abs().max()),
                  "min cos", float(torch.nn.functional.cosine_similarity(cls16.float(), cls32, dim=1).min()))
        except RuntimeError as e:   # half kernels missing on this CPU build
            print("fp16 CPU run unavailable:", e)
    np.savez_compressed(HERE / "clip_vit_b32.npz", **blob)
    print("wrote clip_vit_b32.npz", {k: v.shape for k, v in blob.items()})


if __name__ == "__main__":
    main()
