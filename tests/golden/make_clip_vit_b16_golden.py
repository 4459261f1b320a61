"""Golden for the ViT-B/16 CLIP image tower, the checkpoint the reference ships (models/model_3detr.py:325, :373):
the REFERENCE's own `VisionTransformer` (CLIP/clip/model.py:593-659) at ViT-B/16 geometry (12 layers, width 768,
12 heads, patch 16, 197 tokens), with the same seeded, name-keyed, fp16-rounded weights and the same 32 crops as the
ViT-B/32 golden (make_clip_vit_golden.py), run on CPU

  * in fp32 arithmetic on those fp16 weights  -> `cls32` / `tok32` (tokens subsampled as for B/32),
  * in fp16 arithmetic                          -> `cls16`: the reference's own half-precision distance from `cls32`.

    python tests/golden/make_clip_vit_b16_golden.py        (writes tests/golden/clip_vit_b16.npz)
"""
import numpy as np
import torch

from make_clip_vit_golden import GEOM, HERE, SEED, H, crops, fill_by_name

GEOM_B16 = dict(GEOM, patch_size=16)


def main():
    M = H.load("CLIP.clip.model")
    torch.manual_seed(0)
    vit = M.VisionTransformer(**GEOM_B16).eval()
    fill_by_name(vit, seed=SEED)
    M.convert_weights(vit)              # Linear / conv / in_proj / proj -> fp16 (LayerNorm stays fp32)
    x16 = crops()
    with torch.no_grad():
        # .float() keeps the fp16-ROUNDED values: fp32 arithmetic on the weights the GPU run uses
        cls32, tok32 = vit.float()(x16.float())
        blob = {"cls32": cls32.numpy(), "tok32": tok32[:, ::7, ::8].numpy().copy()}
        fill_by_name(vit, seed=SEED)
        M.convert_weights(vit)
        cls16, _ = vit(x16)
        blob["cls16"] = cls16.float().numpy()
        d = cls16.float() - cls32
        print("reference fp16-on-CPU vs fp32: max rel", float(d.abs().max() / cls32.abs().max()),
              "min cos", float(torch.nn.functional.cosine_similarity(cls16.float(), cls32, dim=1).min()))
    np.savez_compressed(HERE / "clip_vit_b16.npz", **blob)
    print("wrote clip_vit_b16.npz", {k: v.shape for k, v in blob.items()})


if __name__ == "__main__":
    main()
