"""CLIP ViT image tower + text transformer for the distillation targets.

Behavioural mirror of the classes of reference CLIP/clip/model.py that the
registered CoDA models exercise (`VisionTransformer` :585-659 -- which returns
``(cls_embedding, all_token_embeddings)`` --, `ResidualAttentionBlock` :295-316,
`QuickGELU` :263-265, fp32-upcasting `LayerNorm` :254-260, `CLIP.encode_image /
encode_text` :1062-1082, `build_model` :1266-1312, `convert_weights` :1146-1166).
Parameter names follow the OpenAI checkpoints, so a ViT-B/16 or ViT-B/32
``state_dict`` loads unchanged.  Frozen, forward-only, fp16 weights with fp32
LayerNorm -- as the reference runs it -- but the whole batch of crops goes
through in ONE call and attention runs in the fused kernel.
"""
from __future__ import annotations

import os
from collections import OrderedDict
from typing import Optional

import numpy as np
import torch
import torch.nn.functional as F
from torch import nn

from .. import ops


def _linear(x, w, b, quick_gelu=False, residual=None):
    """fp16 activations x fp16 weights on the fp16 wgmma path (fp16 written by the epilogue,
    QuickGELU and the block's residual connection fused); fp32 (CPU checks, small test models) through torch."""
    if x.is_cuda and x.dtype == torch.float16 and x.shape[-1] % 64 == 0:
        return ops.linear(x, w, b, quick_gelu=quick_gelu, residual=residual)
    y = F.linear(x, w, b)
    y = y * torch.sigmoid(1.702 * y) if quick_gelu else y
    return y if residual is None else residual + y


class _MLP(nn.Sequential):
    def forward(self, x, residual=None):
        h = _linear(x, self.c_fc.weight, self.c_fc.bias, quick_gelu=True)
        return _linear(h, self.c_proj.weight, self.c_proj.bias, residual=residual)


class LayerNorm(nn.LayerNorm):
    """LayerNorm computed in fp32 whatever the activation dtype (reference :254-260)."""

    def forward(self, x: torch.Tensor):
        c = x.shape[-1]
        if (x.is_cuda and x.dtype == torch.float16 and c % 128 == 0 and c <= 1024
                and not (torch.is_grad_enabled() and (x.requires_grad or self.weight.requires_grad))):
            return ops.layer_norm_half(x, self.weight, self.bias, self.eps)  # one kernel, no fp32 round trip
        return super().forward(x.float()).to(x.dtype)


class QuickGELU(nn.Module):
    def forward(self, x: torch.Tensor):
        return x * torch.sigmoid(1.702 * x)


class _PackedSelfAttention(nn.Module):
    """Self-attention with `nn.MultiheadAttention`'s parameter names."""

    def __init__(self, d_model: int, n_head: int):
        super().__init__()
        self.embed_dim, self.num_heads = d_model, n_head
        self.in_proj_weight = nn.Parameter(torch.empty(3 * d_model, d_model))
        self.in_proj_bias = nn.Parameter(torch.zeros(3 * d_model))
        self.out_proj = nn.Linear(d_model, d_model)

    def forward(self, x: torch.Tensor, causal: bool = False, residual=None):
        q, k, v = _linear(x, self.in_proj_weight, self.in_proj_bias).split(self.embed_dim, dim=-1)
        if x.is_cuda and x.dtype == torch.float16 and not causal and self.embed_dim // self.num_heads == 64:
            from .. import attention_launch
            # q / k / v stay fp16 slices of the fused projection: the pack kernel reads them in place
            if x.shape[0] <= 64:
                # image tower (50 tokens): fused wgmma attention on HALF operands, the tensor core's native type
                out = attention_launch.forward_half(q, k, v, self.num_heads)
            else:
                # longer sequences: 2 bf16 planes (16 mantissa bits >= fp16's 11)
                out = attention_launch.forward(q, k, v, self.num_heads, nsplit=2, half_out=True)[0].to(x.dtype)
        else:
            out = ops.attention(q, k, v, self.num_heads, 0.0, False, causal=causal)
        return _linear(out, self.out_proj.weight, self.out_proj.bias, residual=residual)


class ResidualAttentionBlock(nn.Module):
    def __init__(self, d_model: int, n_head: int, causal: bool = False):
        super().__init__()
        self.attn = _PackedSelfAttention(d_model, n_head)
        self.ln_1 = LayerNorm(d_model)
        self.mlp = _MLP(OrderedDict([
            ("c_fc", nn.Linear(d_model, d_model * 4)),
            ("gelu", QuickGELU()),
            ("c_proj", nn.Linear(d_model * 4, d_model)),
        ]))
        self.ln_2 = LayerNorm(d_model)
        self.causal = causal

    def forward(self, x: torch.Tensor):  # (L, N, D)
        x = self.attn(self.ln_1(x), causal=self.causal, residual=x)      # x + attn(ln_1(x))
        return self.mlp(self.ln_2(x), residual=x)                         # x + mlp(ln_2(x))


class Transformer(nn.Module):
    def __init__(self, width: int, layers: int, heads: int, causal: bool = False):
        super().__init__()
        self.width, self.layers = width, layers
        self.resblocks = nn.Sequential(*[ResidualAttentionBlock(width, heads, causal) for _ in range(layers)])

    def forward(self, x: torch.Tensor):
        return self.resblocks(x)


class VisionTransformer(nn.Module):
    def __init__(self, input_resolution: int, patch_size: int, width: int, layers: int, heads: int, output_dim: int):
        super().__init__()
        self.input_resolution = input_resolution
        self.output_dim = output_dim
        self.conv1 = nn.Conv2d(3, width, kernel_size=patch_size, stride=patch_size, bias=False)
        scale = width ** -0.5
        self.class_embedding = nn.Parameter(scale * torch.randn(width))
        self.positional_embedding = nn.Parameter(scale * torch.randn((input_resolution // patch_size) ** 2 + 1, width))
        self.ln_pre = LayerNorm(width)
        self.transformer = Transformer(width, layers, heads)
        self.ln_post = LayerNorm(width)
        self.proj = nn.Parameter(scale * torch.randn(width, output_dim))

    def forward(self, x: torch.Tensor, im_name=None, max_w=None, if_pool=True, if_early_feat=False):
        """(N, 3, R, R) -> (cls embedding (N, output_dim), all tokens (N, grid^2 + 1, output_dim))"""
        ps = self.conv1.kernel_size[0]
        if x.dim() == 6:
            # patch-major crops (N, grid, grid, 3, ps, ps) straight from ops.crop_resize_normalize(patch=ps): already
            # the unfolded operand of the patch-embedding GEMM
            n, g = x.shape[0], x.shape[1]
            assert x.shape[2] == g and x.shape[3:] == (3, ps, ps) and x.is_contiguous()
            x = _linear(x.view(n * g * g, 3 * ps * ps), self.conv1.weight.view(self.conv1.weight.shape[0], -1),
                        None).view(n, g * g, -1)
        elif x.is_cuda and x.dtype == torch.float16 and x.shape[-1] % ps == 0 and (3 * ps * ps) % 64 == 0:
            # the patch embedding (kernel = stride = patch size, no bias) is a GEMM over unfolded patches
            n, c, hh, ww = x.shape
            g = hh // ps
            patches = x.view(n, c, g, ps, g, ps).permute(0, 2, 4, 1, 3, 5).reshape(n * g * g, c * ps * ps)
            x = _linear(patches, self.conv1.weight.view(self.conv1.weight.shape[0], -1), None).view(n, g * g, -1)
        else:
            x = self.conv1(x)                               # (N, width, grid, grid)
            x = x.reshape(x.shape[0], x.shape[1], -1).permute(0, 2, 1)
        cls = self.class_embedding.to(x.dtype).expand(x.shape[0], 1, -1)
        x = torch.cat([cls, x], dim=1) + self.positional_embedding.to(x.dtype)
        x = self.ln_pre(x)
        x = self.transformer(x.permute(1, 0, 2)).permute(1, 0, 2)
        all_tokens = self.ln_post(x)
        x = all_tokens[:, 0, :]
        if self.proj is not None:
            x, all_tokens = self._project(x), self._project(all_tokens)
        return x, all_tokens

    def _project(self, x):
        """x @ proj (reference CLIP/clip/model.py:655-657).  fp16 on the device: the wgmma GEMM with the transposed
        projection as its K-major weight (cached; the tower is frozen)."""
        if not (x.is_cuda and x.dtype == torch.float16 and x.shape[-1] % 64 == 0):
            return x @ self.proj
        key = (self.proj.data_ptr(), self.proj._version)
        if getattr(self, "_proj_t_key", None) != key:
            self._proj_t = self.proj.detach().t().contiguous()
            self._proj_t_key = key
        return _linear(x, self._proj_t, None)


class CLIP(nn.Module):
    def __init__(self, embed_dim: int, image_resolution: int, vision_layers: int, vision_width: int,
                 vision_patch_size: int, context_length: int, vocab_size: int, transformer_width: int,
                 transformer_heads: int, transformer_layers: int):
        super().__init__()
        self.context_length = context_length
        self.visual = VisionTransformer(image_resolution, vision_patch_size, vision_width, vision_layers,
                                        vision_width // 64, embed_dim)
        self.transformer = Transformer(transformer_width, transformer_layers, transformer_heads, causal=True)
        self.vocab_size = vocab_size
        self.token_embedding = nn.Embedding(vocab_size, transformer_width)
        self.positional_embedding = nn.Parameter(torch.empty(context_length, transformer_width))
        self.ln_final = LayerNorm(transformer_width)
        self.text_projection = nn.Parameter(torch.empty(transformer_width, embed_dim))
        self.logit_scale = nn.Parameter(torch.ones([]) * np.log(1 / 0.07))
        self.initialize_parameters()

    def initialize_parameters(self):
        nn.init.normal_(self.token_embedding.weight, std=0.02)
        nn.init.normal_(self.positional_embedding, std=0.01)
        for tower in (self.transformer, self.visual.transformer):
            proj_std = (tower.width ** -0.5) * ((2 * tower.layers) ** -0.5)
            attn_std = tower.width ** -0.5
            fc_std = (2 * tower.width) ** -0.5
            for block in tower.resblocks:
                nn.init.normal_(block.attn.in_proj_weight, std=attn_std)
                nn.init.normal_(block.attn.out_proj.weight, std=proj_std)
                nn.init.normal_(block.mlp.c_fc.weight, std=fc_std)
                nn.init.normal_(block.mlp.c_proj.weight, std=proj_std)
        nn.init.normal_(self.text_projection, std=self.transformer.width ** -0.5)

    @property
    def dtype(self):
        return self.visual.conv1.weight.dtype

    def encode_image(self, image, im_name=None, max_w=None, if_pool=True, if_early_feat=False):
        return self.visual(image.type(self.dtype))

    def encode_text(self, text):
        """text (N, context_length) int tokens -> (N, embed_dim); features at the EOT (largest id) token."""
        x = self.token_embedding(text).type(self.dtype) + self.positional_embedding.type(self.dtype)
        x = self.transformer(x.permute(1, 0, 2)).permute(1, 0, 2)
        x = self.ln_final(x).type(self.dtype)
        return x[torch.arange(x.shape[0]), text.argmax(dim=-1)] @ self.text_projection

    def forward(self, image, text):
        image_features = self.encode_image(image)[0]
        text_features = self.encode_text(text)
        image_features = image_features / image_features.norm(dim=1, keepdim=True)
        text_features = text_features / text_features.norm(dim=1, keepdim=True)
        logits_per_image = self.logit_scale.exp() * image_features @ text_features.t()
        return logits_per_image, logits_per_image.t()


def convert_weights(model: nn.Module):
    """Linear / conv / attention / projection parameters to fp16; LayerNorm and embeddings stay fp32."""
    def to_half(m):
        if isinstance(m, (nn.Conv1d, nn.Conv2d, nn.Linear)):
            m.weight.data = m.weight.data.half()
            if m.bias is not None:
                m.bias.data = m.bias.data.half()
        if isinstance(m, _PackedSelfAttention):
            m.in_proj_weight.data = m.in_proj_weight.data.half()
            m.in_proj_bias.data = m.in_proj_bias.data.half()
        for name in ("text_projection", "proj"):
            attr = getattr(m, name, None)
            if isinstance(attr, torch.Tensor):
                attr.data = attr.data.half()
    model.apply(to_half)


def build_model(state_dict: dict) -> CLIP:
    """Infers the ViT architecture from tensor shapes (reference model.py:1266-1312)."""
    if "visual.proj" not in state_dict:
        raise NotImplementedError("only ViT image towers are on the CoDA path")
    vision_width = state_dict["visual.conv1.weight"].shape[0]
    vision_layers = len([k for k in state_dict if k.startswith("visual.") and k.endswith(".attn.in_proj_weight")])
    vision_patch_size = state_dict["visual.conv1.weight"].shape[-1]
    grid = round((state_dict["visual.positional_embedding"].shape[0] - 1) ** 0.5)
    embed_dim = state_dict["text_projection"].shape[1]
    context_length = state_dict["positional_embedding"].shape[0]
    vocab_size = state_dict["token_embedding.weight"].shape[0]
    width = state_dict["ln_final.weight"].shape[0]
    layers = len({k.split(".")[2] for k in state_dict if k.startswith("transformer.resblocks")})
    model = CLIP(embed_dim, vision_patch_size * grid, vision_layers, vision_width, vision_patch_size,
                 context_length, vocab_size, width, width // 64, layers)
    sd = {k: v for k, v in state_dict.items() if k not in ("input_resolution", "context_length", "vocab_size")}
    convert_weights(model)
    model.load_state_dict(sd)
    return model.eval()


VIT_B32 = dict(embed_dim=512, image_resolution=224, vision_layers=12, vision_width=768, vision_patch_size=32,
               context_length=77, vocab_size=49408, transformer_width=512, transformer_heads=8,
               transformer_layers=12)
VIT_B16 = dict(VIT_B32, vision_patch_size=16)


def load(path: Optional[str], device="cuda", arch: str = "ViT-B/32", seed: int = 0) -> CLIP:
    """Loads an OpenAI CLIP checkpoint (TorchScript archive or plain state-dict) if
    `path` exists; otherwise builds a random-init model of `arch` (there are no
    pretrained weights offline -- throughput runs use random weights of the right
    architecture, and say so)."""
    if path is not None and os.path.exists(path):
        try:
            sd = torch.jit.load(path, map_location="cpu").state_dict()
        except RuntimeError:
            sd = torch.load(path, map_location="cpu")
        model = build_model(sd)
    else:
        gen_state = torch.random.get_rng_state()
        torch.manual_seed(seed)
        model = CLIP(**(VIT_B16 if arch.endswith("16") else VIT_B32))
        torch.random.set_rng_state(gen_state)
        convert_weights(model)
        model.eval()
    if str(device) == "cpu":
        model.float()
    for p in model.parameters():
        p.requires_grad = False
    return model.to(device)
