"""The ViT-B/16 CLIP image tower -- the checkpoint the reference ships (models/model_3detr.py:325, :373): 197 tokens per
crop, so its attention runs on the resident fp16 kernel of coda_attention_fwd_half (64 < l <= 256), which reads
q / k / v by TMA straight out of the fused in-projection.

  * the tower against the REFERENCE's own VisionTransformer at B/16 geometry (tests/golden/clip_vit_b16.npz, made by
    tests/golden/make_clip_vit_b16_golden.py), with the bar of tests/test_clip_gpu.py, and never on the bf16
    route (attention_launch.forward);
  * the kernel against fp64 at 1 - 4 key tiles, full and partial last tiles, on fused-projection slices and on
    contiguous tensors, with nothing written past the output;
  * run-to-run bits, a CUDA-graph replay of the tower, the 16-pixel patch-major crops, the model's crop path and a
    captured training step with clip_arch = ViT-B/16;
  * the C entry's refusals (l > 256, hd != 64, a row stride TMA cannot take)."""
import ctypes
import warnings
from pathlib import Path

import numpy as np
import pytest
import torch

from param_fill import fill_by_name

pytestmark = pytest.mark.gpu
GOLDEN = Path(__file__).resolve().parent / "golden" / "clip_vit_b16.npz"

# l of the resident kernel: 2, 3 and 4 key tiles, full and partial last tiles, both ends of 64 < l <= 256
# (tests/test_clip_b16_cpu.py checks this list covers every case)
KERNEL_L = [65, 100, 127, 128, 129, 192, 193, 197, 255, 256]
KERNEL_CASES = [(l, b, h) for l in KERNEL_L for b, h in ((1, 1), (3, 4))] + [(197, 256, 12)]
SENTINEL = -12345.0


def _crops(n=32):
    g = torch.Generator().manual_seed(77)     # tests/golden/make_clip_vit_golden.py:crops
    x = torch.randn(n, 3, 224, 224, generator=g)
    x[:, :, :40, :] = 1.9
    return x.half()


def _vit_b16():
    from coda_neurips2023_b200.clip import model as cm

    vit = cm.VisionTransformer(input_resolution=224, patch_size=16, width=768, layers=12, heads=12, output_dim=512)
    fill_by_name(vit, seed=21)
    cm.convert_weights(vit)
    return vit.cuda().eval()


def _no_bf16_route(monkeypatch):
    from coda_neurips2023_b200 import attention_launch

    def refuse(*a, **k):
        raise AssertionError("the B/16 tower took the bf16 attention route")

    monkeypatch.setattr(attention_launch, "forward", refuse)


def _ref64(q, k, v, h):
    """fp64 softmax(q k^T / 8) v per head, (l, b, h * 64) in and out"""
    l, b, e = q.shape
    qd, kd, vd = (t.double().reshape(l, b, h, 64).permute(1, 2, 0, 3) for t in (q, k, v))
    p = torch.softmax(qd @ kd.transpose(-1, -2) / 8.0, dim=-1)
    return (p @ vd).permute(2, 0, 1, 3).reshape(l, b, e)


def _fwd_half_c(q, k, v, h, out, lds, hd=64):
    from coda_neurips2023_b200._lib import lib, ptr, stream_of

    l, b, _ = q.shape
    cl = ctypes.c_longlong
    with torch.cuda.device(q.device):
        return lib().coda_attention_fwd_half(ctypes.c_int(b), ctypes.c_int(h), ctypes.c_int(l), ctypes.c_int(hd),
                                             ptr(q), ptr(k), ptr(v), cl(lds[0]), cl(lds[1]), cl(lds[2]), ptr(out),
                                             ctypes.c_void_p(0), stream_of(q))


def test_vit_b16_fp16_tower_matches_reference_golden(built_lib, monkeypatch):
    from coda_neurips2023_b200 import _lib

    gold = np.load(GOLDEN)
    vit = _vit_b16()
    _no_bf16_route(monkeypatch)
    n0 = _lib.LAUNCHES
    with torch.no_grad():
        cls, tok = vit(_crops().cuda())
    assert _lib.LAUNCHES - n0 >= 12 * 6, "the tower did not run on the package's own kernels"
    assert cls.dtype == torch.float16 and tok.shape == (32, 197, 512)
    cls = cls.float().cpu().numpy()
    tok = tok.float().cpu().numpy()[:, ::7, ::8]
    exact, ref16 = gold["cls32"], gold["cls16"]
    scale = np.abs(exact).max()
    ref_err = np.abs(ref16 - exact).max() / scale
    our_err = np.abs(cls - exact).max() / scale
    cos = (cls * exact).sum(1) / (np.linalg.norm(cls, axis=1) * np.linalg.norm(exact, axis=1))
    tok_err = np.abs(tok - gold["tok32"]).max() / np.abs(gold["tok32"]).max()
    print(f"PARITY clip_vit_b16: ours max-rel {our_err:.2e} (reference fp16 run {ref_err:.2e}), min cosine "
          f"{cos.min():.7f}, tokens max-rel {tok_err:.2e}")
    assert our_err <= min(2.0 * ref_err, 4e-3)
    assert cos.min() >= 0.99999
    assert tok_err <= 4e-3


@pytest.mark.parametrize("layout", ["fused", "contiguous"])
@pytest.mark.parametrize("l,b,h", KERNEL_CASES)
def test_resident_half_attention_matches_fp64(built_lib, l, b, h, layout):
    """fp16 probabilities carry 11 mantissa bits (as the reference's all-half nn.MultiheadAttention): 2e-3 relative,
    the bar of the l <= 64 instance.  Output rows past l * b * h * 64 halves stay as they were."""
    from coda_neurips2023_b200 import attention_launch

    torch.manual_seed(l * 31 + b)
    e = h * 64
    qkv = (torch.randn(l, b, 3 * e, device="cuda") * 0.8).half()
    if layout == "fused":
        q, k, v = qkv.split(e, dim=-1)
        lds = [3 * e] * 3
    else:
        q, k, v = (t.contiguous() for t in qkv.split(e, dim=-1))
        lds = [e] * 3
    n = l * b * e
    buf = torch.full((n + 4096,), SENTINEL, dtype=torch.float16, device="cuda")
    assert _fwd_half_c(q, k, v, h, buf, lds) == 0
    torch.cuda.synchronize()
    out = buf[:n].view(l, b, e)
    ref = _ref64(q, k, v, h)
    err = ((out.double() - ref).abs().max() / ref.abs().max()).item()
    assert err < 2e-3, err
    assert bool((buf[n:] == SENTINEL).all()), "the kernel wrote past row l - 1"
    # the Python launcher runs the same kernel
    assert torch.equal(attention_launch.forward_half(q, k, v, h), out)


def test_resident_half_attention_is_deterministic_and_needs_no_workspace(built_lib):
    from coda_neurips2023_b200 import attention_launch

    torch.manual_seed(5)
    l, b, h = 197, 256, 12
    e = h * 64
    q, k, v = (torch.randn(l, b, 3 * e, device="cuda") * 0.8).half().split(e, dim=-1)
    a = attention_launch.forward_half(q, k, v, h)
    before = torch.cuda.memory_allocated()
    c = attention_launch.forward_half(q, k, v, h)
    assert torch.cuda.memory_allocated() - before == a.numel() * 2      # the output, nothing else
    assert torch.equal(a, c)


def test_vit_b16_tower_graph_replay_equals_eager(built_lib, monkeypatch):
    vit = _vit_b16()
    _no_bf16_route(monkeypatch)
    x = _crops().cuda()
    with torch.no_grad():
        cls_e, tok_e = vit(x)
        cls_2, _ = vit(x)
        assert torch.equal(cls_e, cls_2)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            cls_g, tok_g = vit(x)
        graph.replay()
        graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(cls_g, cls_e) and torch.equal(tok_g, tok_e)


@pytest.mark.parametrize("hw", [(531, 730), (968, 1296)])
@pytest.mark.parametrize("dtype", [torch.float16, torch.float32])
def test_crop_patch16_is_the_nchw_crop_unfolded(built_lib, hw, dtype):
    from coda_neurips2023_b200 import ops

    rng = np.random.default_rng(hw[0])
    h, w = hw
    imgs = torch.from_numpy(rng.integers(0, 256, size=(8, h, w, 3), dtype=np.uint8)).cuda()
    n = 256
    x0 = rng.integers(0, w - 2, n); y0 = rng.integers(0, h - 2, n)
    x1 = np.minimum(x0 + rng.integers(1, w, n), w); y1 = np.minimum(y0 + rng.integers(1, h, n), h)
    boxes = torch.from_numpy(np.stack([x0, y0, x1, y1], 1).astype(np.int32)).cuda()
    scene = torch.from_numpy(np.repeat(np.arange(8), 32).astype(np.int32)).cuda()
    valid = torch.from_numpy(rng.random(n) > 0.1).cuda()
    nchw = ops.crop_resize_normalize(imgs, scene, boxes, valid, 224, dtype=dtype)
    pm = ops.crop_resize_normalize(imgs, scene, boxes, valid, 224, dtype=dtype, patch=16)
    assert pm.shape == (n, 14, 14, 3, 16, 16)
    assert torch.equal(pm, nchw.view(n, 3, 14, 16, 14, 16).permute(0, 2, 4, 1, 3, 5))


def _b16_model():
    from coda_neurips2023_b200 import synthetic
    from coda_neurips2023_b200.criterion import build_criterion
    from coda_neurips2023_b200.models import build_model

    args = synthetic.make_args(clip_arch="ViT-B/16")
    cfg = synthetic.SyntheticDatasetConfig(args)
    torch.manual_seed(0)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        model, _ = build_model(args, cfg)
    return args, model.cuda().train(), build_criterion(args, cfg).cuda()


def test_model_crop_path_equals_the_tower_on_nchw_crops(built_lib, monkeypatch):
    from coda_neurips2023_b200 import ops, synthetic

    _, model, _ = _b16_model()
    assert model.clip_model.visual.conv1.kernel_size[0] == 16
    _no_bf16_route(monkeypatch)
    inputs = synthetic.to_device(synthetic.make_batch(8, 2000, seed=3), "cuda")
    h, w = inputs["input_image"].shape[1:3]
    g = torch.Generator(device="cuda").manual_seed(1)
    nq, ns = 64, 32
    xy0 = torch.rand(8, nq, 2, device="cuda", generator=g) * torch.tensor([w - 8, h - 8], device="cuda")
    wh = torch.rand(8, nq, 2, device="cuda", generator=g) * torch.tensor([w / 2, h / 2], device="cuda") + 2
    xy1 = torch.minimum(xy0 + wh, torch.tensor([w, h], device="cuda"))
    boxes = torch.cat([xy0, xy1], -1).to(torch.int32)
    valid = torch.rand(8, nq, device="cuda", generator=g) > 0.2
    sel = torch.stack([torch.randperm(nq, device="cuda", generator=g)[:ns] for _ in range(8)])
    feats, vd = model._clip_embed_boxes(inputs, boxes, valid, sel)
    bx = torch.gather(boxes, 1, sel.unsqueeze(-1).expand(-1, -1, 4)).reshape(-1, 4).contiguous()
    scene = torch.arange(8, device="cuda", dtype=torch.int32).repeat_interleave(ns)
    crops = ops.crop_resize_normalize(inputs["input_image"], scene, bx, vd.reshape(-1), 224, dtype=torch.float16)
    with torch.no_grad():
        cls, _ = model.clip_model.visual(crops)
    assert torch.equal(feats, cls.float().reshape(8, ns, -1))


def test_b16_train_step_captures_and_replays(built_lib):
    from coda_neurips2023_b200 import synthetic
    from coda_neurips2023_b200.engine import TrainStep

    args, model, crit = _b16_model()
    step = TrainStep(args, model, crit, torch.device("cuda", 0))
    data = synthetic.to_device(synthetic.make_batch(8, 20000, seed=0), "cuda")
    np.random.seed(0)
    step.capture(data, warmup=2)
    losses = [float(step(data, 0.0)[0]) for _ in range(3)]
    print(f"B/16 step: graph losses {losses}")
    assert all(np.isfinite(losses)), losses


def test_fwd_half_refuses_what_the_kernels_cannot_take(built_lib):
    e = 12 * 64
    qkv = torch.zeros(257, 2, 3 * e + 8, dtype=torch.float16, device="cuda")
    out = torch.empty(257 * 2 * e, dtype=torch.float16, device="cuda")

    def qkv_of(l, ld):
        flat = qkv.view(-1)[: l * 2 * ld].view(l, 2, ld)
        return flat[..., :e], flat[..., e:2 * e], flat[..., 2 * e:3 * e]

    q, k, v = qkv_of(257, 3 * e)
    assert _fwd_half_c(q, k, v, 12, out, [3 * e] * 3) == -1                     # l = 257
    q, k, v = qkv_of(197, 3 * e)
    assert _fwd_half_c(q, k, v, 6, out, [3 * e] * 3, hd=128) == -1              # hd = 128
    q, k, v = qkv_of(197, 3 * e + 4)
    assert _fwd_half_c(q, k, v, 12, out, [3 * e + 4] * 3) == -1                 # row stride not a multiple of 8
    q, k, v = qkv_of(197, 3 * e)
    assert _fwd_half_c(q, k, v, 12, out, [3 * e] * 3) == 0                      # the same call, well formed
    torch.cuda.synchronize()
