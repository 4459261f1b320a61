"""ScanNet camera on the H100: ops.boxes_in_image(camera="scannet") against the reference's fp64 chain restated in
tests/scannet_ref.py (torch.linalg.inv of the camera-to-world pose), the step against the reference's goldens of the
ScanNet cases (tests/scannet_parity_common.py), and the whole training step on ScanNet batches, captured as one CUDA
graph."""
import tempfile
import warnings

import numpy as np
import pytest
import torch

import model_parity_common as mpc
import scannet_parity_common as spc
import scannet_ref
from coda_neurips2023_b200 import ops, synthetic

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module", autouse=True)
def _lib(built_lib):
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False


@pytest.mark.parametrize("name", list(spc.CASES))
def test_scannet_step_matches_reference_golden(name):
    """Same bars as test_model_gpu.py: 1e-4 relative forward / loss; gradients 5e-3 or 4 x the fp32-vs-fp32 noise."""
    torch.manual_seed(0)
    model, out, loss, loss_dict, golden = spc.run(name, "cuda")
    errs = mpc.compare(model, out, loss, loss_dict, golden, rtol=1e-4, atol=1e-5, grad_rtol=5e-3,
                       noise=mpc.cpu_noise(name))
    fwd = {k: v for k, v in errs.items() if not k.startswith("grad.")}
    grd = {k: v for k, v in errs.items() if k.startswith("grad.")}
    wf, wg = max(fwd, key=fwd.get), max(grd, key=grd.get)
    print(f"PARITY {name}: forward worst {wf} = {fwd[wf]:.2e}; gradient worst {wg} = {grd[wg]:.2e}")


def _scene_boxes(batch, b, q, seed):
    """Boxes around points of each scene's cloud (sizes 0.1 .. 2 m): in front of, beside and behind the camera."""
    gen = torch.Generator().manual_seed(seed)
    pc = torch.from_numpy(batch["point_clouds"])
    idx = torch.randint(0, pc.shape[1], (b, q), generator=gen)
    ctr = torch.gather(pc, 1, idx.unsqueeze(-1).expand(-1, -1, 3)).unsqueeze(2)
    half = torch.rand(b, q, 1, 3, generator=gen) * 0.95 + 0.05
    sign = torch.tensor([[1, 1, 1], [1, 1, -1], [1, -1, 1], [1, -1, -1], [-1, 1, 1], [-1, 1, -1], [-1, -1, 1],
                         [-1, -1, -1]], dtype=torch.float32)
    corners = (ctr + half * sign).contiguous()
    size = (2 * half[:, :, 0]).contiguous()
    size[:, -1] = 0                                                 # zero-size box -> not usable
    return corners, size


@pytest.mark.parametrize("b,q,hw,seed", [(8, 256, (968, 1296), 0), (2, 7, (240, 320), 1), (3, 100, (968, 1296), 2)])
def test_boxes_in_image_scannet_matches_reference_projection_chain(b, q, hw, seed):
    batch = synthetic.make_batch(b, 3000, seed=seed, image_hw=hw, camera="scannet")
    batch["x_offset"] = np.arange(b, dtype=np.int64) * 3
    batch["y_offset"] = np.arange(b, dtype=np.int64) * 5 + 1
    inputs = {k: torch.from_numpy(v) for k, v in batch.items()}
    corners, size = _scene_boxes(batch, b, q, seed)
    exp_boxes, exp_valid, exp_ext = scannet_ref.boxes_in_image(corners, size, inputs, camera="scannet", extent=True)
    got_boxes, got_valid, got_ext = ops.boxes_in_image(corners.cuda(), size.cuda(), {k: v.cuda() for k, v in inputs.items()},
                                                       camera="scannet", extent=True)
    got_boxes, got_valid, got_ext = got_boxes.cpu(), got_valid.cpu(), got_ext.cpu()
    assert got_valid.dtype == torch.bool and got_boxes.dtype == torch.int32
    # the projected (clipped, offset, flipped) extents: the in-kernel inverse is not LAPACK's, so not bit-equal
    rel = ((got_ext - exp_ext).abs() / exp_ext.abs().clamp(min=1.0)).max().item()
    assert rel <= 1e-9, rel
    # integer boxes: equal wherever the restated coordinate is not within 1e-6 px of an integer (a coordinate that is
    # an integer exactly -- clipped to an image edge -- is the same in both)
    off = (exp_ext - exp_ext.round()).abs()
    near = ((off > 0) & (off < 1e-6)).any(-1)
    print(f"SCANNET boxes_in_image b={b} q={q}: max rel extent diff {rel:.2e}; {int(near.sum())} boxes with a "
          f"coordinate within 1e-6 px of an integer; {int(exp_valid.sum())} of {b * q} usable")
    assert torch.equal(got_boxes[~near], exp_boxes[~near])
    assert torch.equal(got_valid, exp_valid)
    assert 0 < int(exp_valid.sum()) < b * q
    # every scene sees the same inverse pose: the boxes of one scene do not depend on which block computes them
    again = ops.boxes_in_image(corners[:1].repeat(b, 1, 1, 1).cuda(), size[:1].repeat(b, 1, 1).cuda(),
                               {k: v[:1].repeat(b, *([1] * (v.dim() - 1))).cuda() for k, v in inputs.items()},
                               camera="scannet", extent=True)[2].cpu()
    assert all(torch.equal(again[i], again[0]) for i in range(b))


def test_boxes_in_image_rejects_a_mismatched_camera_on_the_device():
    batch = synthetic.to_device(synthetic.make_batch(2, 500, seed=0, camera="scannet"), "cuda")
    corners, size = torch.zeros(2, 4, 8, 3, device="cuda"), torch.ones(2, 4, 3, device="cuda")
    with pytest.raises(ValueError, match="K .* and Rtilt"):
        ops.boxes_in_image(corners, size, batch)                      # 4 x 4 matrices, SUN RGB-D camera
    sun = synthetic.to_device(synthetic.make_batch(2, 500, seed=0), "cuda")
    with pytest.raises(ValueError, match="K .* and Rtilt"):
        ops.boxes_in_image(corners, size, sun, camera="scannet")


def test_boxes_in_image_sunrgbd_unchanged_by_extent():
    batch = synthetic.make_batch(2, 3000, seed=3)
    inputs = {k: torch.from_numpy(v).cuda() for k, v in batch.items()}
    corners, size = _scene_boxes(batch, 2, 64, 3)
    a = ops.boxes_in_image(corners.cuda(), size.cuda(), inputs)
    b_, v_, ext = ops.boxes_in_image(corners.cuda(), size.cuda(), inputs, camera="sunrgbd", extent=True)
    assert torch.equal(a[0], b_) and torch.equal(a[1], v_)
    assert torch.equal(ext.to(torch.int32), b_)


def test_scannet_stage2_step_graph_replays_equal_the_eager_step():
    """The stage-2 script's shape (8 scenes x 40 000 points, 1296 x 968 images, 128 queries, 60 prompts, discovery on)
    on ScanNet batches: TrainStep.capture + three replays give finite losses, and with dropout 0 the first replay's
    loss equals the eager step's from the same state."""
    from coda_neurips2023_b200 import attention_launch
    from coda_neurips2023_b200.criterion import build_criterion
    from coda_neurips2023_b200.engine import TrainStep
    from coda_neurips2023_b200.models import build_model

    args = synthetic.make_args(
        dataset_name="scannet_anonymous_aligned_image_with_novel_cate_confi", nqueries=128, train_range_max=10,
        test_range_max=60, image_size_width=1296, image_size_height=968, matcher_giou_cost=2.0,
        matcher_center_cost=0.0, matcher_objectness_cost=0.0, loss_no_object_weight=0.25, base_lr=1.4142e-4,
        if_clip_weak_labels=True, loss_feat_seen_softmax_weakly_loss_with_novel_cate_confi_weight=1.0,
        online_nms_update_save_novel_label_clip_driven_with_cate_confidence=True, save_objectness=0.3,
        clip_driven_keep_thres=0.3, online_nms_update_save_epoch=50, distillation_box_num=32,
        enc_dropout=0.0, dec_dropout=0.0, mlp_dropout=0.0)
    cfg = synthetic.SyntheticDatasetConfig(args)

    def make():
        torch.manual_seed(0)
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            model, _ = build_model(args, cfg)
        return model.cuda().train(), build_criterion(args, cfg).cuda()

    tmp = tempfile.mkdtemp(prefix="coda_scannet_pseudo_")
    batches = []
    for s in range(3):
        bt = synthetic.to_device(synthetic.make_batch(8, 40000, seed=20 + s, image_hw=(968, 1296), camera="scannet"),
                                 "cuda")
        bt["pseudo_box_path"] = [f"{tmp}/s{s}_scene{i}.npy" for i in range(8)]
        batches.append(bt)
    model, crit = make()
    seed0 = int(attention_launch.seed_counter(torch.device("cuda", 0)))
    step = TrainStep(args, model, crit, torch.device("cuda", 0))
    np.random.seed(11)
    step.capture(batches[0], warmup=2)
    losses = []
    for i, bt in enumerate(batches):
        np.random.seed(12 + i)
        loss, _ = step(bt, 0.0)
        losses.append(float(loss))
    assert all(np.isfinite(losses)), losses
    model2, crit2 = make()
    attention_launch.seed_counter(torch.device("cuda", 0)).fill_(seed0)
    step2 = TrainStep(args, model2, crit2, torch.device("cuda", 0))
    step2.prepare(batches[0])
    np.random.seed(12)
    loss_e = float(step2(batches[0], 0.0)[0])
    print(f"SCANNET stage-2 step: graph losses {losses}, eager {loss_e}")
    assert abs(loss_e - losses[0]) <= 1e-5 * abs(losses[0])
