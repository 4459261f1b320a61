"""CoDA's 3DETR detector with the CLIP alignment head, H100-native.

Mirror of the registered model classes of reference models/model_3detr.py:
`Model3DETRPredictedBoxDistillationHead` (:130-1833, CoDA proper),
`BoxProcessor` (:56-127), the builders `build_preencoder / build_encoder /
build_decoder / build_3detr_predictedbox_distillation_head` (:3935-4050).
Same constructor keywords, same `forward(inputs, encoder_only, if_test,
if_real_test, curr_epoch, if_cmp_class)` signature, same output-dict keys and
the same parameter names, so `main.py` / `engine.py` and released checkpoints
work unchanged.

What is different is how the step executes:
  * FPS / ball-query / grouping: cluster + ballot kernels (pointnet2/),
  * attention: fused wgmma kernel, LayerNorm / Fourier encoding: warp kernels,
  * the CLIP crop pipeline (reference :984-1103: a Python double loop with four
    host syncs per box and one CLIP call per scene) is one batched projection in
    fp64 tensor ops, ONE crop+pad+bicubic-resize+normalise kernel for all B x 32
    boxes and ONE CLIP forward -- no device->host synchronisation at all.
"""
from __future__ import annotations

import math
import os
import warnings
from functools import partial

import numpy as np
import torch
import torch.nn as nn

from .. import clip as clip_mod
from .. import ops
from ..pointnet2.pointnet2_modules import PointnetSAModuleVotes
from ..pointnet2.pointnet2_utils import furthest_point_sample
from ..utils.pc_util import scale_points, shift_scale_points
from .helpers import GenericMLP
from .position_embedding import PositionEmbeddingCoordsSine
from .transformer import (MaskedTransformerEncoder, TransformerDecoder, TransformerDecoderLayer, TransformerEncoder,
                          TransformerEncoderLayer)

CLIP_CHECKPOINT = "./CLIP/pretrain_models/ViT-B-16.pt"  # path the reference hard-codes (:325)
ALL_CLASS_PATH_V1 = "datasets/all_classes_trainval_v1.npy"
ALL_CLASS_PATH_V2 = "datasets/all_classes_trainval_v2_revised_del_val_less_than_5_classes.npy"
ALL_SUPERCLASS_PATH = "datasets/lvis_1204.npy"
ALL_CMP_CLASS_PATH = "datasets/ov_3detr.npy"                  # the OV-3DET paper's comparison classes, SUN RGB-D
ALL_CMP_CLASS_PATH_SCANNET = "datasets/ov_3detr_scannet.npy"  # ... and ScanNet
SCANNET_CLASS_NAMES_PATH = "datasets/scannet_200_classname_no_wall_floor.npy"   # the text rows, in order
SCANNET_CLASS_IDS_PATH = "datasets/scannet_200_class2id.npy"                     # {name: ScanNet-200 class id}


class BoxProcessor(object):
    """Converts the MLP-head outputs into boxes (reference :56-127)."""

    def __init__(self, dataset_config):
        self.dataset_config = dataset_config

    def compute_predicted_center(self, center_offset, query_xyz, point_cloud_dims):
        center_unnormalized = query_xyz + center_offset
        center_normalized = shift_scale_points(center_unnormalized, src_range=point_cloud_dims)
        return center_normalized, center_unnormalized

    def compute_predicted_size(self, size_normalized, point_cloud_dims):
        scene_scale = torch.clamp(point_cloud_dims[1] - point_cloud_dims[0], min=1e-1)
        return scale_points(size_normalized, mult_factor=scene_scale)

    def compute_predicted_angle(self, angle_logits, angle_residual):
        if angle_logits.shape[-1] == 1:
            # datasets without rotation: keep both heads in the graph (DDP), angle = 0
            angle = angle_logits * 0 + angle_residual * 0
            return angle.squeeze(-1).clamp(min=0)
        angle_per_cls = 2 * np.pi / self.dataset_config.num_angle_bin
        pred_angle_class = angle_logits.argmax(dim=-1).detach()
        angle_center = angle_per_cls * pred_angle_class
        angle = angle_center + angle_residual.gather(2, pred_angle_class.unsqueeze(-1)).squeeze(-1)
        return torch.where(angle > np.pi, angle - 2 * np.pi, angle)

    def compute_objectness_and_cls_prob(self, cls_logits):
        cls_prob = torch.nn.functional.softmax(cls_logits, dim=-1)
        return cls_prob[..., :-1], 1 - cls_prob[..., -1]

    def compute_objectness_and_cls_prob_sigmoid(self, cls_logits):
        cls_prob = torch.sigmoid(cls_logits)
        return cls_prob[..., :-1], 1 - cls_prob[..., -1]

    def box_parametrization_to_corners(self, box_center_unnorm, box_size_unnorm, box_angle):
        return self.dataset_config.box_parametrization_to_corners(box_center_unnorm, box_size_unnorm, box_angle)

    def box_parametrization_to_corners_np(self, box_center_unnorm, box_size_unnorm, box_angle):
        return self.dataset_config.box_parametrization_to_corners_np(box_center_unnorm, box_size_unnorm, box_angle)

    def box_parametrization_to_corners_xyz(self, box_center_unnorm, box_size_unnorm, box_angle):
        return self.dataset_config.box_parametrization_to_corners_xyz(box_center_unnorm, box_size_unnorm, box_angle)


def _prompt(name) -> str:
    return "a photo of a " + str(name).replace("_", " ").lower() + " in the scene"


def scannet_class_rows(names, name_to_id) -> dict:
    """ScanNet-200 class id -> its row in `names` (the class names without wall and floor), matched by name."""
    row_of = {str(n): r for r, n in enumerate(names)}
    return {int(i): row_of[str(n)] for n, i in name_to_id.items() if str(n) in row_of}


def scannet_prompt_class_ids(train_ids, test_ids, reset_num: int) -> list:
    """Class ids of the evaluated ScanNet prompts (reference :228-242): the seen classes, then the unseen classes of
    `test_ids` in their order until `reset_num` of them have been added (at least one), sorted by id."""
    ids, added = list(train_ids), 0
    for c in test_ids:
        if c in train_ids:
            continue
        ids.append(c)
        added += 1
        if added >= reset_num:
            break
    return sorted(ids)


def _scannet_class_names(args, evaluated: bool):
    if not (os.path.exists(SCANNET_CLASS_NAMES_PATH) and os.path.exists(SCANNET_CLASS_IDS_PATH)):
        return None
    names = np.load(SCANNET_CLASS_NAMES_PATH)
    rows = scannet_class_rows(names, np.load(SCANNET_CLASS_IDS_PATH, allow_pickle=True).item())
    train = [int(i) for i in args.train_range_list]
    if evaluated:
        ids = scannet_prompt_class_ids(train, [int(i) for i in args.test_range_list], int(args.reset_scannet_num))
    else:
        ids = train                                  # the seen classes, in the order given
    return [names[rows[i]] for i in ids]


def _class_prompts(args, evaluated=None):
    """'a photo of a {class} in the scene' prompts of the seen (`evaluated` False) or evaluated classes (None: as
    --if_clip_more_prompts says)
    (reference :197-279, :1923-1988).  Needs the class lists of a CoDA checkout (relative paths, as
    in the reference); returns None when they are not reachable (synthetic runs).
    SUN RGB-D: the first train_range_max / test_range_max names of the class dictionary.
    ScanNet (dataset_name contains "scannet"): the ScanNet-200 names picked by class id through
    train_range_list / test_range_list / reset_scannet_num."""
    if evaluated is None:
        evaluated = getattr(args, "if_clip_more_prompts", False)
    if getattr(args, "dataset_name", "").find("scannet") != -1:
        names = _scannet_class_names(args, evaluated)
        return None if names is None else [_prompt(c) for c in names]
    path = ALL_CLASS_PATH_V1 if getattr(args, "if_use_v1", True) else ALL_CLASS_PATH_V2
    if not os.path.exists(path):
        return None
    names = list(np.load(path, allow_pickle=True).item().keys())
    n = args.test_range_max if evaluated else args.train_range_max
    return [_prompt(c) for c in names[:n]]


def superset_prompts(args):
    """The 'superset' prompts of --if_clip_superset (reference :282-323): the seen classes' prompts, then the LVIS
    names of ALL_SUPERCLASS_PATH (its first entry is the column header "name"), each prompt once.  The seen prompts are
    the first 10 of the evaluated prompts for SUN RGB-D, and for ScanNet the seen classes' rows of the evaluated
    prompts, in their order.  None when the class lists are not reachable (synthetic runs); FileNotFoundError when
    they are and the LVIS list is not."""
    evaluated = _class_prompts(args, True)
    if evaluated is None:
        return None
    if not os.path.exists(ALL_SUPERCLASS_PATH):
        raise FileNotFoundError(f"--if_clip_superset needs the LVIS class list {ALL_SUPERCLASS_PATH}, which is "
                                "missing: refusing to stand random rows in for the superset text features")
    if getattr(args, "dataset_name", "").find("scannet") != -1:
        train = [int(i) for i in args.train_range_list]
        ids = scannet_prompt_class_ids(train, [int(i) for i in args.test_range_list], int(args.reset_scannet_num))
        seen = [evaluated[r] for r, c in enumerate(ids) if c in train]
    else:
        seen = evaluated[:10]
    out = []
    for p in seen + [_prompt(c) for c in list(np.load(ALL_SUPERCLASS_PATH, allow_pickle=True))[1:]]:
        if p not in out:
            out.append(p)
    return out


def cmp_prompts(args):
    """The prompts of the comparison classes of forward(if_cmp_class=True) (reference :1971-2000): the names of
    ALL_CMP_CLASS_PATH (ALL_CMP_CLASS_PATH_SCANNET when dataset_name contains "scannet") in file order.  None when the
    class lists are not reachable (synthetic runs); FileNotFoundError when they are and the comparison list is not."""
    if _class_prompts(args, True) is None:
        return None
    path = ALL_CMP_CLASS_PATH_SCANNET if getattr(args, "dataset_name", "").find("scannet") != -1 else ALL_CMP_CLASS_PATH
    if not os.path.exists(path):
        raise FileNotFoundError(f"the comparison-class evaluation (if_cmp_class) needs the class list {path}, "
                                "which is missing")
    return [_prompt(c) for c in np.load(path)]


class Model3DETRPredictedBoxDistillationHead(nn.Module):
    """pre_encoder (PointNet++ SA) -> encoder -> query sampling -> decoder -> MLP heads,
    plus CLIP embeddings of the predicted boxes' image crops as distillation targets."""

    def __init__(self, pre_encoder, encoder, decoder, dataset_config, image_text_encoder=None,
                 encoder_dim=256, decoder_dim=256, position_embedding="fourier", mlp_dropout=0.3,
                 num_queries=256, if_with_clip=False, if_use_gt_box=False, if_expand_box=False,
                 if_with_clip_embed=False, if_with_clip_train=True, num_cls_predict=1,
                 if_with_fake_classes=False, pooling_methods="average", if_clip_more_prompts=False,
                 if_keep_box=False, if_select_box_by_objectness=False, keep_objectness=0.5,
                 online_nms_update_novel_label=False, online_nms_update_accumulate_novel_label=False,
                 online_nms_update_accumulate_epoch=10, distillation_box_num=32, args=None, has_clip=None):
        super().__init__()
        self.if_with_fake_classes = if_with_fake_classes
        self.num_cls_predict = num_cls_predict
        self.pre_encoder = pre_encoder
        self.encoder = encoder
        self.args = args
        self.if_with_clip = if_with_clip
        self.if_clip_more_prompts = if_clip_more_prompts
        self.if_with_clip_train = if_with_clip_train
        self.has_clip = if_with_clip_train if has_clip is None else has_clip     # a frozen CLIP and the text features
        self.box_idx_list = np.arange(128, dtype=np.int8)  # reference :191 (fixed, whatever nqueries is)
        self.external_selection = None  # device (B, 32) int64 tensor when the step is CUDA-graph captured
        self.if_keep_box = if_keep_box
        self.if_select_box_by_objectness = if_select_box_by_objectness
        self.if_use_gt_box, self.if_expand_box = if_use_gt_box, if_expand_box
        self.device = "cuda" if torch.cuda.is_available() else "cpu"
        self.train_range_max = args.train_range_max
        self.test_range_max = args.test_range_max
        self.if_clip_superset = getattr(args, "if_clip_superset", False)

        if self.has_clip:
            self._build_clip(args, dataset_config)

        self.encoder_to_decoder_projection = GenericMLP(
            input_dim=self._projection_dims(encoder_dim)[0], hidden_dims=self._projection_dims(encoder_dim)[1],
            output_dim=decoder_dim, norm_fn_name="bn1d", activation="relu", use_conv=True,
            output_use_activation=True, output_use_norm=True, output_use_bias=False)
        self.pos_embedding = PositionEmbeddingCoordsSine(d_pos=decoder_dim, pos_type=position_embedding,
                                                         normalize=True)
        self.query_projection = GenericMLP(
            input_dim=decoder_dim, hidden_dims=[decoder_dim], output_dim=decoder_dim, use_conv=True,
            output_use_activation=True, hidden_use_bias=True)
        self.decoder = decoder
        self.build_mlp_heads(dataset_config, decoder_dim, mlp_dropout)

        self.num_queries = num_queries
        self.box_processor = BoxProcessor(dataset_config)
        self.keep_objectness = keep_objectness
        self.online_nms_update_save_novel_label_clip_driven_with_cate_confidence = getattr(
            args, "online_nms_update_save_novel_label_clip_driven_with_cate_confidence", False)
        self.save_objectness = getattr(args, "save_objectness", 0.75)
        self.online_nms_update_save_epoch = getattr(args, "online_nms_update_save_epoch", 10)
        self.clip_driven_keep_thres = getattr(args, "clip_driven_keep_thres", 1e6)
        self.online_nms_update_accumulate_epoch = online_nms_update_accumulate_epoch
        self.distillation_box_num = distillation_box_num
        self.eval_layer_id = getattr(args, "eval_layer_id", -1)
        self.dataset_name = "scannet" if args.dataset_name.find("scannet") != -1 else "sunrgbd"
        self.if_clip_weak_labels = getattr(args, "if_clip_weak_labels", False)
        self.if_accumulate_former_pseudo_labels = getattr(args, "if_accumulate_former_pseudo_labels", False)
        self._pending_pseudo = None

    def _projection_dims(self, encoder_dim):
        """(input_dim, hidden_dims) of encoder_to_decoder_projection: the reference hard-codes 256, [512, 512] in
        this head (:409-412)."""
        return 256, [512, 512]

    # ------------------------------------------------------------------ CLIP side
    # True: the prompts of the evaluated classes (test_range_max); False: the seen ones (train_range_max).  The CoDA
    # head follows --if_clip_more_prompts
    def _evaluated_prompts(self, args):
        return getattr(args, "if_clip_more_prompts", False)

    # True: normalise the text features in CLIP's own dtype (fp16 on the GPU), then cast to fp32
    TEXT_NORM_IN_CLIP_DTYPE = False

    def _build_clip(self, args, dataset_config):
        """Frozen CLIP + L2-normalised text features of the class prompts (reference :197-399).
        The reference loads the same checkpoint twice (`clip_model`, `test_clip_model`);
        both are frozen and identical, so one set of weights is shared."""
        ckpt = getattr(args, "clip_checkpoint", CLIP_CHECKPOINT)
        arch = getattr(args, "clip_arch", "ViT-B/32")
        if not os.path.exists(ckpt):
            warnings.warn(f"CLIP checkpoint {ckpt} not found: using a RANDOM-INIT {arch} "
                          "(valid for throughput / parity runs only)")
        self.clip_model = clip_mod.load(ckpt, device=self.device, arch=arch)
        self.test_clip_model = self.clip_model
        self.res_encoder = self.clip_model.visual
        self.logit_scale = self.clip_model.logit_scale
        self.test_logit_scale = self.clip_model.logit_scale.exp()
        res = self.clip_model.visual.input_resolution
        self.clip_resolution = res

        evaluated = self._evaluated_prompts(args)
        prompts = _class_prompts(args, evaluated)
        if self.if_clip_superset:
            self.superset_all_classes_keys = superset_prompts(args)
        tokens = None
        if prompts is not None:
            try:
                from ..clip.tokenizer import tokenize
                tokens = tokenize(prompts).to(self.device)
            except FileNotFoundError as e:
                if os.path.exists(ckpt):
                    raise RuntimeError("a real CLIP checkpoint was loaded but the BPE vocabulary of the tokenizer is "
                                       f"missing ({e}): refusing to substitute random text features") from e
                tokens = None
        self.all_classes_keys = prompts
        self.text_features_synthetic = tokens is None
        with torch.no_grad():
            if tokens is not None:
                raw = self.clip_model.encode_text(tokens)
                feats = raw.to(torch.float32)
            else:
                # synthetic run: random unit rows stand in for the text embeddings (SURVEY.md 8d)
                if os.path.exists(ckpt):
                    raise RuntimeError(f"CLIP checkpoint {ckpt} found but the class list / tokenizer vocabulary is not: "
                                       "the text features would be meaningless")
                warnings.warn("class prompts unavailable: RANDOM unit rows stand in for the CLIP text features "
                              "(throughput / parity runs only; class scores and weak labels are meaningless)")
                n = args.test_range_max if evaluated else args.train_range_max
                g = torch.Generator().manual_seed(1234)
                feats = raw = torch.randn(n, self.clip_model.visual.output_dim, generator=g).to(self.device)
            self.text_features_fg = feats
            src = raw if self.TEXT_NORM_IN_CLIP_DTYPE else feats
            self.text_features_fg_norm = (src / src.norm(dim=1, keepdim=True)).to(torch.float32)
            if self.if_clip_superset:
                if self.superset_all_classes_keys is not None and tokens is not None:
                    self.superset_text_features_fg_norm = self.encode_prompts(self.superset_all_classes_keys)
                else:       # synthetic run (no class lists): seeded random rows, warned about above
                    nsup = getattr(args, "superset_size", 1201)
                    g = torch.Generator().manual_seed(4321)
                    sup = torch.randn(nsup, feats.shape[1], generator=g).to(self.device)
                    sup[: min(10, feats.shape[0])] = feats[: min(10, feats.shape[0])]
                    self.superset_text_features_fg_norm = sup / sup.norm(dim=1, keepdim=True)
            self.test_text_features_fg_norm = (self.superset_text_features_fg_norm if self.if_clip_superset
                                               else self.text_features_fg_norm)

    @torch.no_grad()
    def encode_prompts(self, prompts):
        """(len(prompts), D) fp32 L2-normalised CLIP text features of `prompts` (reference :356-360): the text tower's
        output cast to fp32, then normalised in fp32."""
        from ..clip.tokenizer import tokenize

        feats = self.clip_model.encode_text(tokenize(prompts).to(self.device)).to(torch.float32)
        return feats / feats.norm(dim=1, keepdim=True)

    def to_device(self, device):
        """`.to(device)` plus the plain-tensor attributes the reference keeps outside buffers
        (text features), and the device string the CLIP branch allocates on."""
        self.to(device)
        self.device = str(device)
        for name in ("text_features_fg", "text_features_fg_norm", "superset_text_features_fg_norm",
                     "test_text_features_fg_norm", "cmp_text_features_fg", "cmp_text_features_fg_norm",
                     "test_logit_scale", "logit_scale"):
            if isinstance(getattr(self, name, None), torch.Tensor) and name not in self._parameters:
                setattr(self, name, getattr(self, name).to(device))
        if str(device) == "cpu" and self.has_clip:
            self.clip_model.float()
        return self

    def build_mlp_heads(self, dataset_config, decoder_dim, mlp_dropout):
        mlp_func = partial(GenericMLP, norm_fn_name="bn1d", activation="relu", use_conv=True,
                           hidden_dims=[decoder_dim, decoder_dim], dropout=mlp_dropout, input_dim=decoder_dim)
        if self.if_with_fake_classes:
            self.num_cls_predict += 1
        # +1: background / not-an-object class
        semcls_head = mlp_func(output_dim=self.num_cls_predict + 1)
        text_correlation_head = mlp_func(output_dim=512)
        center_head = mlp_func(output_dim=3)
        size_head = mlp_func(output_dim=3)
        angle_cls_head = mlp_func(output_dim=dataset_config.num_angle_bin)
        angle_reg_head = mlp_func(output_dim=dataset_config.num_angle_bin)
        self.mlp_heads = nn.ModuleDict([
            ("sem_cls_head", semcls_head),
            ("center_head", center_head),
            ("size_head", size_head),
            ("angle_cls_head", angle_cls_head),
            ("angle_residual_head", angle_reg_head),
            ("text_correlation_head", text_correlation_head),
        ])

    # ------------------------------------------------------------------ geometry side
    def get_query_embeddings(self, encoder_xyz, point_cloud_dims):
        query_inds = furthest_point_sample(encoder_xyz, self.num_queries).long()
        query_xyz = torch.gather(encoder_xyz, 1, query_inds.unsqueeze(-1).expand(-1, -1, 3))
        pos_embed = self.pos_embedding(query_xyz, input_range=point_cloud_dims)
        query_embed = self.query_projection(pos_embed)
        return query_xyz, query_embed

    @staticmethod
    def _break_up_pc(pc):
        xyz = pc[..., 0:3].contiguous()
        features = pc[..., 3:].transpose(1, 2).contiguous() if pc.size(-1) > 3 else None
        return xyz, features

    def run_encoder(self, point_clouds):
        xyz, features = self._break_up_pc(point_clouds)
        pre_enc_xyz, pre_enc_features, pre_enc_inds = self.pre_encoder(xyz, features)
        pre_enc_features = pre_enc_features.permute(2, 0, 1)  # (npoints, batch, channel)
        enc_xyz, enc_features, enc_inds = self.encoder(pre_enc_features, xyz=pre_enc_xyz)
        if enc_inds is None:
            enc_inds = pre_enc_inds
        else:
            enc_inds = torch.gather(pre_enc_inds, 1, enc_inds)
        return enc_xyz, enc_features, enc_inds

    def get_box_predictions(self, query_xyz, point_cloud_dims, box_features, point_clouds, inputs):
        """box_features (num_layers, nqueries, batch, channel) -> per-layer prediction dicts
        (reference :1634-1740)."""
        num_layers, num_queries, batch, channel = box_features.shape
        # the reference runs the heads on (num_layers*batch, channel, nqueries) conv maps; as rows
        # (layer, batch, query) x channel the six heads share ONE packed GEMM operand and their outputs
        # land directly in (num_layers, batch, nqueries, out) order
        rows = box_features.permute(0, 2, 1, 3).reshape(num_layers * batch * num_queries, channel)
        # six heads read the same rows: their six input gradients meet in one n-ary sum (ops.fanout)
        taps = iter(ops.fanout(rows, len(self.mlp_heads)))

        def head(name):
            return self.mlp_heads[name].forward_rows(next(taps)).view(num_layers, batch, num_queries, -1)

        cls_logits = head("sem_cls_head")
        text_correlation_embedding = head("text_correlation_head") if "text_correlation_head" in self.mlp_heads else None
        center_offset = head("center_head").sigmoid() - 0.5
        size_normalized = head("size_head").sigmoid()
        angle_logits = head("angle_cls_head")
        angle_residual_normalized = head("angle_residual_head")
        angle_residual = angle_residual_normalized * (np.pi / angle_residual_normalized.shape[-1])

        # box decoding for ALL decoder layers at once: (layer, batch) is one flat batch axis of N = L * B scenes
        n = num_layers * batch
        flat = lambda t: t.reshape(n, num_queries, t.shape[-1])  # noqa: E731
        q_rep = query_xyz.repeat(num_layers, 1, 1)
        dims_rep = [d.repeat(num_layers, 1) for d in point_cloud_dims]
        center_normalized, center_unnormalized = self.box_processor.compute_predicted_center(
            flat(center_offset), q_rep, dims_rep)
        angle_continuous = self.box_processor.compute_predicted_angle(flat(angle_logits), flat(angle_residual))
        size_unnormalized = self.box_processor.compute_predicted_size(flat(size_normalized), dims_rep)
        box_corners = self.box_processor.box_parametrization_to_corners(
            center_unnormalized, size_unnormalized, angle_continuous)
        box_corners_xyz = self.box_processor.box_parametrization_to_corners_xyz(
            center_unnormalized, size_unnormalized, angle_continuous)
        with torch.no_grad():
            semcls_prob, objectness_prob = self.box_processor.compute_objectness_and_cls_prob(flat(cls_logits))
        lay = lambda t: t.reshape(num_layers, batch, *t.shape[1:])  # noqa: E731
        stacked = {
            "sem_cls_logits": cls_logits,
            "center_normalized": lay(center_normalized.contiguous()),
            "center_unnormalized": lay(center_unnormalized),
            "size_normalized": size_normalized,
            "size_unnormalized": lay(size_unnormalized),
            "angle_logits": angle_logits,
            "angle_residual": angle_residual,
            "angle_residual_normalized": angle_residual_normalized,
            "angle_continuous": lay(angle_continuous),
            "objectness_prob": lay(objectness_prob),
            "sem_cls_prob": lay(semcls_prob),
            "box_corners": lay(box_corners),
            "box_corners_xyz": lay(box_corners_xyz),
        }
        if text_correlation_embedding is not None:
            stacked["text_correlation_embedding"] = text_correlation_embedding
        outputs = []
        for l in range(num_layers):   # the reference's per-layer dicts are views into the stacked tensors
            d = {k: v[l] for k, v in stacked.items()}
            d["point_clouds"] = point_clouds
            outputs.append(d)
        # "stacked_layers" lets the criterion take every auxiliary layer in one call (criterion.SetCriterion.forward)
        return {"outputs": outputs[-1], "aux_outputs": outputs[:-1], "stacked_layers": stacked}

    # ------------------------------------------------------------------ CLIP crops
    def draw_box_selection(self, bsz: int) -> np.ndarray:
        """(bsz, distillation_box_num) int64: one `np.random.choice(arange(128), 32, replace=False)`
        per scene, the reference's draw sequence (:991)."""
        return np.stack([np.random.choice(self.box_idx_list, self.distillation_box_num, replace=False)
                         for _ in range(bsz)]).astype(np.int64)

    def _select_boxes(self, objectness_prob, curr_epoch):
        """(sel (B, S) box indices, chosen (B, S) bool).  Stage 1 (and < epoch 540): S = distillation_box_num,
        `np.random.choice(arange(128), 32, replace=False)` per scene on the host RNG, exactly the reference's draw
        sequence (:991), all chosen.  With `if_select_box_by_objectness` from epoch 540 on (reference :993-1004): every
        box with objectness > 0.05, topped up to distillation_box_num with randomly drawn background boxes when there
        are fewer -- here S = nqueries with a mask, so the crop batch keeps a static shape.  The top-up draw uses the
        device RNG (the reference draws it from numpy on host-copied indices: a host sync per scene)."""
        bsz, nq = objectness_prob.shape
        dev = objectness_prob.device
        if (not self.if_select_box_by_objectness) or curr_epoch < 540:
            if self.external_selection is not None:   # drawn ahead of the (graph-captured) step
                sel = self.external_selection
            else:
                sel = torch.from_numpy(self.draw_box_selection(bsz)).to(dev, non_blocking=True)
            return sel, torch.ones_like(sel, dtype=torch.bool)
        is_obj = objectness_prob > 0.05
        n_obj = is_obj.sum(dim=1, keepdim=True)
        # background boxes in random order; the first (distillation_box_num - n_obj) of them are drawn
        prio = torch.rand((bsz, nq), device=dev).masked_fill(is_obj, 2.0)
        rank_bg = prio.argsort(dim=1).argsort(dim=1)                   # 0 .. n_bg-1 among background boxes
        fill = (~is_obj) & (rank_bg < (self.distillation_box_num - n_obj))
        sel = torch.arange(nq, device=dev).unsqueeze(0).expand(bsz, -1)
        return sel, is_obj | fill

    @torch.no_grad()
    def _boxes_in_image(self, inputs, outputs):
        """Every predicted box projected into the image: int32 (B, Q, 4) [xmin, ymin, xmax, ymax] (the reference's
        `int(torch.min/max(.))` truncation of non-negative fp64 values) and the boxes that are usable as crops
        (non-degenerate, in front of the camera, non-zero size; reference :912-968, :1034-1051) -- one kernel, with
        the dataset's camera model (reference :461-466)."""
        # SUN RGB-D is the op's default camera: that call keeps its original form
        camera = {"camera": "scannet"} if self.dataset_name == "scannet" else {}
        return ops.boxes_in_image(outputs["box_corners_xyz"].detach(), outputs["size_unnormalized"].detach(), inputs,
                                  **camera)

    @torch.no_grad()
    def _clip_embed_boxes(self, inputs, boxes, valid, sel, chosen=None):
        """CLIP image embeddings of the crops under boxes[b, sel[b, s]] -> (B, S, D) fp32 (garbage where invalid)."""
        bsz, nsel = sel.shape
        bx = torch.gather(boxes, 1, sel.unsqueeze(-1).expand(-1, -1, 4)).reshape(-1, 4).contiguous()
        vd = torch.gather(valid, 1, sel)
        if chosen is not None:
            vd = vd & chosen
        vd = vd.reshape(-1)
        scene = torch.arange(bsz, device=boxes.device, dtype=torch.int32).repeat_interleave(nsel)
        feats = self._encode_crops(inputs["input_image"], scene, bx, vd)
        return feats.reshape(bsz, nsel, -1), vd.reshape(bsz, nsel)

    @torch.no_grad()
    def _encode_crops(self, images, scene, boxes, valid):
        """CLIP image features (N, D) fp32 of the crops boxes (N, 4) of images[scene] (garbage where not valid)."""
        extra = {}
        visual = getattr(self.clip_model, "visual", None)
        if (images.is_cuda and self.clip_model.dtype == torch.float16
                and isinstance(visual, clip_mod.model.VisionTransformer)):
            ps = visual.conv1.kernel_size[0]
            if self.clip_resolution % ps == 0 and (3 * ps * ps) % 64 == 0:
                extra["patch"] = ps        # crops come out as the unfolded patches the ViT's first GEMM reads
        crops = ops.crop_resize_normalize(images, scene, boxes, valid, self.clip_resolution,
                                          dtype=self.clip_model.dtype, **extra)
        feats = self.clip_model.encode_image(crops)
        if isinstance(feats, tuple):
            feats = feats[0]
        return feats.to(torch.float32)

    @torch.no_grad()
    def get_predicted_box_clip_embedding(self, inputs, outputs, thres_obj=0.05, if_use_gt_box=False,
                                         if_expand_box=False, if_padding_input=True, test=False, curr_epoch=-1,
                                         random_selection_only=False):
        """CLIP image embeddings of the crops under `distillation_box_num` predicted boxes per
        scene -> outputs['gt_text_correlation_embedding'(_mask)] (+ weak labels).
        Same semantics as reference :902-1210, without host synchronisation."""
        bsz, nq = outputs["box_corners_xyz"].shape[:2]
        dev = outputs["box_corners_xyz"].device
        boxes, valid_all = self._boxes_in_image(inputs, outputs)
        sel, chosen = self._select_boxes(outputs["objectness_prob"].detach(),
                                         -1 if random_selection_only else curr_epoch)      # (B, S)
        feats, valid = self._clip_embed_boxes(inputs, boxes, valid_all, sel, chosen)
        vmask = valid.to(torch.float32).unsqueeze(-1)
        emb = torch.zeros((bsz, nq, feats.shape[-1]), device=dev)
        mask = torch.zeros((bsz, nq, 1), device=dev)
        emb.scatter_(1, sel.unsqueeze(-1).expand(-1, -1, feats.shape[-1]), feats * vmask)
        mask.scatter_(1, sel.unsqueeze(-1), vmask)
        outputs["gt_text_correlation_embedding"] = emb
        outputs["gt_text_correlation_embedding_mask"] = mask

        if self.if_keep_box and curr_epoch >= 540 and not random_selection_only:
            self._keep_novel_boxes_as_gt(inputs, outputs, sel, valid, feats)

        if self.if_clip_weak_labels:
            text = outputs["text_features_clip"].to(torch.float32)
            e = emb / (emb.norm(dim=-1, keepdim=True) + 1e-32)
            corr = torch.bmm(e, text.permute(0, 2, 1)) * outputs["logit_scale"]
            scores = ops.softmax_rows(corr)
            max_score, max_id = torch.max(scores, dim=-1)
            outputs["weak_box_cate_label"] = max_id
            outputs["weak_confidence_weight"] = torch.where(mask[:, :, 0] < 1, torch.zeros_like(max_score), max_score)
        else:
            outputs["weak_box_cate_label"] = torch.zeros((bsz, nq), device=dev, dtype=torch.int64)
            outputs["weak_confidence_weight"] = torch.zeros((bsz, nq), device=dev)
        return outputs

    @torch.no_grad()
    def _keep_novel_boxes_as_gt(self, inputs, outputs, sel, valid, feats):
        """`if_keep_box` from epoch 540 on (reference :1106-1150): a selected, croppable box with objectness >
        keep_objectness whose CLIP class over the training prompts is novel (probability > 0.5, class id > 9) is
        APPENDED to the scene's ground truth (slots gt_box_present.sum() .. 63, in selection order) with the model's
        own prediction as the label.  Mutates `inputs` in place like the reference; tensor ops only, no host sync."""
        obj = torch.gather(outputs["objectness_prob"].detach(), 1, sel)
        text = outputs["text_features_clip"].to(torch.float32)
        e = feats / (feats.norm(dim=-1, keepdim=True) + 1e-32)
        scores = ops.softmax_rows(torch.bmm(e, text.permute(0, 2, 1)) * outputs["logit_scale"])
        max_score, max_id = torch.max(scores, dim=-1)
        novel = valid & (obj > self.keep_objectness) & (max_score > 0.5) & (max_id > 9)        # (B, S), selection order
        begin = inputs["gt_box_present"].sum(dim=1).long().view(-1, 1)
        dest = begin + torch.cumsum(novel.long(), dim=1) - 1
        ngt = inputs["gt_box_present"].shape[1]
        ok = novel & (dest < ngt)                      # `begin_idx > 63 -> break`
        dest = torch.where(ok, dest, torch.full_like(dest, ngt))      # rejected entries go to a scratch slot

        def put(key, values):
            """inputs[key][b, dest[b, s]] = values[b, s] for the accepted (b, s)"""
            tgt = inputs[key]
            vals = values.to(tgt.dtype)
            pad = torch.cat((tgt, tgt.new_zeros((tgt.shape[0], 1) + tuple(tgt.shape[2:]))), dim=1)
            idx = dest.view(dest.shape + (1,) * (tgt.dim() - 2)).expand(-1, -1, *tgt.shape[2:])
            pad.scatter_(1, idx, vals)
            tgt.copy_(pad[:, :ngt])

        take = lambda t: torch.gather(t.detach(), 1, sel.view(sel.shape + (1,) * (t.dim() - 2)).expand(-1, -1, *t.shape[2:]))  # noqa: E731
        angle_cls = take(outputs["angle_logits"]).softmax(dim=-1).argmax(dim=-1)
        put("gt_box_present", torch.ones_like(dest))
        put("gt_angle_class_label", angle_cls)
        put("gt_angle_residual_label", torch.gather(take(outputs["angle_residual"]), 2, angle_cls.unsqueeze(-1)).squeeze(-1))
        put("gt_box_sizes_normalized", take(outputs["size_normalized"]))
        put("gt_box_sizes", take(outputs["size_unnormalized"]))
        put("gt_box_corners", take(outputs["box_corners"]))
        if "gt_box_corners_xyz" in inputs:
            put("gt_box_corners_xyz", take(outputs["box_corners_xyz"]))
        put("gt_box_angles", take(outputs["angle_continuous"]))
        put("gt_box_centers_normalized", take(outputs["center_normalized"]))
        put("gt_box_centers", take(outputs["center_unnormalized"]))

    # ------------------------------------------------------------------ stage 2: novel-box discovery
    DISCOVERY_CAPACITY = 32     # candidates per scene that get a CLIP crop (fixed: keeps the step graph-capturable)

    @torch.no_grad()
    def get_predicted_box_clip_embedding_nms_iou_save_keep_clip_driven_with_cate_confidence(
            self, inputs, outputs, thres_obj=0.05, if_use_gt_box=False, if_expand_box=False, if_padding_input=True,
            test=False, curr_epoch=-1, if_test=False):
        """Stage-2 variant of the crop pipeline (reference :1212-1632).  On the epochs that are multiples of
        `online_nms_update_save_epoch` it additionally DISCOVERS novel boxes: class-agnostic 2-D NMS of the projected
        boxes (IoU 0.25), rejection of boxes whose axis-aligned 3-D IoU with a ground-truth box exceeds 0.25,
        objectness >= save_objectness, then CLIP on the crops of the survivors; a survivor whose best class (over the
        `test_range_max` / superset prompts) is a NOVEL one with probability > clip_driven_keep_thres becomes a pseudo
        label row (center(3), size(3), angle, class, class prob, objectness) in the un-augmented frame.

        Everything up to the rows runs on the device without host synchronisation (ops.novel_candidates + one
        batched CLIP call over a fixed capacity of candidates); the rows are parked in `self._pending_pseudo` and
        written to the per-scene .npy files by `flush_pseudo_labels()` -- the only host work, as in the reference
        (np.save, :1524-1540)."""
        discover = (not if_test) and (curr_epoch % self.online_nms_update_save_epoch == 0)
        if discover:
            self._discover_novel_boxes(inputs, outputs)
        # distillation targets: always the random 32-of-128 draw in this variant (reference :1545)
        return self.get_predicted_box_clip_embedding(inputs, outputs, curr_epoch=curr_epoch,
                                                     random_selection_only=True)

    @torch.no_grad()
    def _discover_novel_boxes(self, inputs, outputs):
        self.flush_pseudo_labels()       # rows of the previous discovery step, if nobody fetched them yet
        boxes, valid = self._boxes_in_image(inputs, outputs)
        obj = outputs["objectness_prob"].detach()
        cap = self.DISCOVERY_CAPACITY
        # reference box2d order is (ymin, xmin, ymax, xmax): IoU does not depend on the axis naming
        cand, count = ops.novel_candidates(boxes, valid, obj, outputs["box_corners"].detach(),
                                           inputs["gt_box_corners"], inputs["gt_box_present"], 0.25, 0.25,
                                           float(self.save_objectness), cap)
        cvalid = cand >= 0
        sel = cand.clamp(min=0).long()
        feats, _ = self._clip_embed_boxes(inputs, boxes, valid, sel)
        text = outputs["maybe_novel_text_features_clip"].to(torch.float32)
        e = feats / (feats.norm(dim=-1, keepdim=True) + 1e-32)
        corr = torch.matmul(e, text.t()) * outputs["logit_scale"]
        scores = ops.softmax_rows(corr)
        max_score, max_idx = torch.max(scores, dim=-1)
        cond = cvalid & (max_score > self.clip_driven_keep_thres) & (max_idx >= self.train_range_max)
        # box parameters back in the un-augmented frame (reference :1236-1252), fp64 like the reference's promotion
        scale = inputs["scale_array"].to(torch.double)                       # (B, 1, 3)
        center = outputs["center_unnormalized"].detach().to(torch.double) * scale
        size = outputs["size_unnormalized"].detach().to(torch.double) * scale
        center = torch.matmul(center, inputs["rot_array"].to(torch.double))
        angle = outputs["angle_continuous"].detach().to(torch.double) + inputs["rot_angle"].to(torch.double).view(-1, 1)
        if "zx_flip_array" in inputs:
            zx = inputs["zx_flip_array"].to(torch.double).view(-1, 1)
            center = torch.cat((center[..., :1], center[..., 1:2] * zx.unsqueeze(-1), center[..., 2:]), dim=-1)
            angle = torch.where(zx < 0, math.pi - angle, angle)
        flip = inputs["flip_array"].to(torch.double).view(-1, 1)
        center = torch.cat((center[..., :1] * flip.unsqueeze(-1), center[..., 1:]), dim=-1)
        angle = torch.where(flip < 0, math.pi - angle, angle)
        info = torch.cat((center, size, angle.unsqueeze(-1)), dim=-1).to(torch.float32)      # (B, Q, 7)
        rows = torch.cat((torch.gather(info, 1, sel.unsqueeze(-1).expand(-1, -1, 7)),
                          max_idx.to(torch.float32).unsqueeze(-1), max_score.unsqueeze(-1),
                          torch.gather(obj, 1, sel).unsqueeze(-1)), dim=-1)               # (B, cap, 10)
        room = (inputs["gt_ori_box_num"].view(-1, 1) <= 63) if "gt_ori_box_num" in inputs else torch.ones_like(cond)
        self._pending_pseudo = {"rows": rows, "mask": cond & room, "count": count,
                                "paths": inputs.get("pseudo_box_path")}
        outputs["novel_box_rows"], outputs["novel_box_mask"] = rows, cond & room

    def flush_pseudo_labels(self):
        """Writes the pseudo-label rows of the last discovery step to the scenes' .npy files (reference :1524-1540;
        the one device->host copy of the stage-2 path).  Returns the per-scene arrays."""
        pending, self._pending_pseudo = getattr(self, "_pending_pseudo", None), None
        if pending is None:
            return None
        rows = pending["rows"].cpu().numpy()
        mask = pending["mask"].cpu().numpy().astype(bool)
        count = pending["count"].cpu().numpy()
        if (count[:, 1] > count[:, 0]).any():
            warnings.warn(f"novel-box discovery: {int((count[:, 1] - count[:, 0]).max())} candidates beyond the "
                          f"capacity of {self.DISCOVERY_CAPACITY} per scene were dropped")
        out = []
        for b in range(rows.shape[0]):
            new = rows[b][mask[b]]
            out.append(new)
            paths = pending["paths"]
            if paths is None or len(new) == 0:
                continue
            if self.if_accumulate_former_pseudo_labels and os.path.exists(paths[b]):
                former = np.load(paths[b])
                new = new if former.shape[0] == 0 else np.concatenate((former, new), axis=0)
            np.save(paths[b], new)
        return out

    def get_class_scores(self, box_predictions):
        """Multi-class scores from the text embeddings (reference :1743-1763)."""
        if self.eval_layer_id != -1:
            for key in box_predictions["aux_outputs"][self.eval_layer_id].keys():
                box_predictions["outputs"][key] = box_predictions["aux_outputs"][self.eval_layer_id][key]
        outputs = box_predictions["outputs"]
        text = outputs["text_features_clip"].to(torch.float32)
        e = outputs["text_correlation_embedding"]
        e = e / (e.norm(dim=-1, keepdim=True) + 1e-32)
        corr = torch.bmm(e, text.permute(0, 2, 1)) * outputs["logit_scale"]
        outputs["sem_cls_prob"] = torch.nn.functional.softmax(corr, dim=-1)
        return box_predictions, outputs["sem_cls_prob"], outputs["objectness_prob"]

    # ------------------------------------------------------------------ forward
    def forward(self, inputs, encoder_only=False, if_test=False, if_real_test=False, curr_epoch=-1,
                if_cmp_class=False):
        point_clouds = inputs["point_clouds"]
        enc_xyz, enc_features, enc_inds = self.run_encoder(point_clouds)
        proj = self.encoder_to_decoder_projection
        if isinstance(proj.layers[0], nn.Conv1d) and enc_features.is_contiguous():
            # 1x1 convolutions + BatchNorm over (batch, position) do not care about the order of the rows: run the
            # stack on the (position, batch) rows as they lie in memory -- the reference's (B, C, N) round trip
            # (:1774) would cost a transposed copy in and a strided, re-copied memory tensor out
            npos, bsz, _ = enc_features.shape
            enc_features = proj.forward_rows(enc_features.reshape(npos * bsz, -1)).view(npos, bsz, -1)
        else:
            enc_features = proj(enc_features.permute(1, 2, 0)).permute(2, 0, 1)
        if encoder_only:
            return enc_xyz, enc_features.transpose(0, 1)
        point_cloud_dims = [inputs["point_cloud_dims_min"], inputs["point_cloud_dims_max"]]
        query_xyz, query_embed = self.get_query_embeddings(enc_xyz, point_cloud_dims)
        enc_pos = self.pos_embedding(enc_xyz, input_range=point_cloud_dims).permute(2, 0, 1)
        query_embed = query_embed.permute(2, 0, 1)
        tgt = torch.zeros_like(query_embed, memory_format=torch.contiguous_format)
        box_features = self.decoder(tgt, enc_features, query_pos=query_embed, pos=enc_pos)[0]
        box_predictions = self.get_box_predictions(query_xyz, point_cloud_dims, box_features, point_clouds, inputs)
        return self._clip_outputs(inputs, box_predictions, if_test, if_real_test, if_cmp_class, curr_epoch)

    def _clip_outputs(self, inputs, box_predictions, if_test, if_real_test, if_cmp_class, curr_epoch):
        """The CLIP side of forward (reference :1776-1831): distillation targets in training, class scores at test."""
        point_clouds = inputs["point_clouds"]
        out = box_predictions["outputs"]
        if self.if_with_clip_train:
            out["logit_scale"] = torch.clip(self.logit_scale.exp(), min=None, max=100)

        if self.if_with_clip_train and (not if_real_test) and (not if_cmp_class) and (not if_test):
            bsz = point_clouds.shape[0]
            if self.if_clip_superset:
                # every scene reads the same (C, D) superset matrix: a view, not B copies of it
                out["text_features_clip"] = self.superset_text_features_fg_norm.unsqueeze(0).expand(bsz, -1, -1)
            else:
                out["text_features_clip"] = self.text_features_fg_norm[: self.train_range_max, :].unsqueeze(0).repeat(
                    bsz, 1, 1)
            if self.online_nms_update_save_novel_label_clip_driven_with_cate_confidence:
                out["maybe_novel_text_features_clip"] = (self.superset_text_features_fg_norm if self.if_clip_superset
                                                         else self.text_features_fg_norm[: self.test_range_max, :])
                box_predictions["outputs"] = \
                    self.get_predicted_box_clip_embedding_nms_iou_save_keep_clip_driven_with_cate_confidence(
                        inputs, out, curr_epoch=curr_epoch, if_test=if_test)
            else:
                box_predictions["outputs"] = self.get_predicted_box_clip_embedding(inputs, out, curr_epoch=curr_epoch)
        if if_real_test:
            out["text_features_clip"] = self.text_features_fg_norm.unsqueeze(0).repeat(point_clouds.shape[0], 1, 1)
            box_predictions, _, _ = self.get_class_scores(box_predictions)
        return box_predictions


def read_scannet_matrix(path) -> np.ndarray:
    """The 4 x 4 matrix of a ScanNet calibration text file (intrinsic/intrinsic_color.txt, pose/<frame>.txt): 16
    numbers, row by row, as the reference's load_txt reads them (datasets/scannet_utils.py:69-79)."""
    path = str(path)
    if not os.path.isfile(path):
        raise FileNotFoundError(f"ScanNet calibration file not found: {path}")
    with open(path) as f:
        vals = [float(x) for x in f.read().split()]
    if len(vals) != 16:
        raise ValueError(f"{path}: expected the 16 numbers of a 4 x 4 matrix, found {len(vals)}")
    return np.array(vals, dtype=np.float64).reshape(4, 4)


class ScanNetCalibration:
    """The colour intrinsics and camera-to-world poses of ScanNet scenes, read from `<calib_name>/intrinsic/
    intrinsic_color.txt` and `<calib_name>/pose/<squence_name>.txt` as the reference's SCANNET_Calibration does
    (datasets/scannet_utils.py:110-130); each file is read once."""

    def __init__(self):
        self._cache = {}

    def matrix(self, path) -> np.ndarray:
        path = str(path)
        if path not in self._cache:
            self._cache[path] = read_scannet_matrix(path)
        return self._cache[path]

    def __call__(self, calib_names, squence_names):
        """-> (K (B, 4, 4), pose (B, 4, 4)) fp64 host arrays for the scenes of a batch."""
        K = [self.matrix(os.path.join(str(c), "intrinsic", "intrinsic_color.txt")) for c in calib_names]
        pose = [self.matrix(os.path.join(str(c), "pose", f"{s}.txt")) for c, s in zip(calib_names, squence_names)]
        return np.stack(K), np.stack(pose)


class Model3DETRMultiClassHead(Model3DETRPredictedBoxDistillationHead):
    """The 3DETR + CLIP baseline of the paper (reference Model3DETRMultiClassHead, :1838-3932): the 3DETR heads
    with a class-agnostic objectness head and no text-correlation head, and a frozen CLIP that classifies every
    predicted box by its image crop at test time (`forward(if_real_test=True)`, reference clip_to_class_training
    :2810-3085).  Training never crops."""

    # crops per CLIP tower call at test time: bounds the tower's activations (the ViT-B/16 MLP hidden activation alone
    # is 1.2 MB per crop in fp16) whatever the batch size
    CROPS_PER_CALL = 1024
    TEXT_NORM_IN_CLIP_DTYPE = True          # reference :2088-2090: fp16 features normalised in fp16, then fp32

    def __init__(self, pre_encoder, encoder, decoder, dataset_config, encoder_dim=256, decoder_dim=256,
                 position_embedding="fourier", mlp_dropout=0.3, num_queries=256, if_use_gt_box=False,
                 if_expand_box=False, args=None):
        for flag, on in (("if_use_gt_box", if_use_gt_box), ("if_expand_box", if_expand_box),
                         ("if_only_novel_prompt", getattr(args, "if_only_novel_prompt", False)),
                         ("online_nms_update_save_novel_label_clip_driven_with_cate_confidence",
                          getattr(args, "online_nms_update_save_novel_label_clip_driven_with_cate_confidence", False))):
            if on:
                raise NotImplementedError(f"the baseline head does not implement --{flag}")
        self._masked_encoder = hasattr(encoder, "masking_radius")
        super().__init__(pre_encoder, encoder, decoder, dataset_config, encoder_dim=encoder_dim,
                         decoder_dim=decoder_dim, position_embedding=position_embedding, mlp_dropout=mlp_dropout,
                         num_queries=num_queries, if_with_clip_train=False, num_cls_predict=1, args=args,
                         has_clip=True)
        # reference :2082: a plain tensor (not a parameter, so no state-dict entry), used unclipped at test time
        del self.logit_scale
        self.logit_scale = self.test_logit_scale
        # the reference's baseline holds CLIP once, as clip_model: no aliases, so that its checkpoints load strictly
        del self.test_clip_model, self.res_encoder
        self.scannet_calibration = ScanNetCalibration()

    def _projection_dims(self, encoder_dim):
        # reference :1886-1900
        return encoder_dim, ([encoder_dim] if self._masked_encoder else [encoder_dim, encoder_dim])

    def _evaluated_prompts(self, args):
        return True                          # reference :1923-1988: always the test_range_max / evaluated classes

    # seed of the random comparison-class rows of synthetic runs
    CMP_SYNTHETIC_SEED = 2468

    def _build_clip(self, args, dataset_config):
        super()._build_clip(args, dataset_config)
        self.build_cmp_text(args)

    @torch.no_grad()
    def build_cmp_text(self, args):
        """The text matrix of forward(if_cmp_class=True), encoded once (reference :2092-2095) and normalised as
        text_features_fg_norm is (in CLIP's dtype, then fp32): `cmp_text_features_fg` and `cmp_text_features_fg_norm`
        (C, D), plain tensors, so that checkpoints gain no state-dict key.  Where the class text is synthetic (warned
        about by _build_clip), C seeded random rows stand in: 20 for SUN RGB-D, 19 for ScanNet.  A missing comparison
        list does not stop the build, which serves every other evaluation: the first if_cmp_class forward raises."""
        self.all_cmp_classes_keys = self.cmp_text_features_fg = self.cmp_text_features_fg_norm = None
        self._cmp_text_error = None
        if self.text_features_synthetic:
            n = 19 if getattr(args, "dataset_name", "").find("scannet") != -1 else 20
            g = torch.Generator().manual_seed(self.CMP_SYNTHETIC_SEED)
            raw = torch.randn(n, self.clip_model.visual.output_dim, generator=g).to(self.device)
        else:
            try:
                self.all_cmp_classes_keys = cmp_prompts(args)
            except FileNotFoundError as e:
                self._cmp_text_error = str(e)
                return
            from ..clip.tokenizer import tokenize

            raw = self.clip_model.encode_text(tokenize(self.all_cmp_classes_keys).to(self.device))
        self.cmp_text_features_fg = raw.to(torch.float32)
        self.cmp_text_features_fg_norm = (raw / raw.norm(dim=1, keepdim=True)).to(torch.float32)

    def build_mlp_heads(self, dataset_config, decoder_dim, mlp_dropout):
        # reference :2145-2176: objectness (1 + 1 logits) and the box geometry
        mlp_func = partial(GenericMLP, norm_fn_name="bn1d", activation="relu", use_conv=True,
                           hidden_dims=[decoder_dim, decoder_dim], dropout=mlp_dropout, input_dim=decoder_dim)
        self.mlp_heads = nn.ModuleDict([
            ("sem_cls_head", mlp_func(output_dim=1 + 1)),
            ("center_head", mlp_func(output_dim=3)),
            ("size_head", mlp_func(output_dim=3)),
            ("angle_cls_head", mlp_func(output_dim=dataset_config.num_angle_bin)),
            ("angle_residual_head", mlp_func(output_dim=dataset_config.num_angle_bin)),
        ])

    def _clip_outputs(self, inputs, box_predictions, if_test, if_real_test, if_cmp_class, curr_epoch):
        # reference :3903-3930
        out = box_predictions["outputs"]
        out["logit_scale"] = torch.clip(self.logit_scale.exp(), min=None, max=100)
        if not (if_real_test or if_cmp_class or if_test):
            text = (self.superset_text_features_fg_norm if self.if_clip_superset
                    else self.text_features_fg_norm[: self.train_range_max, :])
            out["text_features_clip"] = text.unsqueeze(0).repeat(inputs["point_clouds"].shape[0], 1, 1)
        if if_real_test:
            self.classify_boxes(inputs, out)
        if if_cmp_class:
            if self.cmp_text_features_fg_norm is None:
                raise FileNotFoundError(self._cmp_text_error)
            self.classify_boxes(inputs, out, text=self.cmp_text_features_fg_norm)
        return box_predictions

    def _camera_inputs(self, inputs, bsz: int, dev):
        """The batch's camera with identity augmentation: the reference's test path projects the predicted boxes
        with the scene's calibration alone (:2905-2938).  ScanNet test batches carry no K / Rtilt: their
        calibration files are read (reference SCANNET_Calibration)."""
        if "K" in inputs and "Rtilt" in inputs:
            K, Rtilt = inputs["K"], inputs["Rtilt"]
        elif self.dataset_name == "scannet":
            K, Rtilt = (torch.from_numpy(a).to(dev) for a in
                        self.scannet_calibration(inputs["calib_name"], inputs["squence_name"]))
        else:
            raise KeyError("the baseline head's test-time classification needs the batch's K and Rtilt")
        f64 = dict(device=dev, dtype=torch.double)
        # the test path clamps the projected extent to [0, width] x [0, height] (:2935-2938) where the training path,
        # which the kernel follows, clamps to [0, width - 1] x [0, height - 1]
        cam = {k: inputs[k] + 1 for k in ("ori_width", "ori_height")}
        cam.update({k: inputs[k] for k in ("x_offset", "y_offset")})
        cam.update(K=K, Rtilt=Rtilt, scale_array=torch.ones((bsz, 1, 3), **f64),
                   rot_array=torch.eye(3, **f64).expand(bsz, 3, 3), flip_array=torch.ones((bsz, 1), **f64),
                   image_flip_array=torch.ones((bsz, 1), **f64), flip_length=torch.zeros((bsz,), **f64))
        return cam

    @torch.no_grad()
    def project_boxes(self, inputs, out, extent=False):
        """ops.boxes_in_image of every predicted box as the reference's test path projects it: the scene's
        calibration, no augmentation, the dataset's camera."""
        bsz = out["box_corners_xyz"].shape[0]
        corners, camera = out["box_corners_xyz"], {}
        if self.dataset_name == "scannet":
            camera = {"camera": "scannet"}
            # the ScanNet test path turns the box by +angle (datasets/scannet_utils.py:402, rotz(box_angle)); the
            # corner builder, like SUN RGB-D's projection (sunrgbd_utils.py:364), turns it by -angle
            corners = self.box_processor.box_parametrization_to_corners_xyz(
                out["center_unnormalized"], out["size_unnormalized"], -out["angle_continuous"])
        return ops.boxes_in_image(corners, out["size_unnormalized"],
                                  self._camera_inputs(inputs, bsz, corners.device), extent=extent, **camera)

    @torch.no_grad()
    def classify_boxes(self, inputs, out, text=None):
        """out['sem_cls_prob'] (B, Q, C) = softmax(logit_scale * f_hat . text^T) of the CLIP feature f of each box's
        crop, zeros for a box without a usable crop; out['sem_cls_logits'] zeros (reference :2810-3085).  `text` is
        the (C, D) normalised text matrix: by default the evaluated classes' (C = test_range_max).
        The usable boxes are compacted on the device (one read of their count per batch) and only their crops go
        through the tower, CROPS_PER_CALL at a time."""
        bsz, nq = out["box_corners_xyz"].shape[:2]
        dev = out["box_corners_xyz"].device
        boxes, valid = self.project_boxes(inputs, out)
        idx = valid.reshape(-1).nonzero().squeeze(1)
        n = idx.numel()
        row_map = torch.full((bsz * nq,), -1, dtype=torch.int32, device=dev)
        row_map[idx] = torch.arange(n, dtype=torch.int32, device=dev)
        if text is None:
            text = self.text_features_fg_norm
        feats = torch.empty((n, text.shape[1]), dtype=torch.float32, device=dev)
        flat_boxes = boxes.reshape(-1, 4)
        for s in range(0, n, self.CROPS_PER_CALL):
            sel = idx[s: s + self.CROPS_PER_CALL]
            scene = torch.div(sel, nq, rounding_mode="floor").to(torch.int32)
            feats[s: s + sel.numel()] = self._encode_crops(inputs["input_image"], scene, flat_boxes[sel],
                                                          torch.ones_like(sel, dtype=torch.bool))
        out["sem_cls_prob"], out["sem_cls_logits"] = ops.clip_classify(feats, text, self.logit_scale, row_map,
                                                                       (bsz, nq))
        out["clip_usable_mask"] = valid
        out["clip_boxes_2d"] = boxes
        out["clip_crop_features"] = feats
        return out


def build_preencoder(args):
    mlp_dims = [3 * int(args.use_color), 64, 128, args.enc_dim]
    return PointnetSAModuleVotes(radius=0.2, nsample=64, npoint=args.preenc_npoints, mlp=mlp_dims,
                                 normalize_xyz=True)


def build_encoder(args):
    # reference models/model_3detr.py:3946-3984
    layer = TransformerEncoderLayer(d_model=args.enc_dim, nhead=args.enc_nhead, dim_feedforward=args.enc_ffn_dim,
                                    dropout=args.enc_dropout, activation=args.enc_activation)
    if args.enc_type == "vanilla":
        return TransformerEncoder(encoder_layer=layer, num_layers=args.enc_nlayers)
    if args.enc_type == "masked":
        interim_downsampling = PointnetSAModuleVotes(radius=0.4, nsample=32, npoint=args.preenc_npoints // 2,
                                                     mlp=[args.enc_dim, 256, 256, args.enc_dim], normalize_xyz=True)
        masking_radius = [math.pow(x, 2) for x in [0.4, 0.8, 1.2]]
        return MaskedTransformerEncoder(encoder_layer=layer, num_layers=3, interim_downsampling=interim_downsampling,
                                        masking_radius=masking_radius)
    raise ValueError(f"Unknown encoder type {args.enc_type}")


def build_decoder(args):
    layer = TransformerDecoderLayer(d_model=args.dec_dim, nhead=args.dec_nhead, dim_feedforward=args.dec_ffn_dim,
                                    dropout=args.dec_dropout)
    return TransformerDecoder(layer, num_layers=args.dec_nlayers, return_intermediate=True)


def build_3detr_predictedbox_distillation_head(args, dataset_config):
    g = lambda name, default=False: getattr(args, name, default)  # noqa: E731
    model = Model3DETRPredictedBoxDistillationHead(
        build_preencoder(args), build_encoder(args), build_decoder(args), dataset_config,
        encoder_dim=args.enc_dim, decoder_dim=args.dec_dim, mlp_dropout=args.mlp_dropout,
        num_queries=args.nqueries, if_with_clip=g("if_with_clip"), if_with_clip_embed=g("if_with_clip_embed"),
        if_use_gt_box=g("if_use_gt_box"), if_expand_box=g("if_expand_box"),
        if_with_fake_classes=g("if_with_fake_classes"), pooling_methods=g("pooling_methods", "average"),
        if_clip_more_prompts=g("if_clip_more_prompts"), if_keep_box=g("if_keep_box"),
        if_select_box_by_objectness=g("if_select_box_by_objectness"), keep_objectness=g("keep_objectness", 0.5),
        online_nms_update_novel_label=g("online_nms_update_novel_label"),
        online_nms_update_accumulate_novel_label=g("online_nms_update_accumulate_novel_label"),
        online_nms_update_accumulate_epoch=g("online_nms_update_accumulate_epoch", 10),
        distillation_box_num=g("distillation_box_num", 32), args=args)
    return model, BoxProcessor(dataset_config)


def build_3detr_multiclasshead(args, dataset_config):
    """The 3DETR + CLIP baseline head (reference Model3DETRMultiClassHead, :1838-3932, built as :4052-4072)."""
    g = lambda name, default=False: getattr(args, name, default)  # noqa: E731
    model = Model3DETRMultiClassHead(
        build_preencoder(args), build_encoder(args), build_decoder(args), dataset_config,
        encoder_dim=args.enc_dim, decoder_dim=args.dec_dim, mlp_dropout=args.mlp_dropout,
        num_queries=args.nqueries, if_use_gt_box=g("if_use_gt_box"), if_expand_box=g("if_expand_box"), args=args)
    return model, BoxProcessor(dataset_config)
