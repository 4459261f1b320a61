"""The PointNet++ shared MLP + max over neighbours as ONE autograd node (training mode, CUDA).

Mirror of `SharedMLP` (third_party_pointnet2/pointnet2/pytorch_utils.py:8-33: Conv2d 1x1 -> BatchNorm2d ->
ReLU blocks) followed by the `F.max_pool2d(kernel_size=[1, nsample])` of `PointnetSAModuleVotes.forward`
(pointnet2_modules.py:247-254), on channels-last rows (B * npoint * nsample, C):

    layer 0      rows_linear_small_k (C_in = 3: exact fp32 FMAs)            -> y0
    layer l > 0  wgmma split-bf16 GEMM on the planes written by layer l-1 -> y_l
    between      BatchNorm statistics (one read of y_l), then normalise + ReLU + split into bf16 operand
                 planes in one pass (the fp32 activation is never written); the last layer instead folds
                 the max over the `nsample` rows of each seed in and returns (B * npoint, C) + arg-max
    backward     per layer: masked BatchNorm-backward sums (one read of y_l and the incoming gradient), then
                 dy written directly as the operand planes of the two gradient GEMMs (dW = dy^T a_{l-1} on
                 MN-major operands, dz_{l-1} = dy W_l); layer 0 accumulates its (C_out x 3) dW in that pass.

Kernels: csrc/sa_mlp_kernels.cu (include/coda_sa_mlp.h).  There is no CPU / eager fallback in here: callers
(`SharedMLP.forward_max_pooled`) check `applicable()` first and use the module-by-module path otherwise.

Inference (eval-mode BatchNorm, nothing for autograd to record): `shared_mlp_max_infer` runs the pre-encoder's
whole 3 -> 64 -> 128 -> 256 MLP + max as one kernel (csrc/sa_infer_sm90.cu) that writes only the pooled rows;
`SharedMLP.forward_max_pooled_infer` checks `infer_applicable()` first.
"""
from __future__ import annotations

import ctypes

import torch
import torch.nn as nn

from . import ops
from ._lib import check, lib, ptr, stream_of

_i, _ll, _f = ctypes.c_int, ctypes.c_longlong, ctypes.c_float
BACKWARD_PLANES = 2


def _channels_ok(c: int) -> bool:
    return 4 <= c <= 1024 and c % 4 == 0 and 256 % (c // 4) == 0


def applicable(x: torch.Tensor, blocks, group: int) -> bool:
    """blocks: list of (conv, bn) module pairs in execution order (each followed by ReLU)."""
    if not (x.is_cuda and x.dtype == torch.float32 and 1 <= group <= 256) or len(blocks) == 0:
        return False
    cin = x.shape[-1]
    if cin > 8 and cin % 64 != 0:
        return False
    if cin <= 8 and x.requires_grad and torch.is_grad_enabled():
        return False                      # the tiny-K first layer does not produce an input gradient
    for li, (conv, bn) in enumerate(blocks):
        cout = conv.weight.shape[0]
        if conv.bias is not None or not bn.training or not bn.affine or not _channels_ok(cout):
            return False
        if li < len(blocks) - 1 and cout % 64 != 0:
            return False
        if cout > 256 and (li > 0 or cin > 8):
            # a GEMM layer's column statistics (16 x cout floats) share the fp32-A GEMM's shared memory with its
            # stages: every instance fits them up to 256 columns (launch_a32 in gemm_a32_sm90.cu)
            return False
    return True


def _scratch(c: int, device) -> torch.Tensor:
    lib().coda_bn_rows_scratch_floats.restype = ctypes.c_longlong
    return torch.empty(int(lib().coda_bn_rows_scratch_floats(_i(c))), dtype=torch.float32, device=device)


def _stats(y: torch.Tensor, bn: nn.modules.batchnorm._BatchNorm):
    rows, c = y.shape
    momentum = 0.0 if bn.momentum is None else float(bn.momentum)
    track = bn.track_running_stats and bn.running_mean is not None
    if track and bn.num_batches_tracked is not None:
        bn.num_batches_tracked.add_(1)
        if bn.momentum is None:
            raise NotImplementedError("cumulative-average BatchNorm momentum is not on the CoDA path")
    mean = torch.empty(c, dtype=torch.float32, device=y.device)
    invstd = torch.empty(c, dtype=torch.float32, device=y.device)
    with torch.cuda.device(y.device):
        st = lib().coda_bn_rows_stats(_ll(rows), _i(c), ptr(y), _f(bn.eps), _f(momentum),
                                      ptr(bn.running_mean if track else None), ptr(bn.running_var if track else None),
                                      ptr(mean), ptr(invstd), ptr(_scratch(c, y.device)), stream_of(y))
    check(st, "bn_rows_stats")
    return mean, invstd


def _stats_affine(y: torch.Tensor, bn, gamma, beta):
    """Batch statistics of y (rows, c) + the folded BatchNorm map (scale, shift) for the next GEMM's prologue."""
    rows, c = y.shape
    momentum, track = _bn_bookkeeping(bn)
    dev = y.device
    group = ops.bn_sync_group(bn)
    if group is not None:
        return ops.bn_stats_synced(group, rows, c, bn, momentum, track, gamma, beta, True, y=y)
    cpad = ops._pad64(c)
    mean = torch.empty(c, dtype=torch.float32, device=dev)
    invstd = torch.empty(c, dtype=torch.float32, device=dev)
    scale = torch.empty(cpad, dtype=torch.float32, device=dev)
    shift = torch.empty(cpad, dtype=torch.float32, device=dev)
    with torch.cuda.device(dev):
        st = lib().coda_bn_rows_stats_affine(_ll(rows), _i(c), ptr(y), _f(bn.eps), _f(momentum),
                                             ptr(bn.running_mean if track else None),
                                             ptr(bn.running_var if track else None), ptr(gamma), ptr(beta), ptr(mean),
                                             ptr(invstd), ptr(scale), ptr(shift), ptr(_scratch(c, dev)), stream_of(y))
    check(st, "bn_rows_stats_affine")
    return mean, invstd, scale, shift


def _bn_bookkeeping(bn):
    momentum = 0.0 if bn.momentum is None else float(bn.momentum)
    track = bn.track_running_stats and bn.running_mean is not None
    if track and bn.num_batches_tracked is not None:
        bn.num_batches_tracked.add_(1)
        if bn.momentum is None:
            raise NotImplementedError("cumulative-average BatchNorm momentum is not on the CoDA path")
    return momentum, track


def _stats_from_partials(partials: torch.Tensor, rows: int, bn, gamma, beta, want_affine: bool):
    """Finalise the column-sum partials a GEMM epilogue wrote (no pass over the activation)."""
    nblocks, _, c = partials.shape
    momentum, track = _bn_bookkeeping(bn)
    dev = partials.device
    group = ops.bn_sync_group(bn)
    if group is not None:
        return ops.bn_stats_synced(group, rows, c, bn, momentum, track, gamma, beta, want_affine, partials=partials)
    mean = torch.empty(c, dtype=torch.float32, device=dev)
    invstd = torch.empty(c, dtype=torch.float32, device=dev)
    scale = shift = None
    if want_affine:
        scale = torch.empty(ops._pad64(c), dtype=torch.float32, device=dev)
        shift = torch.empty(ops._pad64(c), dtype=torch.float32, device=dev)
    with torch.cuda.device(dev):
        st = lib().coda_bn_stats_finalize(_i(nblocks), _ll(rows), _i(c), ptr(partials), _f(bn.eps), _f(momentum),
                                          ptr(bn.running_mean if track else None),
                                          ptr(bn.running_var if track else None), ptr(gamma), ptr(beta), ptr(mean),
                                          ptr(invstd), ptr(scale), ptr(shift), stream_of(partials))
    check(st, "bn_stats_finalize")
    return mean, invstd, scale, shift


class _SharedMLPMax(torch.autograd.Function):
    """forward(x_rows (R, C0), group, nsplit, bns, W0, g0, b0, W1, g1, b1, ...) -> pooled (R / group, C_last)

    Forward data flow (HBM): y_l is written ONCE as fp32 by GEMM l, whose epilogue also produces the BatchNorm
    statistics of y_l; GEMM l+1 reads y_l in place and applies BatchNorm + ReLU + the bf16 split in its prologue
    (ops.gemm_a32, CODA_A32_AFFINE_RELU).  No operand planes, no separate statistics pass."""

    @staticmethod
    def forward(ctx, x, group, nsplit, bns, *params):
        L = lib()
        nl = len(bns)
        rows, c0 = x.shape
        dev = x.device
        ys, means, invstds, scales, shifts = [], [], [], [], []
        small_k = c0 <= 8
        scale = shift = None
        with torch.cuda.device(dev):
            for li in range(nl):
                w, gamma, beta = params[3 * li: 3 * li + 3]
                cout, cin = w.shape
                last = li == nl - 1
                if li == 0 and small_k:
                    y = torch.empty((rows, cout), dtype=torch.float32, device=dev)
                    check(L.coda_rows_linear_small_k(_ll(rows), _i(cin), _i(cout), ptr(x), ptr(w.contiguous()), ptr(y),
                                                     stream_of(x)), "rows_linear_small_k")
                    mean, invstd, scale, shift = _stats_affine(y, bns[li], gamma, beta)
                else:
                    wp = ops._packed_weight(w, False, nsplit)
                    if li == 0:
                        y, part = ops.gemm_a32(x, wp, cout, want_stats=True)
                    else:
                        y, part = ops.gemm_a32(ys[-1], wp, cout, mode=ops.A32_AFFINE_RELU, scale=scale, shift=shift,
                                               want_stats=True)
                    mean, invstd, scale, shift = _stats_from_partials(part, rows, bns[li], gamma, beta, True)
                ys.append(y); means.append(mean); invstds.append(invstd); scales.append(scale); shifts.append(shift)
                if last:
                    groups = rows // group
                    pooled = torch.empty((groups, cout), dtype=torch.float32, device=dev)
                    argmax = torch.empty((groups, cout), dtype=torch.uint8, device=dev)
                    check(L.coda_bn_relu_maxpool_rows(_ll(groups), _i(group), _i(cout), ptr(y), ptr(mean), ptr(invstd),
                                                      ptr(gamma), ptr(beta), ptr(pooled), ptr(argmax), stream_of(x)),
                          "bn_relu_maxpool_rows")
        ctx.nl, ctx.group, ctx.small_k, ctx.nsplit = nl, group, small_k, nsplit
        ctx.groups = [ops.bn_sync_group(bn) for bn in bns]
        ctx.save_for_backward(x, argmax, *ys, *means, *invstds, *scales, *shifts, *params)
        ctx.mark_non_differentiable(argmax)
        return pooled, argmax

    @staticmethod
    def backward(ctx, dpooled, _dargmax):
        L = lib()
        nl, group = ctx.nl, ctx.group
        saved = ctx.saved_tensors
        x, argmax = saved[0], saved[1]
        ys = saved[2: 2 + nl]
        means = saved[2 + nl: 2 + 2 * nl]
        invstds = saved[2 + 2 * nl: 2 + 3 * nl]
        scales = saved[2 + 3 * nl: 2 + 4 * nl]
        shifts = saved[2 + 4 * nl: 2 + 5 * nl]
        params = saved[2 + 5 * nl:]
        rows = x.shape[0]
        dev = x.device
        ns = BACKWARD_PLANES
        grads = [None] * (3 * nl)
        dx = None
        dz = None
        dpooled = dpooled.contiguous()
        with torch.cuda.device(dev):
            for li in range(nl - 1, -1, -1):
                w, gamma, beta = params[3 * li: 3 * li + 3]
                cout, cin = w.shape
                y, mean, invstd = ys[li], means[li], invstds[li]
                sg, sb = ops._sink(gamma), ops._sink(beta)       # dgamma / dbeta straight into the flat gradient buffer
                if sg is None or sb is None:
                    sg = sb = None
                s1 = torch.empty(cout, dtype=torch.float32, device=dev) if sb is None else sb
                s2 = torch.empty(cout, dtype=torch.float32, device=dev) if sg is None else sg
                scratch = _scratch(cout, dev)
                pooled_form = li == nl - 1
                if pooled_form:
                    # dprime: the pooled gradient already masked by the ReLU of its arg-max row and scaled by gamma *
                    # invstd -- the GEMM prologues below only place it
                    dprime = torch.empty_like(dpooled)
                    check(L.coda_bn_relu_bwd_reduce_pooled(_ll(rows // group), _i(group), _i(cout), ptr(y), ptr(dpooled),
                                                           ptr(argmax), ptr(mean), ptr(invstd), ptr(gamma), ptr(beta),
                                                           ptr(s1), ptr(s2), ptr(scratch), ptr(dprime), stream_of(x)),
                          "bn_relu_bwd_reduce_pooled")
                else:
                    check(L.coda_bn_relu_bwd_reduce(_ll(rows), _i(cout), ptr(y), ptr(dz), ptr(mean), ptr(invstd),
                                                    ptr(gamma), ptr(beta), ptr(s1), ptr(s2), ptr(scratch), stream_of(x)),
                          "bn_relu_bwd_reduce")
                loc1, loc2 = s1, s2
                if ctx.groups[li] is not None:
                    # the input gradient needs the means over every rank's rows; dgamma / dbeta stay the local sums.
                    # Taken BEFORE the sink is notified: the notification may start the all-reduce of that range of
                    # the flat gradient on the side stream, which rewrites s1 / s2 in place
                    s1, s2 = ops.bn_sync_backward_sums(s1, s2, ctx.groups[li])
                if sg is None:
                    grads[3 * li + 1], grads[3 * li + 2] = loc2, loc1    # dgamma, dbeta
                else:
                    ops._sunk(sg), ops._sunk(sb)
                sw = ops._sink(w)
                if li == 0 and ctx.small_k:
                    if nl == 1:   # single block: expand the pooled gradient (not a CoDA configuration)
                        dz = torch.zeros((rows // group, group, cout), dtype=torch.float32, device=dev)
                        dz.scatter_(1, argmax.long().unsqueeze(1), dpooled.unsqueeze(1))
                        dz = dz.view(rows, cout)
                    L.coda_bn_rows_small_k_scratch_floats.restype = ctypes.c_longlong
                    sc = torch.empty(int(L.coda_bn_rows_small_k_scratch_floats(_i(cin), _i(cout))), dtype=torch.float32,
                                     device=dev)
                    dw = torch.empty((cout, cin), dtype=torch.float32, device=dev) if sw is None else sw
                    check(L.coda_bn_relu_bwd_small_k(_ll(rows), _i(cin), _i(cout), ptr(y), ptr(dz), ptr(mean), ptr(invstd),
                                                     ptr(gamma), ptr(beta), ptr(s1), ptr(s2), ptr(x), ptr(dw), ptr(sc),
                                                     stream_of(x)), "bn_relu_bwd_small_k")
                    grads[0] = dw if sw is None else ops._sunk(sw)
                    break
                if sw is not None and cin % 4 != 0:
                    sw = None
                # BatchNorm(+ReLU) backward as a GEMM prologue: dy = [z > 0] * scale * d + alpha * y + beta
                cpad = ops._pad64(cout)
                alpha = torch.empty(cpad, dtype=torch.float32, device=dev)
                bcoef = torch.empty(cpad, dtype=torch.float32, device=dev)
                check(L.coda_bn_bwd_coefs(_i(cout), _ll(rows), ptr(mean), ptr(invstd), ptr(gamma), ptr(s1), ptr(s2),
                                          ptr(alpha), ptr(bcoef), stream_of(x)), "bn_bwd_coefs")
                pro = dict(a_scale=scales[li], a_shift=shifts[li], a_alpha=alpha, a_beta=bcoef)
                if pooled_form and group % 32 == 0 and (128 % group == 0 or group % 128 == 0) and cout % 128 == 0:
                    # the arg-max rows / pooled gradient of a tile's groups travel with the raw tiles (TMA)
                    mode, a2 = ops.A32_BN_BWD_POOLED_PRE, dprime
                    extra = dict(argmax=argmax, group=group)
                elif pooled_form:
                    # group sizes that do not tile the kernels' 32-row slabs: expand the pooled gradient once
                    dz = torch.zeros((rows // group, group, cout), dtype=torch.float32, device=dev)
                    dz.scatter_(1, argmax.long().unsqueeze(1), dpooled.unsqueeze(1))
                    dz = dz.view(rows, cout)
                    mode, a2, extra = ops.A32_BN_BWD, dz, {}
                else:
                    mode, a2, extra = ops.A32_BN_BWD, dz, {}
                # dW = dy^T a_{l-1}: both operands are read as fp32 rows; a_{l-1} = relu(bn(y_{l-1})) (or x)
                if li > 0:
                    grads[3 * li] = ops.gemm_tn32(y, ys[li - 1], a_mode=mode, a2=a2, b_mode=ops.A32_AFFINE_RELU,
                                                  b_scale=scales[li - 1], b_shift=shifts[li - 1], out=sw, **pro, **extra)
                else:
                    grads[3 * li] = ops.gemm_tn32(y, x, a_mode=mode, a2=a2, out=sw, **pro, **extra)
                if sw is not None:
                    grads[3 * li] = ops._sunk(sw)
                if li > 0 or ctx.needs_input_grad[0]:
                    # dz_{l-1} = dy W_l: the forward weight planes as an MN-major operand
                    dz_new = ops.gemm_a32(y, ops._packed_weight(w, False, ctx.nsplit), cin, mode=mode, scale=scales[li],
                                          shift=shifts[li], alpha=alpha, beta=bcoef, a2=a2, b_mn=True, nsplit=ns,
                                          **extra)
                    dz = dz_new
                    if li == 0:
                        dx = dz
        return (dx, None, None, None, *grads)


def shared_mlp_max(x_rows: torch.Tensor, blocks, group: int, nsplit: int | None = None) -> torch.Tensor:
    """x_rows (R, C0) channels-last grouped features -> (R / group, C_last): max over each run of `group` rows of
    relu(bn(conv(...))).  `blocks` = [(conv, bn), ...] (1x1 Conv2d without bias, BatchNorm2d or SyncBatchNorm in
    training mode)."""
    params = []
    for conv, bn in blocks:
        params += [conv.weight.reshape(conv.weight.shape[0], -1), bn.weight, bn.bias]
    pooled, _ = _SharedMLPMax.apply(x_rows.contiguous(), int(group), ops.DEFAULT_NSPLIT if nsplit is None else nsplit,
                                    [bn for _, bn in blocks], *params)
    return pooled


# --------------------------------------------------------------------------- inference (eval-mode BatchNorm)
# The one layout the inference kernel covers (csrc/sa_infer_sm90.cu): the 3DETR pre-encoder, xyz (+ rgb) input.
INFER_WIDTHS = (64, 128, 256)
INFER_GROUP = 64
INFER_PLANES = 3          # bf16 planes packed per weight (coda_sa_mlp_max_infer's w2_planes / w3_planes)


def infer_applicable(x: torch.Tensor, blocks, group: int) -> bool:
    """Can the inference kernel compute `blocks` + max over `group` on x (B, C0, npoint, nsample)?  Only with every
    BatchNorm in eval mode with running statistics, and only when autograd would record nothing."""
    if not (x.is_cuda and x.dtype == torch.float32 and x.dim() == 4 and group == INFER_GROUP
            and x.shape[3] == group and x.shape[1] in (3, 6) and len(blocks) == len(INFER_WIDTHS)):
        return False
    if x.stride(3) != 1:
        return False
    params = [t for conv, bn in blocks for t in (conv.weight, bn.weight, bn.bias)]
    if torch.is_grad_enabled() and (x.requires_grad or any(p is not None and p.requires_grad for p in params)):
        return False
    cin = x.shape[1]
    for (conv, bn), cout in zip(blocks, INFER_WIDTHS):
        if conv.bias is not None or tuple(conv.weight.shape) != (cout, cin, 1, 1):
            return False
        if bn.training or not bn.affine or bn.running_mean is None or bn.running_var is None:
            return False
        if any(t.dtype != torch.float32 or t.device != x.device
               for t in (conv.weight, bn.weight, bn.bias, bn.running_mean, bn.running_var)):
            return False
        cin = cout
    return True


def _folded_affine(blocks) -> torch.Tensor:
    """[scale1 | shift1 | scale2 | shift2 | scale3 | shift3] of the eval-mode BatchNorms, from the current running
    statistics (recomputed every call: a changed statistic is never stale)."""
    parts = []
    with torch.no_grad():
        for _, bn in blocks:
            scale = bn.weight * torch.rsqrt(bn.running_var + bn.eps)
            parts += [scale, bn.bias - bn.running_mean * scale]
        return torch.cat(parts)


def shared_mlp_max_infer(x: torch.Tensor, blocks, group: int) -> torch.Tensor:
    """x (B, C0, npoint, nsample) grouped features, read in place -> (B * npoint, 256): max over the neighbours of
    relu(bn(conv(...))) with eval-mode BatchNorm, in one kernel.  Call infer_applicable() first."""
    b, c0, npoint, nsample = x.shape
    (conv1, _), (conv2, _), (conv3, _) = blocks
    w1 = conv1.weight.detach().reshape(INFER_WIDTHS[0], c0).contiguous()
    # the kernel reads 3 planes of W2 and planes 0 and 1 of W3, whatever ops.DEFAULT_NSPLIT says
    w2 = ops._packed_weight(conv2.weight.reshape(INFER_WIDTHS[1], -1), False, INFER_PLANES)
    w3 = ops._packed_weight(conv3.weight.reshape(INFER_WIDTHS[2], -1), False, INFER_PLANES)
    affine = _folded_affine(blocks)
    out = torch.empty((b * npoint, INFER_WIDTHS[2]), dtype=torch.float32, device=x.device)
    with torch.cuda.device(x.device):
        st = lib().coda_sa_mlp_max_infer(_ll(b), _i(c0), _i(npoint), _i(nsample), ptr(x), _ll(x.stride(0)),
                                         _ll(x.stride(1)), _ll(x.stride(2)), ptr(w1), ptr(w2), _ll(w2.stride(0)),
                                         ptr(w3), _ll(w3.stride(0)), ptr(affine), ptr(out), _ll(out.stride(0)),
                                         stream_of(x))
    check(st, "sa_mlp_max_infer")
    return out
