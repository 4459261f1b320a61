"""torch-facing wrappers (autograd where needed) around the C-ABI kernels of
include/coda_detr.h and include/coda_attention.h.  Every function here launches
hand-written sm_90a code on the current stream; none has a CPU or PyTorch
fallback -- a CPU tensor raises.
"""
from __future__ import annotations

import ctypes

import torch

from ._lib import check, lib, ptr, stream_of

_i = ctypes.c_int
_ll = ctypes.c_longlong
_f = ctypes.c_float


def _need_cuda(t: torch.Tensor, name: str) -> None:
    if not t.is_cuda:
        raise RuntimeError(f"{name}: CPU not supported (coda_b200 kernels are CUDA-only)")


def _f32c(t: torch.Tensor) -> torch.Tensor:
    if t.dtype != torch.float32:
        t = t.float()
    return t.contiguous()


# --------------------------------------------------------------------------- gradient sink
class GradSink:
    """Lets the backward kernels write PARAMETER gradients straight into the flat gradient buffer of
    engine.FlatParameters instead of returning them to autograd (which would run one `grad += new` kernel per
    parameter and zero-filled scatter kernels for sliced weights).  A parameter tensor -- or a contiguous slice /
    reshape of one, e.g. the q / k / v row blocks of a packed in-projection -- is recognised by its address inside
    the flat parameter buffer; only regions that receive exactly ONE gradient contribution per step are eligible
    (measured on the probe pass), the others keep going through autograd's accumulation.

    mode "count": record which regions the backward touches (probe pass, nothing is redirected);
    mode "write": `lookup` returns the gradient view to write into, `wrote` notifies the all-reduce bucketing."""

    def __init__(self):
        self.mode = "count"
        self.uses: dict = {}            # (param index, byte offset inside the parameter, numel) -> contributions
        self._by_storage: dict = {}     # untyped storage address -> (param index, param)
        self.base = self.end = 0
        self.flat_grad = None
        self.allowed: set = set()       # (byte offset in the flat buffer, numel)
        self.on_write = None

    # -- probe pass (parameters still own their storages)
    def watch(self, params):
        self._by_storage = {p.untyped_storage().data_ptr(): (i, p) for i, p in enumerate(params)}

    def _note(self, w):
        hit = self._by_storage.get(w.untyped_storage().data_ptr())
        if hit is not None and w.is_contiguous():
            key = (hit[0], w.data_ptr() - hit[1].data_ptr(), w.numel())
            self.uses[key] = self.uses.get(key, 0) + 1

    # -- steady state
    def arm(self, flat_param, flat_grad, param_byte_offsets):
        """param_byte_offsets[i]: byte offset of probe-time parameter i inside the flat buffers"""
        self.base, self.end = flat_param.data_ptr(), flat_param.data_ptr() + flat_param.numel() * 4
        self.flat_param = flat_param      # kept alive: its address range must not be recycled while this sink is armed
        self.flat_grad = flat_grad
        per_param: dict = {}
        for (i, rel, numel), n in self.uses.items():
            per_param.setdefault(i, []).append((rel, numel, n))
        self.allowed = set()
        for i, regions in per_param.items():
            # eligible: every region of the parameter written once, regions pairwise disjoint
            regions.sort()
            ok = all(n == 1 for _, _, n in regions) and all(
                a[0] + a[1] * 4 <= b[0] for a, b in zip(regions, regions[1:]))
            if ok:
                for rel, numel, _ in regions:
                    self.allowed.add((param_byte_offsets[i] + rel, numel))
        self.mode = "write"

    def lookup(self, w):
        if self.mode == "count":
            self._note(w)
            return None
        ptr_ = w.data_ptr()
        if not (self.base <= ptr_ < self.end) or not w.is_contiguous():
            return None
        off = ptr_ - self.base
        if (off, w.numel()) not in self.allowed:
            return None
        return self.flat_grad.as_strided(w.shape, w.stride(), off // 4)

    def wrote(self, view):
        if self.on_write is not None:
            self.on_write((view.data_ptr() - self.flat_grad.data_ptr()) // 4)


_SINK: GradSink | None = None


def set_grad_sink(sink) -> None:
    global _SINK
    _SINK = sink


def _sink(w):
    """Gradient destination of parameter(-slice) `w` in the flat buffer, or None (-> return the gradient to autograd)."""
    return None if (_SINK is None or w is None) else _SINK.lookup(w)


def _sunk(view):
    _SINK.wrote(view)
    return None      # what the backward returns to autograd for this input


# --------------------------------------------------------------------------- LayerNorm
class _LayerNorm(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, weight, bias, eps):
        _need_cuda(x, "layer_norm")
        xc = _f32c(x)
        c = xc.shape[-1]
        rows = xc.numel() // c
        y = torch.empty_like(xc)
        mean = torch.empty(rows, dtype=torch.float32, device=x.device)
        rstd = torch.empty(rows, dtype=torch.float32, device=x.device)
        with torch.cuda.device(x.device):
            st = lib().coda_layer_norm_fwd(_ll(rows), _i(c), _f(eps), ptr(xc), ptr(weight), ptr(bias), ptr(y),
                                           ptr(mean), ptr(rstd), stream_of(x))
        check(st, "layer_norm_fwd")
        ctx.save_for_backward(xc, weight, bias, mean, rstd)
        return y

    @staticmethod
    def backward(ctx, dy):
        xc, weight, bias, mean, rstd = ctx.saved_tensors
        dyc = _f32c(dy)
        c = xc.shape[-1]
        rows = xc.numel() // c
        dx = torch.empty_like(xc)
        sg, sb = _sink(weight), _sink(bias)
        if sg is None or sb is None:
            sg = sb = None
        dgamma = torch.empty_like(weight) if sg is None else sg
        dbeta = torch.empty_like(weight) if sb is None else sb
        nscratch = lib().coda_layer_norm_bwd_scratch(_ll(rows), _i(c))
        partial = torch.empty(max(int(nscratch), 1), dtype=torch.float32, device=xc.device)
        with torch.cuda.device(xc.device):
            st = lib().coda_layer_norm_bwd(_ll(rows), _i(c), ptr(dyc), ptr(xc), ptr(weight), ptr(mean), ptr(rstd),
                                           ptr(dx), ptr(dgamma), ptr(dbeta), ptr(partial), stream_of(xc))
        check(st, "layer_norm_bwd")
        if sg is not None:
            return dx, _sunk(sg), _sunk(sb), None
        return dx, dgamma, dbeta, None


def layer_norm(x: torch.Tensor, weight: torch.Tensor, bias: torch.Tensor, eps: float = 1e-5) -> torch.Tensor:
    """LayerNorm over the last dim (multiple of 128, <= 1024); fp32."""
    return _LayerNorm.apply(x, weight, bias, float(eps))


@torch.no_grad()
def layer_norm_half(x: torch.Tensor, weight: torch.Tensor, bias: torch.Tensor, eps: float = 1e-5) -> torch.Tensor:
    """Forward-only LayerNorm on fp16 activations with fp32 statistics (frozen CLIP towers)."""
    _need_cuda(x, "layer_norm_half")
    assert x.dtype == torch.float16
    xc = x.contiguous()
    c = xc.shape[-1]
    y = torch.empty_like(xc)
    w32, b32 = _f32c(weight), _f32c(bias)      # held until the launch (see boxes_in_image)
    with torch.cuda.device(x.device):
        st = lib().coda_layer_norm_fwd_half(_ll(xc.numel() // c), _i(c), _f(eps), ptr(xc), ptr(w32), ptr(b32), ptr(y),
                                            stream_of(x))
    check(st, "layer_norm_fwd_half")
    return y


class LayerNorm(torch.nn.LayerNorm):
    """nn.LayerNorm with the same parameters / state-dict keys, running the
    warp-per-row kernel (reference NORM_DICT["ln"], models/helpers.py:27-32)."""

    def forward(self, x):
        return layer_norm(x, self.weight, self.bias, self.eps)


def _ln_backward(rows, c, dy, dmap, dy2, add, xc, weight, bias, mean, rstd, dx, dgamma=None, dbeta=None):
    """one coda_layer_norm_bwd_ex launch (+ its finalize); dgamma / dbeta: destination or None -> (sink | new).
    Returns (dgamma, dbeta) as they go back to autograd (None when written into the flat gradient buffer)."""
    own = dgamma is not None
    sg = sb = None
    if not own:
        sg, sb = _sink(weight), _sink(bias)
        if sg is None or sb is None:
            sg = sb = None
        dgamma = torch.empty_like(weight) if sg is None else sg
        dbeta = torch.empty_like(weight) if sb is None else sb
    nscratch = lib().coda_layer_norm_bwd_scratch(_ll(rows), _i(c))
    partial = torch.empty(max(int(nscratch), 1), dtype=torch.float32, device=xc.device)
    inner, so, si = dmap
    with torch.cuda.device(xc.device):
        st = lib().coda_layer_norm_bwd_ex(_ll(rows), _i(c), ptr(dy), _i(inner), _ll(so), _ll(si), ptr(dy2), ptr(add),
                                          ptr(xc), ptr(weight), ptr(mean), ptr(rstd), ptr(dx), ptr(dgamma), ptr(dbeta),
                                          ptr(partial), stream_of(xc))
    check(st, "layer_norm_bwd_ex")
    if sg is not None:
        return _sunk(sg), _sunk(sb)
    return dgamma, dbeta


class _LayerNormBranch(torch.autograd.Function):
    """The head of a pre-norm transformer sub-block as ONE autograd node:

        x  ->  (x, norm(x), norm(x) + pos)

    `x` passes through so that the gradient of the residual branch arrives at this node and is added to the norm's
    input gradient inside the backward kernel; `norm(x) + pos` (the q = k operand, reference
    models/transformer.py:556-580 `with_pos_embed`) is a second store of the forward kernel and a second load of the
    backward one.  Autograd's own wiring runs an `a + b` kernel for each of those joins."""

    @staticmethod
    def forward(ctx, x, weight, bias, eps, pos, want_y):
        _need_cuda(x, "layer_norm_branch")
        ctx.set_materialize_grads(False)
        xc = _f32c(x)
        c = xc.shape[-1]
        rows = xc.numel() // c
        y = torch.empty_like(xc) if want_y else None
        pc = ypos = None
        if pos is not None:
            assert pos.shape == x.shape, "pos must have the shape of x"
            pc = _f32c(pos)
            ypos = torch.empty_like(xc)
        mean = torch.empty(rows, dtype=torch.float32, device=x.device)
        rstd = torch.empty(rows, dtype=torch.float32, device=x.device)
        with torch.cuda.device(x.device):
            st = lib().coda_layer_norm_fwd_ex(_ll(rows), _i(c), _f(eps), ptr(xc), ptr(weight), ptr(bias), ptr(y), _i(0),
                                              _ll(0), _ll(0), ptr(pc), ptr(ypos), ptr(mean), ptr(rstd), stream_of(x))
        check(st, "layer_norm_fwd_ex")
        ctx.save_for_backward(xc, weight, bias, mean, rstd)
        ctx.pos_grad = pos is not None and pos.requires_grad
        # the residual operand: `x` itself, or its contiguous copy when one had to be made (the consumer would
        # otherwise copy it again)
        return (x if xc.data_ptr() == x.data_ptr() else xc), y, ypos

    @staticmethod
    def backward(ctx, g_id, g_y, g_ypos):
        xc, weight, bias, mean, rstd = ctx.saved_tensors
        c = xc.shape[-1]
        rows = xc.numel() // c
        ds = [_f32c(g) for g in (g_y, g_ypos) if g is not None]
        if not ds:                                # the norm's outputs were not used: only the by-pass gradient
            ds = [torch.zeros_like(xc)]
        add = None if g_id is None else _f32c(g_id)
        dx = torch.empty_like(xc)
        dgamma, dbeta = _ln_backward(rows, c, ds[0], (0, 0, 0), ds[1] if len(ds) > 1 else None, add, xc, weight, bias,
                                     mean, rstd, dx)
        return dx, dgamma, dbeta, None, (g_ypos if ctx.pos_grad else None), None


def layer_norm_branch(x: torch.Tensor, norm: torch.nn.Module, pos: torch.Tensor | None = None, want_y: bool = True):
    """-> (x_resid, y, y_pos): x_resid is `x` (use it as the residual operand), y = norm(x) (None unless want_y),
    y_pos = y + pos (y itself when pos is None).  Any other norm module takes the plain sequence of ops."""
    if not (isinstance(norm, LayerNorm) and x.is_cuda and x.dtype == torch.float32
            and norm.weight.shape[0] % 128 == 0 and norm.weight.shape[0] <= 1024
            and (pos is None or (pos.shape == x.shape and pos.dtype == torch.float32))):
        y = norm(x)
        return x, (y if want_y else None), (y if pos is None else y + pos)
    if pos is None:
        x_id, y, _ = _LayerNormBranch.apply(x, norm.weight, norm.bias, float(norm.eps), None, True)
        return x_id, y, y
    return _LayerNormBranch.apply(x, norm.weight, norm.bias, float(norm.eps), pos, bool(want_y))


class _NormStack(torch.autograd.Function):
    """norm(x_l) of every decoder layer's output (reference models/transformer.py:122-137 `intermediate`), written
    straight into ONE (layers, batch, query, channel) buffer -- the order the prediction heads read
    (models/model_3detr.py:1634-1650 permutes the (layers, query, batch, channel) stack) -- so that neither the
    torch.stack copy, nor the permuting copy, nor their strided gradient slices exist."""

    @staticmethod
    def forward(ctx, weight, bias, eps, *xs):
        nl = len(xs)
        q, b, c = xs[0].shape
        rows = q * b
        dev = xs[0].device
        xcs = [_f32c(x) for x in xs]
        out = torch.empty((nl, b, q, c), dtype=torch.float32, device=dev)
        mean = torch.empty((nl, rows), dtype=torch.float32, device=dev)
        rstd = torch.empty((nl, rows), dtype=torch.float32, device=dev)
        with torch.cuda.device(dev):
            for l, xc in enumerate(xcs):
                st = lib().coda_layer_norm_fwd_ex(_ll(rows), _i(c), _f(eps), ptr(xc), ptr(weight), ptr(bias), ptr(out[l]),
                                                  _i(b), _ll(c), _ll(q * c), None, None, ptr(mean[l]), ptr(rstd[l]),
                                                  stream_of(xc))
                check(st, "layer_norm_fwd_ex")
        ctx.save_for_backward(weight, bias, mean, rstd, *xcs)
        return out

    @staticmethod
    def backward(ctx, dout):
        weight, bias, mean, rstd = ctx.saved_tensors[:4]
        xcs = ctx.saved_tensors[4:]
        nl = len(xcs)
        q, b, c = xcs[0].shape
        rows = q * b
        dc = _f32c(dout)
        dev = dc.device
        dgam = torch.empty((nl, c), dtype=torch.float32, device=dev)
        dbet = torch.empty((nl, c), dtype=torch.float32, device=dev)
        dxs = []
        for l, xc in enumerate(xcs):
            dx = torch.empty_like(xc)
            _ln_backward(rows, c, dc[l], (b, c, q * c), None, None, xc, weight, bias, mean[l], rstd[l], dx,
                         dgamma=dgam[l], dbeta=dbet[l])
            dxs.append(dx)
        sg, sb = _sink(weight), _sink(bias)
        if sg is None or sb is None:
            sg = sb = None
        dgamma = sum_tensors([dgam[l] for l in range(nl)], out=sg)
        dbeta = sum_tensors([dbet[l] for l in range(nl)], out=sb)
        if sg is not None:
            dgamma, dbeta = _sunk(sg), _sunk(sb)
        return (dgamma, dbeta, None, *dxs)


def norm_stack(norm: torch.nn.Module, xs) -> torch.Tensor:
    """[(Q, B, C)] * layers -> (layers, B, Q, C) = norm of every entry; see _NormStack"""
    return _NormStack.apply(norm.weight, norm.bias, float(norm.eps), *xs)


def norm_stack_applicable(norm, xs) -> bool:
    return (isinstance(norm, LayerNorm) and len(xs) > 0 and all(x.is_cuda and x.dtype == torch.float32 and x.dim() == 3
                                                               and x.shape == xs[0].shape for x in xs)
            and xs[0].shape[-1] % 128 == 0 and xs[0].shape[-1] <= 1024)


# --------------------------------------------------------------------------- gradient fan-in
_SUM_MAX = 16


def sum_tensors(ts, out: torch.Tensor | None = None) -> torch.Tensor:
    """sum of same-shape fp32 CUDA tensors in one pass per 16 operands (coda_sum_n); `out` may be one of them"""
    ts = [_f32c(t) for t in ts]
    if out is None:
        out = torch.empty_like(ts[0])
    assert out.is_contiguous() and all(t.shape == ts[0].shape for t in ts)
    if any(t.data_ptr() == out.data_ptr() for t in ts[_SUM_MAX:]):
        # the first pass would overwrite an operand of a later pass before that pass reads it
        return sum_tensors([sum_tensors(ts)], out=out)
    n = ts[0].numel()
    with torch.cuda.device(out.device):
        while True:
            head, ts = ts[:_SUM_MAX], ts[_SUM_MAX:]
            arr = (ctypes.c_void_p * len(head))(*[t.data_ptr() for t in head])
            check(lib().coda_sum_n(_ll(n), _i(len(head)), arr, ptr(out), stream_of(out)), "sum_n")
            if not ts:
                return out
            ts = [out] + ts


class _FanOut(torch.autograd.Function):
    """x -> n aliases of x whose gradients meet in ONE n-ary sum (autograd's accumulation: n - 1 binary adds, each
    re-reading and re-writing the running sum)."""

    @staticmethod
    def forward(ctx, x, n):
        ctx.set_materialize_grads(False)
        return tuple(x.detach() for _ in range(n))

    @staticmethod
    def backward(ctx, *gs):
        gs = [g for g in gs if g is not None]
        if not gs:
            return None, None
        if len(gs) == 1:
            return gs[0], None
        return sum_tensors(gs), None


def fanout(x: torch.Tensor, n: int):
    """n handles on `x` for n consumers; use when a large activation feeds several branches"""
    if n <= 1 or not (x.is_cuda and x.dtype == torch.float32 and x.requires_grad and torch.is_grad_enabled()):
        return (x,) * max(n, 1)
    return _FanOut.apply(x, n)


# --------------------------------------------------------------------------- masked L1 (alignment loss)
class _MaskedL1(torch.autograd.Function):
    @staticmethod
    def forward(ctx, pred, target, w):
        nl = pred.shape[0]
        d = pred.shape[-1]
        rows = pred[0].numel() // d
        out = torch.empty(nl, dtype=torch.float32, device=pred.device)
        scratch = torch.empty(nl * 128, dtype=torch.float32, device=pred.device)
        with torch.cuda.device(pred.device):
            check(lib().coda_masked_l1_fwd(_i(nl), _ll(rows), _i(d), ptr(pred), ptr(target), ptr(w), ptr(out),
                                           ptr(scratch), stream_of(pred)), "masked_l1_fwd")
        ctx.save_for_backward(pred, target, w)
        return out

    @staticmethod
    def backward(ctx, g):
        pred, target, w = ctx.saved_tensors
        nl = pred.shape[0]
        d = pred.shape[-1]
        rows = pred[0].numel() // d
        gc = _f32c(g)
        dpred = torch.empty_like(pred)
        with torch.cuda.device(pred.device):
            check(lib().coda_masked_l1_bwd(_i(nl), _ll(rows), _i(d), ptr(pred), ptr(target), ptr(w), ptr(gc), ptr(dpred),
                                           stream_of(pred)), "masked_l1_bwd")
        return dpred, None, None


def masked_l1(pred: torch.Tensor, target: torch.Tensor, w: torch.Tensor) -> torch.Tensor:
    """(layers,) sums of |pred * w - target * w| with pred (layers, ..., d), target (..., d) broadcast over the layers and
    w (..., 1) or (...) one weight per row (reference criterion.py:924-943); target and w carry no gradient."""
    _need_cuda(pred, "masked_l1")
    d = pred.shape[-1]
    assert d % 4 == 0 and pred.shape[1:] == target.shape and w.numel() == target.numel() // d
    assert not target.requires_grad and not w.requires_grad
    return _MaskedL1.apply(_f32c(pred), _f32c(target), _f32c(w).reshape(-1))


# --------------------------------------------------------------------------- dropout / residual
_uint = ctypes.c_uint


def _seed_dev(device):
    from . import attention_launch

    return attention_launch.seed_counter(device)   # advanced once per step, inside the step's CUDA graph


def _next_salt() -> int:
    from . import attention_launch

    return attention_launch.next_salt()


class _DropoutAdd(torch.autograd.Function):
    """out = resid + dropout(x): the residual connection of every transformer sub-block in ONE pass; the mask is
    counter-based and regenerated by the backward (nothing saved)."""

    @staticmethod
    def forward(ctx, x, resid, p, salt):
        xc = _f32c(x)
        rc = None if resid is None else _f32c(resid)
        out = torch.empty_like(xc)
        with torch.cuda.device(x.device):
            st = lib().coda_dropout_add_fwd(_ll(xc.numel()), ptr(xc), ptr(rc), _f(p), _uint(salt),
                                            ptr(_seed_dev(x.device) if p > 0 else None), ptr(out), stream_of(x))
        check(st, "dropout_add_fwd")
        ctx.p, ctx.salt, ctx.has_resid = p, salt, resid is not None
        return out

    @staticmethod
    def backward(ctx, dout):
        dc = _f32c(dout)
        if ctx.p > 0.0:
            dx = torch.empty_like(dc)
            with torch.cuda.device(dc.device):
                st = lib().coda_dropout_bwd(_ll(dc.numel()), ptr(dc), _f(ctx.p), _uint(ctx.salt),
                                            ptr(_seed_dev(dc.device)), ptr(dx), stream_of(dc))
            check(st, "dropout_bwd")
        else:
            dx = dc
        return dx, (dc if ctx.has_resid else None), None, None


def dropout_add(x: torch.Tensor, resid: torch.Tensor, p: float, training: bool) -> torch.Tensor:
    """resid + dropout(x, p) (reference: `src = src + self.dropout1(src2)`, models/transformer.py:461-479)."""
    _need_cuda(x, "dropout_add")
    p = float(p) if training else 0.0
    return _DropoutAdd.apply(x, resid, p, _next_salt() if p > 0.0 else 0)


def dropout(x: torch.Tensor, p: float, training: bool) -> torch.Tensor:
    """nn.Dropout with the counter-based mask (no mask tensor, no ATen kernel)."""
    if not training or p <= 0.0:
        return x
    _need_cuda(x, "dropout")
    return _DropoutAdd.apply(x, None, float(p), _next_salt())


# --------------------------------------------------------------------------- BatchNorm on rows (GenericMLP blocks)
def _bn_scratch(c: int, device) -> torch.Tensor:
    lib().coda_bn_rows_scratch_floats.restype = ctypes.c_longlong
    return torch.empty(int(lib().coda_bn_rows_scratch_floats(_i(c))), dtype=torch.float32, device=device)


def bn_channels_ok(c: int) -> bool:
    return 4 <= c <= 1024 and c % 4 == 0 and 256 % (c // 4) == 0


# ---- synchronised BatchNorm (reference main.py:993 convert_sync_batchnorm).  Which group, if any, a BatchNorm
# synchronises over is decided per module by bn_sync_group(): an nn.SyncBatchNorm follows the rules of torch's
# SyncBatchNorm.forward (its own process_group); a plain BatchNorm follows this package's global option, off by default
# (per-GPU statistics and exactly one gradient all-reduce per step, DESIGN.md section 7).  A synchronised BatchNorm
# executed by bn_act_rows / sa_mlp takes its batch statistics over the group's ranks: one 16*C-byte fp64 all-reduce
# per layer forward, one 8*C-byte fp32 all-reduce backward.  Every rank of the group is assumed to hold the same
# number of rows (the finalize divides by rows * world): the reference's DistributedSampler pads the dataset so that
# every rank gets the same batch size.  No collective checks it.
_BN_SYNC = {"on": False, "group": None}


def set_bn_sync(enabled: bool, group=None) -> None:
    """The global option for plain (unconverted) BatchNorm modules; nn.SyncBatchNorm modules ignore it."""
    _BN_SYNC["on"], _BN_SYNC["group"] = bool(enabled), group


def bn_sync_world() -> int:
    """Ranks the global option synchronises plain BatchNorm modules over (1: off, or no process group)."""
    import torch.distributed as dist

    if not _BN_SYNC["on"] or not dist.is_available() or not dist.is_initialized():
        return 1
    return dist.get_world_size(_BN_SYNC["group"])


def bn_sync_group(bn):
    """The process group whose ranks' rows `bn` takes its batch statistics over, or None for statistics of this rank's
    rows alone.  An nn.SyncBatchNorm synchronises, as torch's SyncBatchNorm.forward does, in training mode with a process
    group initialised and more than one rank in `bn.process_group` (None: the default group); otherwise it takes the
    statistics of this rank's rows.  A plain BatchNorm synchronises whenever it takes batch statistics (training mode,
    or eval mode without running statistics) while the global option is on (set_bn_sync / TrainStep(sync_bn=True))
    over more than one rank."""
    import torch.distributed as dist

    if not dist.is_available() or not dist.is_initialized():
        return None
    if isinstance(bn, torch.nn.SyncBatchNorm):
        if not bn.training:
            return None
        group = bn.process_group
    elif _BN_SYNC["on"] and (bn.training or bn.running_mean is None):
        group = _BN_SYNC["group"]
    else:
        return None
    group = dist.group.WORLD if group is None else group
    return group if dist.get_world_size(group) > 1 else None


def bn_stats_synced(group, rows: int, c: int, bn, momentum: float, track: bool, gamma, beta, want_affine: bool, *,
                    y=None, partials=None):
    """Batch statistics over the ranks of `group` (bn_sync_group): local fp64 column sums (from y, or from a GEMM
    epilogue's partials) -> all-reduce -> finalize over rows * world.  Returns (mean, invstd, scale | None,
    shift | None)."""
    import torch.distributed as dist

    src = y if y is not None else partials
    dev = src.device
    world = dist.get_world_size(group)
    sums = torch.empty(2 * c, dtype=torch.float64, device=dev)
    mean = torch.empty(c, dtype=torch.float32, device=dev)
    invstd = torch.empty(c, dtype=torch.float32, device=dev)
    scale = shift = None
    if want_affine:
        scale = torch.empty(_pad64(c), dtype=torch.float32, device=dev)
        shift = torch.empty(_pad64(c), dtype=torch.float32, device=dev)
    L = lib()
    with torch.cuda.device(dev):
        if y is not None:
            check(L.coda_bn_rows_sums(_ll(rows), _i(c), ptr(y), ptr(sums), ptr(_bn_scratch(c, dev)), stream_of(y)),
                  "bn_rows_sums")
        else:
            check(L.coda_bn_partials_sums(_i(partials.shape[0]), _i(c), ptr(partials), ptr(sums), stream_of(partials)),
                  "bn_partials_sums")
        dist.all_reduce(sums, group=group)
        check(L.coda_bn_stats_finalize_sums(_ll(rows * world), _i(c), ptr(sums), _f(bn.eps), _f(momentum),
                                            ptr(bn.running_mean if track else None),
                                            ptr(bn.running_var if track else None), ptr(gamma), ptr(beta), ptr(mean),
                                            ptr(invstd), ptr(scale), ptr(shift), stream_of(src)), "bn_stats_finalize_sums")
    return mean, invstd, scale, shift


def bn_sync_backward_sums(s1: torch.Tensor, s2: torch.Tensor, group):
    """(s1, s2) = local sums of dz and dz * xhat (they ARE dbeta / dgamma and stay local, as in torch's SyncBatchNorm);
    the input gradient needs the means over the ranks of `group`: returns the rank-averaged copies (the kernels divide
    by the local row count, so average = global sum / global count)."""
    import torch.distributed as dist

    t = torch.stack((s1, s2))
    dist.all_reduce(t, op=dist.ReduceOp.AVG, group=group)
    return t[0], t[1]


class _BNActRows(torch.autograd.Function):
    """drop(relu(batch_norm(y))) on channels-last rows with batch statistics (training mode): statistics, one
    forward pass; backward = masked reduction + one pass (csrc/step_kernels.cu)."""

    @staticmethod
    def forward(ctx, y, gamma, beta, bn, relu, p, salt):
        yc = _f32c(y)
        rows, c = yc.shape
        dev = yc.device
        track = bn.track_running_stats and bn.running_mean is not None
        if track and bn.num_batches_tracked is not None:
            bn.num_batches_tracked.add_(1)
        if bn.momentum is None:
            raise NotImplementedError("cumulative-average BatchNorm momentum is not on the CoDA path")
        out = torch.empty_like(yc)
        L = lib()
        ctx.group = bn_sync_group(bn)
        with torch.cuda.device(dev):
            if ctx.group is not None:
                mean, invstd, _, _ = bn_stats_synced(ctx.group, rows, c, bn, float(bn.momentum), track, gamma, beta,
                                                     False, y=yc)
            else:
                mean = torch.empty(c, dtype=torch.float32, device=dev)
                invstd = torch.empty(c, dtype=torch.float32, device=dev)
                check(L.coda_bn_rows_stats(_ll(rows), _i(c), ptr(yc), _f(bn.eps), _f(bn.momentum),
                                           ptr(bn.running_mean if track else None),
                                           ptr(bn.running_var if track else None), ptr(mean), ptr(invstd),
                                           ptr(_bn_scratch(c, dev)), stream_of(yc)), "bn_rows_stats")
            check(L.coda_bn_act_rows_fwd(_ll(rows), _i(c), ptr(yc), ptr(mean), ptr(invstd), ptr(gamma), ptr(beta),
                                         _i(1 if relu else 0), _f(p), _uint(salt),
                                         ptr(_seed_dev(dev) if p > 0 else None), ptr(out), stream_of(yc)),
                  "bn_act_rows_fwd")
        ctx.save_for_backward(yc, gamma, beta, mean, invstd)
        ctx.relu, ctx.p, ctx.salt = relu, p, salt
        return out

    @staticmethod
    def backward(ctx, dout):
        y, gamma, beta, mean, invstd = ctx.saved_tensors
        dc = _f32c(dout)
        rows, c = y.shape
        dev = y.device
        sg, sb = _sink(gamma), _sink(beta)
        if sg is None or sb is None:
            sg = sb = None
        s1 = torch.empty(c, dtype=torch.float32, device=dev) if sb is None else sb      # dbeta
        s2 = torch.empty(c, dtype=torch.float32, device=dev) if sg is None else sg      # dgamma
        dy = torch.empty_like(y)
        L = lib()
        seed = ptr(_seed_dev(dev) if ctx.p > 0 else None)
        args = (_ll(rows), _i(c), ptr(y), ptr(dc), ptr(mean), ptr(invstd), ptr(gamma), ptr(beta),
                _i(1 if ctx.relu else 0), _f(ctx.p), _uint(ctx.salt), seed)
        with torch.cuda.device(dev):
            check(L.coda_bn_act_rows_bwd_reduce(*args, ptr(s1), ptr(s2), ptr(_bn_scratch(c, dev)), stream_of(y)),
                  "bn_act_rows_bwd_reduce")
            t1, t2 = bn_sync_backward_sums(s1, s2, ctx.group) if ctx.group is not None else (s1, s2)
            check(L.coda_bn_act_rows_bwd(*args, ptr(t1), ptr(t2), ptr(dy), stream_of(y)), "bn_act_rows_bwd")
        if sg is not None:
            return dy, _sunk(sg), _sunk(sb), None, None, None, None
        return dy, s2, s1, None, None, None, None      # dgamma = sum dz * xhat, dbeta = sum dz


def bn_act_rows(h: torch.Tensor, bn: torch.nn.modules.batchnorm._BatchNorm, relu: bool, drop_p: float,
                training: bool) -> torch.Tensor:
    """drop(relu(bn(h))) for h (rows, C): the BatchNorm1d -> ReLU -> Dropout run of a GenericMLP block
    (reference models/helpers.py:82-99) as two kernels.  Training-mode statistics come from the batch (and update
    the running buffers, over the ranks of bn_sync_group(bn) when it names a group); eval mode normalises with the
    running statistics.  `bn` may be an nn.BatchNorm1d or the nn.SyncBatchNorm convert_sync_batchnorm made of one."""
    _need_cuda(h, "bn_act_rows")
    c = h.shape[-1]
    if not (bn.affine and bn_channels_ok(c)):
        raise NotImplementedError(f"BatchNorm over {c} channels without affine parameters is not on the CoDA path")
    p = float(drop_p) if training else 0.0
    if bn.training or bn.running_mean is None:
        return _BNActRows.apply(h, bn.weight, bn.bias, bn, bool(relu), p, _next_salt() if p > 0.0 else 0)
    # eval: a per-channel affine map with constants (running statistics)
    scale = bn.weight * torch.rsqrt(bn.running_var + bn.eps)
    out = h * scale + (bn.bias - bn.running_mean * scale)
    return torch.relu(out) if relu else out


# --------------------------------------------------------------------------- softmax
def softmax_rows(x: torch.Tensor, log: bool = False) -> torch.Tensor:
    """softmax / log-softmax over the last dimension (no autograd)."""
    _need_cuda(x, "softmax_rows")
    xc = _f32c(x.detach())
    c = xc.shape[-1]
    y = torch.empty_like(xc)
    with torch.cuda.device(x.device):
        st = lib().coda_softmax_rows(_ll(xc.numel() // c), _i(c), _i(1 if log else 0), ptr(xc), ptr(y), stream_of(x))
    check(st, "softmax_rows")
    return y


# --------------------------------------------------------------------------- Fourier pos-enc
@torch.no_grad()
def fourier_pos_embed(xyz: torch.Tensor, gauss_B: torch.Tensor, d_out: int, input_range=None) -> torch.Tensor:
    """xyz (B, N, 3) -> (B, 2*d_out, N) = [sin | cos](2 pi x_hat @ gauss_B[:, :d_out]);
    x_hat is xyz mapped to [0, 1] by `input_range` = [min (B, 3), max (B, 3)] if given."""
    _need_cuda(xyz, "fourier_pos_embed")
    xc = _f32c(xyz)
    gb = _f32c(gauss_B)
    b, n, _ = xc.shape
    out = torch.empty((b, 2 * d_out, n), dtype=torch.float32, device=xyz.device)
    rmin = rmax = None
    if input_range is not None:
        rmin, rmax = _f32c(input_range[0]), _f32c(input_range[1])
    with torch.cuda.device(xyz.device):
        st = lib().coda_fourier_pos_embed(_i(b), _i(n), _i(d_out), _i(gb.shape[1]), _i(0 if rmin is None else 1),
                                          ptr(xc), ptr(rmin), ptr(rmax), ptr(gb), ptr(out), stream_of(xyz))
    check(st, "fourier_pos_embed")
    return out


# --------------------------------------------------------------------------- GIoU / matcher
@torch.no_grad()
def giou3d(corners1: torch.Tensor, corners2: torch.Tensor, nums_k2: torch.Tensor, rotated,
           rot_k2_limit: int | None = None) -> torch.Tensor:
    """(B, K1, 8, 3), (B, K2, 8, 3), (B,) -> generalised IoU (B, K1, K2).
    `rotated` is a bool, or a 1-element device tensor (read by the kernel: no host sync)."""
    _need_cuda(corners1, "giou3d")
    c1, c2 = _f32c(corners1), _f32c(corners2)
    b, k1, k2 = c1.shape[0], c1.shape[1], c2.shape[1]
    nk = nums_k2.to(device=c1.device, dtype=torch.int32).contiguous()
    out = torch.empty((b, k1, k2), dtype=torch.float32, device=c1.device)
    lim = k2 if rot_k2_limit is None else int(rot_k2_limit)
    rdev = None
    if isinstance(rotated, torch.Tensor):
        rdev = rotated.to(device=c1.device, dtype=torch.int32).reshape(1).contiguous()
        rotated = False
    with torch.cuda.device(c1.device):
        st = lib().coda_giou3d(_i(b), _i(k1), _i(k2), _i(1 if rotated else 0), ptr(rdev), _i(lim), ptr(c1), ptr(c2),
                               ptr(nk), ptr(out), stream_of(c1))
    check(st, "giou3d")
    return out


@torch.no_grad()
def hungarian(cost: torch.Tensor, nactual: torch.Tensor):
    """cost (B, nprop, ngt) fp32, nactual (B,) -> (per_prop_gt_inds int64 (B, nprop),
    proposal_matched_mask fp32 (B, nprop)); same assignment as scipy's
    linear_sum_assignment on cost[b, :, :nactual[b]]."""
    _need_cuda(cost, "hungarian")
    cc = _f32c(cost)
    b, nprop, ngt = cc.shape
    na = nactual.to(device=cc.device, dtype=torch.int32).contiguous()
    inds = torch.empty((b, nprop), dtype=torch.int64, device=cc.device)
    mask = torch.empty((b, nprop), dtype=torch.float32, device=cc.device)
    with torch.cuda.device(cc.device):
        st = lib().coda_hungarian(_i(b), _i(nprop), _i(ngt), ptr(cc), ptr(na), ptr(inds), ptr(mask), stream_of(cc))
    check(st, "hungarian")
    return inds, mask


CAMERAS = {"sunrgbd": 0, "scannet": 1}      # include/coda_detr.h CODA_CAMERA_*; K / Rtilt are n x n per scene
_CAMERA_DIM = {"sunrgbd": 3, "scannet": 4}


@torch.no_grad()
def boxes_in_image(corners_xyz: torch.Tensor, size_unnorm: torch.Tensor, inputs: dict, camera: str = "sunrgbd",
                   extent: bool = False):
    """Predicted boxes (B, Q, 8, 3) -> (int32 (B, Q, 4) [xmin, ymin, xmax, ymax] in the image, bool (B, Q) usable as
    a crop): include/coda_detr.h coda_boxes_in_image, fp64 like the reference's projection; no host sync.
    `camera` is the dataset's camera model: "sunrgbd" (K, Rtilt 3 x 3 intrinsics and tilt) or "scannet" (K the 4 x 4
    colour intrinsics, Rtilt the 4 x 4 camera-to-world pose).  With `extent`, also the fp64 (B, Q, 4)
    [umin, vmin, umax, vmax] the integer box truncates."""
    if camera not in CAMERAS:
        raise ValueError(f"boxes_in_image: unknown camera {camera!r} (expected one of {sorted(CAMERAS)})")
    b, q = corners_xyz.shape[:2]
    n = _CAMERA_DIM[camera]
    kshape, tshape = tuple(inputs["K"].shape), tuple(inputs["Rtilt"].shape)
    if kshape != (b, n, n) or tshape != (b, n, n):
        raise ValueError(f"boxes_in_image: the {camera} camera needs K and Rtilt of shape ({b}, {n}, {n}); "
                         f"got K {kshape} and Rtilt {tshape}")
    _need_cuda(corners_xyz, "boxes_in_image")
    dev = corners_xyz.device
    f64 = lambda t, shape: t.to(device=dev, dtype=torch.double).reshape(shape).contiguous()  # noqa: E731
    i64 = lambda t: t.to(device=dev, dtype=torch.int64).reshape(b).contiguous()  # noqa: E731
    scale = f64(inputs["scale_array"], (b, 3))
    rot, K, Rtilt = f64(inputs["rot_array"], (b, 9)), f64(inputs["K"], (b, n * n)), f64(inputs["Rtilt"], (b, n * n))
    flip, img_flip = f64(inputs["flip_array"], (b,)), f64(inputs["image_flip_array"], (b,))
    flip_len = f64(inputs["flip_length"], (b,))
    zx = f64(inputs["zx_flip_array"], (b,)) if "zx_flip_array" in inputs else None
    boxes = torch.empty((b, q, 4), dtype=torch.int32, device=dev)
    valid = torch.empty((b, q), dtype=torch.uint8, device=dev)
    ext = torch.empty((b, q, 4), dtype=torch.double, device=dev) if extent else None
    # every converted operand is held in a local until the launch has been issued (a temporary that dies inside the
    # argument list would hand its block to the next conversion)
    cx, su = _f32c(corners_xyz), _f32c(size_unnorm)
    ow, oh, xo, yo = (i64(inputs[k]) for k in ("ori_width", "ori_height", "x_offset", "y_offset"))
    with torch.cuda.device(dev):
        st = lib().coda_boxes_in_image(_i(b), _i(q), _i(CAMERAS[camera]), ptr(cx), ptr(su), ptr(scale), ptr(rot),
                                       ptr(flip), ptr(zx), ptr(K), ptr(Rtilt), ptr(ow), ptr(oh), ptr(xo), ptr(yo),
                                       ptr(img_flip), ptr(flip_len), ptr(boxes), ptr(valid), ptr(ext),
                                       stream_of(corners_xyz))
    check(st, "boxes_in_image")
    return (boxes, valid.bool(), ext) if extent else (boxes, valid.bool())


@torch.no_grad()
def novel_candidates(boxes2d: torch.Tensor, valid: torch.Tensor, objectness: torch.Tensor, pred_corners: torch.Tensor,
                     gt_corners: torch.Tensor, gt_present: torch.Tensor, nms_iou: float, gt_iou: float,
                     min_objectness: float, cap: int):
    """Stage-2 discovery, candidate selection per scene (include/coda_detr.h coda_novel_candidates): 2-D NMS of the
    projected boxes, ground-truth overlap rejection, objectness threshold -> (cand_idx (B, cap) int32 in descending
    score order, -1 padded; cand_count (B, 2) int32 = written, untruncated total).  No host synchronisation."""
    _need_cuda(boxes2d, "novel_candidates")
    b, q, _ = boxes2d.shape
    g = gt_corners.shape[1]
    bx = boxes2d.to(torch.int32).contiguous()
    vd = valid.to(torch.uint8).contiguous()
    cand = torch.empty((b, cap), dtype=torch.int32, device=bx.device)
    count = torch.empty((b, 2), dtype=torch.int32, device=bx.device)
    ob, pc, gc, gp = _f32c(objectness), _f32c(pred_corners), _f32c(gt_corners), _f32c(gt_present)
    with torch.cuda.device(bx.device):
        st = lib().coda_novel_candidates(_i(b), _i(q), _i(g), _i(cap), ptr(bx), ptr(vd), ptr(ob), ptr(pc), ptr(gc),
                                         ptr(gp), _f(nms_iou), _f(gt_iou), _f(min_objectness), ptr(cand), ptr(count),
                                         stream_of(bx))
    check(st, "novel_candidates")
    return cand, count


# --------------------------------------------------------------------------- attention
def attention(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, nhead: int, dropout_p: float = 0.0,
              training: bool = False, causal: bool = False, mask=None) -> torch.Tensor:
    """Multi-head scaled-dot-product attention on projected, sequence-first tensors.

    q (Lq, B, E), k / v (Lk, B, E) -> (Lq, B, E).  The scale 1/sqrt(E/nhead) is applied to
    q; the forward kernel never materialises the probabilities in HBM.
    """
    _need_cuda(q, "attention")
    from . import attention_sm100  # wgmma kernels (include/coda_attention.h)

    return attention_sm100.attention(q, k, v, nhead, dropout_p, training, causal, mask)


def attention_mask_bits(mask: torch.Tensor, batch: int):
    """boolean attention mask (True = not visible), (1 | B, Lq, Lk) -> packed (bits_q, bits_k) for ops.attention."""
    _need_cuda(mask, "attention_mask_bits")
    from . import attention_launch

    return attention_launch.mask_bits(mask, batch)


def radius_mask_bits(xyz: torch.Tensor, radius: float):
    """packed mask of `cdist(xyz, xyz) >= radius` for points xyz (B, L, 3): the masked encoder's radius masks."""
    _need_cuda(xyz, "radius_mask_bits")
    from . import attention_launch

    return attention_launch.radius_mask_bits(xyz, radius)


def attention_fused(a: torch.Tensor, b, layout: str, nhead: int, dropout_p: float = 0.0, training: bool = False,
                    mask=None) -> torch.Tensor:
    """Self-attention straight from fused projections -- "qkv": a = (L, B, 3E); "qk_v": a = (L, B, 2E) q|k and
    b = v (L, B, E).  Slices are read in place; the backward writes one packed gradient per fused projection."""
    _need_cuda(a, "attention")
    from . import attention_sm100

    return attention_sm100.attention_fused(a, b, layout, nhead, dropout_p, training, mask)


# --------------------------------------------------------------------------- CLIP crops
CLIP_MEAN = (0.48145466, 0.4578275, 0.40821073)
CLIP_STD = (0.26862954, 0.26130258, 0.27577711)


@torch.no_grad()
def crop_resize_normalize(images: torch.Tensor, scene: torch.Tensor, boxes: torch.Tensor, valid: torch.Tensor,
                          res: int, dtype=torch.float16, mean=CLIP_MEAN, std=CLIP_STD, patch: int = 0,
                          tile_rows: int = 0) -> torch.Tensor:
    """images (B, H, W, 3) uint8, scene (N,) int32, boxes (N, 4) int32 [xmin, ymin, xmax, ymax],
    valid (N,) bool -> (N, 3, res, res) CLIP-normalised crops (white-padded to square, antialiased
    bicubic resize with torchvision's uint8 semantics); with patch = ps > 0 the crops come out patch-major,
    (N, res / ps, res / ps, 3, ps, ps): the operand of the ViT's patch-embedding GEMM, no unfold copy."""
    _need_cuda(images, "crop_resize_normalize")
    if images.dtype != torch.uint8:
        raise RuntimeError("images must be uint8 (HWC)")
    img = images.contiguous()
    nimg, h, w, _ = img.shape
    n = boxes.shape[0]
    sc = scene.to(torch.int32).contiguous()
    bx = boxes.to(torch.int32).contiguous()
    vd = valid.to(torch.uint8).contiguous()
    if dtype not in (torch.float16, torch.float32):
        raise RuntimeError("output dtype must be float16 or float32")
    if patch > 0:
        assert res % patch == 0
        out = torch.empty((n, res // patch, res // patch, 3, patch, patch), dtype=dtype, device=img.device)
    else:
        out = torch.empty((n, 3, res, res), dtype=dtype, device=img.device)
    work = torch.empty(nimg * h * w, dtype=torch.int32, device=img.device)      # RGBX copy of the images
    m = (ctypes.c_float * 3)(*mean)
    s = (ctypes.c_float * 3)(*std)
    with torch.cuda.device(img.device):
        st = lib().coda_crop_resize_normalize_ex(_i(nimg), _i(h), _i(w), _i(n), _i(res), ptr(img), ptr(sc), ptr(bx),
                                                 ptr(vd), m, s, _i(1 if dtype == torch.float16 else 0), _i(patch),
                                                 _i(tile_rows), ptr(work), ptr(out), stream_of(img))
    check(st, "crop_resize_normalize")
    return out


@torch.no_grad()
def clip_classify(feats: torch.Tensor, text: torch.Tensor, scale: torch.Tensor, row_map: torch.Tensor,
                  shape) -> tuple:
    """Class probabilities of every (scene, query) row from its crop's CLIP feature (include/coda_image.h
    coda_clip_classify).  feats (n, 512) fp32 of the compacted crops, text (C, 512) normalised fp32, scale a
    one-element device tensor, row_map (B * Q) int32 (-1 = no crop) -> (sem_cls_prob (*shape, C): softmax of
    scale * f_hat . text^T, zeros where skipped; sem_cls_logits (*shape, C): zeros).  No host synchronisation."""
    _need_cuda(text, "clip_classify")
    for name, t in (("feats", feats), ("scale", scale), ("row_map", row_map)):
        if t.device != text.device:
            raise ValueError(f"clip_classify: {name} is on {t.device}, the text features on {text.device}")
    fc, tc, sc = _f32c(feats), _f32c(text), _f32c(scale.reshape(1))
    rm = row_map.to(torch.int32).contiguous()
    c, d = tc.shape
    if fc.shape[1:] != (d,):
        raise ValueError(f"clip_classify: features of width {tuple(fc.shape[1:])} against text of width {d}")
    prob = torch.empty((*shape, c), dtype=torch.float32, device=tc.device)
    logits = torch.empty_like(prob)
    if prob.numel() // c != rm.numel():
        raise ValueError(f"clip_classify: {rm.numel()} row-map entries for output rows {tuple(shape)}")
    with torch.cuda.device(tc.device):
        st = lib().coda_clip_classify(_ll(rm.numel()), _i(fc.shape[0]), _i(c), _i(d), ptr(fc), ptr(tc), ptr(sc),
                                      ptr(rm), ptr(prob), ptr(logits), stream_of(tc))
    check(st, "clip_classify")
    return prob, logits


# --------------------------------------------------------------------------- wgmma GEMM
# bf16 planes per fp32 operand.  3 -> six cross products, all 24 mantissa bits: fp32-class accuracy, which the
# 1e-4 parity bar needs through 13 layers (2 planes / 3 products measured 1.4e-4 on the class logits).
DEFAULT_NSPLIT = 3


def _pad64(k: int) -> int:
    return (k + 63) // 64 * 64


def pack_split(x: torch.Tensor, rows: int, k: int, row_stride: int, k_stride: int, nsplit: int = DEFAULT_NSPLIT,
               scale: float = 1.0, batch: int = 1, batch_stride: int = 0) -> torch.Tensor:
    """fp32 matrix/matrices addressed as x[b*batch_stride + r*row_stride + c*k_stride] -> bf16 planes
    (nsplit, batch, rows, kpad), K zero-padded to a multiple of 64 (operand format of gemm_nt)."""
    _need_cuda(x, "pack_split")
    assert x.dtype == torch.float32
    kpad = _pad64(k)
    out = torch.empty((nsplit, batch, rows, kpad), dtype=torch.bfloat16, device=x.device)
    base = x.data_ptr()
    with torch.cuda.device(x.device):
        for b in range(batch):
            # planes of one batch entry are (batch * rows * kpad) apart: pack plane-by-plane views
            st = lib().coda_pack_split_bf16_strided(
                _ll(rows), _i(k), _i(kpad), _ll(row_stride), _ll(k_stride),
                ctypes.c_void_p(base + 4 * b * batch_stride), _f(scale), _i(nsplit),
                ctypes.c_void_p(out.data_ptr() + 2 * b * rows * kpad), _ll(batch * rows * kpad), stream_of(x))
            check(st, "pack_split_bf16")
    return out


def gemm_nt(a_planes: torch.Tensor, b_planes: torch.Tensor, m: int, n: int, bias=None, relu: bool = False,
            out: torch.Tensor | None = None, act: int | None = None, out_dtype=torch.float32,
            residual: torch.Tensor | None = None) -> torch.Tensor:
    """C[b] = A[b] @ B[b]^T (+ bias) from packed planes (nsplit, batch, rows, kpad); B may have batch 1
    (shared weights).  fp16 planes (nsplit == 1) select the fp16 tensor-core path.  Returns fp32 (batch, m, n)."""
    _need_cuda(a_planes, "gemm_nt")
    nsplit, batch, _, kpad = a_planes.shape
    assert b_planes.shape[0] == nsplit and b_planes.shape[3] == kpad and a_planes.dtype == b_planes.dtype
    is_fp16 = a_planes.dtype == torch.float16
    bb = b_planes.shape[1]
    assert bb in (1, batch)
    if out is None:
        out = torch.empty((batch, m, n), dtype=out_dtype, device=a_planes.device)
    if act is None:
        act = 1 if relu else 0
    if residual is not None:
        assert residual.dtype == torch.float16 and residual.shape == (m, n) and residual.stride(1) == 1
    with torch.cuda.device(a_planes.device):
        st = lib().coda_gemm_nt_res(
            _i(nsplit), _i(1 if is_fp16 else 0), _i(batch), _i(m), _i(n), _i(kpad), ptr(a_planes),
            _ll(a_planes.stride(0)), _ll(a_planes.stride(1)), ptr(b_planes), _ll(b_planes.stride(0)),
            _ll(b_planes.stride(1) if bb > 1 else 0), ptr(bias), _i(act), _i(1 if out.dtype == torch.float16 else 0),
            ptr(residual), _ll(residual.stride(0) if residual is not None else 0),
            ptr(out), _ll(out.stride(1)), _ll(out.stride(0)), stream_of(a_planes))
    check(st, "gemm_nt")
    return out


A32_PLAIN, A32_AFFINE_RELU, A32_BN_BWD, A32_BN_BWD_POOLED = 0, 1, 2, 3
A32_BN_BWD_POOLED_PRE = 4     # a2 = pre-masked, pre-scaled pooled gradient (coda_bn_relu_bwd_reduce_pooled `dprime`)


def a32_ok(a: torch.Tensor) -> bool:
    """Can `a` (2-D fp32) be the in-place A operand of gemm_a32 (TMA row rules)?"""
    return (a.dim() == 2 and a.dtype == torch.float32 and a.is_cuda and a.stride(1) == 1 and a.stride(0) % 4 == 0
            and a.stride(0) >= a.shape[1] and a.data_ptr() % 16 == 0 and a.shape[1] >= 1)


def gemm_a32(a: torch.Tensor, b_planes: torch.Tensor, n: int, *, mode: int = A32_PLAIN, scale=None, shift=None,
             alpha=None, beta=None, a2=None, argmax=None, group: int = 0, b_mn: bool = False, bias=None,
             relu: bool = False, out: torch.Tensor | None = None, want_stats: bool = False, nsplit: int | None = None):
    """C (m, n) = T(a) @ B^T with the fp32 activation `a` (m, k) read IN PLACE: the split into bf16 operand planes
    happens inside the kernel (csrc/gemm_a32_sm90.cu), `T` is the prologue selected by `mode`
    (include/coda_gemm.h).  b_planes: packed weight planes (nsplit, 1, rows, ld) -- K-major (rows = n) or, with
    b_mn, the forward planes of a weight (rows = k) reused for the input gradient.  Returns C, or (C, partials) with
    want_stats: per-CTA column sum / sum-of-squares partials of C for coda_bn_stats_finalize."""
    _need_cuda(a, "gemm_a32")
    m, k = a.shape
    ns = b_planes.shape[0] if nsplit is None else nsplit
    assert a32_ok(a) and 2 <= ns <= b_planes.shape[0] and b_planes.dtype == torch.bfloat16
    ld = b_planes.shape[3]
    if out is None:
        out = torch.empty((m, n), dtype=torch.float32, device=a.device)
    L = lib()
    stats = None
    if want_stats:
        # rows = upper bound of the grid; CTAs that do not exist / columns a CTA never owns stay zero
        stats = torch.zeros((int(L.coda_gemm_a32_grid(_i(m), _i(n))), 2, n), dtype=torch.float32, device=a.device)
    lda2 = 0
    if mode == A32_BN_BWD:
        assert a32_ok(a2) and a2.shape == a.shape
        lda2 = a2.stride(0)
    elif mode in (A32_BN_BWD_POOLED, A32_BN_BWD_POOLED_PRE):
        assert a2.is_contiguous() and argmax.is_contiguous() and a2.shape == (m // group, k)
    with torch.cuda.device(a.device):
        st = L.coda_gemm_a32(_i(ns), _i(m), _i(n), _i(k), ptr(a), _ll(a.stride(0)), _i(mode), ptr(scale), ptr(shift),
                             ptr(alpha), ptr(beta), ptr(a2), _ll(lda2), ptr(argmax), _i(group), ptr(b_planes),
                             _ll(b_planes.stride(0)), _i(ld), _i(1 if b_mn else 0), ptr(bias), _i(1 if relu else 0),
                             ptr(out), _ll(out.stride(0)), ptr(stats), stream_of(a))
    check(st, "gemm_a32")
    return (out, stats) if want_stats else out


def tn32_ok(a: torch.Tensor) -> bool:
    return a32_ok(a) and a.shape[1] % 4 == 0


def gemm_tn32(a: torch.Tensor, b: torch.Tensor, *, a_mode: int = A32_PLAIN, a_scale=None, a_shift=None, a_alpha=None,
              a_beta=None, a2=None, argmax=None, group: int = 0, b_mode: int = A32_PLAIN, b_scale=None,
              b_shift=None, out: torch.Tensor | None = None, colsum_out: torch.Tensor | None = None) -> torch.Tensor:
    """C (m, n) = sum_r TA(a)[r, :]^T TB(b)[r, :] from the fp32 activations a (R, m), b (R, n) read in place
    (csrc/gemm_tn32_sm90.cu): the weight-gradient GEMM with the BatchNorm-backward / BatchNorm-forward
    prologues applied inside the kernel.  Two bf16 planes per operand.  colsum_out (m,): receives sum_r TA(a)[r, :]
    (the bias gradient) from the same pass."""
    _need_cuda(a, "gemm_tn32")
    rows, m = a.shape
    n = b.shape[1]
    assert tn32_ok(a) and tn32_ok(b) and b.shape[0] == rows
    if out is None:
        out = torch.empty((m, n), dtype=torch.float32, device=a.device)
    assert out.shape == (m, n) and out.stride(1) == 1 and out.stride(0) % 4 == 0 and out.data_ptr() % 16 == 0
    lda2 = 0
    if a_mode == A32_BN_BWD:
        assert a32_ok(a2) and a2.shape == a.shape
        lda2 = a2.stride(0)
    elif a_mode in (A32_BN_BWD_POOLED, A32_BN_BWD_POOLED_PRE):
        assert a2.is_contiguous() and argmax.is_contiguous() and a2.shape == (rows // group, m)
    with torch.cuda.device(a.device):
        st = lib().coda_gemm_tn32(_ll(rows), _i(m), _i(n), ptr(a), _ll(a.stride(0)), _i(a_mode), ptr(a_scale),
                                  ptr(a_shift), ptr(a_alpha), ptr(a_beta), ptr(a2), _ll(lda2), ptr(argmax), _i(group),
                                  ptr(b), _ll(b.stride(0)), _i(b_mode), ptr(b_scale), ptr(b_shift), ptr(out),
                                  _ll(out.stride(0)), ptr(colsum_out), stream_of(a))
    check(st, "gemm_tn32")
    return out


def gemm_tn(a_planes: torch.Tensor, b_planes: torch.Tensor, m: int, n: int) -> torch.Tensor:
    """C (m, n) = sum_r A[r, :m]^T B[r, :n] from ROW-packed planes (nsplit, 1, rows, pad64(cols)):
    the weight-gradient form dW = dY^T X on MN-major tensor-core operands (no transposed copies)."""
    _need_cuda(a_planes, "gemm_tn")
    nsplit, _, mc, lda = a_planes.shape
    assert b_planes.shape[0] == nsplit and b_planes.shape[2] == mc
    ldb = b_planes.shape[3]
    out = torch.empty((m, n), dtype=torch.float32, device=a_planes.device)
    with torch.cuda.device(a_planes.device):
        st = lib().coda_gemm_tn(_i(nsplit), _i(mc), _i(m), _i(n), ptr(a_planes), _ll(a_planes.stride(0)), _i(lda),
                                ptr(b_planes), _ll(b_planes.stride(0)), _i(ldb), ptr(out), _ll(n), stream_of(a_planes))
    check(st, "gemm_tn")
    return out


BACKWARD_NSPLIT = 2
USE_TN_WGRAD = True  # weight gradients from the row-packed operands (MN-major MMA); False: transposed packs


# --------------------------------------------------------------------------- Linear on the wgmma GEMM
_WEIGHT_EPOCH = 0
_WEIGHT_CACHE: dict = {}
# Weight planes depend on nothing but the parameters: a step can pack ALL of them up front on a side stream, under
# the furthest-point sampling that opens the forward (64 CTAs, 1.1 ms, nothing else to run beside it) instead of one
# ~4 us launch in front of every GEMM.  _PACK_LOG records the (weight, transposed, nsplit) requests of a step;
# _PACK_JOIN is the side stream the first consumer of a step has to wait for.
_PACK_LOG: list | None = None
_PACK_JOIN = None


def record_weight_packs(on: bool):
    """start recording / stop and return the list of weight-plane requests"""
    global _PACK_LOG
    if on:
        _PACK_LOG = []
        return None
    log, _PACK_LOG = _PACK_LOG, None
    return log


def prepack_weights(requests, side_stream) -> None:
    """pack every requested weight on `side_stream` (which has been ordered after the parameter update); the first
    _packed_weight call of the step joins it."""
    global _PACK_JOIN
    with torch.cuda.stream(side_stream):
        for w, transposed, nsplit in requests:
            _packed_weight(w, transposed, nsplit)
    _PACK_JOIN = side_stream


_ACT_CACHE: dict = {}   # packed planes of activations that several layers consume within one step


def invalidate_weight_cache() -> None:
    """Call after parameters were updated through storage the tensors' version counters do not see
    (the flat-buffer optimiser step of engine.TrainStep, eager or replayed from its CUDA graph: a replay runs no
    Python, so TrainStep.__call__ calls this after every replay).  Also ends the per-step activation-pack cache.
    Host-only: no synchronisation, no launch."""
    global _WEIGHT_EPOCH
    _WEIGHT_EPOCH += 1
    _WEIGHT_CACHE.clear()
    _ACT_CACHE.clear()


def _packed_rows(x: torch.Tensor, nsplit: int) -> torch.Tensor:
    """Row-packed planes of a 2-D activation, shared by every layer that consumes the SAME tensor in
    this step (the six prediction heads read one box-feature tensor, the eight decoder layers project
    the same encoder memory).  The entry keeps `x` alive, so its address cannot be recycled."""
    key = (x.data_ptr(), tuple(x.shape), x.stride(0), x._version, nsplit)
    hit = _ACT_CACHE.get(key)
    if hit is None:
        planes = pack_split(x, x.shape[0], x.shape[1], x.stride(0), 1, nsplit)
        if len(_ACT_CACHE) > 64:
            _ACT_CACHE.clear()
        _ACT_CACHE[key] = (planes, x)
        return planes
    return hit[0]


def _packed_weight(w: torch.Tensor, transposed: bool, nsplit: int) -> torch.Tensor:
    """Planes of W (N, K) as a B operand: rows = N, k = K; or of W^T (rows = K, k = N) when transposed."""
    global _PACK_JOIN
    if _PACK_JOIN is not None and torch.cuda.current_stream(w.device) != _PACK_JOIN:
        torch.cuda.current_stream(w.device).wait_stream(_PACK_JOIN)      # once per step: planes packed up front
        _PACK_JOIN = None
    key = (w.data_ptr(), tuple(w.shape), w._version, _WEIGHT_EPOCH, transposed, nsplit)
    hit = _WEIGHT_CACHE.get(key)
    if hit is None:
        if _PACK_LOG is not None:
            # detached: a recorded slice of a parameter must not keep the recording step's autograd graph alive
            _PACK_LOG.append((w.detach(), transposed, nsplit))
        n, k = w.shape
        wd = w.detach()
        planes = pack_split(wd, k, n, 1, k, nsplit) if transposed else pack_split(wd, n, k, k, 1, nsplit)
        if len(_WEIGHT_CACHE) > 512:
            _WEIGHT_CACHE.clear()
        # the entry keeps the weight's storage alive: a freed weight's address could otherwise be handed to a
        # new parameter of the same shape and hit this entry with stale planes
        hit = _WEIGHT_CACHE[key] = (planes, wd)
    return hit[0]


def colsum(x: torch.Tensor, out: torch.Tensor | None = None) -> torch.Tensor:
    """sum over the rows of a contiguous (rows, c) fp32 matrix (bias gradients).  Channel counts the row kernel does
    not cover (the 2- / 3- / 12-wide prediction heads) take the plain tensor reduction."""
    rows, c = x.shape
    if not (x.is_cuda and x.dtype == torch.float32 and x.is_contiguous() and rows > 0
            and 4 <= c <= 1024 and c % 4 == 0 and 256 % (c // 4) == 0):
        if out is None:
            return x.sum(dim=0)
        return torch.sum(x, dim=0, out=out)
    if out is None:
        out = torch.empty(c, dtype=torch.float32, device=x.device)
    scratch = torch.empty(132 * 4 * 2 * c, dtype=torch.float32, device=x.device)
    with torch.cuda.device(x.device):
        st = lib().coda_rows_colsum(_ll(rows), _i(c), ptr(x), ptr(out), ptr(scratch), stream_of(x))
    check(st, "rows_colsum")
    return out


class _Linear(torch.autograd.Function):
    """y = x W^T + b on the wgmma GEMM.  The activation is read IN PLACE as fp32 (gemm_a32: the bf16 split happens
    in the kernel's prologue); only the weight is packed (once per step, cached).  Backward: dX = dY W reuses the
    FORWARD weight planes as an MN-major operand (no transposed copy), dW = dY^T X runs on row-packed planes."""

    @staticmethod
    def forward(ctx, x, weight, bias, relu, nsplit):
        m, k = x.shape
        n = weight.shape[0]
        wp = _packed_weight(weight, False, nsplit)
        if not a32_ok(x):
            x = x.contiguous()
        if a32_ok(x) and n % 4 == 0:
            y = gemm_a32(x, wp, n, bias=bias, relu=relu)
        else:          # rows TMA cannot address in place (k or n not a multiple of 4: the 2-/3-wide heads): packed operands
            y = gemm_nt(_packed_rows(x, nsplit), wp, m, n, bias=bias, relu=relu)[0]
        ctx.save_for_backward(x, weight, y if relu else None, bias)
        ctx.has_bias, ctx.relu, ctx.nsplit = bias is not None, relu, nsplit
        return y

    @staticmethod
    def backward(ctx, dy):
        x, weight, y, bias = ctx.saved_tensors
        # gradients are held to a looser bar than the forward (5e-3 vs 1e-4): two planes suffice
        nsplit = min(ctx.nsplit, BACKWARD_NSPLIT)
        dy = dy.contiguous()
        m, k = x.shape
        n = weight.shape[0]
        dx = dw = db = None
        want_db = ctx.has_bias and ctx.needs_input_grad[2]
        # ReLU backward: dZ = [y > 0] * dY.  Both consumers of dZ are GEMMs whose A prologue can evaluate it from
        # (y, dY) while splitting the operand (the BatchNorm-backward prologue with scale 1, everything else 0), so
        # the masked gradient is never written: no compare / cast / multiply kernels in front of the GEMMs.
        pro = None
        if ctx.relu:
            if (a32_ok(dy) and a32_ok(y) and tn32_ok(dy) and tn32_ok(x) and k % 4 == 0 and nsplit == 2
                    and ctx.needs_input_grad[1]):
                one, zero = _unit_vectors(n, dy.device)
                pro = dict(scale=one, shift=zero, alpha=zero, beta=zero)
            else:
                dy = dy * (y > 0).to(dy.dtype)
        if pro is not None:
            if ctx.needs_input_grad[0]:
                dx = gemm_a32(y, _packed_weight(weight, False, ctx.nsplit), k, mode=A32_BN_BWD, a2=dy, b_mn=True,
                              nsplit=nsplit, **pro)
            sw, sb = _sink(weight), None
            if want_db:
                sb = _sink(bias)
                db = torch.empty(n, dtype=torch.float32, device=dy.device) if sb is None else sb
            dw = gemm_tn32(y, x, a_mode=A32_BN_BWD, a2=dy, a_scale=one, a_shift=zero, a_alpha=zero, a_beta=zero,
                           out=sw, colsum_out=db)
            if sw is not None:
                dw = _sunk(sw)
            if sb is not None:
                db = _sunk(sb)
            return dx, dw, db, None, None
        if ctx.needs_input_grad[0]:
            if a32_ok(dy) and k % 4 == 0:
                # dX (m, k) = dY (m, n) @ W (n, k): contraction over the ROWS of the forward weight planes
                dx = gemm_a32(dy, _packed_weight(weight, False, ctx.nsplit), k, b_mn=True, nsplit=nsplit)
            else:
                dx = gemm_nt(pack_split(dy, m, n, n, 1, nsplit), _packed_weight(weight, True, nsplit), m, k)[0]
        if ctx.needs_input_grad[1]:
            # dW (n, k) = sum_m dY[m, n] X[m, k]: contraction over the ROWS of both operands
            if tn32_ok(dy) and tn32_ok(x) and nsplit == 2:
                sw = _sink(weight) if k % 4 == 0 else None
                sb = None
                if want_db:      # the bias gradient (column sums of dY) comes out of the same pass
                    sb = _sink(bias)
                    db = torch.empty(n, dtype=torch.float32, device=dy.device) if sb is None else sb
                dw = gemm_tn32(dy, x, out=sw, colsum_out=db)    # fp32 rows in place, split inside the kernel
                if sw is not None:
                    dw = _sunk(sw)
                if sb is not None:
                    db = _sunk(sb)
                want_db = False
            else:
                dya = pack_split(dy, m, n, n, 1, nsplit)
                xa = _packed_rows(x, nsplit)     # shared by every layer that consumed the same x (the six heads)
                dw = gemm_tn(dya, xa, n, k)
        if want_db:
            sb = _sink(bias)
            db = colsum(dy, out=sb)
            if sb is not None:
                db = _sunk(sb)
        return dx, dw, db, None, None


_UNIT: dict = {}


def _unit_vectors(n: int, device):
    """(ones, zeros) of n floats rounded up to 128: the per-column coefficient vectors that turn the BatchNorm-backward prologue
    into a plain ReLU mask"""
    key = ((n + 127) // 128 * 128, device)
    hit = _UNIT.get(key)
    if hit is None:
        hit = _UNIT[key] = (torch.ones(key[0], dtype=torch.float32, device=device),
                            torch.zeros(key[0], dtype=torch.float32, device=device))
    return hit


_BIAS32: dict = {}


def _bias_fp32(bias):
    """fp32 copy of a (frozen, fp16) bias, cached: the epilogue adds the bias in fp32.  The entry keeps the
    source tensor alive so that its address cannot be recycled for another parameter while the entry exists."""
    key = (bias.data_ptr(), tuple(bias.shape), bias._version)
    hit = _BIAS32.get(key)
    if hit is None:
        if len(_BIAS32) > 256:
            _BIAS32.clear()
        hit = _BIAS32[key] = (bias.detach().float(), bias)
    return hit[0]


def linear(x: torch.Tensor, weight: torch.Tensor, bias=None, relu: bool = False, nsplit: int | None = None,
           quick_gelu: bool = False, residual: torch.Tensor | None = None):
    """y = x @ weight^T + bias over the last dim of x, on the wgmma GEMM (fp32 in / out, bf16
    split-operand accumulation); fp16 x / weight take the fp16 tensor-core path (inference only)."""
    _need_cuda(x, "linear")
    lead = x.shape[:-1]
    k = x.shape[-1]
    n = weight.shape[0]
    x2 = x.reshape(-1, k)
    if x2.dtype == torch.float16:
        assert weight.dtype == torch.float16 and k % 64 == 0, "fp16 path needs fp16 weights and K % 64 == 0"
        x2 = x2.contiguous()
        res2 = None
        if residual is not None:      # y = act(x W^T + b) + residual, added in the GEMM epilogue
            res2 = residual.reshape(-1, n)
            if res2.dtype != torch.float16 or res2.stride(1) != 1 or res2.stride(0) % 8 != 0 or n % 8 != 0:
                res2 = None
        y = gemm_nt(x2.view(1, 1, x2.shape[0], k), weight.detach().contiguous().view(1, 1, n, k), x2.shape[0], n,
                    bias=None if bias is None else _bias_fp32(bias), act=2 if quick_gelu else (1 if relu else 0),
                    out_dtype=torch.float16, residual=res2)[0]
        y = y.reshape(*lead, n)
        return y + residual if (residual is not None and res2 is None) else y
    if residual is not None:
        raise NotImplementedError("fused residual exists on the fp16 inference path only")
    if x2.stride(-1) != 1:
        x2 = x2.contiguous()
    w2 = weight.reshape(n, -1)
    y = _Linear.apply(x2.float(), w2, bias, relu, DEFAULT_NSPLIT if nsplit is None else nsplit)
    return y.reshape(*lead, n)


class Linear(torch.nn.Linear):
    """nn.Linear (same parameters / state-dict keys) running on the wgmma GEMM."""

    def forward(self, x):
        return linear(x, self.weight, self.bias)


# --------------------------------------------------------------------------- contrastive CE over a text matrix
class _TextCE(torch.autograd.Function):
    @staticmethod
    def forward(ctx, s, e, label, w, scale, c):
        rows, ld = s.shape
        d = e.shape[1]
        loss = torch.empty(rows, dtype=torch.float32, device=s.device)
        lse, inv = torch.empty_like(loss), torch.empty_like(loss)
        with torch.cuda.device(s.device):
            check(lib().coda_text_ce_fwd(_ll(rows), _i(c), _i(ld), _i(d), ptr(s), ptr(e), ptr(label), ptr(w),
                                         ptr(scale), ptr(loss), ptr(lse), ptr(inv), stream_of(s)), "text_ce_fwd")
        ctx.save_for_backward(s, e, label, w, scale, lse, inv)
        ctx.c = c
        return loss

    @staticmethod
    def backward(ctx, g):
        s, e, label, w, scale, lse, inv = ctx.saved_tensors
        rows, ld = s.shape
        d = e.shape[1]
        gc = _f32c(g)
        ds, dnorm = torch.empty_like(s), torch.empty_like(e)
        with torch.cuda.device(s.device):
            check(lib().coda_text_ce_bwd(_ll(rows), _i(ctx.c), _i(ld), _i(d), ptr(s), ptr(e), ptr(label), ptr(w),
                                         ptr(scale), ptr(lse), ptr(inv), ptr(gc), ptr(ds), ptr(dnorm), stream_of(s)),
                  "text_ce_bwd")
        return ds, dnorm, None, None, None, None


def text_ce_rows(s: torch.Tensor, e: torch.Tensor, label: torch.Tensor, w: torch.Tensor, scale: torch.Tensor,
                 c: int) -> torch.Tensor:
    """(rows,) w_r * CE(scale * S_r / (||e_r|| + 1e-32), label_r) from the raw logits S (rows, ld) = e T^T, columns
    [0, c) used, and the embeddings e (rows, d) they came from (include/coda_step.h coda_text_ce_fwd).  Gradients flow
    to S and, through the normalisation, to e; label -100 is ignored, other labels outside [0, c) give NaN."""
    _need_cuda(s, "text_ce_rows")
    assert s.dim() == 2 and e.dim() == 2 and s.shape[0] == e.shape[0] and s.shape[1] % 4 == 0 and 1 <= c <= s.shape[1]
    assert label.numel() == s.shape[0] and w.numel() == s.shape[0] and scale.numel() == 1
    assert not w.requires_grad and not scale.requires_grad
    return _TextCE.apply(_f32c(s), _f32c(e), label.to(torch.int64).contiguous(), _f32c(w).reshape(-1),
                         _f32c(scale.reshape(1)), c)


_PADDED_TEXT: dict = {}


def _rows_padded4(t: torch.Tensor) -> torch.Tensor:
    """(C, D) -> (pad4(C), D) with zero rows appended, cached: the padded text matrix is a GEMM B operand whose
    output rows TMA can store in place.  The entry keeps the source alive so that its address is not recycled."""
    c = t.shape[0]
    if c % 4 == 0:
        return t
    key = (t.data_ptr(), tuple(t.shape), t.stride(), t._version)
    hit = _PADDED_TEXT.get(key)
    if hit is None:
        if len(_PADDED_TEXT) > 8:
            _PADDED_TEXT.clear()
        padded = torch.zeros(((c + 3) // 4 * 4, t.shape[1]), dtype=torch.float32, device=t.device)
        padded[:c].copy_(t.detach())
        hit = _PADDED_TEXT[key] = (padded, t)
    return hit[0]


def text_contrastive_ce(e: torch.Tensor, text: torch.Tensor, label: torch.Tensor, w: torch.Tensor,
                        scale: torch.Tensor) -> torch.Tensor:
    """(rows,) weighted cross-entropy of the stage-2 contrastive loss over ONE shared text matrix (criterion.py
    loss_feat_seen_softmax_weakly_loss_with_novel_cate_confi): e (rows, D) the head's embeddings, text (C, D) the
    normalised text features (no gradient).  The raw logits e T^T come from the wgmma GEMM (ops.linear, whose backward
    gives dS T), the normalisation, scale, softmax and label pick from coda_text_ce_fwd / _bwd."""
    _need_cuda(e, "text_contrastive_ce")
    c = text.shape[0]
    s = linear(e, _rows_padded4(text.to(torch.float32)))
    return text_ce_rows(s, e, label, w, scale, c)


# --------------------------------------------------------------------------- decoder memory K / V bank
def pack_weights_concat(ws, nsplit: int) -> torch.Tensor:
    """Operand planes of the row-wise concatenation of the weights `ws` (each (n_i, k), row stride free):
    (nsplit, 1, sum n_i, kpad) -- each weight is packed straight into its rows of the shared buffer."""
    k = ws[0].shape[1]
    kpad = _pad64(k)
    total = sum(int(w.shape[0]) for w in ws)
    out = torch.empty((nsplit, 1, total, kpad), dtype=torch.bfloat16, device=ws[0].device)
    off = 0
    with torch.cuda.device(out.device):
        for w in ws:
            wd = w.detach()
            assert wd.dtype == torch.float32 and wd.stride(1) == 1 and wd.shape[1] == k
            st = lib().coda_pack_split_bf16_strided(
                _ll(wd.shape[0]), _i(k), _i(kpad), _ll(wd.stride(0)), _ll(1), ptr(wd), _f(1.0), _i(nsplit),
                ctypes.c_void_p(out.data_ptr() + 2 * off * kpad), _ll(total * kpad), stream_of(wd))
            check(st, "pack_split_bf16")
            off += int(wd.shape[0])
    return out


class KVBank:
    """Keys and values of the decoder's cross-attention for ALL layers at once.  The memory does not change across the
    decoder layers (reference models/transformer.py:97-143: every layer projects the same `memory + pos` / `memory`
    with its own weights), so the sixteen (16384 x 512 x 512) projections are two (16384 x 512 x 4096) GEMMs, and in the
    backward the sixteen input-gradient GEMMs + fourteen full-size gradient accumulations on `memory` are two GEMMs
    with a 4096-long contraction (the sum over layers happens in the tensor core's accumulator).

    Autograd wiring: `_KVBankFn` returns a one-element TOKEN; each layer's cross-attention (`_AttentionBank`) takes the
    token as a differentiable input and reads its K / V slice from the bank.  In the backward every attention node
    writes its dK / dV slice into the bank's gradient buffers in place and returns a zero for the token, so autograd
    runs `_KVBankFn.backward` exactly once, after the last layer that used the bank.  A layer whose output does not
    reach the loss runs no attention backward: `written` records the layers that did, and `_KVBankFn.backward` zeroes
    the column blocks of the others."""

    def __init__(self):
        self.k_all = self.v_all = self.dk_all = self.dv_all = None
        self.nlayers = self.e = 0
        self.written = set()


class _KVBankFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, mem_key, memory, bank, nsplit, *params):
        # params = (wk_0, bk_0, wv_0, bv_0, wk_1, ...): row slices of each layer's packed in-projection
        nl = len(params) // 4
        lk, b, e = memory.shape
        xk = mem_key.reshape(lk * b, e)
        xv = memory.reshape(lk * b, e)
        if not a32_ok(xk):
            xk = xk.contiguous()
        if not a32_ok(xv):
            xv = xv.contiguous()
        wk, bk, wv, bv = params[0::4], params[1::4], params[2::4], params[3::4]
        pk, pv = pack_weights_concat(wk, nsplit), pack_weights_concat(wv, nsplit)
        bank.k_all = gemm_a32(xk, pk, nl * e, bias=torch.cat([t.detach() for t in bk]))
        bank.v_all = gemm_a32(xv, pv, nl * e, bias=torch.cat([t.detach() for t in bv]))
        bank.nlayers, bank.e = nl, e
        bank.dk_all = bank.dv_all = None
        bank.written = set()
        ctx.bank, ctx.nsplit, ctx.shape = bank, nsplit, (lk, b, e)
        ctx.save_for_backward(xk, xv, pk, pv, *params)
        return torch.zeros(1, dtype=torch.float32, device=memory.device)

    @staticmethod
    def backward(ctx, dtoken):
        bank = ctx.bank
        xk, xv, pk, pv = ctx.saved_tensors[:4]
        params = ctx.saved_tensors[4:]
        lk, b, e = ctx.shape
        nl = bank.nlayers
        dk_all, dv_all = bank.dk_all, bank.dv_all
        assert dk_all is not None and dv_all is not None, "no cross-attention used the K / V bank"
        for i in range(nl):
            if i not in bank.written:      # this layer's output did not reach the loss: its dK / dV are zero
                dk_all[:, i * e: (i + 1) * e].zero_()
                dv_all[:, i * e: (i + 1) * e].zero_()
        ns = min(ctx.nsplit, BACKWARD_NSPLIT)
        d_key = d_mem = None
        if ctx.needs_input_grad[0]:
            d_key = gemm_a32(dk_all, pk, e, b_mn=True, nsplit=ns).view(lk, b, e)
        if ctx.needs_input_grad[1]:
            d_mem = gemm_a32(dv_all, pv, e, b_mn=True, nsplit=ns).view(lk, b, e)
        grads = []
        for i in range(nl):
            for x, d_all, w, bias in ((xk, dk_all, params[4 * i], params[4 * i + 1]),
                                      (xv, dv_all, params[4 * i + 2], params[4 * i + 3])):
                dy = d_all[:, i * e: (i + 1) * e]                   # (rows, e) view, row stride nl * e
                sw, sb = _sink(w), _sink(bias)
                db = torch.empty(e, dtype=torch.float32, device=dy.device) if sb is None else sb
                dw = gemm_tn32(dy, x, out=sw, colsum_out=db)
                grads += [dw if sw is None else _sunk(sw), db if sb is None else _sunk(sb)]
        bank.k_all = bank.v_all = bank.dk_all = bank.dv_all = None
        bank.written = set()
        return (d_key, d_mem, None, None, *grads)


class _AttentionBank(torch.autograd.Function):
    @staticmethod
    def forward(ctx, q, token, bank, idx, nhead, dropout_p, salt):
        from . import attention_launch

        lk_b, ne = bank.k_all.shape
        e = bank.e
        lq, b, _ = q.shape
        k = bank.k_all.view(lk_b // b, b, ne)[..., idx * e: (idx + 1) * e]
        v = bank.v_all.view(lk_b // b, b, ne)[..., idx * e: (idx + 1) * e]
        out, lse = attention_launch.forward(q, k, v, nhead, dropout_p, salt)
        ctx.save_for_backward(q, k, v, out, lse)
        ctx.bank, ctx.idx, ctx.nhead, ctx.dropout_p, ctx.salt = bank, idx, nhead, dropout_p, salt
        return out

    @staticmethod
    def backward(ctx, dout):
        from . import attention_launch

        q, k, v, out, lse = ctx.saved_tensors
        bank, idx, e = ctx.bank, ctx.idx, ctx.bank.e
        lk, b, _ = k.shape
        if bank.dk_all is None:          # a layer that runs this backward writes its whole block: no zero fill
            bank.dk_all = torch.empty((lk * b, bank.nlayers * e), dtype=torch.float32, device=q.device)
            bank.dv_all = torch.empty((lk * b, bank.nlayers * e), dtype=torch.float32, device=q.device)
        dk = bank.dk_all.view(lk, b, -1)[..., idx * e: (idx + 1) * e]
        dv = bank.dv_all.view(lk, b, -1)[..., idx * e: (idx + 1) * e]
        dq = torch.empty(q.shape, dtype=torch.float32, device=q.device)
        attention_launch.backward(q, k, v, out, dout, lse, ctx.nhead, ctx.dropout_p, ctx.salt, grads=(dq, dk, dv))
        bank.written.add(idx)
        return dq, torch.zeros(1, dtype=torch.float32, device=q.device), None, None, None, None, None


def attention_operand_planes() -> int:
    """bf16 planes on which the fused attention consumes q / k / v in the forward (and its producers compute them)"""
    from . import attention_launch

    return min(DEFAULT_NSPLIT, max(attention_launch.FORWARD_NSPLIT, BACKWARD_NSPLIT))


def kv_bank(mem_key: torch.Tensor, memory: torch.Tensor, attn_modules, nsplit: int | None = None):
    """-> (bank, token) for `attention_bank`; attn_modules: the layers' cross-attention modules (packed in_proj)"""
    _need_cuda(memory, "kv_bank")
    bank = KVBank()
    params = []
    for m in attn_modules:
        e = m.embed_dim
        w, bvec = m.in_proj_weight, m.in_proj_bias
        params += [w[e: 2 * e], bvec[e: 2 * e], w[2 * e:], bvec[2 * e:]]
    # the attention kernels consume K / V on attention_launch.FORWARD_NSPLIT planes: projecting them more precisely
    # than that is work whose result the consumer rounds away
    if nsplit is None:
        nsplit = attention_operand_planes()
    token = _KVBankFn.apply(mem_key, memory, bank, nsplit, *params)
    return bank, token


def attention_bank(q: torch.Tensor, bank: KVBank, token: torch.Tensor, idx: int, nhead: int, dropout_p: float,
                   training: bool) -> torch.Tensor:
    from . import attention_launch

    p = float(dropout_p) if training else 0.0
    return _AttentionBank.apply(q, token, bank, idx, nhead, p, attention_launch.next_salt() if p > 0.0 else 0)


def kv_bank_applicable(memory: torch.Tensor, attn_modules) -> bool:
    if not (memory.is_cuda and memory.dtype == torch.float32 and len(attn_modules) > 1):
        return False
    e = attn_modules[0].embed_dim
    hd = e // attn_modules[0].num_heads
    return hd in (64, 128) and e % 64 == 0 and all(m.embed_dim == e and m.num_heads == attn_modules[0].num_heads
                                                    for m in attn_modules)
