"""One data-parallel training step: the body of the reference's training loop
(engine.py:120-165 `train_one_epoch`: H2D of the batch, forward, criterion,
backward with the gradient all-reduce, clip_grad_norm_, AdamW) as a reusable
object, laid out for the H100:

  * all trainable parameters live in ONE flat fp32 buffer and their gradients in another, ordered by
    the moment their gradient becomes final during the backward (measured once, on a probe pass), so
    that the data-parallel exchange is a handful of NCCL all-reduces over contiguous ranges, each
    launched on NCCL's stream the moment its range is final -- the exchange of the prediction heads
    and the upper decoder layers overlaps the rest of the backward, and only the last, small range
    (encoder + set abstraction, ~7 MB) is exposed.  The reference's DDP does the same with 25 MB buckets;
  * the global-norm clip and AdamW are two kernels over the flat buffers (`FlatAdamW`,
    csrc/step_kernels.cu: one deterministic norm reduction, one update pass with the clip coefficient,
    bias corrections and the 1/world scaling folded in).  Parameter groups of the reference
    (optimizer.py:4-36: `filter_biases_wd` -> no decay on 1-D parameters and biases) are per-range
    weight-decay values; parameters that never receive a gradient are left out of the update, as
    torch's AdamW skips `grad is None` parameters;
  * the caller's torch.optim.AdamW can be adopted (`TrainStep(optimizer=...)`): its moments and step count are
    imported into the flat buffers and its per-parameter state becomes views of them, so the reference's
    save_checkpoint / resume_if_possible carry the optimizer state through unchanged;
  * rank 0's parameters and buffers are broadcast before the first step (what DDP's constructor does;
    the reference seeds every rank differently, main.py:982-985);
  * BatchNorm statistics stay per GPU (no SyncBatchNorm): the step's only other collective is the
    4-byte box-count all-reduce of the criterion;
  * the batch is copied from pinned host memory on the compute stream and the loss is left on the
    device: the caller decides when to synchronise.
"""
from __future__ import annotations

import ctypes
import math
import weakref

import torch
import torch.distributed as dist

from . import ops
from .utils.dist import get_world_size, is_distributed, is_primary


def adjust_learning_rate(args, optimizer, curr_epoch: float) -> float:
    """Cosine schedule with linear warm-up (reference engine.py:33-55)."""
    lr = _lr_at(args, curr_epoch)
    for group in optimizer.param_groups:
        group["lr"] = lr
    return lr


def _lr_at(a, curr_epoch: float) -> float:
    if curr_epoch <= a.warm_lr_epochs and a.warm_lr_epochs > 0:
        return a.warm_lr + (curr_epoch / a.warm_lr_epochs) * (a.base_lr - a.warm_lr)
    return a.final_lr + 0.5 * (a.base_lr - a.final_lr) * (1 + math.cos(math.pi * curr_epoch / a.max_epoch))


def allreduce_mean_(flat: torch.Tensor) -> torch.Tensor:
    """Mean over ranks of one flat tensor (NCCL over NVLink on GPUs)."""
    if is_distributed() and get_world_size() > 1:
        dist.all_reduce(flat)
        flat.div_(get_world_size())
    return flat


def broadcast_module_state(module: torch.nn.Module, src: int = 0) -> None:
    """Every parameter and buffer of `module` from rank `src` (DistributedDataParallel's constructor does this;
    without it, ranks that were seeded differently would average the gradients of DIFFERENT models)."""
    if not (is_distributed() and get_world_size() > 1):
        return
    with torch.no_grad():
        for t in list(module.parameters()) + list(module.buffers()):
            dist.broadcast(t.data, src)


class FlatParameters:
    """Re-homes every trainable parameter of `module` (and its gradient) into one contiguous fp32 buffer each.
    `order` (a permutation of the trainable parameters) fixes the layout; default = registration order."""

    ALIGN = 64   # elements

    def __init__(self, module: torch.nn.Module, order=None):
        named = [(n, p) for n, p in module.named_parameters() if p.requires_grad]
        params = [p for _, p in named] if order is None else list(order)
        assert params and all(p.dtype == torch.float32 for p in params)
        assert {id(p) for p in params} == {id(p) for _, p in named}, "order must be a permutation of the parameters"
        name_of = {id(p): n for n, p in named}
        dev = params[0].device
        # every parameter starts on a 256-byte boundary: kernels read per-channel vectors (BatchNorm / LayerNorm
        # scales, biases) with 16-byte loads and TMA addresses weight rows; the few padding elements stay zero
        pad = lambda n: (n + self.ALIGN - 1) // self.ALIGN * self.ALIGN  # noqa: E731
        total = sum(pad(p.numel()) for p in params)
        self.flat_param = torch.nn.Parameter(torch.zeros(total, dtype=torch.float32, device=dev))
        self.flat_grad = torch.zeros(total, dtype=torch.float32, device=dev)
        self.offsets, self.names = [], []
        off = 0
        with torch.no_grad():
            for p in params:
                n = p.numel()
                self.flat_param.data[off:off + n].copy_(p.data.reshape(-1))
                p.data = self.flat_param.data[off:off + n].view_as(p)
                p.grad = self.flat_grad[off:off + n].view_as(p)
                self.offsets.append(off)
                self.names.append(name_of[id(p)])
                off += pad(n)
        self.flat_param.grad = self.flat_grad
        self.params = params

    def zero_grad(self):
        self.flat_grad.zero_()

    def nbytes(self) -> int:
        return self.flat_grad.numel() * 4


class BucketedAllReduce:
    """Mean of the flat gradient over ranks as `nbuckets` all-reduces over contiguous ranges, each started (async,
    on the process group's stream) the moment its range has received all of its gradient writes -- counted as
    EVENTS: a post-accumulate hook of a parameter that autograd accumulates, or a direct write of a backward kernel
    into the flat buffer (ops.GradSink).  The number of events per range is either the number of active parameters
    (default) or measured on a calibration pass (`calibrate`).  `finish()` starts whatever is left and joins.  With
    the flat buffer laid out in gradient-ready order the ranges complete front to back."""

    def __init__(self, flat: FlatParameters, nbuckets: int = 4, active=None):
        self.flat, self.world = flat, get_world_size()
        self.enabled = is_distributed() and self.world > 1
        n = len(flat.params)
        active = [True] * n if active is None else list(active)
        total = flat.flat_grad.numel()
        # bucket boundaries at parameter boundaries, ~equal element counts
        bounds, target = [0], total / max(nbuckets, 1)
        for i in range(n - 1):
            if flat.offsets[i + 1] >= target * len(bounds) and len(bounds) < nbuckets:
                bounds.append(flat.offsets[i + 1])
        bounds.append(total)
        self.ranges = list(zip(bounds[:-1], bounds[1:]))
        self._starts = [lo for lo, _ in self.ranges]
        self.bucket_of = [self.bucket_at(flat.offsets[i]) for i in range(n)]
        self.expected = [0] * len(self.ranges)
        for i in range(n):
            if active[i]:
                self.expected[self.bucket_of[i]] += 1
        self.count = [0] * len(self.ranges)
        self.launched = [False] * len(self.ranges)
        self.works = []
        self.calibrating = False
        self._avg = dist.ReduceOp.AVG if (self.enabled and dist.get_backend() == "nccl") else None
        if self.enabled:
            for i, p in enumerate(flat.params):
                p.register_post_accumulate_grad_hook(self._make_hook(self.bucket_of[i]))

    def bucket_at(self, elem_offset: int) -> int:
        import bisect

        return bisect.bisect_right(self._starts, elem_offset) - 1

    def _make_hook(self, b):
        def hook(_param):
            self.event(b)
        return hook

    def event(self, b: int):
        self.count[b] += 1
        if not self.calibrating and self.count[b] == self.expected[b]:
            self._launch(b)

    def event_at(self, elem_offset: int):
        """a backward kernel wrote the gradient region that starts at `elem_offset` of the flat buffer"""
        if self.enabled:
            self.event(self.bucket_at(elem_offset))

    def calibrate(self, run_backward):
        """Counts the gradient events per range on one forward/backward (`run_backward()`)."""
        self.start()
        self.calibrating = True
        try:
            run_backward()
        finally:
            self.calibrating = False
        self.expected = list(self.count)
        self.start()

    def _launch(self, b):
        if self.launched[b] or not self.enabled:
            return
        self.launched[b] = True
        lo, hi = self.ranges[b]
        if hi > lo:
            view = self.flat.flat_grad[lo:hi]
            self.works.append((dist.all_reduce(view, op=self._avg or dist.ReduceOp.SUM, async_op=True), view))

    def start(self):
        self.count = [0] * len(self.ranges)
        self.launched = [False] * len(self.ranges)
        self.works = []

    def finish(self):
        if not self.enabled:
            return
        for b in range(len(self.ranges)):
            self._launch(b)
        for work, view in self.works:
            work.wait()
            if self._avg is None:
                view.div_(self.world)
        self.works = []


class FlatAdamW:
    """clip_grad_norm_ + torch.optim.AdamW on the flat buffers: coda_grad_norm + coda_adamw_update
    (include/coda_step.h).  `weight_decay[i]` / `active[i]` per parameter of `flat`."""

    CHUNK = 16384

    class _Chunk(ctypes.Structure):
        _fields_ = [("offset", ctypes.c_longlong), ("len", ctypes.c_int), ("weight_decay", ctypes.c_float)]

    def __init__(self, flat: FlatParameters, lr: torch.Tensor, weight_decay, active=None, betas=(0.9, 0.999),
                 eps: float = 1e-8, max_norm: float = 0.0):
        self.flat, self.lr, self.betas, self.eps, self.max_norm = flat, lr, betas, eps, float(max_norm)
        dev = flat.flat_param.device
        self.exp_avg = torch.zeros_like(flat.flat_grad)
        self.exp_avg_sq = torch.zeros_like(flat.flat_grad)
        self.state = torch.zeros(8, dtype=torch.float32, device=dev)   # step, norm, clip coef, bc1, sqrt(bc2)
        L = ops.lib()
        L.coda_grad_norm_scratch_floats.restype = ctypes.c_longlong
        self.scratch = torch.empty(int(L.coda_grad_norm_scratch_floats()), dtype=torch.float32, device=dev)
        self.active = [True] * len(flat.params) if active is None else list(active)
        raw, self.nchunks = self._chunk_table(weight_decay)
        self.chunks = raw.to(dev)

    def _chunk_table(self, weight_decay):
        """(offset, len, weight_decay) of every CHUNK-element piece of the active parameters, as raw bytes."""
        f = self.flat
        n = len(f.params)
        wds = [float(weight_decay)] * n if not isinstance(weight_decay, (list, tuple)) else list(weight_decay)
        chunks = []
        for i, p in enumerate(f.params):
            if not self.active[i]:
                continue
            off, left = f.offsets[i], p.numel()
            while left > 0:
                ln = min(left, self.CHUNK)
                chunks.append((off, ln, wds[i]))
                off += ln
                left -= ln
        arr = (self._Chunk * max(len(chunks), 1))()
        for k, (off, ln, wd) in enumerate(chunks):
            arr[k].offset, arr[k].len, arr[k].weight_decay = off, ln, wd
        return torch.frombuffer(bytearray(bytes(arr)), dtype=torch.uint8).clone(), len(chunks)

    def set_weight_decay(self, weight_decay):
        """New per-parameter weight decay, written into the chunk table in place (a captured step reads it there)."""
        raw, _ = self._chunk_table(weight_decay)
        self.chunks.copy_(raw)

    def step(self, grad_scale: float = 1.0):
        f = self.flat
        L = ops.lib()
        _f, _i, _ll, ptr = ctypes.c_float, ctypes.c_int, ctypes.c_longlong, ops.ptr
        with torch.cuda.device(f.flat_param.device):
            ops.check(L.coda_grad_norm(_ll(f.flat_grad.numel()), ptr(f.flat_grad), _f(grad_scale), _f(self.max_norm),
                                       _f(self.betas[0]), _f(self.betas[1]), ptr(self.scratch), ptr(self.state),
                                       ops.stream_of(f.flat_grad)), "grad_norm")
            ops.check(L.coda_adamw_update(_i(self.nchunks), ptr(self.chunks), ptr(f.flat_param.data), ptr(f.flat_grad),
                                          ptr(self.exp_avg), ptr(self.exp_avg_sq), ptr(self.lr), _f(grad_scale),
                                          _f(self.betas[0]), _f(self.betas[1]), _f(self.eps), ptr(self.state),
                                          ops.stream_of(f.flat_grad)), "adamw_update")

    @property
    def grad_norm(self) -> torch.Tensor:
        """Total gradient norm of the last step (device scalar; what clip_grad_norm_ returns)."""
        return self.state[1]

    def state_tensors(self):
        return [self.exp_avg, self.exp_avg_sq, self.state]


def _no_decay(name: str, p: torch.Tensor) -> bool:
    """optimizer.py:19: `len(param.shape) == 1 or name.endswith("bias")`"""
    return p.dim() == 1 or name.endswith("bias")


# ------------------------------------------------------------------ torch.optim.AdamW state <-> the flat layout
# A torch optimizer's state_dict numbers its parameters in param_groups order; `index[i]` is that number for the i-th
# parameter of a FlatParameters layout.  FlatAdamW keeps one step count for every parameter it updates (the active
# ones); the moments of every parameter, inactive ones included, sit in its flat buffers at the parameter's offset.

def _names(names, idx, most: int = 4) -> str:
    picked = [names[i] for i in idx]
    return ", ".join(picked[:most]) + (f" and {len(picked) - most} more" if len(picked) > most else "")


def adamw_flat_index(optimizer, flat: FlatParameters) -> list:
    """`index[i]`: the state_dict number of `flat.params[i]` in `optimizer`.  ValueError unless `optimizer` is a
    torch.optim.AdamW over exactly the trainable parameters of the layout, each once."""
    if not isinstance(optimizer, torch.optim.AdamW):
        raise ValueError(f"TrainStep adopts a torch.optim.AdamW, not a {type(optimizer).__name__}")
    ordered = [p for g in optimizer.param_groups for p in g["params"]]
    number = {}
    for k, p in enumerate(ordered):
        number.setdefault(id(p), k)
    mine = {id(p) for p in flat.params}
    missing = [i for i, p in enumerate(flat.params) if id(p) not in number]
    foreign = [k for k, p in enumerate(ordered) if id(p) not in mine]
    if missing or foreign or len(number) != len(ordered):
        raise ValueError("the optimizer's parameters must be exactly the model's trainable parameters: "
                         + "; ".join(s for s in (
                             f"not in the optimizer: {_names(flat.names, missing)}" if missing else "",
                             f"{len(foreign)} optimizer parameters that are not trainable parameters of the model "
                             f"(state_dict numbers {foreign[:8]})" if foreign else "",
                             f"{len(ordered) - len(number)} listed twice" if len(number) != len(ordered) else "") if s))
    return [number[id(p)] for p in flat.params]


_ADAMW_RULE_OPTIONS = ("amsgrad", "maximize", "differentiable")


def adamw_hyperparameters(param_groups, index: list):
    """(weight decay of each parameter of the layout, betas, eps) from the optimizer's param_groups.  ValueError for
    an option that changes the update rule, and for betas / eps that differ between groups (the flat step has one
    of each)."""
    for g_i, g in enumerate(param_groups):
        bad = [k for k in _ADAMW_RULE_OPTIONS if g.get(k, False)]
        if not g.get("decoupled_weight_decay", True):
            bad.append("decoupled_weight_decay=False")
        if bad:
            raise ValueError(f"param_groups[{g_i}] sets {', '.join(bad)}: the flat step implements plain AdamW")
    rules = {(tuple(float(b) for b in g["betas"]), float(g["eps"])) for g in param_groups}
    if len(rules) != 1:
        raise ValueError(f"param_groups differ in betas / eps {sorted(rules)}: the flat step takes one of each")
    (betas, eps), = rules
    decay = [float(g["weight_decay"]) for g in param_groups for _ in g["params"]]
    return [decay[k] for k in index], betas, eps


def adamw_state_to_flat(state: dict, index: list, flat: FlatParameters, active: list, exp_avg: torch.Tensor,
                        exp_avg_sq: torch.Tensor):
    """Copies the per-parameter moments of `state` (a state_dict's "state": number -> {"step", "exp_avg",
    "exp_avg_sq"}) into the flat moment buffers, zero elsewhere.  Returns (the active parameters' common step count,
    0 without state; {i: step} of the inactive parameters that have state, carried unchanged).  Everything is checked
    before anything is written: ValueError for a state entry without a step count, for moments that do not fit their
    parameter, for active parameters with different step counts, or for state on some active parameters but not on
    others.  The moments may be views of the flat buffers themselves (an optimizer that reloads its own state_dict
    in memory keeps them: torch's load_state_dict does not copy a tensor that is already on the right device)."""
    steps = {}
    for i, p in enumerate(flat.params):
        st = state.get(index[i])
        if not st:
            continue
        if "step" not in st:
            raise ValueError(f"optimizer state of {flat.names[i]} has no step count")
        for key in ("exp_avg", "exp_avg_sq"):
            if key not in st or tuple(st[key].shape) != tuple(p.shape):
                got = tuple(st[key].shape) if key in st else "none"
                raise ValueError(f"optimizer state of {flat.names[i]}: {key} {got} does not fit the parameter "
                                 f"{tuple(p.shape)}")
        steps[i] = float(st["step"])
    act = [i for i, a in enumerate(active) if a]
    with_state = [i for i in act if i in steps]
    if with_state and len(with_state) != len(act):
        without = [i for i in act if i not in steps]
        raise ValueError("the optimizer holds state for some of the parameters that receive a gradient but not for "
                         f"others (with: {_names(flat.names, with_state)}; without: {_names(flat.names, without)}); "
                         "the flat step keeps one step count for all of them")
    counts = sorted({steps[i] for i in with_state})
    if len(counts) > 1:
        first = {s: next(i for i in with_state if steps[i] == s) for s in counts}
        raise ValueError("the parameters that receive a gradient have different AdamW step counts ("
                         + ", ".join(f"{flat.names[i]}: {s:g}" for s, i in first.items())
                         + "); the flat step keeps one step count for all of them")
    own = {exp_avg.untyped_storage().data_ptr(), exp_avg_sq.untyped_storage().data_ptr()}

    def source(t):      # read before the buffers are cleared
        return t.clone() if t.untyped_storage().data_ptr() in own else t

    with torch.no_grad():
        sources = {i: (source(state[index[i]]["exp_avg"]), source(state[index[i]]["exp_avg_sq"])) for i in steps}
        exp_avg.zero_()
        exp_avg_sq.zero_()
        for i, (m, v) in sources.items():
            off, n = flat.offsets[i], flat.params[i].numel()
            exp_avg[off:off + n].copy_(m.reshape(-1))
            exp_avg_sq[off:off + n].copy_(v.reshape(-1))
    return (counts[0] if counts else 0.0), {i: s for i, s in steps.items() if not active[i]}


def adamw_state_from_flat(param_groups, index: list, flat: FlatParameters, active: list, exp_avg: torch.Tensor,
                          exp_avg_sq: torch.Tensor, step: float, carried: dict) -> dict:
    """The inverse: a state_dict's "state" whose moments are VIEWS of the flat buffers.  Active parameters have state
    once `step` > 0 (torch creates it on the first update); inactive ones where `carried` has their step.  `step` is
    a float32 tensor on the CPU, or on the parameter's device for capturable / fused groups, as torch keeps it."""
    on_device = [bool(g.get("capturable", False) or g.get("fused", False)) for g in param_groups for _ in g["params"]]
    state = {}
    for i, p in enumerate(flat.params):
        s = step if active[i] else carried.get(i)
        if s is None or (active[i] and s <= 0):
            continue
        off, n = flat.offsets[i], p.numel()
        state[index[i]] = {
            "step": torch.tensor(float(s), dtype=torch.float32, device=p.device if on_device[index[i]] else "cpu"),
            "exp_avg": exp_avg[off:off + n].view_as(p),
            "exp_avg_sq": exp_avg_sq[off:off + n].view_as(p)}
    return dict(sorted(state.items()))


def bind_adamw_state(optimizer, index: list, flat: FlatParameters, active: list, exp_avg: torch.Tensor,
                     exp_avg_sq: torch.Tensor, step: float, carried: dict) -> None:
    """Replaces the optimizer's per-parameter state by `adamw_state_from_flat`: its state_dict() then reads the flat
    buffers."""
    state = adamw_state_from_flat(optimizer.param_groups, index, flat, active, exp_avg, exp_avg_sq, step, carried)
    for k, p in enumerate(p for g in optimizer.param_groups for p in g["params"]):
        if k in state:
            optimizer.state[p] = state[k]
        else:
            optimizer.state.pop(p, None)


# adopted optimizer -> (the TrainStep that holds it, the handles of its state_dict / load_state_dict hooks)
_ADOPTED = weakref.WeakKeyDictionary()


def adamw_numbered_state(optimizer) -> dict:
    """optimizer.state keyed by state_dict number (what state_dict() packs, without running its hooks)."""
    ordered = [p for g in optimizer.param_groups for p in g["params"]]
    return {k: optimizer.state[p] for k, p in enumerate(ordered) if optimizer.state.get(p)}


class TrainStep:
    """The step runs either eagerly or, after `capture()`, as ONE CUDA graph: the ~6 000 kernel
    launches of a step (8 decoder layers x many small ops) are launch-bound on the host otherwise.
    Everything inside the step is static-shaped and free of host synchronisation (the criterion
    matches on the GPU); the only per-step host work -- the learning rate, the random choice of the
    32 boxes per scene that get CLIP crops, the batch upload -- happens before the replay and is
    handed over through persistent device buffers.

    Preparation (first call or `capture`): one probe forward/backward on the first batch records which
    parameters receive a gradient and in which order; the flat buffers are laid out in that order, rank 0's
    state is broadcast, the optimizer is built.  The probe and the graph warm-up leave NO trace: parameters,
    optimizer state, BatchNorm buffers and the dropout counter are restored afterwards."""

    def __init__(self, args, model, criterion, device, nbuckets: int = 4, sync_bn: bool | None = None,
                 optimizer: torch.optim.AdamW | None = None):
        """sync_bn: synchronise BatchNorm statistics over the ranks (the reference converts to SyncBatchNorm when
        ngpus > 1, main.py:993).  Default (None -> args.sync_bn, else False): per-GPU statistics and exactly one
        gradient all-reduce per step, as the north-star asks; True adds one small all-reduce per BatchNorm layer
        and direction (DESIGN.md section 7) and makes N ranks x B scenes equal one rank x N*B scenes.

        optimizer: the caller's torch.optim.AdamW over the model's trainable parameters (the reference's
        build_optimizer), possibly holding a loaded state.  `prepare` adopts it: its moments and step count become
        the flat step's, its per-group weight decay, betas and eps replace the values derived from `args` (the
        learning rate still follows the schedule), and its per-parameter moments become views of the flat buffers,
        so that its state_dict() is what the step runs with and a later load_state_dict() is what it runs on.  The
        optimizer's hooks keep this step alive as long as the optimizer lives; a step that adopts the same optimizer
        later takes it over."""
        self.args, self.model, self.criterion, self.device = args, model, criterion, device
        self.adamw = optimizer
        self.world = get_world_size()
        self.sync_bn = bool(getattr(args, "sync_bn", False) if sync_bn is None else sync_bn)
        ops.set_bn_sync(self.sync_bn and self.world > 1)
        self.nbuckets = nbuckets
        self.lr = torch.tensor(float(args.base_lr), device=device)
        self.flat = None
        self.optimizer = None
        self.reducer = None
        self.graph = None
        self.graph_branch = None
        self.launches_per_step = None
        self.static_batch = None
        self.static_out = None
        self._sel_host = None
        self._nsel = getattr(model, "distillation_box_num", 32)
        self._pack_requests = None          # (weight, transposed, nsplit) planes a step asks for; recorded on step one
        self._pack_stream = None

    # ------------------------------------------------------------------ host-side per-step work
    def to_device(self, batch_host: dict) -> dict:
        """engine.py:125-129: every tensor of the collated batch to the device (async from pinned memory)."""
        return {k: (v.to(self.device, non_blocking=True) if isinstance(v, torch.Tensor) else v)
                for k, v in batch_host.items()}

    def _set_lr(self, curr_epoch: float):
        lr = _lr_at(self.args, curr_epoch)
        self.lr.fill_(lr)
        return lr

    def _draw_selection(self, bsz: int):
        """Host RNG draw of the CLIP-crop boxes for the coming step -> persistent device buffer."""
        m = self.model
        if not getattr(m, "if_with_clip_train", False):
            return
        sel = torch.from_numpy(m.draw_box_selection(bsz))
        if self._sel_host is None or self._sel_host.shape != sel.shape:
            self._sel_host = torch.empty_like(sel).pin_memory()
            m.external_selection = torch.empty_like(sel, device=self.device)
        self._sel_host.copy_(sel)
        m.external_selection.copy_(self._sel_host, non_blocking=True)

    def _branch(self, curr_epoch: float):
        """Python-level branches of the model's forward that depend on the epoch: a captured graph is valid for
        one value of this key only."""
        m = self.model
        late = int(curr_epoch) >= 540
        discover = (getattr(m, "online_nms_update_save_novel_label_clip_driven_with_cate_confidence", False)
                    and int(curr_epoch) % max(int(getattr(m, "online_nms_update_save_epoch", 1)), 1) == 0)
        return (late and getattr(m, "if_select_box_by_objectness", False), late and getattr(m, "if_keep_box", False),
                discover)

    # ------------------------------------------------------------------ state that a dry run must not change
    def _volatile(self):
        from . import attention_launch

        ts = [b for b in self.model.buffers()] + [b for b in self.criterion.buffers()]
        ts.append(attention_launch.seed_counter(self.device))
        if self.flat is not None:
            ts.append(self.flat.flat_param.data)
        if self.optimizer is not None:
            ts += self.optimizer.state_tensors()
        return ts

    def _snapshot(self):
        return [(t, t.clone()) for t in self._volatile()]

    @staticmethod
    def _restore(snap):
        with torch.no_grad():
            for t, saved in snap:
                t.copy_(saved)

    def _drop_dry_run_pseudo_labels(self):
        """Stage-2 discovery rows of a probe or warm-up step are not a step's result: they are dropped instead of
        being written to the scenes' files (the next discovery step would flush them, inside a graph capture too)."""
        if getattr(self.model, "_pending_pseudo", None) is not None:
            self.model._pending_pseudo = None

    # ------------------------------------------------------------------ preparation
    def prepare(self, example_batch: dict):
        if self.flat is not None:
            return self
        broadcast_module_state(self.model)          # DDP-constructor semantics (rank 0 wins)
        named = [(n, p) for n, p in self.model.named_parameters() if p.requires_grad]
        order, fired = [], set()

        def hook(p):
            if id(p) not in fired:
                fired.add(id(p))
                order.append(p)

        handles = [p.register_post_accumulate_grad_hook(hook) for _, p in named]
        sink = ops.GradSink()            # count mode: which parameter regions does the backward write, how often
        sink.watch([p for _, p in named])
        ops.set_grad_sink(sink)
        snap = self._snapshot()
        for _, p in named:
            p.grad = None

        def dry_run():
            self._draw_selection(example_batch["point_clouds"].shape[0])
            outputs = self.model(example_batch, curr_epoch=0)
            loss, _ = self.criterion(outputs, dict(example_batch))
            loss.backward()

        dry_run()
        for h in handles:
            h.remove()
        self._restore(snap)
        self._drop_dry_run_pseudo_labels()
        inactive = [p for _, p in named if id(p) not in fired]
        if is_distributed() and self.world > 1:
            # every rank must lay the buffers out identically: compare the ready order with rank 0's
            index = {id(p): i for i, (_, p) in enumerate(named)}
            mine = torch.tensor([index[id(p)] for p in order] + [-1] * len(inactive), device=self.device)
            ref = mine.clone()
            dist.broadcast(ref, 0)
            if not torch.equal(mine, ref):
                raise RuntimeError("gradient-ready order differs between ranks: the model's graph is not the same "
                                   "on every rank")
        for _, p in named:
            p.grad = None
        self.flat = FlatParameters(self.model, order=order + inactive)
        active = [True] * len(order) + [False] * len(inactive)
        a = self.args
        wds = []
        for name, p in zip(self.flat.names, self.flat.params):
            wds.append(0.0 if (getattr(a, "filter_biases_wd", False) and _no_decay(name, p)) else float(a.weight_decay))
        self.optimizer = FlatAdamW(self.flat, self.lr, wds, active, max_norm=float(a.clip_gradient))
        if self.adamw is not None:
            # one step at a time holds an optimizer: a step that adopts it later takes it over, from the step count
            # the holder has reached (the optimizer's own copy is refreshed only when a state_dict is taken)
            holder = _ADOPTED.get(self.adamw)
            if holder is not None:
                holder[0]._export()
            self._adopt_on_every_rank()
            if holder is not None:
                for h in holder[1]:
                    h.remove()
            _ADOPTED[self.adamw] = (self, (self.adamw.register_state_dict_pre_hook(lambda _opt: self._export()),
                                           self.adamw.register_load_state_dict_post_hook(self._reload)))
        self.reducer = BucketedAllReduce(self.flat, self.nbuckets, active)
        self.inactive_names = [n for n, f in zip(self.flat.names, active) if not f]
        # from now on the backward kernels write single-use parameter gradients straight into flat_grad
        flat_off = {id(p): off for p, off in zip(self.flat.params, self.flat.offsets)}
        sink.arm(self.flat.flat_param, self.flat.flat_grad, [flat_off[id(p)] * 4 for _, p in named])
        sink.on_write = self.reducer.event_at
        self.sink = sink
        ops.invalidate_weight_cache()
        if self.reducer.enabled:
            # gradient events per all-reduce range (hooks + direct writes), measured once
            snap = self._snapshot()
            self.flat.zero_grad()
            self.reducer.calibrate(dry_run)
            self._restore(snap)
            self.flat.zero_grad()
            ops.invalidate_weight_cache()
        return self

    # ------------------------------------------------------------------ the caller's AdamW
    def _adopt(self):
        """The adopted optimizer's options, moments and step count -> FlatAdamW; then its state is bound to the flat
        buffers.  Every check runs before FlatAdamW changes."""
        fa, opt = self.optimizer, self.adamw
        index = adamw_flat_index(opt, self.flat)
        wds, betas, eps = adamw_hyperparameters(opt.param_groups, index)
        if self.graph is not None and (betas, eps) != (tuple(fa.betas), fa.eps):
            raise ValueError(f"betas {betas} / eps {eps} differ from the captured step's {tuple(fa.betas)} / {fa.eps}: "
                             "load the optimizer state before capture")
        step, carried = adamw_state_to_flat(adamw_numbered_state(opt), index, self.flat, fa.active, fa.exp_avg,
                                            fa.exp_avg_sq)
        fa.state[0].fill_(step)
        fa.set_weight_decay(wds)
        fa.betas, fa.eps = betas, eps
        self._adamw_index, self._carried = index, carried
        self._adamw_groups = [{k: v for k, v in g.items() if k not in ("params", "lr")} for g in opt.param_groups]
        self._export(step)

    def _export(self, step: float | None = None):
        """Binds the adopted optimizer's per-parameter state to the flat buffers.  Without `step`, the step count is
        read from the device: the one device -> host read of a state_dict(), none per step."""
        fa = self.optimizer
        if step is None:
            step = float(fa.state[0])
        bind_adamw_state(self.adamw, self._adamw_index, self.flat, fa.active, fa.exp_avg, fa.exp_avg_sq, step,
                         self._carried)

    def _reload(self, opt):
        """After optimizer.load_state_dict: import the loaded state in place (a captured step reads the flat buffers,
        no re-capture).  If it is refused, the optimizer goes back to describing the state the step runs with."""
        try:
            self._adopt()
        except ValueError:
            for g, kept in zip(opt.param_groups, self._adamw_groups):
                g.update(kept)
            self._export()
            raise

    def _adopt_on_every_rank(self):
        """`_adopt` at prepare.  With several ranks, all of them learn whether any rank refused its optimizer state
        before rank 0's state is broadcast: a refusal on one rank alone would leave the others waiting in the
        broadcast."""
        err = None
        try:
            self._adopt()
        except ValueError as e:
            err = e
        if is_distributed() and self.world > 1:
            refused = torch.zeros(self.world, device=self.device)
            refused[dist.get_rank()] = float(err is not None)
            dist.all_reduce(refused)
            ranks = refused.nonzero().flatten().tolist()
            if ranks:
                raise err or ValueError(f"the optimizer state was refused on rank(s) {ranks}")
            self._broadcast_adopted()
        elif err is not None:
            raise err

    def _broadcast_adopted(self):
        """Rank 0's moments and step counts on every rank (DDP-constructor semantics, as for the parameters)."""
        fa = self.optimizer
        for t in (fa.exp_avg, fa.exp_avg_sq, fa.state):
            dist.broadcast(t, 0)
        inactive = [i for i, f in enumerate(fa.active) if not f]
        if inactive:
            steps = torch.tensor([self._carried.get(i, -1.0) for i in inactive], dtype=torch.float64,
                                 device=self.device)
            dist.broadcast(steps, 0)
            self._carried = {i: s for i, s in zip(inactive, steps.tolist()) if s >= 0}
        self._export()

    def capture(self, example_batch: dict, warmup: int = 3, curr_epoch: float = 0.0):
        """Captures the whole step into a CUDA graph (static copy of `example_batch` as input).  The warm-up
        iterations run real steps; everything they touch is restored before the capture."""
        self.static_batch = {k: (v.clone() if isinstance(v, torch.Tensor) else v) for k, v in example_batch.items()}
        self.prepare(self.static_batch)
        bsz = self.static_batch["point_clouds"].shape[0]
        snap = self._snapshot()
        side = torch.cuda.Stream(device=self.device)
        side.wait_stream(torch.cuda.current_stream(self.device))
        with torch.cuda.stream(side):
            for _ in range(warmup):
                self._draw_selection(bsz)
                self._body(self.static_batch, curr_epoch)
        torch.cuda.current_stream(self.device).wait_stream(side)
        torch.cuda.synchronize(self.device)
        self._restore(snap)
        self._drop_dry_run_pseudo_labels()
        self._draw_selection(bsz)
        ops.invalidate_weight_cache()
        from . import _lib

        n0 = _lib.LAUNCHES
        self.graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self.graph):
            self.static_out = self._body(self.static_batch, curr_epoch)
        self.launches_per_step = _lib.LAUNCHES - n0  # C-ABI kernel launches recorded in the graph
        self.graph_branch = self._branch(curr_epoch)
        return self

    def __call__(self, batch: dict, curr_epoch: float = 0.0):
        """One optimiser step on a batch that is already on the device.  Returns (loss, loss_dict)."""
        self.prepare(batch)
        self._set_lr(curr_epoch)
        bsz = batch["point_clouds"].shape[0]
        if self.graph is not None and self._branch(curr_epoch) != self.graph_branch:
            # the model takes a different Python branch from this epoch on: the captured graph is stale
            self.graph = None
            self.capture(self.static_batch, warmup=1, curr_epoch=curr_epoch)
            self._set_lr(curr_epoch)
        self._draw_selection(bsz)
        if self.graph is not None:
            for k, v in batch.items():
                if isinstance(v, torch.Tensor):
                    self.static_batch[k].copy_(v, non_blocking=True)
                elif k == "pseudo_box_path":
                    self.static_batch[k] = v
            self.graph.replay()
            # the replayed AdamW wrote the parameters through the flat buffer: neither their version counters nor the
            # weight-plane epoch moved, so planes an eager forward (evaluation) packed since the last step are stale
            ops.invalidate_weight_cache()
            out = self.static_out
        else:
            out = self._body(batch, curr_epoch)
        if self._branch(curr_epoch)[2]:
            # stage-2 discovery epoch: the pseudo-label rows of this step go to the scenes' .npy files now (the one
            # device->host copy of the path; every other epoch the step stays free of host synchronisation)
            if self.graph is not None and getattr(self.model, "_pending_pseudo", None) is not None:
                self.model._pending_pseudo["paths"] = batch.get("pseudo_box_path")
            self.model.flush_pseudo_labels()
        return out

    def _body(self, batch: dict, curr_epoch: float):
        from . import attention_launch

        attention_launch.advance_seed(self.device)
        self.flat.zero_grad()
        self.reducer.start()
        # operand planes of every weight the step will ask for, packed on a side stream while the main stream runs the
        # furthest-point sampling; the request list is recorded on the first step
        recording = self._pack_requests is None
        if recording:
            ops.record_weight_packs(True)
        else:
            if self._pack_stream is None:
                self._pack_stream = torch.cuda.Stream(device=self.device)
            self._pack_stream.wait_stream(torch.cuda.current_stream(self.device))
            ops.prepack_weights(self._pack_requests, self._pack_stream)
        outputs = self.model(batch, curr_epoch=int(curr_epoch))
        loss, loss_dict = self.criterion(outputs, batch)
        loss.backward()                                # range all-reduces start from the gradient hooks
        if recording:
            self._pack_requests = ops.record_weight_packs(False)
        elif ops._PACK_JOIN is not None:               # no consumer joined (cannot happen with packed weights in use)
            torch.cuda.current_stream(self.device).wait_stream(self._pack_stream)
            ops._PACK_JOIN = None
        self.reducer.finish()
        self.optimizer.step()                          # global-norm clip + AdamW, two kernels
        ops.invalidate_weight_cache()  # packed bf16 weight planes are stale now
        return loss.detach(), loss_dict


@torch.no_grad()
def evaluate(args, curr_epoch, model, criterion, dataset_config, dataset_loader, logger=None, curr_train_iter=0,
             if_real_test=False, if_cmp_class=False):
    """Evaluation loop (reference engine.py:2553-2661): model in eval mode -> (optional loss) -> APCalculator.
    Differences are implementation-only: the AP bookkeeping of a batch runs on the device (utils/ap_calculator.py,
    five kernel launches, no host copies), and under data parallelism the ranks do not all-gather their point
    clouds and outputs (`all_gather_dict`, :2634-2636): the calculator is rank-local, each rank matches its own
    scenes, and `compute_metrics()` on the returned calculator is a collective that exchanges the detection records --
    every rank must call it.  The loss is averaged over the ranks as the reference does."""
    from .utils.ap_calculator import APCalculator
    from .utils.dist import all_reduce_average, get_rank, reduce_dict

    world = get_world_size()
    ap_calculator = APCalculator(dataset_config=dataset_config, ap_iou_thresh=[0.25, 0.5],
                                 class2type_map=getattr(dataset_config, "class2type", None), exact_eval=True, args=args,
                                 rank=get_rank(), world_size=world)
    device = next(model.parameters()).device
    model.eval()
    loss_sum, nloss = 0.0, 0
    loss_dict_reduced = None
    for batch in dataset_loader:
        batch = {k: (v.to(device, non_blocking=True) if isinstance(v, torch.Tensor) else v) for k, v in batch.items()}
        outputs = model(batch, if_real_test=if_real_test, if_cmp_class=if_cmp_class)
        if criterion is not None:
            loss, loss_dict = criterion(outputs, batch)
            if world > 1:
                loss = all_reduce_average(loss)
                loss_dict_reduced = reduce_dict(loss_dict)
            loss_sum, nloss = loss_sum + loss.detach(), nloss + 1
        ap_calculator.step_meter(outputs, batch)
    if logger is not None and nloss and is_primary():
        if loss_dict_reduced is not None:
            logger.log_scalars(loss_dict_reduced, curr_train_iter, prefix="Test_details/")
        logger.log_scalars({"loss": float(loss_sum) / nloss}, curr_train_iter, prefix="Test/")
    return ap_calculator
