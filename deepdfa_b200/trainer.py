"""Fused data-parallel train step for ``FlowGNNGGNNModule`` on H100.

One process per GPU.  Per step: forward (T x {gather, GRU}) -> readout+MLP -> labels+BCE ->
hand-written backward -> ONE all-reduce of the flat gradient buffer (NCCL over NVLink/NVSwitch via
``torch.distributed``; the loss rides in the buffer's last element) -> fused Adam over the flat
parameter buffer.  Graphs never exchange messages, so the batch shards across ranks with no
data-path collective (SURVEY.md §8e); the gradient all-reduce is the only exchange step.

Replaces, for the hot path only, Lightning's ``Trainer.fit`` loop around
``BaseModule.training_step`` (base_module.py:171-199) + ``torch.optim.Adam`` (config_default.yaml:43-47).
``FusedTrainer.optimizer`` (:class:`FusedAdam`) is the ``torch.optim.Optimizer`` face of the fused Adam: checkpoints in
``torch.optim.Adam``'s (or, with parameter groups / decoupled weight decay, ``torch.optim.AdamW``'s) format and LR schedulers
that reach captured steps.
"""
from __future__ import annotations

from typing import Optional

import numbers
import os

import torch
import torch.distributed as dist

from . import _lib
from . import engine as E
from .capture import CapturedBatches, cache_graph
from .encoder_cache import CachedRows, encoder_names
from .module import FlowGNNGGNNModule, _ENGINES

_ALIGN = 64  # elements; keeps every parameter 256-byte aligned inside the flat buffers


def flat_offsets(plist):
    """Element offset of every tensor of ``plist`` (``module.param_list()`` order) inside the flat buffers, and their length:
    every slot is rounded up to ``_ALIGN`` elements."""
    offs, total = [], 0
    for p in plist:
        offs.append(total)
        total += (p.numel() + _ALIGN - 1) // _ALIGN * _ALIGN
    return offs, total


def flat_param_list(module):
    """The tensors the flat buffers hold, in ``module.param_list()`` order: every parameter of the module.  In
    label_style="node" the two gate slots of ``param_list()`` are non-persistent zero buffers, not parameters (the style has no
    pooling), and are left out; the graph-style list is ``param_list()`` itself."""
    plist = module.param_list()
    if module.hparams.label_style == "node":
        k = len(module._tables())
        plist = plist[:k + 6] + plist[k + 8:]
    return plist


def trainable_ranges(plist):
    """The ``[begin, end)`` element ranges of the flat buffers (laid out by :func:`flat_offsets`) whose tensors have
    ``requires_grad``, each slot with its alignment padding, adjacent slots merged; the bounds are multiples of ``_ALIGN``.
    Raises ``ValueError`` when no tensor is trainable."""
    offs, total = flat_offsets(plist)
    ranges = []
    for p, lo, hi in zip(plist, offs, offs[1:] + [total]):
        if not p.requires_grad:
            continue
        if ranges and ranges[-1][1] == lo:
            ranges[-1] = (ranges[-1][0], hi)
        else:
            ranges.append((lo, hi))
    if not ranges:
        raise ValueError("FusedTrainer: no parameter of the module has requires_grad=True: there is nothing to train")
    return ranges


def exchange_for_frozen(exchange: str, world: int, frozen: bool):
    """``(exchange, note)``: the gradient exchange a trainer with frozen parameters uses over ``world`` ranks.  The peer-memory
    exchange (``"p2p"``) runs Adam over every element of its shard, so with frozen parameters ``"auto"`` picks NCCL (``note``
    says why) and ``"p2p"`` raises ``NotImplementedError``.  Without frozen parameters or on one rank, nothing changes."""
    if not frozen or world <= 1 or exchange == "nccl":
        return exchange, None
    if exchange == "p2p":
        raise NotImplementedError("exchange='p2p' with frozen parameters: the peer-memory exchange's sharded Adam updates every "
                                  "parameter; use exchange='nccl' (or 'auto')")
    return "nccl", "auto: frozen parameters (the peer-memory exchange updates every parameter): NCCL all-reduce"


def owned_range(numel: int, rank: int, world: int):
    """``[lo, hi)``: the elements of the flat buffers whose Adam moments rank ``rank`` of ``world`` keeps up to date under
    ``exchange="p2p"``.  Mirrors ``allreduce_adam_p2p_kernel``: the buffers are cut into 16-byte units and every rank owns
    ``per = ceil(numel / 4 / world)`` consecutive units (the last rank fewer, possibly none)."""
    n4 = numel // 4
    per = (n4 + world - 1) // world
    lo = min(n4, rank * per)
    return 4 * lo, 4 * min(n4, lo + per)


_FIRST, _ADD, _APPLY = "first", "add", "apply"     # what a micro-batch does with its gradient (FusedTrainer._phase)

_ADAM_FLAGS = dict(amsgrad=False, maximize=False, foreach=None, capturable=False, differentiable=False, fused=None,
                   decoupled_weight_decay=False)
_UNSUPPORTED = ("amsgrad", "maximize", "decoupled_weight_decay")
# the keys a param_groups entry of FusedTrainer may carry: torch's Adam / AdamW group keys (amsgrad and maximize only when False;
# foreach, capturable, differentiable and fused choose torch's implementation and mean nothing to the fused kernels)
_GROUP_KEYS = ("lr", "betas", "eps", "weight_decay", "decoupled_weight_decay")
_IGNORED_KEYS = ("amsgrad", "maximize", "foreach", "capturable", "differentiable", "fused")


def resolve_param_groups(module, param_groups):
    """Checks torch-style ``param_groups`` (a list of ``{"params": [...], <lr, betas, eps, weight_decay,
    decoupled_weight_decay>}``) against ``module`` and returns them as new dicts with ``params`` as lists.  Raises
    ``ValueError`` for: no group, more than ``ADAM_MAX_GROUPS`` groups, a group without ``params``, an unknown key, AMSGrad or
    ``maximize``, a tensor that is not a parameter of the module, a parameter in two groups (or twice in one), and a trainable
    parameter in no group (named).  Frozen parameters may appear in a group or be left out."""
    if isinstance(param_groups, dict) or not isinstance(param_groups, (list, tuple)) or not param_groups:
        raise ValueError("param_groups must be a non-empty list of dicts, as torch.optim.AdamW takes them")
    if len(param_groups) > _lib.ADAM_MAX_GROUPS:
        raise ValueError(f"param_groups: {len(param_groups)} groups, the fused Adam kernels take at most {_lib.ADAM_MAX_GROUPS}")
    names = {id(p): n for n, p in module.named_parameters()}
    seen, out = {}, []
    for gi, g in enumerate(param_groups):
        if not isinstance(g, dict) or "params" not in g:
            raise ValueError(f"param_groups[{gi}] must be a dict with a 'params' entry")
        unknown = sorted(set(g) - {"params", *_GROUP_KEYS, *_IGNORED_KEYS})
        if unknown:
            raise ValueError(f"param_groups[{gi}]: unknown key(s) {unknown}; a group may set {list(_GROUP_KEYS)}")
        bad = [k for k in ("amsgrad", "maximize") if g.get(k)]
        if bad:
            raise ValueError(f"param_groups[{gi}]: {bad} are not supported by the fused Adam kernels")
        params = [g["params"]] if isinstance(g["params"], torch.Tensor) else list(g["params"])
        for p in params:
            if id(p) not in names:
                raise ValueError(f"param_groups[{gi}] holds a tensor of shape {tuple(p.shape)} that is not a parameter of the module")
            if id(p) in seen:
                raise ValueError(f"parameter {names[id(p)]!r} appears in param_groups[{seen[id(p)]}] and param_groups[{gi}]")
            seen[id(p)] = gi
        out.append(dict(g, params=params))
    missing = [n for n, p in module.named_parameters() if p.requires_grad and id(p) not in seen]
    if missing:
        raise ValueError(f"trainable parameter(s) {missing} are in no group of param_groups (freeze them with "
                         "requires_grad_(False) or add them to a group)")
    return out


def group_ranges(plist, group_of):
    """``[(begin, end, group)]``: the trainable slots of the flat buffers (laid out by :func:`flat_offsets`) with the index of
    their parameter group, each slot with its alignment padding, adjacent slots of one group merged.  ``group_of`` maps
    ``id(tensor)`` to a group index; frozen tensors and tensors in no group are left out."""
    offs, total = flat_offsets(plist)
    ranges = []
    for p, lo, hi in zip(plist, offs, offs[1:] + [total]):
        if not p.requires_grad or id(p) not in group_of:
            continue
        g = group_of[id(p)]
        if ranges and ranges[-1][1] == lo and ranges[-1][2] == g:
            ranges[-1] = (ranges[-1][0], hi, g)
        else:
            ranges.append((lo, hi, g))
    return ranges


def group_row(group) -> tuple:
    """A row of the device group table (``DDFA_ADAM_GROUP_WORDS`` words) for a torch param group: ``[lr, beta1, beta2, eps,
    weight_decay, decoupled, decay, 0]``, ``decay = 1 - lr * weight_decay`` in double (the kernel's fp32 word rounds it once,
    as torch's Python scalar in ``param.mul_(1 - lr * weight_decay)`` is rounded)."""
    lr, wd = float(group["lr"]), float(group["weight_decay"])
    dec = bool(group.get("decoupled_weight_decay", False))
    return (lr, float(group["betas"][0]), float(group["betas"][1]), float(group["eps"]), wd, 1.0 if dec else 0.0,
            1.0 - lr * wd if dec else 1.0, 0.0)


class FusedAdam(torch.optim.Optimizer):
    """The optimizer object of a :class:`FusedTrainer` (``trainer.optimizer``): a ``torch.optim.Optimizer`` whose state is
    the trainer's flat Adam buffers.  It owns no arithmetic — the update runs inside the trainer's step, in
    ``ddfa_adam_flat_hp`` / ``ddfa_allreduce_adam_p2p_hp`` or their ``_groups`` forms — and exists so that the usual tools
    work on a fused run:

    * ``state_dict()`` / ``load_state_dict()`` in ``torch.optim.Adam``'s / ``torch.optim.AdamW``'s format, parameters indexed
      in group order (one group: ``module.parameters()`` order, what ``torch.optim.Adam(module.parameters())`` and a
      Lightning checkpoint's ``optimizer_states[0]`` use; the flat buffers hold them in ``module.param_list()`` order);
    * LR schedulers: ``step()`` copies every group's hyperparameters into device words that the Adam kernels read when they
      run, so a captured CUDA graph picks up a new learning rate on its next replay.

    Two forms, chosen by ``hyper``:

    * ``hyper`` fp32[5] ``[lr, beta1, beta2, eps, weight_decay]``: one parameter group over ``module.parameters()``, coupled
      L2 weight decay (``torch.optim.Adam``) — the trainer's default.
    * ``hyper`` fp32[G, DDFA_ADAM_GROUP_WORDS], the group table (rows from :func:`group_row`): the G groups of
      ``param_groups`` (torch's list, checked by :func:`resolve_param_groups`; None: one group over ``module.parameters()``),
      each coupled (Adam) or decoupled (AdamW) as its ``decoupled_weight_decay`` says, missing keys from the arguments.  The
      groups are fixed: ``add_param_group`` raises.

    No AMSGrad, no ``maximize``.  The buffers may live on any device, so the conversion also runs on CPU tensors."""

    def __init__(self, module, exp_avg: torch.Tensor, exp_avg_sq: torch.Tensor, step_count: torch.Tensor, hyper: torch.Tensor,
                 lr: float = 1e-3, betas=(0.9, 0.999), eps: float = 1e-8, weight_decay: float = 0.0, shard=None,
                 param_groups=None, decoupled_weight_decay: bool = False):
        """``exp_avg`` / ``exp_avg_sq``: flat fp32 moment buffers laid out by :func:`flat_offsets`; ``step_count``: int32[1];
        ``hyper``: the hyperparameter words (see the class).  ``shard = (rank, world, process_group)`` when each rank keeps the
        moments of its :func:`owned_range` only (``exchange="p2p"``)."""
        self._table = hyper.dim() == 2
        if not self._table and (param_groups is not None or decoupled_weight_decay):
            raise ValueError("FusedAdam: param_groups and decoupled_weight_decay need the group table (hyper of shape [G, 8])")
        groups = (resolve_param_groups(module, param_groups) if param_groups is not None
                  else [{"params": list(module.parameters())}])
        if self._table and tuple(hyper.shape) != (len(groups), _lib.ADAM_GROUP_WORDS):
            raise ValueError(f"FusedAdam: group table of shape {tuple(hyper.shape)} for {len(groups)} groups")
        flags = dict(_ADAM_FLAGS, decoupled_weight_decay=bool(decoupled_weight_decay))
        self._sealed = False
        super().__init__(groups, dict(lr=lr, betas=tuple(betas), eps=eps, weight_decay=weight_decay, **flags))
        self._sealed = self._table
        plist = flat_param_list(module)
        offs, total = flat_offsets(plist)
        where = {id(p): o for p, o in zip(plist, offs)}
        params = [p for g in self.param_groups for p in g["params"]]
        if (param_groups is None and len(plist) != len(params)) or any(id(p) not in where for p in params):
            raise ValueError("FusedAdam: module.parameters() and the flat parameter list hold different tensors")
        if exp_avg.numel() != total or exp_avg_sq.numel() != total:
            raise ValueError(f"FusedAdam: moment buffers of {exp_avg.numel()} / {exp_avg_sq.numel()} elements, layout needs {total}")
        self._slots = [(where[id(p)], p.numel()) for p in params]      # per state_dict index: (flat offset, numel)
        # frozen parameters (requires_grad=False when the trainer was built) get no state, as torch.optim.Adam gives them none
        self._trainable = [bool(p.requires_grad) for p in params]
        self._flat = (exp_avg, exp_avg_sq, step_count, hyper)
        self._shard = shard
        self._pushed = None
        self._push()

    def add_param_group(self, param_group):
        """The group table's layout is fixed when the trainer is built: adding a group to it raises ``ValueError``."""
        if self._sealed:
            raise ValueError("FusedAdam: add_param_group after construction is not supported (the flat buffers and the group "
                             "table are laid out when the trainer is built); pass every group to FusedTrainer(param_groups=...)")
        super().add_param_group(param_group)

    def _groups(self):
        if not self._table and len(self.param_groups) != 1:
            raise ValueError("FusedAdam supports exactly one parameter group (build the trainer with param_groups= for several)")
        if len(self.param_groups) != len(self._flat[3]) and self._table:
            raise ValueError("FusedAdam: the parameter groups no longer match the group table")
        for g in self.param_groups:
            bad = [k for k in (_UNSUPPORTED if not self._table else ("amsgrad", "maximize")) if g.get(k)]
            if bad:
                raise ValueError(f"FusedAdam: {bad} are not supported (the fused kernels implement torch.optim.Adam with coupled L2"
                                 + ("" if self._table else "; build the trainer with decoupled_weight_decay=True or param_groups= "
                                    "for AdamW") + ")")
        return self.param_groups

    def _push(self):
        """Writes the hyperparameters that changed since the last push into the device words, by value, in stream order
        (no staging buffer the host could overwrite while the device lags behind)."""
        groups = self._groups()
        hyper = self._flat[3]
        if self._table:
            rows = [group_row(g) for g in groups]
            for i, row in enumerate(rows):
                for j, x in enumerate(row):
                    if self._pushed is None or self._pushed[i][j] != x:
                        hyper[i, j].fill_(x)
            self._pushed = rows
            return
        g = groups[0]
        vals = (float(g["lr"]), float(g["betas"][0]), float(g["betas"][1]), float(g["eps"]), float(g["weight_decay"]))
        for i, x in enumerate(vals):
            if self._pushed is None or self._pushed[i] != x:
                hyper[i].fill_(x)
        self._pushed = vals

    def step(self, closure=None):
        """Hands every group's lr / betas / eps / weight_decay (and, with the group table, decoupled_weight_decay) to the
        kernels of the NEXT trainer step that updates the parameters (the trainer calls this at the start of every such step —
        with gradient accumulation, the last micro-batch of a window and ``flush()`` — so a scheduler stepped once per optimizer
        step follows the windows; a value is written only when it changed).  Computes nothing itself."""
        if closure is not None:
            raise ValueError("FusedAdam.step takes no closure: FusedTrainer.step runs forward and backward")
        self._push()

    def _gathered(self, t: torch.Tensor) -> torch.Tensor:
        if self._shard is None:
            return t
        rank, world, group = self._shard
        lo, hi = owned_range(t.numel(), rank, world)
        out = torch.zeros_like(t)
        out[lo:hi].copy_(t[lo:hi])
        dist.all_reduce(out, op=dist.ReduceOp.SUM, group=group)    # every element is nonzero on its owner only: exact
        return out

    def state_dict(self):
        """What ``torch.optim.Adam(groups).state_dict()`` (``torch.optim.AdamW`` for decoupled groups) returns after the same
        steps: per parameter index — assigned in group order — ``{"step": float32 CPU tensor, "exp_avg", "exp_avg_sq"}``
        (copies, shaped like the parameter, on its device), empty before the first step and for parameters frozen when the
        trainer was built, and every group with its keys.  Reads the step counter from the device: one synchronisation.
        With sharded moments (``exchange="p2p"``) this is a collective: every rank must call it, and every rank gets the
        full state (each rank's owned slice, all-reduced)."""
        groups = self._groups()
        exp_avg, exp_avg_sq, step_count, _ = self._flat
        step = int(step_count.item())
        m, v = self._gathered(exp_avg), self._gathered(exp_avg_sq)
        params = [p for g in groups for p in g["params"]]
        state = {}
        if step > 0:
            for i, (p, (o, n)) in enumerate(zip(params, self._slots)):
                if not self._trainable[i]:
                    continue
                state[i] = {"step": torch.tensor(float(step), dtype=torch.float32),
                            "exp_avg": m[o:o + n].view_as(p).clone(), "exp_avg_sq": v[o:o + n].view_as(p).clone()}
        packed, start = [], 0
        for g in groups:
            pg = {k: val for k, val in g.items() if k != "params"}
            pg["params"] = list(range(start, start + len(g["params"])))
            start += len(g["params"])
            packed.append(pg)
        return {"state": state, "param_groups": packed}

    def load_state_dict(self, state_dict):
        """Loads ``torch.optim.Adam``'s format (from :meth:`state_dict`, ``torch.optim.Adam.state_dict()`` or a Lightning
        checkpoint's ``optimizer_states[0]``), older forms included: ``step`` as int or tensor, group keys such as
        ``foreach`` / ``capturable`` / ``fused`` / ``differentiable`` missing; an empty ``state`` means step 0 and zero
        moments.  With the group table, ``torch.optim.AdamW``'s too: each group's ``decoupled_weight_decay`` is loaded with its
        other keys.  Writes IN PLACE into the flat moment buffers, the step counter and the hyperparameter words, so CUDA
        graphs captured before the load replay from the loaded state.  Every rank loads the full moments, whatever world size
        wrote them.  Raises ``ValueError`` (as torch does) for a different number of groups or of parameters in a group, and
        for a shape mismatch, AMSGrad, ``maximize``, ``decoupled_weight_decay`` without the group table, or per-parameter
        steps that differ.  Entries of parameters frozen when the trainer was built are accepted and ignored; the step count
        comes from the trainable parameters only."""
        groups = state_dict.get("param_groups")
        cur_groups = self._groups()
        if not isinstance(groups, (list, tuple)) or len(groups) != len(cur_groups):
            raise ValueError(f"FusedAdam has {len(cur_groups)} parameter group(s), the checkpoint "
                             f"{len(groups) if isinstance(groups, (list, tuple)) else None}")
        unsupported = _UNSUPPORTED if not self._table else ("amsgrad", "maximize")
        ids = []
        for gi, (saved, cur) in enumerate(zip(groups, cur_groups)):
            bad = [k for k in unsupported if saved.get(k)]
            if bad:
                raise ValueError(f"FusedAdam cannot load an optimizer with {bad} set"
                                 + ("" if self._table else " (build the trainer with decoupled_weight_decay=True or param_groups= "
                                    "to load AdamW)"))
            gids = list(saved.get("params", []))
            if len(gids) != len(cur["params"]):
                raise ValueError(f"parameter group {gi}: the checkpoint has {len(gids)} parameters, the optimizer {len(cur['params'])}")
            ids += gids
        cur = [p for g in cur_groups for p in g["params"]]
        state = state_dict.get("state", {})
        if set(state) - set(ids):
            raise ValueError(f"state entries {sorted(set(state) - set(ids))} belong to no parameter of the groups")
        steps, entries = set(), []
        for i, (pid, p) in enumerate(zip(ids, cur)):
            st = state.get(pid)
            if not self._trainable[i]:
                entries.append(None)              # frozen: its saved state, if any, is ignored
            elif st:
                for key in ("exp_avg", "exp_avg_sq"):
                    if key not in st or tuple(st[key].shape) != tuple(p.shape):
                        raise ValueError(f"parameter {i}: {key} of shape {tuple(st[key].shape) if key in st else None}, "
                                         f"the parameter has {tuple(p.shape)}")
                s = st.get("step", 0)
                s = float(s.item()) if torch.is_tensor(s) else float(s)
                if s != int(s) or not 0 <= s < 2 ** 31:
                    raise ValueError(f"parameter {i}: step {s} is not a step count")
                steps.add(int(s))
                entries.append(st)
            else:
                steps.add(0)                          # no state yet: the parameter has never been updated
                entries.append(None)
        if len(steps) > 1:
            raise ValueError(f"per-parameter steps differ ({sorted(steps)}): the fused optimizer keeps one step counter")
        step = steps.pop() if steps else 0
        exp_avg, exp_avg_sq, step_count, _ = self._flat
        with torch.no_grad():
            exp_avg.zero_()
            exp_avg_sq.zero_()
            for (o, n), st in zip(self._slots, entries):
                if st is not None:
                    exp_avg[o:o + n].copy_(st["exp_avg"].reshape(-1))
                    exp_avg_sq[o:o + n].copy_(st["exp_avg_sq"].reshape(-1))
            step_count.fill_(step)
        for saved, group in zip(groups, cur_groups):
            group.update({k: val for k, val in saved.items() if k != "params"})
        self._push()


def _group_property(key, convert=None):
    """A :class:`FusedTrainer` attribute that reads and writes ``optimizer.param_groups[0][key]``."""
    def get(self):
        return self.optimizer.param_groups[0][key]

    def set(self, value):
        self.optimizer.param_groups[0][key] = value if convert is None else convert(value)
    return property(get, set)


class FusedTrainer(CapturedBatches):
    def __init__(self, module: FlowGNNGGNNModule, lr: float = 1e-3, betas=(0.9, 0.999), eps: float = 1e-8,
                 weight_decay: float = 1e-2, process_group=None, use_cuda_graph: bool = False, max_graph_shapes: int = 8,
                 max_resident_graphs: int = 64, distributed: bool = True, bucket_nodes: int = 0, bucket_edges: int = 0,
                 bucket_min_pad_nodes: int = 64, overlap_allreduce: bool = True, exchange: str = "auto",
                 max_grad_norm: Optional[float] = None, skip_nonfinite: bool = False, node_sample_seed: int = 0,
                 track_metrics: bool = False, accumulate_grad_batches: int = 1, param_groups=None,
                 decoupled_weight_decay: bool = False):
        """``distributed=False`` makes this a single-rank trainer even inside an initialised process group (no all-reduce).
        ``bucket_nodes`` / ``bucket_edges`` > 0 switch on shape bucketing for HOST batches under ``use_cuda_graph``: every batch
        is padded with ONE dummy graph of isolated nodes up to the next multiple of ``bucket_nodes`` nodes (at least
        ``bucket_min_pad_nodes`` of them, which also carry the padding edges as self loops) and ``bucket_edges`` edges, so that a
        shuffled stream of ever-new ``(N, E)`` (the reference reshuffles every epoch, datamodule.py:123-129) replays a handful of
        captured graphs.  The dummy graph has zero loss weight (``ddfa_graph_label_bce_valid``): no gradient comes from it.

        Gradient guard (opt-in; with both arguments at their defaults the step enqueues exactly what it did without them):
        ``max_grad_norm`` clips the total L2 norm of the exchanged gradients as ``torch.nn.utils.clip_grad_norm_(params,
        max_grad_norm)`` would, between the exchange and Adam, inside the (captured) step; ``float("inf")`` measures the norm
        without clipping.  ``skip_nonfinite=True`` makes a step whose norm is not finite leave parameters, moments and the Adam
        step count bit-unchanged (GradScaler's rule) and count it in ``skipped_steps``.  ``grad_norm`` holds the last step's
        pre-clip norm; ``max_grad_norm`` can be changed later, also after capture.

        label_style="node": the loss is the mean BCE over per-node logits, on every valid node, or with
        ``undersample_node_on_loss_factor`` on every vulnerable node plus ``round(n_vuln * factor)`` non-vulnerable ones drawn on
        the device inside the step (``ddfa_node_sample``: Philox keys from ``node_sample_seed`` and the draw counter
        ``node_sample_draws``).  The head runs over that row list only.  A draw that asks for more non-vulnerable nodes than the
        batch has takes them all and raises ``ValueError`` at the next step or at ``check_inputs()`` (``random.sample`` raises
        on the module path).  Several ranks (an NCCL group): R ranks over the shards of a global batch do what one rank does over
        the shards concatenated in rank order — the same rows, drawn over the global batch (``engine.NodeDrawDP``: 1 or 6 small
        NCCL collectives on a side stream under the GGNN forward), each rank keeping its own, and the mean over the rows of all
        ranks.  ``global_batch`` is ignored; ``node_sample_seed`` must be the same on every rank (``ValueError``);
        :meth:`last_node_offset` and :meth:`last_num_rows_global` map the rows to the global batch.  Other backends: one rank.

        Frozen parameters: a parameter with ``requires_grad=False`` when the trainer is built is not trained — Adam runs over the
        trainable elements only (``ddfa_adam_flat_ranges``), its gradient slot is zeroed before the norm, and it gets no optimizer
        state, as with ``torch.optim.Adam(module.parameters())``.  With the embedding tables and the six GatedGraphConv tensors
        all frozen the GGNN runs in its inference form and the backward stops after the readout (graph style) or the head
        (node style); with only the tables frozen the embedding backward is skipped.  The trainable set is fixed: changing
        ``requires_grad`` later raises ``ValueError`` at the next step, and a module with nothing trainable raises at once.  With
        more than one rank, frozen parameters need the NCCL exchange (``exchange="auto"`` picks it, ``"p2p"`` raises
        ``NotImplementedError``).

        ``track_metrics=True``: the step ends with one ``ddfa_eval_metrics_*`` call on its own logits — graph style over the valid
        graphs, node style over the drawn loss rows (what base_module.py:178-190 feeds ``train_metrics``) — each step weighted by
        its number of graphs; :meth:`metrics` / :meth:`reset_metrics` mirror ``training_epoch_end``.  This rank's samples only.
        With the default ``False`` the step enqueues nothing for it.

        ``accumulate_grad_batches=k`` (Lightning's ``accumulate_grad_batches``, the ``--gradient_accumulation_steps`` of HF-style
        loops): every :meth:`step` / :meth:`step_ids` call is one micro-batch whose gradient is that of its loss divided by ``k``;
        the gradients of ``k`` consecutive micro-batches (a window) are summed in fp32, in micro-batch order, and the window's last
        micro-batch runs the exchange, the guard and Adam over that sum — once per window, as DDP's ``no_sync`` does.  The other
        micro-batches run no collective, no norm and no Adam, and do not call ``optimizer.step()``; the step count advances once
        per window.  The returned loss is the micro-batch's own mean loss, not divided by ``k``; on a micro-batch that does not
        end its window, with more than one rank, it is this rank's share of it (no collective runs).  :attr:`accumulated` counts
        the micro-batches of the open window; :meth:`flush` applies a partial one (the end of an epoch).  Node-row draws,
        ``track_metrics``, bucketing and input checks stay per micro-batch.  ``optimizer.state_dict()`` may be taken during an
        open window: it holds no partial sum (as Lightning does not checkpoint ``.grad``), so a resumed run starts a fresh
        window.  ``k`` is fixed for the trainer's life.  With the default ``k = 1`` the step enqueues exactly what it did without
        the argument.

        Parameter groups and AdamW: ``param_groups`` is torch's list ``[{"params": [...], <lr, betas, eps, weight_decay,
        decoupled_weight_decay>}, ...]`` (at most 64 groups), keys a group leaves out taking this constructor's arguments;
        ``decoupled_weight_decay=True`` is ``torch.optim.AdamW`` / ``Adam(decoupled_weight_decay=True)`` — ``p *= 1 - lr *
        weight_decay`` before the Adam step instead of L2 in the gradient — for every group that does not say otherwise.
        Every trainable parameter must be in exactly one group (``ValueError`` names the one that is not); frozen parameters
        may be in a group, and are skipped as torch skips them.  ``optimizer.state_dict()`` is then ``torch.optim.AdamW(groups)``'s
        (``Adam``'s for coupled groups), indices in group order, and a ``LambdaLR`` with one lambda per group reaches captured
        steps.  The update runs ``ddfa_adam_flat_groups`` / ``ddfa_allreduce_adam_p2p_groups[_guarded]`` on every step path.
        With neither argument the step enqueues exactly what it did without them."""
        k = accumulate_grad_batches
        if isinstance(k, bool) or not isinstance(k, numbers.Integral) or k < 1:
            raise ValueError(f"accumulate_grad_batches must be an integer >= 1, got {accumulate_grad_batches!r}")
        self._k = int(k)
        self._accumulated = 0
        if module.device.type != "cuda":
            raise _lib.DdfaError("FusedTrainer needs the module on a CUDA device (no CPU fallback)")
        self._node = module.hparams.label_style == "node"
        if module.hparams.label_style not in ("graph", "node") or module.hparams.encoder_mode or module._num_layers == 0:
            raise NotImplementedError("FusedTrainer trains a classifier head (label_style='graph' or 'node', not encoder_mode); train "
                                      "other modules through module.training_step + torch.optim")
        seed = int(node_sample_seed)
        if not 0 <= seed < 2 ** 64:
            raise ValueError(f"node_sample_seed must be in [0, 2**64), got {node_sample_seed!r}")
        self.node_sample_seed = seed
        self.module = module
        self.device = module.device
        self.pg = process_group
        self._guard = max_grad_norm is not None or bool(skip_nonfinite)
        self.skip_nonfinite = bool(skip_nonfinite)
        self._max_grad_norm = float("inf") if max_grad_norm is None else self._check_max_norm(max_grad_norm)
        self.world = dist.get_world_size(process_group) if (distributed and dist.is_available() and dist.is_initialized()) else 1
        self.bucket_nodes, self.bucket_edges, self.bucket_min_pad_nodes = int(bucket_nodes), int(bucket_edges), int(bucket_min_pad_nodes)
        # The gradient exchange is split in two: everything except the four GGNN weight matrices' gradients is final before the
        # batched weight-gradient GEMM starts, so those ranges are all-reduced on a side stream WHILE that launch runs; only
        # [w_msg, b_msg, w_ih, w_hh] (0.46 MB of the 1.5 MB) is reduced after it.  False: one all-reduce of the whole buffer.
        self.overlap_allreduce = bool(overlap_allreduce)
        self._ar_stream = None
        # exchange = "p2p": no NCCL call in the step — the flat parameter and gradient buffers live in symmetric (peer-mapped)
        # memory and ONE kernel per rank does reduce-scatter + Adam + all-gather over NVLink (ddfa_allreduce_adam_p2p); optimizer
        # moments are sharded (each rank keeps them for its 1/R slice only).  Single node.  "nccl": all-reduce + ddfa_adam_flat.
        # "auto" (default): "p2p" when every rank of the group is on this node and the symmetric-memory set-up succeeds on ALL
        # ranks, else "nccl" (the reason is kept in ``exchange_note``).  Measured at N = 2 / 4 / 8: profiles/r03k, r03n, r03o.
        if exchange not in ("auto", "nccl", "p2p"):
            raise ValueError(f"exchange must be 'auto', 'nccl' or 'p2p', got {exchange!r}")
        # Frozen parameters (requires_grad=False when the trainer is built): Adam runs over the trainable ranges only, frozen
        # gradient slots are zeroed before the norm, and the backward is pruned to what the trainable parameters need.
        plist = module.param_list()
        flat = flat_param_list(module)
        # parameter groups / AdamW: the group table and [begin, end, group] ranges of the grouped Adam entry points
        self._grouped = param_groups is not None or bool(decoupled_weight_decay)
        groups = resolve_param_groups(module, param_groups) if param_groups is not None else None
        self._flat_params = flat
        self._trainable = tuple(bool(p.requires_grad) for p in flat)
        self._ranges = trainable_ranges(flat)
        self._frozen = not all(self._trainable)
        ntab = len(module._tables())
        self._grad_ggnn = any(self._trainable[:ntab + 6])    # False: tables and all six GatedGraphConv tensors frozen
        self._grad_tables = any(self._trainable[:ntab])      # False: no embedding backward
        exchange, self.exchange_note = exchange_for_frozen(exchange, self.world, self._frozen)
        auto = exchange == "auto"
        if auto:
            exchange = "p2p"
            local = int(os.environ.get("LOCAL_WORLD_SIZE", "0") or 0)
            if self.world > 1 and (dist.get_backend(process_group) != "nccl" or (local and local != self.world)
                                   or torch.cuda.device_count() < self.world):
                exchange, self.exchange_note = "nccl", "auto: ranks span more than this node (or a non-NCCL group): NCCL all-reduce"
        self.exchange = exchange if self.world > 1 else "nccl"
        if self._node and self.world > 1 and dist.get_backend(process_group) != "nccl":
            # several ranks draw the loss rows of the global batch through NCCL collectives captured in the step graph
            raise NotImplementedError("FusedTrainer: label_style='node' over several ranks needs an NCCL process group; with this "
                                      "backend it trains on one rank (distributed=False or a one-rank group)")
        self.use_cuda_graph = use_cuda_graph
        # a captured graph bakes in the batch SHAPE (and, for resident batches, the batch object): cap how many are kept so a
        # stream of ever-new shapes (un-bucketed real data) degrades to eager launches instead of growing without bound
        self.max_graph_shapes = max_graph_shapes
        self.max_resident_graphs = max_resident_graphs
        offs, total = flat_offsets(flat)
        self.numel = total
        self._frozen_ranges = [(a[1], b[0]) for a, b in zip([(0, 0)] + self._ranges, self._ranges + [(total, total)]) if a[1] < b[0]]
        self._gemm_grad_range = (offs[ntab], offs[ntab + 4])     # flat offsets of [w_msg, b_msg, w_ih, w_hh]
        with torch.cuda.device(self.device):
            if self.exchange == "p2p":
                try:
                    self._setup_p2p(total)
                    ok, why = 1, None
                except _lib.DdfaError as exc:
                    if not auto:
                        raise
                    ok, why = 0, str(exc)
                # all ranks take the same path: one failed set-up sends every rank to NCCL.  (The set-up itself contains collectives —
                # symmetric-memory rendezvous — so this covers failures every rank sees alike: the module missing, peer access
                # unavailable, an allocation refused; a rank that dies alone is a job failure either way.)
                if auto:
                    flag = torch.tensor([ok], dtype=torch.int32, device=self.device)
                    dist.all_reduce(flag, op=dist.ReduceOp.MIN, group=process_group)
                    if int(flag.item()) == 0:
                        self.exchange = "nccl"
                        self.exchange_note = "auto: symmetric-memory set-up failed on a rank (" + (why or "another rank") + "): NCCL all-reduce"
            if self.exchange != "p2p":
                self.flat_p = torch.zeros(total, dtype=torch.float32, device=self.device)
                self.flat_g = torch.zeros(total + _ALIGN, dtype=torch.float32, device=self.device)  # [+ loss slot]
            self.exp_avg = torch.zeros(total, dtype=torch.float32, device=self.device)
            self.exp_avg_sq = torch.zeros(total, dtype=torch.float32, device=self.device)
            # the window's gradient sum (ddfa_grad_accumulate), laid out as flat_g without its loss slot; only with k > 1
            self._acc = torch.zeros(total, dtype=torch.float32, device=self.device) if self._k > 1 else None
            self.step_count = torch.zeros(1, dtype=torch.int32, device=self.device)
            # [lr, beta1, beta2, eps, weight_decay] — with parameter groups one such row per group, plus [decoupled, decay, pad]
            # (group_row) — read by the Adam kernels when they run; written by self.optimizer.step()
            if self._grouped:
                ngroups = len(groups) if groups is not None else 1
                self.hyper = torch.zeros(ngroups, _lib.ADAM_GROUP_WORDS, dtype=torch.float32, device=self.device)
                group_of = ({id(p): gi for gi, g in enumerate(groups) for p in g["params"]} if groups is not None
                            else {id(p): 0 for p in flat})
                self._group_ranges = group_ranges(flat, group_of)
                self._ranges_dev = torch.tensor(self._group_ranges, dtype=torch.int64, device=self.device).reshape(-1)
            else:
                self.hyper = torch.zeros(5, dtype=torch.float32, device=self.device)
                if self._frozen:
                    self._ranges_dev = torch.tensor(self._ranges, dtype=torch.int64, device=self.device).reshape(-1)
            shard = (self._p2p_rank, self.world, self.pg) if self.exchange == "p2p" else None
            self.optimizer = FusedAdam(module, self.exp_avg, self.exp_avg_sq, self.step_count, self.hyper, lr=lr, betas=betas, eps=eps,
                                       weight_decay=weight_decay, shard=shard, param_groups=groups,
                                       decoupled_weight_decay=decoupled_weight_decay)
            if self._guard:
                # the bound (a device word of its own, read when the step runs: not a param_groups key, so state_dict() stays
                # torch.optim.Adam's), [norm, coef, nonfinite] of the last step, the skip counter and the norm's scratch
                self._max_norm_dev = torch.full((1,), self._max_grad_norm, dtype=torch.float32, device=self.device)
                self._gstate = torch.zeros(4, dtype=torch.float32, device=self.device)
                self._skipped = torch.zeros(1, dtype=torch.int32, device=self.device)
                L = _lib.lib()
                if self.exchange == "p2p":
                    self._guard_ws = torch.zeros(L.call("ddfa_p2p_guard_state_bytes"), dtype=torch.uint8, device=self.device)
                else:
                    self._guard_ws = torch.empty(L.call("ddfa_grad_norm_workspace_bytes", total), dtype=torch.uint8, device=self.device)
        gviews = []
        for p, o in zip(flat, offs):
            view = self.flat_p[o:o + p.numel()].view_as(p)
            view.copy_(p.data)
            p.data = view                      # module parameters now alias the flat buffer
            gviews.append(self.flat_g[o:o + p.numel()].view_as(p))
        K, nl = len(module._tables()), module._num_layers
        pviews = [p.data for p in flat]
        if self._node:
            # the gate slots of the ParamPack: the module's zero buffers, and gradients nothing reads (the node head has no gate)
            gate = plist[K + 6:K + 8]
            self._gate_grad_sink = [torch.zeros_like(t) for t in gate]
            pviews = pviews[:K + 6] + [t.data for t in gate] + pviews[K + 6:]
            gviews = gviews[:K + 6] + self._gate_grad_sink + gviews[K + 6:]
            with torch.cuda.device(self.device):
                self._draw = torch.zeros(1, dtype=torch.int64, device=self.device)         # draws made (ddfa_node_sample advances it)
                self._num_rows = torch.zeros(1, dtype=torch.int32, device=self.device)     # S of the last step
                self._sample_status = torch.zeros(1, dtype=torch.int32, device=self.device)
            self._status_host = torch.zeros(1, dtype=torch.int32).pin_memory()
            self._status_pending = None
            self._last_rows = None
            if self.world > 1:
                self._node_dp_setup(process_group)
        self.params = E.ParamPack.from_flat_list(pviews, K, nl)
        self.grads = E.ParamPack.from_flat_list(gviews, K, nl)
        self.loss_slot = self.flat_g[total:total + 1]          # this rank's share of the loss goes here (the kernels' loss_out)
        if self.exchange == "p2p":                                # ... and the global loss into a local word (peers read the slot above)
            self._loss_local = self.loss_slot
            self.loss_slot = torch.zeros(1, dtype=torch.float32, device=self.device)
        # with the guard a step may go non-finite and the run continues: images whose padding rows a producer leaves unwritten
        # get their last tile cleared every step, so no NaN of a skipped step can sit in rows a later, smaller batch pads with
        self.ws = E.Workspace(self.device, scrub_image_tails=self._guard)
        self.track_metrics = bool(track_metrics)
        if self.track_metrics:
            with torch.cuda.device(self.device):
                self._metric_state = torch.zeros(_lib.EVAL_STATE_WORDS, dtype=torch.float64, device=self.device)
                self._metric_ws = torch.empty(_lib.lib().call("ddfa_eval_metrics_workspace_bytes"), dtype=torch.uint8, device=self.device)
        self._update = self._update_calls()
        super().__init__()

    # The Adam hyperparameters live in self.optimizer.param_groups[0], which is what an LR scheduler changes; the next step
    # (eager or replayed) uses whatever is there when it starts.
    lr = _group_property("lr")
    betas = _group_property("betas", tuple)
    eps = _group_property("eps")
    weight_decay = _group_property("weight_decay")

    # ---- gradient guard ----------------------------------------------------------------------------------------------------
    @staticmethod
    def _check_max_norm(value) -> float:
        v = float(value)
        if not v >= 0.0:
            raise ValueError(f"max_grad_norm must be >= 0 (float('inf') measures without clipping), got {value!r}")
        return v

    @property
    def max_grad_norm(self) -> Optional[float]:
        """The clipping bound (``float('inf')``: measure, don't clip); None when the trainer was built without the guard."""
        return self._max_grad_norm if self._guard else None

    @max_grad_norm.setter
    def max_grad_norm(self, value):
        """Written by value into the bound's device word in stream order, so the next step — eager or a replayed graph —
        uses it.  ``None`` means ``inf``.  Turning the guard on or off is a construction-time choice."""
        if not self._guard:
            raise ValueError("this FusedTrainer was built without a gradient guard: pass max_grad_norm= (float('inf') to start "
                             "unclipped) or skip_nonfinite=True to FusedTrainer(...)")
        v = float("inf") if value is None else self._check_max_norm(value)
        if v != self._max_grad_norm:
            self._max_norm_dev.fill_(v)
        self._max_grad_norm = v

    @property
    def grad_norm(self) -> Optional[torch.Tensor]:
        """fp32[1] device tensor: the last step's total gradient L2 norm before clipping (after the data-parallel exchange;
        ``clip_grad_norm_``'s return value).  Valid once that step's stream work has completed; None without the guard."""
        return self._gstate[0:1] if self._guard else None

    @property
    def skipped_steps(self) -> int:
        """Steps skipped because their gradient norm was not finite (reads the device counter: one synchronisation)."""
        return int(self._skipped.item()) if self._guard else 0

    # ---- gradient accumulation ---------------------------------------------------------------------------------------------
    @property
    def accumulated(self) -> int:
        """Micro-batches in the open accumulation window: 0 right after an update (always 0 with ``accumulate_grad_batches=1``)."""
        return self._accumulated

    def _phase(self) -> str:
        """What the next micro-batch does with its gradient: ``"first"`` (starts the window's sum), ``"add"`` (adds to it) or
        ``"apply"`` (adds the sum to its own gradient, then exchange, guard and Adam — every step with ``k = 1``)."""
        if self._accumulated == self._k - 1:
            return _APPLY
        return _FIRST if self._accumulated == 0 else _ADD

    def _phase_key(self, phase: str) -> tuple:
        """Part of every captured-graph key: a graph bakes in its phase's launches.  Empty with ``k = 1`` (the keys stay as they were)."""
        return () if self._k == 1 else (phase,)

    def _begin(self) -> str:
        """Start of a micro-batch: the checks of every step, and the optimizer's ``step()`` when this one updates the parameters."""
        self._check_trainable()
        self._raise_deferred_sample_errors()
        phase = self._phase()
        if phase == _APPLY:
            self.optimizer.step()
        return phase

    def _end(self, phase: str) -> torch.Tensor:
        """Counts the enqueued micro-batch into the window and returns its loss word.  Under peer memory, where the exchange kernel
        writes the global loss into a local word, a micro-batch that runs no exchange returns this rank's own loss slot."""
        self._accumulated = 0 if phase == _APPLY else self._accumulated + 1
        if phase != _APPLY and self.exchange == "p2p":
            return self._loss_local
        return self.loss_slot

    def flush(self) -> None:
        """Applies the open window now, short as it is: the exchange, the guard and Adam over the gradients accumulated so far
        (each still scaled by ``1 / accumulate_grad_batches``), with no forward pass — what Lightning does on the last batch of an
        epoch.  Calls ``optimizer.step()`` first, as a full window does.  Does nothing when the window is empty.  Collective when
        the exchange is: every rank must call it.  The loss slot is not touched, so on one rank the last micro-batch's returned
        loss keeps its value."""
        if self._accumulated == 0:
            return
        self._check_trainable()
        self.optimizer.step()
        with torch.cuda.device(self.device):
            self.flat_g[:self.numel].zero_()
            self._finish(_APPLY)
        self._accumulated = 0

    def _add_window(self, lo: int, hi: int) -> None:
        """The applying micro-batch: adds the window's sum to flat_g[lo:hi) (nothing with k = 1)."""
        if self._acc is not None:
            E.grad_accumulate(self._acc, self.flat_g, lo, hi, _lib.GRAD_ACC_APPLY)

    def _finish(self, phase: str, split: bool = False) -> None:
        """After a micro-batch's backward: its gradient goes into the window's sum, or — on the applying micro-batch — the sum
        is added to it and the exchange, the guard and Adam follow.  ``split``: the small-gradient ranges were already summed and
        handed to the side-stream all-reduce (``_reduce_small_grads``); the GEMM range remains."""
        if phase != _APPLY:
            mode = _lib.GRAD_ACC_SET if phase == _FIRST else _lib.GRAD_ACC_ADD
            E.grad_accumulate(self._acc, self.flat_g, 0, self.numel, mode)
            return
        if split:
            lo, hi = self._gemm_grad_range
            self._add_window(lo, hi)
            dist.all_reduce(self.flat_g[lo:hi], op=dist.ReduceOp.SUM, group=self.pg)
            torch.cuda.current_stream().wait_stream(self._ar_stream)     # both halves are in before the norm and Adam
        else:
            self._add_window(0, self.numel)
            if self.exchange != "p2p" and self.world > 1:     # under p2p the exchange is the update kernel itself
                dist.all_reduce(self.flat_g, op=dist.ReduceOp.SUM, group=self.pg)
        self._enqueue_update()

    # ---- label_style="node"------------------------------------------------------------------------------------------------
    def _require_node(self, what):
        if not self._node:
            raise ValueError(f"{what}: this FusedTrainer trains a label_style='graph' module")

    @property
    def node_sample_draws(self) -> int:
        """Undersampling draws made so far (the Philox counter of the next draw).  Reading it synchronises.  Setting it writes
        the device word in stream order, so a resumed run that restores it draws what the uninterrupted run would have drawn."""
        self._require_node("node_sample_draws")
        return int(self._draw.item())

    @node_sample_draws.setter
    def node_sample_draws(self, value: int):
        self._require_node("node_sample_draws")
        v = int(value)
        if v < 0:
            raise ValueError(f"node_sample_draws must be >= 0, got {value!r}")
        self._draw.fill_(v)

    def last_loss_rows(self) -> torch.Tensor:
        """int32 device tensor: the nodes the last step's loss was taken over, ascending (reads S: one synchronisation).  With
        several ranks: the rows of this rank's shard, in local node ids (add :meth:`last_node_offset` for global ids)."""
        self._require_node("last_loss_rows")
        if self._last_rows is None:
            return torch.zeros(0, dtype=torch.int32, device=self.device)
        return self._last_rows[:int(self._num_rows.item())].clone()

    def last_node_offset(self) -> int:
        """The first node of this rank's shard in the last step's global batch (the shards concatenated in rank order): the
        number of valid nodes on the ranks before it.  0 on one rank.  Reads a device word: one synchronisation."""
        self._require_node("last_node_offset")
        return int(self._node_off.item()) if self.world > 1 else 0

    def last_num_rows_global(self) -> int:
        """S of the last step over the global batch, the divisor of its mean loss: the loss rows of all ranks.  On one rank
        ``last_loss_rows().numel()``.  Reads a device word: one synchronisation."""
        self._require_node("last_num_rows_global")
        return int((self._s_global if self.world > 1 else self._num_rows).item())

    def _node_dp_setup(self, process_group):
        """Several ranks, node style: every rank must draw with the same seed (checked here, collectively: every rank raises
        alike); the device words of the global row count and the shard's node offset; the side stream the draw runs on."""
        seed = self.node_sample_seed
        lo, hi = seed & 0xFFFFFFFF, seed >> 32
        t = torch.tensor([lo, hi, -lo, -hi], dtype=torch.int64, device=self.device)
        dist.all_reduce(t, op=dist.ReduceOp.MAX, group=process_group)     # max == own on every word: the same seed on every rank
        if t.tolist() != [lo, hi, -lo, -hi]:
            raise ValueError(f"node_sample_seed differs between the ranks (this rank: {seed}); every rank draws the loss rows of the "
                             "global batch with the same Philox keys")
        self._s_global = torch.zeros(1, dtype=torch.int32, device=self.device)
        self._node_off = torch.zeros(1, dtype=torch.int32, device=self.device)
        self._sample_stream = torch.cuda.Stream(device=self.device)
        self._node_rank = dist.get_rank(process_group)

    def _sum_ints(self, t: torch.Tensor) -> None:
        dist.all_reduce(t, op=dist.ReduceOp.SUM, group=self.pg)

    def _after_run(self, rows, num_nodes: int):
        """After every step, replays included, node style: remembers its row list and sends the sampler's status word to the
        host behind it."""
        if not self._node:
            return
        self._last_rows = rows
        self._status_host.copy_(self._sample_status, non_blocking=True)
        ev = torch.cuda.Event()
        ev.record()
        self._status_pending = ev

    def _raise_deferred_sample_errors(self, wait: bool = False):
        if not self._node or self._status_pending is None:
            return
        if wait:
            self._status_pending.synchronize()
        elif not self._status_pending.query():
            return
        self._status_pending = None
        if int(self._status_host[0]):
            self._sample_status.zero_()
            self._status_host.zero_()
            raise ValueError("undersample_node_on_loss_factor asked for more non-vulnerable nodes than an earlier batch had "
                             "(random.sample raises 'Sample larger than population'); that step drew all of them")

    def check_inputs(self):
        """Waits for the last step and raises what it deferred: ``ValueError`` when a node-style undersampling draw asked for
        more non-vulnerable nodes than the batch had."""
        self._raise_deferred_sample_errors(wait=True)

    def _check_trainable(self):
        """The trainable set is fixed when the trainer is built: torch keeps a step count per parameter, the fused optimizer one
        for all, so a tensor unfrozen mid-run could not follow torch's bias correction."""
        if tuple(p.requires_grad for p in self._flat_params) != self._trainable:
            raise ValueError("FusedTrainer: requires_grad of a parameter changed after the trainer was built; the trainable set "
                             "is fixed at construction — build a new FusedTrainer (and optimizer state) for the new set")

    # ------------------------------------------------------------------------------------
    def _setup_p2p(self, total: int):
        """Symmetric allocations + rendezvous (torch.distributed._symmetric_memory): every rank gets device pointers to every
        rank's parameter / gradient / flag buffers."""
        try:
            import torch.distributed._symmetric_memory as symm
            group = self.pg if self.pg is not None else dist.group.WORLD
            self.flat_p = symm.empty(total, dtype=torch.float32, device=self.device)
            self.flat_g = symm.empty(total + _ALIGN, dtype=torch.float32, device=self.device)
            # 2 * world words for the barriers; the guarded kernel also needs world norm epochs and 16 fp64 slice sums
            self._flags = symm.empty(128, dtype=torch.int32, device=self.device)      # >= DDFA_P2P_GUARD_FLAG_WORDS
            self.flat_p.zero_(); self.flat_g.zero_(); self._flags.zero_()
            torch.cuda.synchronize(self.device)
            hp, hg, hf = (symm.rendezvous(t, group) for t in (self.flat_p, self.flat_g, self._flags))
            self._peer_ptrs = tuple([int(x) for x in h.buffer_ptrs] for h in (hp, hg, hf))
            self._symm_handles = (hp, hg, hf)
            self._p2p_rank = dist.get_rank(group)
        except Exception as exc:       # no silent downgrade to NCCL: the caller asked for the peer-memory exchange
            raise _lib.DdfaError(f"exchange='p2p': symmetric-memory setup failed ({type(exc).__name__}: {exc})") from exc
        if len(self._peer_ptrs[0]) != self.world or 2 * self.world > 64:
            raise _lib.DdfaError("exchange='p2p': unexpected symmetric-memory world size")
        self._ticket = torch.zeros(1, dtype=torch.int32, device=self.device)
        dist.barrier(group)            # every rank's flag words are zero before anyone's first kernel can write one

    def _update_calls(self):
        """``[(entry point, arguments but the stream)]``: the optimizer update that ends every step.  None of its buffers ever
        moves (``load_state_dict`` writes in place), so the calls are fixed when the trainer is built.  With the guard and
        without peer memory, the norm of the exchanged gradients comes first."""
        skipped = self._skipped.data_ptr() if self.skip_nonfinite else None      # skip_nonfinite implies the guard
        adam = (self.exp_avg.data_ptr(), self.exp_avg_sq.data_ptr(), self.step_count.data_ptr())
        # parameter groups: the ranges with their group index and the group table
        table = (self._ranges_dev.data_ptr(), len(self._group_ranges), self.hyper.data_ptr(), self.hyper.shape[0]) if self._grouped else None
        if self.exchange == "p2p":
            self._peer_arrays = tuple(_lib.ptr_array(p) for p in self._peer_ptrs)      # host arrays the calls point into
            head = (*self._peer_arrays, self._p2p_rank, self.world, *adam, self.numel, self.numel, self.loss_slot.data_ptr())
            if self._grouped and self._guard:
                return [("ddfa_allreduce_adam_p2p_groups_guarded", head + table + (self._max_norm_dev.data_ptr(), self._gstate.data_ptr(),
                                                                                   skipped, self._guard_ws.data_ptr()))]
            if self._grouped:
                return [("ddfa_allreduce_adam_p2p_groups", head + (self._ticket.data_ptr(),) + table)]
            if self._guard:
                return [("ddfa_allreduce_adam_p2p_guarded", head + (self.hyper.data_ptr(), self._max_norm_dev.data_ptr(),
                                                                    self._gstate.data_ptr(), skipped, self._guard_ws.data_ptr()))]
            return [("ddfa_allreduce_adam_p2p_hp", head + (self._ticket.data_ptr(), self.hyper.data_ptr()))]
        flat = (self.flat_p.data_ptr(), self.flat_g.data_ptr(), *adam, self.numel, self.hyper.data_ptr())
        norm = [("ddfa_grad_norm", (self.flat_g.data_ptr(), self.numel, self._max_norm_dev.data_ptr(), self._gstate.data_ptr(),
                                    self._guard_ws.data_ptr(), self._guard_ws.numel()))] if self._guard else []
        if self._grouped:
            return norm + [("ddfa_adam_flat_groups", flat[:6] + table + ((self._gstate.data_ptr(), skipped) if self._guard else (None, None)))]
        if self._frozen:
            ranged = (*flat[:6], self._ranges_dev.data_ptr(), len(self._ranges), self.hyper.data_ptr())
            return norm + [("ddfa_adam_flat_ranges", ranged + ((self._gstate.data_ptr(), skipped) if self._guard else (None, None)))]
        if self._guard:
            return [("ddfa_grad_norm", (self.flat_g.data_ptr(), self.numel, self._max_norm_dev.data_ptr(), self._gstate.data_ptr(),
                                        self._guard_ws.data_ptr(), self._guard_ws.numel())),
                    ("ddfa_adam_flat_guarded", flat + (self._gstate.data_ptr(), skipped))]
        return [("ddfa_adam_flat_hp", flat)]

    def _global_batch(self, global_batch: Optional[int], local_graphs: int) -> int:
        """The divisor of the mean BCE (base_module.py:74,183).  Ranks generally hold different numbers of graphs
        (batched_graph.split_batch balances by nodes), so with more than one rank the caller must say what the global batch is."""
        if self._node:            # node style: the loss is a mean over rows, whose global count the step exchanges itself
            return int(local_graphs)
        if global_batch is not None:
            return int(global_batch)
        if self.world > 1:
            raise _lib.DdfaError("FusedTrainer.step: global_batch is required when world_size > 1 (shards hold different numbers of graphs; "
                                 "the loss is the mean over the GLOBAL batch)")
        return int(local_graphs)

    def _enqueue(self, ctx, prepared, vuln, num_valid: Optional[int], valid_nodes: Optional[torch.Tensor]):
        """Enqueues one step of the batch ``prepared`` (``module._prepare``) with ``ctx = (global_batch, phase)``: one
        micro-batch, ``phase`` as :meth:`_phase` says.  Node style returns the row-list buffer the step's loss rows go to;
        ``valid_nodes``: the int32 device word of its valid node count under bucketing (None: every node is valid)."""
        global_batch, phase = ctx
        g, dg, idx = prepared
        m = self.module
        eng = _ENGINES[m.engine]
        pw = 1.0 if m.hparams.positive_weight is None else float(m.hparams.positive_weight)
        self.flat_g.zero_()
        if self._node:
            rows = self._enqueue_node(dg, idx, vuln, eng, pw, valid_nodes, phase)
            if self.track_metrics:
                self._enqueue_metrics("ddfa_eval_metrics_rows", (E._p(self._last_logits), E._p(vuln), E._p(rows),
                                                                 self._num_rows.data_ptr(), dg.num_nodes),
                                      pw, g.batch_size if num_valid is None else num_valid)
            return rows
        if isinstance(idx, CachedRows):      # an encoder cache's rows: the readout over them, no GGNN launch
            _, logits, saved = E.readout_forward(self.params, dg, idx.x, idx.h, m.hparams.n_steps, training=True, alloc=self.ws)
        else:
            _, logits, saved = E.forward(self.params, dg, idx, m.hparams.n_steps, training=True, engine=eng, alloc=self.ws,
                                         grad_ggnn=self._grad_ggnn)
        prune = dict(grad_ggnn=self._grad_ggnn, grad_tables=self._grad_tables)
        global_batch = self._global_batch(global_batch, dg.batch_size if num_valid is None else num_valid)
        # the gradient of loss / k (k = 1: 1 / global_batch as ever); the loss itself stays the micro-batch's mean
        _, _, dlogits = E.graph_label_bce(dg, vuln, logits, pw, 1.0 / global_batch, 1.0 / (global_batch * self._k), True,
                                          alloc=self.ws, loss_out=self._loss_local if self.exchange == "p2p" else self.loss_slot,
                                          num_valid=num_valid)
        # NCCL over several ranks: the small-gradient ranges are all-reduced on a side stream during the weight-gradient launch
        split = phase == _APPLY and self.exchange != "p2p" and self.world > 1 and self.overlap_allreduce
        E.backward(self.params, dg, saved, self.grads, dlogits=dlogits, engine=eng, alloc=self.ws,
                   on_small_grads_ready=self._reduce_small_grads if split else None, **prune)
        self._finish(phase, split)
        if self.track_metrics:
            B = dg.batch_size
            nv = B if num_valid is None else int(num_valid)
            self._enqueue_metrics("ddfa_eval_metrics_graph", (E._p(logits), E._p(vuln), E._p(dg.graph_ptr), B, nv), pw, nv)

    def _enqueue_metrics(self, name, head, pw, num_graphs):
        """track_metrics: the step's logits into the training metric state (no prediction store), weighted by the graph count."""
        _lib.lib().call(name, *head, pw, float(num_graphs), self._metric_state.data_ptr(), None, None, 0,
                        self._metric_ws.data_ptr(), self._metric_ws.numel(), torch.cuda.current_stream().cuda_stream)

    def metrics(self, prefix: str = "train_") -> dict:
        """The training metrics of the steps since the last :meth:`reset_metrics` (``track_metrics=True``; one synchronisation):
        the keys of ``FusedEvaluator.compute``, the loss being the epoch mean of the step losses weighted by their graph counts.
        Raises ``ValueError`` when no step was tracked."""
        from .evaluator import metrics_from_state, SAMPLES
        if not self.track_metrics:
            raise ValueError("this FusedTrainer was built with track_metrics=False")
        s = self._metric_state.cpu()
        if s[SAMPLES] == 0:
            raise ValueError("FusedTrainer.metrics: no sample was tracked since the last reset_metrics()")
        return metrics_from_state(s, prefix)

    def reset_metrics(self) -> None:
        """Zeroes the training metric state in stream order (``training_epoch_end``)."""
        if not self.track_metrics:
            raise ValueError("this FusedTrainer was built with track_metrics=False")
        self._metric_state.zero_()

    def metric_state(self) -> torch.Tensor:
        """The float64 device training metric state (``ddfa_eval_metrics_*`` layout), for a cross-rank ``all_reduce``."""
        if not self.track_metrics:
            raise ValueError("this FusedTrainer was built with track_metrics=False")
        return self._metric_state

    def _enqueue_update(self):
        """The optimizer update that ends the step.  With frozen parameters their gradient slots are cleared first (the full
        backward of a mixed frozen set writes some of them), so the norm is ``clip_grad_norm_`` over the trainable parameters."""
        for lo, hi in self._frozen_ranges:
            self.flat_g[lo:hi].zero_()
        L, stream = _lib.lib(), torch.cuda.current_stream().cuda_stream
        for name, args in self._update:
            L.call(name, *args, stream)

    def _enqueue_node(self, dg, idx, vuln, eng, pw, valid_nodes, phase):
        """label_style="node": GGNN forward without the readout, the loss rows drawn on the device, the head and the BCE over
        them, the head backward into dh_T / dx, the GGNN backward from there, the update (or, inside an accumulation window, the
        gradient into the window's sum).  Several ranks: the rows are those of the global batch's draw that fall in this shard
        (``engine.NodeDrawDP``), drawn with their collectives on a side stream under the GGNN forward, and the BCE divides by
        the global row count."""
        m, ws = self.module, self.ws
        N = dg.num_nodes
        factor = m.hparams.undersample_node_on_loss_factor
        if self.world > 1:
            return self._enqueue_node_dp(dg, idx, vuln, eng, pw, valid_nodes, phase)
        x, h_T, saved = self._node_rows(dg, idx, eng)
        if valid_nodes is None:
            valid_nodes = ws.get("node_valid", (1,), torch.int32)
            valid_nodes.fill_(N)
        rows = ws.get("node_rows", (N,), torch.int32)
        E.node_sample(vuln, valid_nodes, factor, self.node_sample_seed, self._draw, rows, self._num_rows, self._sample_status, alloc=ws)
        logits, act = E.node_head_fwd(self.params, x, h_T, rows, self._num_rows, alloc=ws)
        self._last_logits = logits
        dlogits = E.node_bce(logits, vuln, rows, self._num_rows, pw, self.loss_slot, alloc=ws,
                             grad_scale=None if self._k == 1 else 1.0 / self._k)
        return self._node_backward(dg, saved, eng, dlogits, x, h_T, rows, act, phase)

    def _enqueue_node_dp(self, dg, idx, vuln, eng, pw, valid_nodes, phase):
        m, ws = self.module, self.ws
        N = dg.num_nodes
        if valid_nodes is None:
            valid_nodes = ws.get("node_valid", (1,), torch.int32)
            valid_nodes.fill_(N)
        rows = ws.get("node_rows", (N,), torch.int32)
        draw = E.NodeDrawDP(vuln, valid_nodes, m.hparams.undersample_node_on_loss_factor, self.node_sample_seed, self._draw, rows,
                            self._num_rows, self._sample_status, self._s_global, self._node_off, self._node_rank, self.world, alloc=ws)
        main = torch.cuda.current_stream()
        self._sample_stream.wait_stream(main)
        with torch.cuda.stream(self._sample_stream):      # it needs _VULN and the valid count only: under the GGNN forward
            draw.run(self._sum_ints)
        x, h_T, saved = self._node_rows(dg, idx, eng)
        main.wait_stream(self._sample_stream)
        logits, act = E.node_head_fwd(self.params, x, h_T, rows, self._num_rows, alloc=ws)
        self._last_logits = logits
        dlogits = E.node_bce_global(logits, vuln, rows, self._num_rows, self._s_global, pw,
                                    self._loss_local if self.exchange == "p2p" else self.loss_slot, grad_scale=1.0 / self._k, alloc=ws)
        return self._node_backward(dg, saved, eng, dlogits, x, h_T, rows, act, phase)

    def _node_rows(self, dg, idx, eng):
        """``(x, h_T, Saved or None)`` of a node-style step: the GGNN forward without the readout, or an encoder cache's rows."""
        if isinstance(idx, CachedRows):
            return idx.x, idx.h, None
        return E.forward(self.params, dg, idx, self.module.hparams.n_steps, training=True, engine=eng, alloc=self.ws, head=False,
                         grad_ggnn=self._grad_ggnn)

    def _node_backward(self, dg, saved, eng, dlogits, x, h_T, rows, act, phase):
        ws = self.ws
        dh, dx = E.node_head_bwd(self.params, self.grads, dlogits, x, h_T, rows, self._num_rows, act, alloc=ws,
                                 input_grads=self._grad_ggnn)
        if self._grad_ggnn:
            E.backward(self.params, dg, saved, self.grads, engine=eng, alloc=ws, dh_final=dh, dx_direct=dx,
                       grad_tables=self._grad_tables)
        self._finish(phase)
        return rows

    def _reduce_small_grads(self):
        """All-reduce of the embedding / bias / readout / MLP gradients and the loss slot on a side stream (engine.backward
        calls this before the weight-gradient launch).  The window's sum goes into those ranges first."""
        lo, hi = self._gemm_grad_range
        self._add_window(0, lo)
        self._add_window(hi, self.numel)
        main = torch.cuda.current_stream()
        if self._ar_stream is None:
            self._ar_stream = torch.cuda.Stream(device=self.device)
        self._ar_stream.wait_stream(main)
        with torch.cuda.stream(self._ar_stream):
            dist.all_reduce(self.flat_g[:lo], op=dist.ReduceOp.SUM, group=self.pg)
            dist.all_reduce(self.flat_g[hi:], op=dist.ReduceOp.SUM, group=self.pg)      # ... b_ih, b_hh, gate, MLP, [loss]

    # ---- the batch paths (capture.CapturedBatches) and their hooks ----------------------------------------------------------
    def num_bucket_shapes(self) -> int:
        # keys start (kind, Nb, Eb, B, det, global batch): the phases of one shape count once
        return len({k[:6] for k in self._stream_slots if k[0] == "bucket"})

    def _prepare(self, batch):
        return self.module._prepare(batch)

    def _prepare_cache(self, cb):
        return cb, E.per_node_view(cb, cache_graph(cb)) if self._node else cache_graph(cb), cb.rows

    def _check_cache(self, cache, who: str) -> None:
        """A cache holds what a FROZEN encoder computes: a trainer that trains any encoder tensor refuses it."""
        if self._grad_ggnn:
            ntab = len(self.module._tables())
            names = [n for n, t in zip(encoder_names(self.module), self._trainable[:ntab + 6]) if t]
            raise ValueError(f"{who}: an EncoderCache holds the output of a frozen graph encoder, but this trainer trains the encoder "
                             f"tensor(s) {names}; freeze the embedding tables and the GatedGraphConv (requires_grad_(False)) before "
                             "building the trainer, or pass a GraphArena")

    def _key_suffix(self, ctx, B: int) -> tuple:
        global_batch, phase = ctx
        return (self._global_batch(global_batch, B),) + self._phase_key(phase)

    def prefetch(self, batch, global_batch: Optional[int] = None) -> None:
        """Starts the host->device copy of a (pinned) host batch on a side stream so that it overlaps the step that is running;
        the following ``step(batch)`` with the SAME batch object picks the staged copy up (with gradient accumulation: the very
        next micro-batch).  No-op without ``use_cuda_graph`` or for device batches."""
        self._prefetch(batch, (global_batch, self._phase()))

    def step_ids(self, arena, ids, global_batch: Optional[int] = None) -> torch.Tensor:
        """One optimisation step on the graphs ``ids`` of a device-resident :class:`deepdfa_b200.arena.GraphArena` (SURVEY.md §8
        f1: the batch producer).  With ``use_cuda_graph`` the batch is assembled into static per-shape buffers by
        ``ddfa_arena_batch`` inside one captured graph, so a step costs the H2D copy of the id list plus one graph launch;
        otherwise it is ``step(arena.batch(ids))``.  One micro-batch, as :meth:`step`.

        ``arena`` may also be an :class:`~deepdfa_b200.encoder_cache.EncoderCache` of this trainer's module when the trainer
        was built over a frozen encoder (embedding tables and GatedGraphConv with ``requires_grad=False``; ``ValueError``
        otherwise, naming the trainable encoder tensors).  The step is then the frozen step with the GGNN forward replaced by
        ``ddfa_cache_batch``, a gather of the graphs' cached rows; everything after it (readout or node head, loss, their
        backward, exchange, guard, Adam, metrics, accumulation) is unchanged.  The cache is checked against the module first
        (``EncoderCache.check``: ``ValueError`` when the encoder changed), so a captured step is never replayed over stale rows."""
        phase = self._begin()
        self._run_ids(arena, ids, (global_batch, phase), "step_ids")
        return self._end(phase)

    def step(self, batch, global_batch: Optional[int] = None) -> torch.Tensor:
        """One optimisation step on this rank's shard.  Returns the device tensor holding the
        global mean loss (valid after the step's stream work completes).  Starts with ``self.optimizer.step()``, which hands
        the current learning rate etc. to this step's Adam launch (an LR scheduler on ``self.optimizer`` sees that call).
        With ``accumulate_grad_batches=k > 1`` the call is one micro-batch: only the last of a window updates the parameters
        and calls ``optimizer.step()`` (see the constructor).  Host batches under ``use_cuda_graph`` run through static
        per-shape buffers (every phase of a shape has a slot of its own), device batches one captured graph per object."""
        phase = self._begin()
        self._run(batch, (global_batch, phase))
        return self._end(phase)

    # ------------------------------------------------------------------------------------
    @staticmethod
    def dp_self_check(engine: str, device, rank: int, world: int, steps: int = 5, graphs_per_rank: int = 24, nodes: int = 60,
                      exchange: str = "auto", label_style: str = "graph", factor: Optional[float] = None) -> dict:
        """On-hardware data-parallel parity (SURVEY.md §8(e) "Determinism"): ``steps`` optimisation steps of a global batch
        sharded over the ``world`` ranks (node-balanced shards of different sizes, NCCL all-reduce) against the same steps of
        the UNSHARDED batch on this rank alone, same seeds.  fp32 summation order is the only difference.  Collective: every
        rank must call it.  Returns the loss curves and the largest parameter difference after the last step.
        ``label_style="node"`` (``factor``: ``undersample_node_on_loss_factor``) also checks that every step's loss rows of
        this rank, mapped to the global batch, are the unsharded run's rows inside this shard (``rows_identical``)."""
        from . import synth
        from .batched_graph import split_batch
        feat = "_ABS_DATAFLOW_api_all_limitall_1000_limitsubkeys_1000"
        node = label_style == "node"
        style = dict(label_style="node", undersample_node_on_loss_factor=factor) if node else {}

        def make(distributed):
            torch.manual_seed(4321)
            m = FlowGNNGGNNModule(feat, 1002, 32, 8, 2, concat_all_absdf=True, positive_weight=4.0, engine=engine, **style).to(device)
            return m, FusedTrainer(m, distributed=distributed, exchange=exchange if distributed else "nccl")
        m_dp, tr_dp = make(True)
        m_1, tr_1 = make(False)
        l_dp, l_1, rows_ok = [], [], True
        for i in range(steps):
            b = synth.make_batch(graphs_per_rank * world, nodes, seed=900 + i, variable=True, vuln_rate=0.3)
            shard = split_batch(b, world)[rank]
            l_dp.append(float(tr_dp.step(shard.to(device), global_batch=b.batch_size)))
            l_1.append(float(tr_1.step(b.to(device), global_batch=b.batch_size)))
            if node:
                off, n = tr_dp.last_node_offset(), shard.num_nodes()
                r1 = tr_1.last_loss_rows().long()
                mine = r1[(r1 >= off) & (r1 < off + n)] - off
                rows_ok = rows_ok and torch.equal(tr_dp.last_loss_rows().long(), mine)
        dparam = max(float((p.data - q.data).abs().max()) for p, q in zip(m_dp.param_list(), m_1.param_list()))
        out = {"steps": steps, "world": world, "global_batch": graphs_per_rank * world, "loss_sharded": l_dp, "loss_single_rank": l_1,
               "max_abs_loss_diff": max(abs(a - b) for a, b in zip(l_dp, l_1)), "max_abs_param_diff": dparam,
               "shard_sizes_differ": True, "exchange": exchange}
        if node:
            out.update(label_style="node", factor=factor, rows_identical=bool(rows_ok))
        return out
