"""``FlowGNNGGNNModule`` — the reference-facing module of the hot path.

Host-side mirror of ``DDFA/code_gnn/models/flow_gnn/ggnn.py:21-109`` (class, ctor argument order,
``forward(graph, extrafeats)``, ``out_dim``, ``hparams.label_style`` / ``hparams.encoder_mode``) and
of the step contract of ``DDFA/code_gnn/models/base_module.py`` (``get_label`` :83-95,
``training_step`` :171-199, ``validation_step`` :211-224, loss :72-74).  Parameters keep the
reference's ``state_dict`` names and shapes, so a reference checkpoint loads unchanged:

    all_embeddings.{api,datatype,literal,operator}.weight [V,H]   (or embedding.weight)
    ggnn.linears.0.{weight [D,D], bias [D]}
    ggnn.gru.{weight_ih [3D,D], weight_hh [3D,D], bias_ih [3D], bias_hh [3D]}      (gate order r,z,n)
    pooling.gate_nn.{weight [1,2D], bias [1]}
    output_layer.{0,2,4,...}.{weight, bias}

All arithmetic runs in libddfa_b200.so (hand-written sm_90a kernels) through the C ABI; the
torch modules below are parameter containers only and raise if called.  No CPU / DGL / PyTorch
compute fallback exists: a CPU graph is moved to the module's CUDA device, a CPU module raises.
"""
from __future__ import annotations

import logging
import os
from types import SimpleNamespace
from typing import Optional

import torch
from torch import nn

from . import engine as E
from ._lib import ENGINE_SIMT, ENGINE_TCGEN05, DdfaError
from .batched_graph import as_batched_cfg

logger = logging.getLogger(__name__)

allfeats = ["api", "datatype", "literal", "operator"]  # reference ggnn.py:17-19

_ENGINES = {"simt": ENGINE_SIMT, "tcgen05": ENGINE_TCGEN05}
MAX_HIDDEN_WIDTH = 512      # readout.cu (kMaxChunks = 4: D <= 512) and the embedding backward (K * H <= 512)
TCGEN05_WIDTH = 128         # the tensor-core GRU kernels with activation images and the fused backward are written for D == 128
# every width the tensor-core engine runs: 128, and the multiples of 64 from 192 up (gru_tc_wide.cu: the SIMT engine's data flow
# with its six GEMMs on the tensor cores)
TCGEN05_WIDTHS = (TCGEN05_WIDTH,) + tuple(range(192, MAX_HIDDEN_WIDTH + 1, 64))


def default_engine(hidden_width: int) -> str:
    """GEMM engine used when none is requested: the tcgen05 engine for the reference configuration (4 x 32 = 128
    hidden columns), the fp32 SIMT engine for every other width."""
    return "tcgen05" if hidden_width == 128 else "simt"


class _ParamsOnly(nn.Module):
    def forward(self, *a, **k):  # pragma: no cover - guard
        raise DdfaError(f"{type(self).__name__} is a parameter container; compute runs in libddfa_b200.so")


class GatedGraphConvParams(_ParamsOnly):
    """Parameter layout + init of dgl.nn.pytorch.GatedGraphConv(n_etypes=1) (call site ggnn.py:57-60)."""

    def __init__(self, in_feats, out_feats, n_steps, n_etypes=1):
        super().__init__()
        if n_etypes != 1:
            raise NotImplementedError("the reference uses n_etypes=1 (ggnn.py:60)")
        if in_feats > out_feats:
            raise ValueError("GatedGraphConv requires in_feats <= out_feats")
        self._in_feats, self._out_feats, self._n_steps = in_feats, out_feats, n_steps
        self.linears = nn.ModuleList([nn.Linear(out_feats, out_feats) for _ in range(n_etypes)])
        self.gru = nn.GRUCell(out_feats, out_feats, bias=True)
        self.reset_parameters()

    def reset_parameters(self):
        gain = nn.init.calculate_gain("relu")
        self.gru.reset_parameters()
        for linear in self.linears:
            nn.init.xavier_normal_(linear.weight, gain=gain)
            nn.init.zeros_(linear.bias)


class GlobalAttentionPoolingParams(_ParamsOnly):
    """Parameter layout of dgl.nn.pytorch.GlobalAttentionPooling(gate_nn) (call site ggnn.py:66-68)."""

    def __init__(self, gate_nn):
        super().__init__()
        self.gate_nn = gate_nn


class _GGNNFunction(torch.autograd.Function):
    """Whole hot path as one autograd node: forward and backward are hand-written kernels."""

    @staticmethod
    def forward(ctx, dg, idx, n_steps, engine, num_tables, num_layers, oob, need_grad, *flat):
        # need_grad is decided by the caller: ctx.needs_input_grad is True for Parameters even under torch.no_grad(), which
        # would run validation / test / inference in the training-mode forward (every per-step buffer kept)
        params = E.ParamPack.from_flat_list([t.detach() for t in flat], num_tables, num_layers)
        pooled, logits, saved = E.forward(params, dg, idx, n_steps, training=need_grad, engine=engine, oob_counter=oob)
        ctx.state = (params, dg, saved, engine, num_layers)
        return logits if num_layers > 0 else pooled

    @staticmethod
    def backward(ctx, dout):
        params, dg, saved, engine, num_layers = ctx.state
        grads = params.zeros_like()
        dout = dout.contiguous().float()
        if num_layers > 0:
            E.backward(params, dg, saved, grads, dlogits=dout, engine=engine)
        else:
            E.backward(params, dg, saved, grads, dpooled=dout, engine=engine)
        ctx.state = None
        return (None,) * 8 + tuple(grads.flat_list())


class _BCEFunction(torch.autograd.Function):
    """mean BCEWithLogits(pos_weight) over graphs with labels = segment-max of _VULN (base_module.py:72-95,183)."""

    @staticmethod
    def forward(ctx, logits, dg, vuln, pos_weight):
        B = dg.batch_size
        labels, loss, dlogits = E.graph_label_bce(dg, vuln, logits.detach().contiguous(), pos_weight, 1.0 / B, 1.0 / B, True)
        ctx.save_for_backward(dlogits)
        ctx.mark_non_differentiable(labels)
        return loss.reshape(()), labels

    @staticmethod
    def backward(ctx, dloss, _dlabels):
        (dlogits,) = ctx.saved_tensors
        return dlogits * dloss, None, None, None


class FlowGNNGGNNModule(nn.Module):
    """Drop-in for ``code_gnn.models.flow_gnn.ggnn.FlowGNNGGNNModule`` (reference ggnn.py:21-109).

    Extra keyword (not in the reference): ``engine`` = "simt" | "tcgen05" selects the GEMM engine of the
    GRU step (default: ``$DDFA_B200_ENGINE`` if set, else ``default_engine(W)``).  The hidden width W (``hidden_dim``, times 4
    with ``concat_all_absdf``) must be a multiple of 4 and at most 512; "tcgen05" runs W = 128 and W = 192, 256, ..., 512
    (``TCGEN05_WIDTHS``).  Both are checked here (``ValueError``).  The default stays "simt" at every width but 128.
    """

    def __init__(self, feat, input_dim, hidden_dim, n_steps, num_output_layers, label_style="graph",
                 concat_all_absdf=False, encoder_mode=False,
                 # BaseModule.__init__ (base_module.py:27-29)
                 undersample_node_on_loss_factor=None, test_every=False, tune_nni=False, positive_weight=None,
                 profile=False, time=False, engine: Optional[str] = None, **kwargs):
        super().__init__()
        if kwargs:
            raise TypeError(f"FlowGNNGGNNModule got unexpected keyword arguments {sorted(kwargs)}")
        self.hparams = SimpleNamespace(  # save_hyperparameters() (ggnn.py:34, base_module.py:30)
            feat=feat, input_dim=input_dim, hidden_dim=hidden_dim, n_steps=n_steps,
            num_output_layers=num_output_layers, label_style=label_style, concat_all_absdf=concat_all_absdf,
            encoder_mode=encoder_mode, undersample_node_on_loss_factor=undersample_node_on_loss_factor,
            test_every=test_every, tune_nni=tune_nni, positive_weight=positive_weight, profile=profile, time=time)
        self.class_threshold = 0.5  # base_module.py:32
        # base_module.py:72-74: the reference keeps BCEWithLogitsLoss(pos_weight) as a submodule, so a checkpoint
        # saved with positive_weight carries the buffer "loss_fn.pos_weight"; keep the same container/key.  The loss
        # itself is computed by ddfa_graph_label_bce.
        self.loss_fn = nn.BCEWithLogitsLoss(
            pos_weight=None if positive_weight is None else torch.tensor([positive_weight]))

        if "_ABS_DATAFLOW" in feat:  # ggnn.py:36-37
            feat = "_ABS_DATAFLOW"
        self.feature_keys = {"feature": feat}
        self.input_dim = input_dim
        self.concat_all_absdf = concat_all_absdf

        embedding_dim = hidden_dim
        if self.concat_all_absdf:  # ggnn.py:47-52
            self.all_embeddings = nn.ModuleDict({of: nn.Embedding(input_dim, embedding_dim) for of in allfeats})
            embedding_dim *= len(allfeats)
            hidden_dim *= len(allfeats)
        else:
            self.embedding = nn.Embedding(input_dim, embedding_dim)
        if embedding_dim % 4 != 0:
            raise ValueError(f"hidden width {embedding_dim} must be a multiple of 4 for the 128-bit kernels")
        self._D = hidden_dim
        self._H = embedding_dim // (len(allfeats) if self.concat_all_absdf else 1)

        self.ggnn = GatedGraphConvParams(in_feats=embedding_dim, out_feats=hidden_dim, n_steps=n_steps, n_etypes=1)
        output_in_size = embedding_dim + hidden_dim
        self.out_dim = output_in_size  # ggnn.py:64

        if label_style == "graph":
            self.pooling = GlobalAttentionPoolingParams(nn.Linear(output_in_size, 1))
        elif label_style == "node":
            # ggnn.py:101-107 without the pooling: the head runs on every node's [ggnn_out | feat_embed] row.  Same kernels:
            # every node is handed to the readout as a one-node graph — softmax over one node is exactly 1, so "pooled" is the
            # row itself — with an all-zero gate that is no parameter (the reference has no pooling module in this style).
            self.register_buffer("_node_gate_w", torch.zeros(1, output_in_size), persistent=False)
            self.register_buffer("_node_gate_b", torch.zeros(1), persistent=False)
        else:
            raise NotImplementedError(
                f"label_style={label_style!r}: the 'graph' (shipped) and 'node' styles are implemented on the CUDA path; the "
                "dataflow_solution_* styles (reference base_module.py:88-91) are not")

        self._num_layers = 0
        if not encoder_mode:  # ggnn.py:70-80
            layers = []
            for i in range(num_output_layers):
                last = i == num_output_layers - 1
                layers.append(nn.Linear(output_in_size, 1 if last else output_in_size))
                if not last:
                    layers.append(nn.ReLU())
            self.output_layer = nn.Sequential(*layers)
            self._num_layers = num_output_layers

        # the kernels cap the width: the readout holds a [h | x] row of 2 * W floats in four 128-float chunks per half, and the
        # embedding backward one K * H row per CTA; checked here rather than as a DdfaError from inside the first forward
        config = f"hidden_dim={self.hparams.hidden_dim}, concat_all_absdf={concat_all_absdf}"
        if hidden_dim > MAX_HIDDEN_WIDTH:
            raise ValueError(f"hidden width {hidden_dim} ({config}) exceeds {MAX_HIDDEN_WIDTH}, the widest the readout and embedding "
                             "kernels run")
        source = "engine argument"
        if engine is None:
            source = "DDFA_B200_ENGINE" if os.environ.get("DDFA_B200_ENGINE") else "default"
            engine = os.environ.get("DDFA_B200_ENGINE") or default_engine(hidden_dim)
        if engine not in _ENGINES:
            raise ValueError(f"engine must be one of {sorted(_ENGINES)}, got {engine!r}")
        if engine == "tcgen05" and hidden_dim not in TCGEN05_WIDTHS:
            widths = ", ".join(str(w) for w in TCGEN05_WIDTHS[:-1]) + f" and {TCGEN05_WIDTHS[-1]}"
            raise ValueError(f"engine='tcgen05' (from the {source}) runs hidden widths {widths} only, got {hidden_dim} ({config}); "
                             "use engine='simt'")
        self.engine = engine
        # Input validation (the reference raises on an out-of-range embedding index; DGL rejects edge ids >= num_nodes):
        #   "deferred" (default)     device-side counters, read without a host sync -> IndexError at the NEXT call / check_inputs()
        #   "sync" ($DDFA_B200_VALIDATE=1)   checked before forward returns (one device sync per call)
        #   "off"  ($DDFA_B200_VALIDATE=0)   indices are clamped / bad edges dropped silently
        self.validate_inputs = {"1": "sync", "0": "off"}.get(os.environ.get("DDFA_B200_VALIDATE", ""), "deferred")
        self._oob = None
        self._oob_host = None
        self._oob_pending = None

    # ---- parameter plumbing -----------------------------------------------------------------
    def _tables(self):
        if self.concat_all_absdf:
            return [self.all_embeddings[of].weight for of in allfeats]
        return [self.embedding.weight]

    def _mlp_linears(self):
        if self._num_layers == 0:
            return []
        return [m for m in self.output_layer if isinstance(m, nn.Linear)]

    def param_list(self):
        """Parameters in ParamPack.flat_list() order."""
        lin, gru = self.ggnn.linears[0], self.ggnn.gru
        gate_w, gate_b = ((self.pooling.gate_nn.weight, self.pooling.gate_nn.bias) if self.hparams.label_style == "graph"
                          else (self._node_gate_w, self._node_gate_b))
        mlp = self._mlp_linears()
        return [*self._tables(), lin.weight, lin.bias, gru.weight_ih, gru.weight_hh, gru.bias_ih, gru.bias_hh,
                gate_w, gate_b, *[m.weight for m in mlp], *[m.bias for m in mlp]]

    @property
    def device(self):
        return self.ggnn.gru.weight_ih.device

    def _prepare(self, graph):
        dev = self.device
        if dev.type != "cuda":
            raise DdfaError("FlowGNNGGNNModule (deepdfa_b200) must live on a CUDA device (H100); move it with .cuda(). "
                            "There is no CPU fallback.")
        g = as_batched_cfg(graph)
        dg = E.prepare_graph(g, dev, need_transpose=True)
        if self.hparams.label_style == "node":
            dg = E.per_node_view(g, dg)
        idx = E.node_indices(g, self.concat_all_absdf, self.feature_keys["feature"], dev)
        return g, dg, idx

    # ---- reference API ----------------------------------------------------------------------
    def forward(self, graph, extrafeats=None):
        """ggnn.py:82-109.  Returns logits [B] (0-d for a single graph, like ``.squeeze()``) or, in
        encoder_mode, the pooled embedding [B, out_dim]."""
        g, dg, idx = self._prepare(graph)
        self._raise_deferred_input_errors()
        if self.validate_inputs != "off" and self._oob is None:
            with torch.cuda.device(self.device):
                self._oob = torch.zeros(1, dtype=torch.int32, device=self.device)
                self._oob_host = torch.zeros(1, dtype=torch.int32).pin_memory()
        flat = self.param_list()
        need_grad = torch.is_grad_enabled() and any(p.requires_grad for p in flat)
        with torch.cuda.device(self.device):
            out = _GGNNFunction.apply(dg, idx, self.hparams.n_steps, _ENGINES[self.engine], len(self._tables()),
                                      self._num_layers, self._oob, need_grad, *flat)
            if self.validate_inputs == "sync":
                self._check_inputs_now(dg)
            elif self.validate_inputs == "deferred":
                # no host sync on the hot path: the counters travel to pinned host memory behind the kernels and are looked at
                # by the NEXT call (or by check_inputs()), which raises for this batch one step late
                self._oob_host.copy_(self._oob, non_blocking=True)
                ev = torch.cuda.Event()
                ev.record()
                self._oob_pending = (ev, dg)
        if self.hparams.encoder_mode:
            return out
        return out.squeeze()

    # ---- input validation ------------------------------------------------------------------
    def _check_inputs_now(self, dg):
        bad = int(self._oob.item())
        dropped = int(dg._csr_ws[:4].view(torch.int32).item()) if getattr(dg, "_csr_ws", None) is not None else 0
        if bad:
            self._oob.zero_()
            raise IndexError(f"{bad} node feature indices outside [0, {self.input_dim})")
        if dropped:
            raise IndexError(f"{dropped} edges with an endpoint outside [0, num_nodes) were dropped by ddfa_build_csr")

    def _raise_deferred_input_errors(self, wait: bool = False):
        pend = self._oob_pending
        if pend is None:
            return
        ev, dg = pend
        if wait:
            ev.synchronize()
        elif not ev.query():
            return
        self._oob_pending = None
        bad = int(self._oob_host[0])
        if bad:
            self._oob.zero_()
            self._oob_host.zero_()
            raise IndexError(f"{bad} node feature indices outside [0, {self.input_dim}) in an earlier batch")
        if getattr(dg, "_csr_ws", None) is not None:
            dropped = int(dg._csr_ws[:4].view(torch.int32).item())      # the event has completed: this read does not wait
            if dropped:
                raise IndexError(f"{dropped} edges with an endpoint outside [0, num_nodes) were dropped by ddfa_build_csr in an earlier batch")

    def check_inputs(self):
        """Waits for the last forward's validation counters and raises IndexError if that batch had out-of-range node
        feature indices or edge endpoints (validate_inputs == "deferred")."""
        self._raise_deferred_input_errors(wait=True)

    def get_label(self, batch):
        """base_module.py:83-95: graph style — per-graph max of ndata['_VULN'] as float, a fused segment-max kernel instead of
        dgl.unbatch + a Python loop; node style — ndata['_VULN'] as float (the same kernel over one-node segments)."""
        g, dg, _ = self._prepare(batch)
        vuln = g.ndata["_VULN"].to(self.device, non_blocking=True)
        with torch.cuda.device(self.device):
            labels, _, _ = E.graph_label_bce(dg, vuln, None, 1.0, 0.0, 0.0, False)
        return labels

    def loss_and_labels(self, batch, out):
        g, dg, _ = self._prepare(batch)
        vuln = g.ndata["_VULN"].to(self.device, non_blocking=True)
        pw = 1.0 if self.hparams.positive_weight is None else float(self.hparams.positive_weight)
        if out.dim() == 0:
            out = out.unsqueeze(0)
        with torch.cuda.device(self.device):
            loss, labels = _BCEFunction.apply(out, dg, vuln, pw)
        return loss, labels

    def resample(self, batch, out, label):
        """base_module.py:96-135 without the Lightning logging (node style): keep every vulnerable node and
        ``round(#vulnerable * undersample_node_on_loss_factor)`` non-vulnerable ones drawn with ``random.sample``.  Like the
        reference this reads the labels on the host (one sync); it is not part of the shipped (graph-style) configuration."""
        import random
        vuln_indices = label.nonzero().flatten().tolist()
        num_indices_to_sample = round(len(vuln_indices) * self.hparams.undersample_node_on_loss_factor)
        nonvuln_indices = random.sample((label == 0).nonzero().flatten().tolist(), num_indices_to_sample)
        indices = vuln_indices + nonvuln_indices
        return out[indices], label[indices]

    def training_step(self, batch_data, batch_idx=0):
        """base_module.py:171-199 without the Lightning logging: returns the loss tensor."""
        batch, extrafeats = batch_data
        out = self.forward(batch, extrafeats)
        if self.hparams.label_style == "node" and self.hparams.undersample_node_on_loss_factor is not None:
            # base_module.py:178-183: the loss over the resampled subset of nodes is the reference's own torch expression on a
            # short vector (self.loss_fn); gradients reach the kernels' backward through the indexing
            out, label = self.resample(batch, out, self.get_label(batch))
            return self.loss_fn(out, label)
        loss, _ = self.loss_and_labels(batch, out)
        return loss

    def validation_step(self, batch_data, batch_idx=0, dataloader_idx=0):
        """base_module.py:211-224: returns (loss, sigmoid(out), int labels)."""
        batch, extrafeats = batch_data
        with torch.no_grad():
            out = self.forward(batch, extrafeats)
            loss, labels = self.loss_and_labels(batch, out)
            if out.dim() == 0:
                out = out.unsqueeze(0)
            return loss, torch.sigmoid(out), labels.int()

    # ---- profiling / timing records in the reference's schema (SURVEY.md §8 f4) --------------------------------------
    def analytic_counts(self, num_nodes: int, batch_size: int):
        """(flops, macs, params) of one forward pass in the REFERENCE formulation (what its DeepSpeed FlopsProfiler run,
        base_module.py:76-77,259-272, reports for the module tree): per node and propagation step D*D MACs for
        GatedGraphConv.linears[0] plus 6*D*D for the GRUCell; the gate Linear(2D, 1) per node; the MLP head per graph.
        Embedding lookups and elementwise work are not counted; flops = 2 * macs."""
        D, T = self._D, self.hparams.n_steps
        macs = num_nodes * T * 7 * D * D + num_nodes * 2 * D
        if not self.hparams.encoder_mode:
            dims = [2 * D] * self._num_layers + [1] if self._num_layers > 0 else []
            macs += batch_size * sum(a * b for a, b in zip(dims[:-1], dims[1:]))
        params = sum(p.numel() for p in self.parameters())
        return 2 * macs, macs, params

    @staticmethod
    def _count_str(x: float) -> str:
        """'<number> <unit>' with the units scripts/report_profiling.py parses (G / M / K)."""
        for unit, scale in (("G", 1e9), ("M", 1e6), ("K", 1e3)):
            if x >= scale:
                return f"{x / scale:.2f} {unit}"
        return f"{x:.2f} K" if x == 0 else f"{x / 1e3:.4f} K"

    def test_step(self, batch_data, batch_idx=0):
        """base_module.py:238-321 without the torchmetrics bookkeeping: returns (loss, sigmoid(out), int labels).  With
        ``time=True`` (``--model.time True``, scripts/run_profiling.sh) every step after the third appends
        ``{"step", "batch_size", "runtime"}`` (CUDA-event milliseconds around ``forward``) to ``timedata.jsonl``; with
        ``profile=True`` it appends ``{"step", "flops", "params", "macs", "batch_size"}`` to ``profiledata.jsonl`` — the files
        ``scripts/report_profiling.py`` reads.  The counts are analytic (``analytic_counts``), not instrumented."""
        import json
        import os
        batch, extrafeats = batch_data
        do_profile = bool(self.hparams.profile) and batch_idx > 2
        do_time = bool(self.hparams.time) and batch_idx > 2
        with torch.no_grad():
            labels = self.get_label(batch)
            if do_time:
                start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                start.record()
            out = self.forward(batch, extrafeats)
            if do_time:
                end.record()
            record, filename = None, None
            if do_profile:
                g = as_batched_cfg(batch)
                flops, macs, params = self.analytic_counts(g.num_nodes(), g.batch_size)
                record = {"step": batch_idx, "flops": self._count_str(flops), "params": self._count_str(params),
                          "macs": self._count_str(macs), "batch_size": int(labels.numel())}
                filename = "profiledata.jsonl"
            elif do_time:
                torch.cuda.synchronize()
                record = {"step": batch_idx, "batch_size": int(labels.numel()), "runtime": start.elapsed_time(end)}
                filename = "timedata.jsonl"
            if filename is not None:
                with open(os.path.join(getattr(self, "profile_output_dir", "."), filename), "a") as f:
                    f.write(json.dumps(record))
                    f.write("\n")
            loss, labels = self.loss_and_labels(batch, out)
            if out.dim() == 0:
                out = out.unsqueeze(0)
            return loss, torch.sigmoid(out), labels.int()

    def configure_optimizers(self, lr=1e-3, weight_decay=1e-2):
        """config_default.yaml:43-47 (torch.optim.Adam, coupled L2).  The fused CUDA optimizer is
        ``deepdfa_b200.trainer.FusedTrainer``; this returns the stock optimizer for drop-in scripts."""
        return torch.optim.Adam(self.parameters(), lr=lr, weight_decay=weight_decay)

    def freeze_graph(self):  # base_module.py:80-81
        logger.warning("freeze_graph not implemented")
