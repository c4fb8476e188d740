"""Fused evaluation of ``FlowGNNGGNNModule``: captured validation / test passes with the metrics accumulated on the device.

Replaces, for evaluation, Lightning's loop around ``BaseModule.validation_step`` / ``test_step`` (base_module.py:211-224,
238-323) and the torchmetrics objects the epoch ends compute (base_module.py:325-346, 348-383).  Per batch: the GGNN forward in
its inference form (``engine.forward(training=False)``: two rotating h buffers, no saved gates, no transposed CSR), the readout +
MLP (graph style) or the node head over every valid node (node style), then ONE metric kernel (``ddfa_eval_metrics_graph`` /
``ddfa_eval_metrics_rows``) that adds the batch's confusion counts, its mean BCE and, optionally, its probabilities and labels to
a persistent fp64 device state.  Nothing syncs with the host until :meth:`FusedEvaluator.compute`.

The batch paths are those of :class:`~deepdfa_b200.capture.CapturedBatches`, which :class:`~deepdfa_b200.trainer.FusedTrainer`
shares: host batches through static per-shape buffers (two sets, ``prefetch``) with optional shape bucketing, resident device
batches (one captured graph per object), graph ids of a :class:`~deepdfa_b200.arena.GraphArena` assembled inside the captured
graph, and eager launches beyond ``max_graph_shapes``.

Statement-level localisation (``statements=``): per batch, a score per node (CFG node = statement) and IVDetect's top-k statement
metric over them (DDFA/sastvd/helpers/evaluate.py:262-322), added by ``ddfa_stmt_metric`` to a second fp64 state.  The scores are
the node head's probability (node style), or, for the function logit of graph style, the readout's attention α_n, the saliency
Σ_d |∂logit/∂x_{n,d}|, the integrated gradients Σ_d x_{n,d} · mean_k ∂logit/∂x_{n,d}(α_k x), DeepLift / DeepLiftShap
Σ_d (x − x̄)_{n,d} · g̃_{n,d} (g̃: the gradient with the MLP head's ReLUs under the rescale rule, against a baseline forward on x̄) or
GradientShap's mean over samples of Σ_d (x̃ − b)_{n,d} · ∂logit/∂x_{n,d}(b + α(x̃ − b)), of the embedding output x.
"""
from __future__ import annotations

import numbers
from typing import Optional

import torch

from . import _lib
from . import engine as E
from .batched_graph import as_batched_cfg
from .capture import CapturedBatches, cache_graph
from .encoder_cache import CachedRows
from .module import FlowGNNGGNNModule, _ENGINES

# the fp64 words of the metric state (include/ddfa_b200.h, DDFA_EVAL_STATE_WORDS)
TP, FP, TN, FN, SAMPLES, BATCHES, LOSS_W, WEIGHT, STORED, OVERFLOW = range(10)
# the fp64 words of the statement metric state (DDFA_STMT_STATE_WORDS): hits at k = 1..10 are words S_HIT1 + k - 1
S_FUNCTIONS, S_VULN, S_HIT1, S_RANK_SUM, S_CLEAN, S_NAN, S_BATCHES = 0, 1, 2, 12, 13, 14, 15
STMT_TOP_K = 10
# statements= -> the label style it scores
STATEMENT_MODES = {"probability": "node", "attention": "graph", "saliency": "graph", "integrated_gradients": "graph",
                   "deeplift": "graph", "deeplift_shap": "graph", "gradient_shap": "graph"}
# the modes that run the dgrad-only backward, and those whose default sample count is captum's / the reference's
_GRADIENT_MODES = ("saliency", "integrated_gradients", "deeplift", "deeplift_shap", "gradient_shap")
_SHAP_SAMPLES = {"deeplift_shap": 16, "gradient_shap": 5}


def _ratio(num: float, den: float) -> float:
    return num / den if den > 0 else 0.0


def metrics_from_state(state, prefix: str = "val_") -> dict:
    """The metrics of a metric state (any float64 tensor or sequence of ``EVAL_STATE_WORDS`` values, e.g. a sum of the states of
    several ranks): torchmetrics < 0.10's binary defaults — micro average, 0 wherever a denominator is 0 — and Lightning's epoch
    mean of the batch losses weighted by the batch size (NaN when no batch had a sample).  Keys: ``{prefix}loss``,
    ``{prefix}Accuracy``, ``{prefix}Precision``, ``{prefix}Recall``, ``{prefix}F1Score``, ``{prefix}confusion`` =
    ``[[TN, FP], [FN, TP]]`` (sklearn's ``confusion_matrix`` layout) and ``{prefix}num_samples``."""
    s = [float(v) for v in (state.tolist() if torch.is_tensor(state) else state)]
    tp, fp, tn, fn = s[TP], s[FP], s[TN], s[FN]
    n = tp + fp + tn + fn
    precision, recall = _ratio(tp, tp + fp), _ratio(tp, tp + fn)
    return {f"{prefix}loss": s[LOSS_W] / s[WEIGHT] if s[WEIGHT] > 0 else float("nan"),
            f"{prefix}Accuracy": _ratio(tp + tn, n),
            f"{prefix}Precision": precision,
            f"{prefix}Recall": recall,
            f"{prefix}F1Score": _ratio(2.0 * tp, 2.0 * tp + fp + fn),
            f"{prefix}confusion": [[int(tn), int(fp)], [int(fn), int(tp)]],
            f"{prefix}num_samples": int(n)}


def _share(num: float, den: float) -> float:
    return num / den if den > 0 else float("nan")


def statement_metrics_from_state(state, prefix: str = "val_", node_style: bool = False) -> dict:
    """The statement metrics of a statement state (any float64 tensor or sequence of ``STMT_STATE_WORDS`` values, e.g. a sum over
    ranks), with the keys of evaluate.py:262-322: ``{prefix}stmt_top{k}`` (k = 1..10, ``eval_statements_list(..., vo=True)``: the
    share of vulnerable functions whose first vulnerable statement ranks among the first k), ``{prefix}stmt_ifa`` (the mean number
    of statements ranked above it, the initial false alarms), ``{prefix}stmt_vuln_functions`` and ``{prefix}stmt_functions``.
    ``node_style`` (scores are probabilities) adds ``{prefix}stmt_nonvuln_clean`` (the share of non-vulnerable functions with no
    probability > 0.5) and ``{prefix}stmt_all_top{k}`` (its product with top-k, ``vo=False``).  Unlike :func:`metrics_from_state`
    (0 wherever a denominator is 0), a share over no function is NaN: the reference divides by zero there."""
    s = [float(v) for v in (state.tolist() if torch.is_tensor(state) else state)]
    nv = s[S_VULN]
    out = {f"{prefix}stmt_top{k}": _share(s[S_HIT1 + k - 1], nv) for k in range(1, STMT_TOP_K + 1)}
    out[f"{prefix}stmt_ifa"] = _share(s[S_RANK_SUM], nv)
    out[f"{prefix}stmt_vuln_functions"] = int(nv)
    out[f"{prefix}stmt_functions"] = int(s[S_FUNCTIONS])
    if node_style:
        clean = _share(s[S_CLEAN], s[S_FUNCTIONS] - nv - s[S_NAN])
        out[f"{prefix}stmt_nonvuln_clean"] = clean
        out.update({f"{prefix}stmt_all_top{k}": out[f"{prefix}stmt_top{k}"] * clean for k in range(1, STMT_TOP_K + 1)})
    return out


# the int64 words of the curve info (include/ddfa_b200.h, DDFA_CURVE_INFO_WORDS)
C_DISTINCT, C_PR_POINTS, C_POSITIVES, C_NEGATIVES, C_NAN, C_BAD_LABELS, C_ONE_CLASS = range(7)


def _bin_thresholds(binned_thresholds, device) -> torch.Tensor:
    """The fp32 device thresholds of the binned curve.  An integer k gives BinnedPrecisionRecallCurve's default as recalled for
    torchmetrics < 0.10 (torchmetrics is not a dependency, so this is not checked against it): ``torch.linspace(0, 1.0, k)``,
    built in fp32 on the host and moved to the device.  Otherwise the given thresholds, compared with the probabilities as given."""
    if isinstance(binned_thresholds, numbers.Integral) and not isinstance(binned_thresholds, bool):
        if int(binned_thresholds) < 1:
            raise ValueError(f"binned_thresholds must be >= 1, got {binned_thresholds!r}")
        host = torch.linspace(0, 1.0, int(binned_thresholds), dtype=torch.float32)
        return host.pin_memory().to(device, non_blocking=True)
    t = torch.as_tensor(binned_thresholds)
    if t.dim() != 1 or t.numel() == 0 or not t.dtype.is_floating_point:
        raise ValueError(f"binned_thresholds: an int or a non-empty 1-D float sequence, got {binned_thresholds!r}")
    return t.to(device=device, dtype=torch.float32).contiguous()


def binary_curves(probs: torch.Tensor, labels: torch.Tensor, binned_thresholds=100) -> dict:
    """The threshold curves of fp32 CUDA probabilities and 0 / 1 labels, computed on the device (``ddfa_curve_sort`` /
    ``ddfa_curve_metrics``) with torchmetrics < 0.10's rules, as ``BaseModule.test_epoch_end`` (base_module.py:348-383) runs them:

    - ``pr_curve``: ``(precision, recall, thresholds)`` of ``PrecisionRecallCurve``.  Cut at the first threshold that reaches
      full recall, thresholds ascending, precision 1 / recall 0 appended (one point more than thresholds).  sklearn's
      ``precision_recall_curve`` does not cut, so it returns more points.
    - ``roc_curve``: ``(fpr, tpr, thresholds)`` of ``ROC``: a leading (0, 0) point at ``thresholds[1] + 1``, thresholds descending.
    - ``pr_curve_binned``: ``(precision, recall, thresholds)`` of ``BinnedPrecisionRecallCurve(1, thresholds=binned_thresholds)``:
      ``(TP + 1e-6) / (TP + FP + 1e-6)`` and ``TP / (TP + FN + 1e-6)`` at ``p >= t``, then 1 / 0 appended.
    - ``AUROC`` (trapezoids over the ROC curve) and ``AveragePrecision`` (``-Σ (r[k+1] - r[k]) · p[k]`` over the PR curve):
      Python floats, fp64 sums in a fixed order, bit-reproducible.

    Precision, recall, fpr and tpr are fp64 device tensors from the exact int64 counts; thresholds are the stored fp32 values bit
    for bit (a zero shows as +0.0: the reference ties -0.0 with +0.0).  One synchronisation.  For several ranks, ``all_gather``
    each rank's ``FusedEvaluator.predictions()`` and call this on the concatenation.  Raises ``DdfaError`` for tensors off the GPU
    and ``ValueError`` for no samples, NaN probabilities, labels other than 0 / 1, or a single class."""
    for name, t in (("probs", probs), ("labels", labels)):
        if not torch.is_tensor(t) or t.device.type != "cuda":
            raise _lib.DdfaError(f"binary_curves: {name} must be a CUDA tensor (there is no CPU path), got "
                                 f"{t.device if torch.is_tensor(t) else type(t).__name__}")
        if t.dtype != torch.float32 or t.dim() != 1:
            raise ValueError(f"binary_curves: {name} must be a 1-D float32 tensor, got {t.dtype} of shape {tuple(t.shape)}")
    if labels.device != probs.device or labels.numel() != probs.numel():
        raise ValueError(f"binary_curves: probs ({probs.numel()} on {probs.device}) and labels ({labels.numel()} on "
                         f"{labels.device}) differ")
    n = probs.numel()
    if n == 0:
        raise ValueError("binary_curves: no samples")
    dev = probs.device
    L = _lib.lib()
    with torch.cuda.device(dev):
        p, y = probs.contiguous(), labels.contiguous()
        bins = _bin_thresholds(binned_thresholds, dev)
        nb = bins.numel()
        ws = torch.empty(L.call("ddfa_curve_workspace_bytes", n), dtype=torch.uint8, device=dev)
        thr = torch.empty(n, dtype=torch.float32, device=dev)
        tps = torch.empty(n, dtype=torch.int64, device=dev)
        fps = torch.empty(n, dtype=torch.int64, device=dev)
        f64 = lambda k: torch.empty(k, dtype=torch.float64, device=dev)   # noqa: E731
        pr_p, pr_r, pr_t = f64(n + 1), f64(n + 1), torch.empty(n, dtype=torch.float32, device=dev)
        fpr, tpr, roc_t = f64(n + 1), f64(n + 1), torch.empty(n + 1, dtype=torch.float32, device=dev)
        bin_p, bin_r = f64(nb + 1), f64(nb + 1)
        words = f64(2 + _lib.CURVE_INFO_WORDS)        # [AUROC, AP] then the info words: one copy to the host
        summary, info = words[:2], words[2:].view(torch.int64)
        st = E._stream_ptr()
        E._call("ddfa_curve_sort", p.data_ptr(), y.data_ptr(), n, thr.data_ptr(), tps.data_ptr(), fps.data_ptr(), info.data_ptr(),
                ws.data_ptr(), ws.numel(), st)
        E._call("ddfa_curve_metrics", thr.data_ptr(), tps.data_ptr(), fps.data_ptr(), n, bins.data_ptr(), nb, pr_p.data_ptr(),
                pr_r.data_ptr(), pr_t.data_ptr(), fpr.data_ptr(), tpr.data_ptr(), roc_t.data_ptr(), bin_p.data_ptr(),
                bin_r.data_ptr(), summary.data_ptr(), info.data_ptr(), ws.data_ptr(), ws.numel(), st)
        host = words.cpu()
    auroc, ap = host[:2].tolist()
    w = host[2:].view(torch.int64).tolist()
    if w[C_NAN]:
        raise ValueError(f"binary_curves: {w[C_NAN]} of {n} probabilities are NaN")
    if w[C_BAD_LABELS]:
        raise ValueError(f"binary_curves: {w[C_BAD_LABELS]} of {n} labels are neither 0 nor 1")
    if w[C_ONE_CLASS]:
        raise ValueError(f"binary_curves: only one class present ({w[C_POSITIVES]} positives, {w[C_NEGATIVES]} negatives): the "
                         "ROC curve and AUROC are undefined")
    m, k = w[C_DISTINCT], w[C_PR_POINTS]
    return {"pr_curve": (pr_p[:k + 1], pr_r[:k + 1], pr_t[:k]),
            "roc_curve": (fpr[:m + 1], tpr[:m + 1], roc_t[:m + 1]),
            "pr_curve_binned": (bin_p, bin_r, bins),
            "AUROC": auroc,
            "AveragePrecision": ap}


class InferencePass(CapturedBatches):
    """The inference forward and the per-statement scores of one batch over the module's current parameters, on the batch paths
    of :class:`~deepdfa_b200.capture.CapturedBatches`: what :class:`FusedEvaluator` and
    :class:`~deepdfa_b200.predictor.FusedPredictor` enqueue before their own per-batch kernels.  The owner's ``__init__`` checks
    the module and calls :meth:`_init_inference`."""

    def _init_inference(self, model: FlowGNNGGNNModule, statements, ig_steps, shap_samples, baseline_stdev, noise_stdev,
                        attribution_seed, use_cuda_graph, bucket_nodes, bucket_edges, max_graph_shapes, bucket_min_pad_nodes,
                        max_resident_graphs) -> None:
        """Checks the statement settings (``FusedEvaluator``'s docstring describes them) against the module and allocates what
        the forward and the scores keep between batches.  An ``encoder_mode`` module (graph style) takes ``"attention"`` only:
        the gradient modes differentiate a logit."""
        who = type(self).__name__
        hp = model.hparams
        if statements is not None:
            if statements not in STATEMENT_MODES:
                raise ValueError(f"{who}: statements={statements!r} is not one of {sorted(STATEMENT_MODES)} or None")
            if hp.encoder_mode and statements != "attention":
                raise ValueError(f"{who}: an encoder_mode module has no logit to attribute: statements='attention' or None, "
                                 f"got {statements!r}")
            if STATEMENT_MODES[statements] != hp.label_style:
                raise ValueError(f"{who}: statements={statements!r} scores label_style={STATEMENT_MODES[statements]!r} "
                                 f"modules, this one has label_style={hp.label_style!r}")
        if int(ig_steps) < 1:
            raise ValueError(f"ig_steps must be >= 1, got {ig_steps!r}")
        if shap_samples is not None and int(shap_samples) < 1:
            raise ValueError(f"shap_samples must be >= 1, got {shap_samples!r}")
        for name, v in (("baseline_stdev", baseline_stdev), ("noise_stdev", noise_stdev)):
            if not float(v) >= 0.0 or float(v) == float("inf"):
                raise ValueError(f"{name} must be a finite value >= 0, got {v!r}")
        if float(baseline_stdev) > 0 and statements not in ("deeplift_shap", "gradient_shap"):
            raise ValueError(f"baseline_stdev applies to statements='deeplift_shap' / 'gradient_shap', not {statements!r}")
        if float(noise_stdev) > 0 and statements != "gradient_shap":
            raise ValueError(f"noise_stdev applies to statements='gradient_shap', not {statements!r}")
        if isinstance(attribution_seed, bool) or not isinstance(attribution_seed, numbers.Integral) or \
                not 0 <= int(attribution_seed) < 2 ** 64:
            raise ValueError(f"attribution_seed must be an integer in [0, 2**64), got {attribution_seed!r}")
        self.statements = statements
        self.ig_steps = int(ig_steps)
        self.shap_samples = int(shap_samples) if shap_samples is not None else _SHAP_SAMPLES.get(statements, 1)
        self.baseline_stdev, self.noise_stdev = float(baseline_stdev), float(noise_stdev)
        self.attribution_seed = int(attribution_seed)
        self.module = model
        self.device = model.device
        self._node = hp.label_style == "node"
        self.use_cuda_graph = bool(use_cuda_graph)
        self.bucket_nodes, self.bucket_edges, self.bucket_min_pad_nodes = int(bucket_nodes), int(bucket_edges), int(bucket_min_pad_nodes)
        self.max_graph_shapes = int(max_graph_shapes)
        self.max_resident_graphs = int(max_resident_graphs)
        dev = self.device
        with torch.cuda.device(dev):
            self._oob = torch.zeros(1, dtype=torch.int32, device=dev)        # out-of-range embedding indices (the owner raises)
            self._num_rows = torch.zeros(1, dtype=torch.int32, device=dev) if self._node else None
            # the gradients the dgrad chain computes inline (MLP, gate, GRU biases / w_hh) land here, never in the module's .grad
            self._grad_scratch = E.ParamPack.from_flat_list([torch.zeros_like(p) for p in model.param_list()], len(model._tables()),
                                                            model._num_layers) if self._attributes else None
            # the batch counter of the attribution draws (advanced once per attributed batch, inside a captured graph too)
            self._draws = torch.zeros(1, dtype=torch.int64, device=dev)
        self.ws = E.Workspace(dev)
        # DeepLift's baseline forwards keep their readout state here, apart from the input pass's saved state in self.ws
        self._ref_ws = E.Workspace(dev) if statements in ("deeplift", "deeplift_shap") else None
        self._param_key = None
        CapturedBatches.__init__(self)

    @property
    def _attributes(self) -> bool:
        return self.statements in _GRADIENT_MODES

    @property
    def attribution_draws(self) -> int:
        """Batches attributed so far by "deeplift", "deeplift_shap" or "gradient_shap" (the Philox batch counter of the next one).
        Reading it synchronises.
        Setting it writes the device word in stream order, so a run that restores it draws what an earlier run drew."""
        return int(self._draws.item())

    @attribution_draws.setter
    def attribution_draws(self, value: int):
        v = int(value)
        if v < 0:
            raise ValueError(f"attribution_draws must be >= 0, got {value!r}")
        self._draws.fill_(v)

    def _params(self):
        """A ParamPack over the module's current parameter storage; a change of storage drops every captured graph."""
        m = self.module
        plist = [p.data for p in m.param_list()]
        key = tuple(p.data_ptr() for p in plist)
        if key != self._param_key:
            if self._param_key is not None:
                self._drop_graphs()
            self._param_key = key
        return E.ParamPack.from_flat_list(plist, len(m._tables()), m._num_layers)

    def _prepare(self, graph):
        """The device graph without the transposed CSR (inference reads none; saliency and integrated gradients run the
        backward and ask for it), the per-node view in node style, the function-level graph_ptr and the embedding indices."""
        m = self.module
        g = as_batched_cfg(graph)
        dg = E.prepare_graph(g, self.device, need_transpose=self._attributes)
        fptr = dg.graph_ptr
        if self._node:
            dg = E.per_node_view(g, dg)
        idx = E.node_indices(g, m.concat_all_absdf, m.feature_keys["feature"], self.device)
        return g, dg, idx, fptr

    def _prepare_cache(self, cb):
        """A batch gathered from an encoder cache: its graph_ptr-only device graph (per node in node style), the function-level
        graph_ptr and the cached rows in place of the embedding indices."""
        dg = cache_graph(cb)
        return cb, E.per_node_view(cb, dg) if self._node else dg, cb.rows, dg.graph_ptr

    def _check_cache(self, cache, who: str) -> None:
        if self._attributes:
            raise ValueError(f"{who}: statements={self.statements!r} differentiates through the GGNN, which an EncoderCache "
                             "skips; pass a GraphArena, or use statements='attention', 'probability' or None")

    def _forward(self, params, prepared, vuln, valid_nodes: Optional[torch.Tensor], scores: Optional[torch.Tensor]):
        """The inference forward of one batch (``prepared``: what :meth:`_prepare` made of it) over ``params``.  Graph style:
        ``(logits [B] or None in encoder_mode, pooled [B, out_dim])``, the readout's attention written into ``scores`` with
        ``statements="attention"``.  Node style: ``(logits, rows)``, the node head over every valid node in order (``valid_nodes``:
        the int32 device word of the valid node count under bucketing, None: every node)."""
        g, dg, idx, fptr = prepared
        m, ws = self.module, self.ws
        eng = _ENGINES[m.engine]
        cached = isinstance(idx, CachedRows)       # an encoder cache's rows: no embedding, no GGNN launch
        if not self._node:
            att = scores if self.statements == "attention" else None
            if cached:
                pooled, logits, _ = E.readout_forward(params, dg, idx.x, idx.h, m.hparams.n_steps, training=False, alloc=ws,
                                                      attention=att)
            else:
                pooled, logits, _ = E.forward(params, dg, idx, m.hparams.n_steps, training=False, engine=eng, alloc=ws,
                                              oob_counter=self._oob, attention=att)
            return logits, pooled
        N = dg.num_nodes
        if cached:
            x, h_T = idx.x, idx.h
        else:
            x, h_T, _ = E.forward(params, dg, idx, m.hparams.n_steps, training=False, engine=eng, alloc=ws, head=False,
                                  oob_counter=self._oob)
        if valid_nodes is None:
            valid_nodes = ws.get("node_valid", (1,), torch.int32)
            valid_nodes.fill_(N)
        rows = ws.get("node_rows", (N,), torch.int32)
        E.node_sample(vuln, valid_nodes, None, 0, None, rows, self._num_rows, None, alloc=ws)
        logits, _ = E.node_head_fwd(params, x, h_T, rows, self._num_rows, alloc=ws)
        return logits, rows

    def _scores(self, params, prepared, logits, scores: Optional[torch.Tensor]) -> None:
        """The per-node scores :meth:`_forward` does not write into ``scores`` (None: none): the node head's probabilities in
        node style (rows = every valid node in order, so logits[n] is node n's), the gradient modes' attributions in graph style."""
        if scores is None:
            return
        g, dg, idx, fptr = prepared
        if self._node:
            E._call("ddfa_stmt_node_probability", E._p(logits), self._num_rows.data_ptr(), dg.num_nodes, E._p(scores), E._stream_ptr())
        elif self._attributes:
            self._attribute(params, dg, idx, scores)

    def _attribute(self, params, dg, idx, scores) -> None:
        """Saliency / integrated gradients / DeepLift(Shap) / GradientShap of every function's logit with respect to the
        embedding output x: training-form forwards and dgrad-only backwards (``grad_weights=False``) with dlogits = 1, the
        gradients of the weights going to a scratch pack.  Integrated gradients start the m forwards from α_k·x (x: the
        inference forward's embedding output, still in the workspace) and accumulate x·g / m; the others start them from the
        rows ``ddfa_stmt_shap_input`` writes and accumulate (x̃ − b)·g over their samples."""
        m, ws = self.module, self.ws
        eng = _ENGINES[m.engine]
        T = m.hparams.n_steps
        N, B = dg.num_nodes, dg.batch_size
        ones = ws.get("stmt_dlogits", (B,))
        ones.fill_(1.0)
        if self.statements == "saliency":
            _, _, saved = E.forward(params, dg, idx, T, training=True, engine=eng, alloc=ws)
            dh, dxd = E.backward(params, dg, saved, self._grad_scratch, dlogits=ones, engine=eng, alloc=ws, grad_weights=False)
            E._call("ddfa_stmt_input_grad_score", None, E._p(dh), E._p(dxd), N, dh.shape[1], _lib.STMT_SCORE_ABS, 1.0, 0,
                    E._p(scores), E._stream_ptr())
            return
        D = len(params.tables) * params.tables[0].shape[1]
        x0 = ws.get("x", (N, D))             # written by the inference forward of this batch; later passes write the same rows or none
        if self.statements == "integrated_gradients":
            steps = self.ig_steps
            for k in range(steps):
                _, _, saved = E.forward(params, dg, idx, T, training=True, engine=eng, alloc=ws, x_in=x0, x_scale=(k + 0.5) / steps)
                dh, dxd = E.backward(params, dg, saved, self._grad_scratch, dlogits=ones, engine=eng, alloc=ws, grad_weights=False)
                E._call("ddfa_stmt_input_grad_score", E._p(x0), E._p(dh), E._p(dxd), N, D, _lib.STMT_SCORE_X_TIMES, 1.0 / steps,
                        int(k > 0), E._p(scores), E._stream_ptr())
            return
        diff = ws.get("attr_diff", (N, D))

        def shap_input(x_src, alpha, noise, sample):
            def fill(out, image):
                E._call("ddfa_stmt_shap_input", E._p(x_src), E._p(dg.graph_ptr), B, N, D, float(alpha), float(noise),
                        self.baseline_stdev, self.attribution_seed, self._draws.data_ptr(), sample, E._p(out), E._p(diff),
                        E._p(image), E._stream_ptr())
            return fill

        if self.statements == "gradient_shap":
            # sample s: the plain gradient at b + α(x̃ − b) (x̃, b and α drawn), times x̃ − b
            S = self.shap_samples
            for s in range(S):
                _, _, saved = E.forward(params, dg, idx, T, training=True, engine=eng, alloc=ws,
                                        x_fill=shap_input(x0, -1.0, self.noise_stdev, s))
                dh, dxd = E.backward(params, dg, saved, self._grad_scratch, dlogits=ones, engine=eng, alloc=ws, grad_weights=False)
                E._call("ddfa_stmt_attribution_score", E._p(diff), E._p(dh), E._p(dxd), N, D, 1.0 / S, int(s > 0), E._p(scores),
                        E._stream_ptr())
        else:
            # DeepLift: one input pass; per baseline a forward from it (GGNN in its inference form, readout state kept in _ref_ws)
            # and the backward of the input pass with the head's ReLUs rescaled against it
            _, _, saved = E.forward(params, dg, idx, T, training=True, engine=eng, alloc=ws)
            J = self.shap_samples if self.statements == "deeplift_shap" and self.baseline_stdev > 0 else 1
            for j in range(J):
                _, _, ref = E.forward(params, dg, idx, T, training=True, grad_ggnn=False, engine=eng, alloc=self._ref_ws,
                                      x_fill=shap_input(saved.x, 0.0, 0.0, j))
                dh, dxd = E.backward(params, dg, saved, self._grad_scratch, dlogits=ones, engine=eng, alloc=ws, grad_weights=False,
                                     mlp_ref=(ref.pooled, ref.mlp_act))
                E._call("ddfa_stmt_attribution_score", E._p(diff), E._p(dh), E._p(dxd), N, D, 1.0 / J, int(j > 0), E._p(scores),
                        E._stream_ptr())
        self._draws.add_(1)

    def prefetch(self, batch) -> None:
        """Starts the host->device copy of a (pinned) host batch on a side stream, overlapping the batch that is running; the
        next call that runs the SAME batch object picks the staged copy up.  No-op without ``use_cuda_graph`` or for device
        batches."""
        self._prefetch(batch, None)


class FusedEvaluator(InferencePass):
    def __init__(self, model: FlowGNNGGNNModule, use_cuda_graph: bool = True, bucket_nodes: int = 0, bucket_edges: int = 0,
                 max_graph_shapes: int = 8, max_predictions: int = 0, bucket_min_pad_nodes: int = 64, max_resident_graphs: int = 64,
                 statements: Optional[str] = None, ig_steps: int = 50, shap_samples: Optional[int] = None,
                 baseline_stdev: float = 0.0, noise_stdev: float = 0.0, attribution_seed: int = 0):
        """``max_predictions`` > 0 keeps the first that many probabilities and labels (``predictions()``; the reference's
        ``test_preds`` / ``test_labels``); more samples than that make :meth:`compute` raise, the counts stay complete.
        ``bucket_nodes`` / ``bucket_edges``: shape bucketing of host batches under ``use_cuda_graph``, as in ``FusedTrainer``
        (one padding graph, excluded from every metric).  The evaluator reads the module's parameters where they live when a
        batch runs and never writes them; graphs captured over other parameter storage (a ``FusedTrainer`` built later moves
        the parameters into its flat buffer) are recaptured.
        ``statements``: the per-statement score of :meth:`last_scores` and of the statement metrics (``STATEMENT_MODES``):
        ``"probability"`` (node style: the node head's sigmoid), ``"attention"`` (graph style: the readout's softmax gate α_n,
        summing to 1 over each function), ``"saliency"`` (graph style: Σ_d |∂logit/∂x_{n,d}| of the embedding output x, captum's
        ``Saliency(abs=True)``) or ``"integrated_gradients"`` (graph style: Σ_d x_{n,d} · (1/m) Σ_{k<m} ∂logit/∂x_{n,d} at
        ((k + ½)/m)·x, m = ``ig_steps``, zero baseline: captum's ``IntegratedGradients(method="riemann_middle")``).  The target is
        each function's own logit; one backward with dlogits = 1 serves every function of the batch.  None (the default)
        enqueues nothing beyond the classification metrics.
        ``"deeplift"`` (graph style): captum's ``DeepLift(multiply_by_inputs=True)`` with a zero baseline x̄: Σ_d (x − x̄)_{n,d} ·
        g̃_{n,d}, g̃ the input gradient with each hidden ReLU of the MLP head under the rescale rule — its derivative replaced by
        (relu(z) − relu(z̄)) / (z − z̄), z̄ the pre-activation of a full forward of the same graph from x̄ — and every other
        nonlinearity (GRU gates, pooling softmax, gate products) a plain gradient at the input pass's activations, as captum
        hooks only ``nn.ReLU`` modules.  ``"deeplift_shap"``: captum's ``DeepLiftShap``, the mean of DeepLift over the baselines
        b_j = ``baseline_stdev`` · ε_j, j < ``shap_samples`` (default 16); with ``baseline_stdev`` = 0 (the default) every baseline
        is zero and DeepLift runs once, bit-identical to ``"deeplift"``.  ``"gradient_shap"``: captum's ``GradientShap``, the mean
        over ``shap_samples`` (default 5) samples s of Σ_d (x̃ − b) · ∂logit/∂x at b + α(x̃ − b), x̃ = x + ``noise_stdev`` · ε,
        b = ``baseline_stdev`` · ε' (zero by default) and α uniform in [0, 1) per function.  The draws are Philox4x32-10 with key
        ``attribution_seed`` and a device batch counter (``ddfa_stmt_shap_input``, :attr:`attribution_draws`), advanced once per
        batch these three modes attribute, so captured replays draw fresh values."""
        if model.device.type != "cuda":
            raise _lib.DdfaError("FusedEvaluator needs the module on a CUDA device (no CPU fallback)")
        hp = model.hparams
        if hp.encoder_mode or model._num_layers == 0:
            raise ValueError("FusedEvaluator: an encoder_mode module returns embeddings, not logits: there is nothing to score")
        if hp.label_style not in ("graph", "node"):
            raise ValueError(f"FusedEvaluator: label_style={hp.label_style!r} is not supported ('graph' or 'node')")
        if int(max_predictions) < 0:
            raise ValueError(f"max_predictions must be >= 0, got {max_predictions!r}")
        self._init_inference(model, statements, ig_steps, shap_samples, baseline_stdev, noise_stdev, attribution_seed, use_cuda_graph,
                             bucket_nodes, bucket_edges, max_graph_shapes, bucket_min_pad_nodes, max_resident_graphs)
        self.max_predictions = int(max_predictions)
        L = _lib.lib()
        dev = self.device
        with torch.cuda.device(dev):
            self._state = torch.zeros(_lib.EVAL_STATE_WORDS, dtype=torch.float64, device=dev)
            self._metric_ws = torch.empty(L.call("ddfa_eval_metrics_workspace_bytes"), dtype=torch.uint8, device=dev)
            cap = max(self.max_predictions, 1)
            self._probs = torch.zeros(cap, dtype=torch.float32, device=dev) if self.max_predictions else None
            self._labels = torch.zeros(cap, dtype=torch.float32, device=dev) if self.max_predictions else None
            self._stmt_state = torch.zeros(_lib.STMT_STATE_WORDS, dtype=torch.float64, device=dev)
            self._stmt_ws = torch.empty(L.call("ddfa_stmt_metric_workspace_bytes"), dtype=torch.uint8, device=dev) if statements else None
        self._last_scores = None

    # ---- the metric state ------------------------------------------------------------------------------------------------
    def reset(self) -> None:
        """Zeroes the metric state and the statement state in stream order (the prediction store starts over at position 0)."""
        self._state.zero_()
        self._stmt_state.zero_()

    def state(self) -> torch.Tensor:
        """The float64 device metric state (``EVAL_STATE_WORDS`` words, layout in include/ddfa_b200.h), a view: the evaluator
        keeps accumulating into it.  Every word is a sum, so ``dist.all_reduce(ev.state())`` adds ranks exactly (integers below
        2**53) and :meth:`metrics_from_state` turns the sum into the global metrics."""
        return self._state

    metrics_from_state = staticmethod(metrics_from_state)
    statement_metrics_from_state = staticmethod(statement_metrics_from_state)

    def statement_state(self) -> torch.Tensor:
        """The float64 device statement state (``STMT_STATE_WORDS`` words, layout in include/ddfa_b200.h, DDFA_STMT_STATE_WORDS),
        a view, separate from :meth:`state`.  Every word is an integer count, so ``dist.all_reduce(ev.statement_state())`` adds
        ranks exactly and :meth:`statement_metrics_from_state` turns the sum into the global statement metrics."""
        return self._stmt_state

    def last_scores(self) -> torch.Tensor:
        """The fp32 device scores ``[N]`` of the last batch's statements, in the batch's node order (without the padding graph's
        nodes under bucketing).  The next :meth:`update` overwrites them: copy them per batch to keep them."""
        if self.statements is None:
            raise ValueError("FusedEvaluator.last_scores: built with statements=None (no per-statement score)")
        if self._last_scores is None:
            raise ValueError("FusedEvaluator.last_scores: no batch was evaluated yet")
        return self._last_scores

    def compute(self, prefix: str = "val_") -> dict:
        """The metrics of everything evaluated since the last :meth:`reset` (one synchronisation).  Raises ``ValueError`` when
        no sample was evaluated or predictions overflowed ``max_predictions``, and ``IndexError`` when a batch had node feature
        indices outside the embedding tables."""
        s = self._state.cpu()
        bad = int(self._oob.item())
        if bad:
            self._oob.zero_()
            raise IndexError(f"{bad} node feature indices outside [0, {self.module.input_dim}) in an evaluated batch")
        n = int(s[TP] + s[FP] + s[TN] + s[FN])
        if n == 0:
            raise ValueError("FusedEvaluator.compute: no sample was evaluated since the last reset()")
        if self._probs is not None and s[OVERFLOW] > 0:
            raise ValueError(f"FusedEvaluator.compute: {n} predictions, max_predictions={self.max_predictions}: build the "
                             f"evaluator with max_predictions >= {n}")
        out = metrics_from_state(s, prefix)
        if self.statements is not None:
            ss = self._stmt_state.cpu()
            if ss[S_NAN] > 0:
                raise ValueError(f"FusedEvaluator.compute: {int(ss[S_NAN])} functions had a NaN statement score "
                                 f"(statements={self.statements!r})")
            out.update(statement_metrics_from_state(ss, prefix, node_style=self._node))
        return out

    def predictions(self):
        """``(probs, labels)``: fp32 device tensors of the first ``min(stored, max_predictions)`` samples in evaluation order
        (graph order, or node order within a batch).  Reads the stored count: one synchronisation."""
        if self._probs is None:
            raise ValueError("FusedEvaluator.predictions: built with max_predictions=0 (no prediction store)")
        k = int(self._state[STORED].item())
        return self._probs[:k], self._labels[:k]

    def curves(self, prefix: str = "test_", binned_thresholds=100) -> dict:
        """:func:`binary_curves` of :meth:`predictions`, with ``{prefix}`` keys: ``{prefix}pr_curve``, ``{prefix}roc_curve``,
        ``{prefix}pr_curve_binned``, ``{prefix}AUROC`` and ``{prefix}AveragePrecision`` — what ``test_epoch_end`` writes to
        ``pr.csv`` / ``pr_binned.csv``, and the two threshold-free scores.  Raises as :meth:`compute` does (no prediction store,
        nothing evaluated, overflow, node feature indices outside the tables) and as :func:`binary_curves` does.  The metric
        state is only read."""
        if self._probs is None:
            raise ValueError("FusedEvaluator.curves: built with max_predictions=0 (no prediction store)")
        s = self._state.cpu()
        bad = int(self._oob.item())
        if bad:
            raise IndexError(f"{bad} node feature indices outside [0, {self.module.input_dim}) in an evaluated batch")
        n = int(s[TP] + s[FP] + s[TN] + s[FN])
        if n == 0:
            raise ValueError("FusedEvaluator.curves: no sample was evaluated since the last reset()")
        if s[OVERFLOW] > 0:
            raise ValueError(f"FusedEvaluator.curves: {n} predictions, max_predictions={self.max_predictions}: build the "
                             f"evaluator with max_predictions >= {n}")
        k = int(s[STORED])
        out = binary_curves(self._probs[:k], self._labels[:k], binned_thresholds)
        return {f"{prefix}{key}": v for key, v in out.items()}

    # ---- per batch -------------------------------------------------------------------------------------------------------
    def _enqueue(self, params, prepared, vuln, num_valid: Optional[int], valid_nodes: Optional[torch.Tensor]):
        """Enqueues one batch (``prepared``: what :meth:`_prepare` made of it) over ``params``: the inference forward and the
        metric kernel, then, with ``statements``, the per-node scores and the statement metric.  ``num_valid``: graphs
        [num_valid, B) are bucket padding (the real ones are the batch's weight in the loss mean); ``valid_nodes``: the int32
        device word of the valid node count in node style under bucketing.  Returns the scores (None without ``statements``):
        a fresh [N] tensor, which a captured graph keeps writing on every replay."""
        g, dg, idx, fptr = prepared
        num_graphs = g.batch_size if num_valid is None else num_valid
        m = self.module
        pw = 1.0 if m.hparams.positive_weight is None else float(m.hparams.positive_weight)
        store = (E._p(self._probs), E._p(self._labels), self.max_predictions)
        mws = (self._metric_ws.data_ptr(), self._metric_ws.numel(), E._stream_ptr())
        L = _lib.lib()
        N = dg.num_nodes
        scores = torch.empty(N, dtype=torch.float32, device=self.device) if self.statements else None
        logits, rows = self._forward(params, prepared, vuln, valid_nodes, scores)
        if not self._node:
            B = dg.batch_size
            L.call("ddfa_eval_metrics_graph", E._p(logits), E._p(vuln), E._p(dg.graph_ptr), B, B if num_valid is None else int(num_valid),
                   pw, float(num_graphs), self._state.data_ptr(), *store, *mws)
        else:
            L.call("ddfa_eval_metrics_rows", E._p(logits), E._p(vuln), E._p(rows), self._num_rows.data_ptr(), N, pw, float(num_graphs),
                   self._state.data_ptr(), *store, *mws)
        self._scores(params, prepared, logits, scores)
        self._statement_metric(scores, vuln, fptr, num_valid)
        return scores

    def _statement_metric(self, scores, vuln, fptr, num_valid: Optional[int]) -> None:
        if self.statements is None:
            return
        B = fptr.numel() - 1
        mode = _lib.STMT_MODE_FULL if self._node else _lib.STMT_MODE_VULN_ONLY
        E._call("ddfa_stmt_metric", E._p(scores), E._p(vuln), E._p(fptr), B, B if num_valid is None else int(num_valid), mode, 0.5,
                self._stmt_state.data_ptr(), self._stmt_ws.data_ptr(), self._stmt_ws.numel(), E._stream_ptr())

    def update(self, batch) -> None:
        """Adds one batch (host, resident device or DGL batch; ``(batch, extrafeats)`` tuples as Lightning hands them over are
        accepted) to the metric state.  No host synchronisation."""
        if isinstance(batch, tuple):
            batch = batch[0]
        self._run(batch, self._params())

    def update_ids(self, arena, ids) -> None:
        """Adds the graphs ``ids`` of a device-resident :class:`~deepdfa_b200.arena.GraphArena` (assembled by
        ``ddfa_arena_batch`` inside the captured graph: the H2D copy of the id list plus one graph launch per batch).
        ``arena`` may also be an :class:`~deepdfa_b200.encoder_cache.EncoderCache` of this module: the batch's cached GGNN rows
        are gathered (``ddfa_cache_batch``) and only the readout / node head and the metrics run.  ``statements=None``,
        ``"attention"`` and ``"probability"`` only (the gradient modes raise ``ValueError``); ``ValueError`` when the module's
        encoder changed since the cache was built."""
        self._run_ids(arena, ids, self._params(), "update_ids")

    def _after_run(self, scores, num_nodes: int) -> None:
        self._last_scores = None if scores is None else scores[:num_nodes]

