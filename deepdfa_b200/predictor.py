"""Fused prediction over unlabeled code: per function its probability, its top-k statements and, for ``encoder_mode`` modules (the
DDFA half of LineVul / CodeT5 combined models), its pooled embedding, appended to a device result store in captured batches.

Per batch: the inference forward and the statement scores of :class:`~deepdfa_b200.evaluator.FusedEvaluator` (the same
kernels, through :class:`~deepdfa_b200.evaluator.InferencePass`), then ONE ``ddfa_predict_store`` call that writes the batch's
functions at a device cursor: the probability (graph style: sigmoid of the logit; node style: the maximum of the node
probabilities), the embedding, and the statements ranked by score with ``ddfa_stmt_metric``'s rule.  Nothing syncs with the host
until :meth:`FusedPredictor.results`, so a captured batch replays and appends.  No ``_VULN`` labels are read.
"""
from __future__ import annotations

from typing import Optional

import torch

from . import _lib
from . import engine as E
from .evaluator import InferencePass
from .module import FlowGNNGGNNModule


class FusedPredictor(InferencePass):
    def __init__(self, model: FlowGNNGGNNModule, capacity: int, statements: Optional[str] = None, top_k: int = 10,
                 use_cuda_graph: bool = True, bucket_nodes: int = 0, bucket_edges: int = 0, max_graph_shapes: int = 8,
                 bucket_min_pad_nodes: int = 64, max_resident_graphs: int = 64, ig_steps: int = 50, shap_samples: Optional[int] = None,
                 baseline_stdev: float = 0.0, noise_stdev: float = 0.0, attribution_seed: int = 0):
        """``capacity``: the functions the result store holds; more make :meth:`results` raise (the count stays complete).
        ``statements``: the per-statement score the top ``top_k`` (1 to 32) statements of each function are ranked by, one of
        ``FusedEvaluator``'s modes with the same meaning and the same ``ig_steps`` / ``shap_samples`` / ``baseline_stdev`` /
        ``noise_stdev`` / ``attribution_seed``: ``"probability"`` for node style, ``"attention"`` or a gradient mode for graph
        style, ``"attention"`` only for ``encoder_mode`` modules (graph style).  None stores no statements.
        ``use_cuda_graph``, ``bucket_nodes`` / ``bucket_edges`` / ``bucket_min_pad_nodes``, ``max_graph_shapes`` and
        ``max_resident_graphs``: the batch paths and capture policy of ``FusedEvaluator``.  The predictor reads the module's
        parameters where they live when a batch runs and never writes them or their ``.grad``; graphs captured over other
        parameter storage are recaptured."""
        if model.device.type != "cuda":
            raise _lib.DdfaError("FusedPredictor needs the module on a CUDA device (no CPU fallback)")
        hp = model.hparams
        if hp.label_style not in ("graph", "node"):
            raise ValueError(f"FusedPredictor: label_style={hp.label_style!r} is not supported ('graph' or 'node')")
        if hp.encoder_mode and hp.label_style != "graph":
            raise ValueError("FusedPredictor: an encoder_mode module with label_style='node' embeds nodes, not functions")
        if isinstance(capacity, bool) or int(capacity) != capacity or int(capacity) < 1:
            raise ValueError(f"capacity must be an integer >= 1, got {capacity!r}")
        if statements is not None and not 1 <= int(top_k) <= _lib.PREDICT_MAX_K:
            raise ValueError(f"top_k must be in [1, {_lib.PREDICT_MAX_K}], got {top_k!r}")
        self._init_inference(model, statements, ig_steps, shap_samples, baseline_stdev, noise_stdev, attribution_seed, use_cuda_graph,
                             bucket_nodes, bucket_edges, max_graph_shapes, bucket_min_pad_nodes, max_resident_graphs)
        self.capacity = int(capacity)
        self.top_k = int(top_k) if statements is not None else 0
        self._encoder = bool(hp.encoder_mode)
        C, k, dev = self.capacity, self.top_k, self.device
        with torch.cuda.device(dev):
            self._cursor = torch.zeros(2, dtype=torch.int64, device=dev)        # [0] stored, [1] dropped
            self._prob = None if self._encoder else torch.zeros(C, dtype=torch.float32, device=dev)
            self._emb = torch.zeros(C, model.out_dim, dtype=torch.float32, device=dev) if self._encoder else None
            self._top_idx = torch.zeros(C, k, dtype=torch.int32, device=dev) if k else None
            self._top_score = torch.zeros(C, k, dtype=torch.float32, device=dev) if k else None

    def reset(self) -> None:
        """Empties the result store in stream order: the next prediction goes to position 0."""
        self._cursor.zero_()

    def results(self) -> dict:
        """The store's device tensors, views of the functions predicted since the last :meth:`reset` in call order (graphs in
        batch order, bucket padding excluded): ``"prob"`` fp32 [F] (not for ``encoder_mode``), ``"embedding"`` fp32 [F, out_dim]
        (``encoder_mode`` only), and with ``statements`` ``"top_statements"`` int32 [F, top_k] (node indices local to each
        function, -1 past its last statement) and ``"top_scores"`` fp32 [F, top_k] (their scores, NaN past the last statement).
        Later predictions after a :meth:`reset` overwrite them.  One synchronisation.  The store is this process's: with several
        ranks, each holds the functions it predicted, and gathering them is the caller's.  Raises ``IndexError`` when a batch
        had node feature indices outside the embedding tables and ``ValueError`` when more functions than ``capacity`` were
        predicted."""
        stored, dropped, bad = torch.cat([self._cursor, self._oob.to(torch.int64)]).tolist()
        if bad:
            self._oob.zero_()
            raise IndexError(f"{bad} node feature indices outside [0, {self.module.input_dim}) in a predicted batch")
        if dropped:
            raise ValueError(f"FusedPredictor.results: {stored + dropped} functions predicted, capacity={self.capacity}: build the "
                             f"predictor with capacity >= {stored + dropped}")
        out = {}
        if self._prob is not None:
            out["prob"] = self._prob[:stored]
        if self._emb is not None:
            out["embedding"] = self._emb[:stored]
        if self.top_k:
            out["top_statements"] = self._top_idx[:stored]
            out["top_scores"] = self._top_score[:stored]
        return out

    def predict(self, batch) -> None:
        """Predicts one batch (host, resident device or DGL batch; ``(batch, extrafeats)`` tuples are accepted), labelled or not.
        No host synchronisation."""
        if isinstance(batch, tuple):
            batch = batch[0]
        self._run(batch, self._params())

    def predict_ids(self, arena, ids) -> None:
        """Predicts the graphs ``ids`` of a device-resident :class:`~deepdfa_b200.arena.GraphArena`, assembled inside the captured
        graph.  ``arena`` may also be an :class:`~deepdfa_b200.encoder_cache.EncoderCache` of this module, as for
        ``FusedEvaluator.update_ids``: only the readout / node head runs over the cached rows (``encoder_mode``: the embedding is
        the readout's pooled vector over them); ``statements=None``, ``"attention"`` or ``"probability"``."""
        self._run_ids(arena, ids, self._params(), "predict_ids")

    # ---- per batch -------------------------------------------------------------------------------------------------------
    def _vuln(self, g):
        return None         # no label is read: node style takes every valid node, and nothing else looks at _VULN

    def _enqueue(self, params, prepared, vuln, num_valid: Optional[int], valid_nodes: Optional[torch.Tensor]):
        """The inference forward and the scores of ``FusedEvaluator``, then ``ddfa_predict_store`` over functions [0, num_valid)
        (None: every graph of the batch)."""
        g, dg, idx, fptr = prepared
        scores = torch.empty(dg.num_nodes, dtype=torch.float32, device=self.device) if (self.statements or self._node) else None
        logits, extra = self._forward(params, prepared, vuln, valid_nodes, scores)
        self._scores(params, prepared, logits, scores)      # node style: the node probabilities, with or without statements
        B = fptr.numel() - 1
        pooled = extra if self._encoder else None
        E._call("ddfa_predict_store", None if self._node else E._p(logits), E._p(scores) if self._node else None, E._p(pooled),
                pooled.shape[1] if pooled is not None else 0, E._p(scores) if self.top_k else None, self.top_k, E._p(fptr), B,
                B if num_valid is None else int(num_valid), E._p(self._prob), E._p(self._emb), E._p(self._top_idx),
                E._p(self._top_score), self._cursor.data_ptr(), self.capacity, E._stream_ptr())
        return scores          # kept with a captured graph, which writes it on every replay

    def _after_run(self, scores, num_nodes: int) -> None:
        pass
