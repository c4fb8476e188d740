"""deepdfa_b200 — H100-native (sm_90a) implementation of DeepDFA's DDFA ``code_gnn`` GGNN hot path.

Public surface (mirrors the reference for this path only):
  FlowGNNGGNNModule   — drop-in for code_gnn.models.flow_gnn.ggnn.FlowGNNGGNNModule
  BatchedCFG, batch, unbatch, graph, add_self_loop, collate — the DGLGraph subset the path touches
  FusedTrainer        — data-parallel fused train step (NCCL gradient all-reduce + fused Adam)
  FusedEvaluator      — captured validation / test passes, metrics accumulated on the device
  binary_curves       — PR / ROC / binned PR curves, AUROC and average precision of device predictions, on the device
  FusedPredictor      — captured prediction over unlabeled functions: probabilities, top-k statements, embeddings
  EncoderCache        — a frozen graph encoder's output over a whole GraphArena, kept on the device for step_ids / update_ids / predict_ids
  synth.make_batch    — synthetic Big-Vul-shaped CFG batches

Importing the package does not load the CUDA library; the first kernel call does, and raises if
``deepdfa_b200/lib/libddfa_b200.so`` is missing (there is no CPU fallback).
"""
from .batched_graph import BatchedCFG, add_self_loop, as_batched_cfg, batch, collate, graph, unbatch  # noqa: F401
from .module import FlowGNNGGNNModule, allfeats  # noqa: F401
from .trainer import FusedTrainer  # noqa: F401
from .evaluator import FusedEvaluator, binary_curves  # noqa: F401
from .predictor import FusedPredictor  # noqa: F401
from .arena import ArenaBatch, GraphArena  # noqa: F401
from .encoder_cache import EncoderCache  # noqa: F401
from ._lib import DdfaError  # noqa: F401
from . import synth  # noqa: F401

__all__ = ["FlowGNNGGNNModule", "FusedTrainer", "FusedEvaluator", "binary_curves", "FusedPredictor", "GraphArena", "ArenaBatch", "EncoderCache", "BatchedCFG", "batch", "unbatch", "graph", "add_self_loop",
           "collate", "as_batched_cfg", "synth", "allfeats", "DdfaError"]
