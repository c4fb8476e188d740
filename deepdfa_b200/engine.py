"""Host-side driver of the hot path: graph preparation, forward, backward — all device work is
done by libddfa_b200.so through the C ABI (deepdfa_b200._lib); torch only owns device memory
and streams.  There is no CPU path: every entry raises if the tensors are not on a CUDA device.

Mirrors the control flow of the reference ``FlowGNNGGNNModule.forward``
(DDFA/code_gnn/models/flow_gnn/ggnn.py:82-109) with DGL's GatedGraphConv / GlobalAttentionPooling
replaced by the kernels documented in include/ddfa_b200.h.
"""
from __future__ import annotations

import os

from dataclasses import dataclass, field
from typing import List, Optional

import torch

from . import _lib
from ._lib import ENGINE_SIMT, ENGINE_TCGEN05, DdfaError, ptr_array
from .batched_graph import ABS_DATAFLOW_SUBKEYS, BatchedCFG, as_batched_cfg


def _stream_ptr() -> int:
    return torch.cuda.current_stream().cuda_stream


def _p(t: Optional[torch.Tensor]) -> int:
    return 0 if t is None else t.data_ptr()


# Execution options of the backward pass (A/B switches for scripts and tests; both settings of each run the CUDA kernels):
#   fuse_gather_bwd: the transposed edge gather of step t+1's ds rides in step t's gate_bwd launch (tcgen05 engine)
#   batched_wgrad:   ONE weight-gradient launch over all T steps instead of a deferred accumulation per step
#   packed_state:    tcgen05 engine: h_t kept only as its activation image and the saved gates as packed 64-bit words (round-2 form, the
#                    default); False = the round-1 form (fp32 copy of every h_t, four fp32 gate planes) for whole-step A/Bs
OPTIONS = {"fuse_gather_bwd": os.environ.get("DDFA_FUSE_GATHER_BWD", "1") != "0",
           "batched_wgrad": os.environ.get("DDFA_BATCHED_WGRAD", "1") != "0",
           "packed_state": os.environ.get("DDFA_PACKED_STATE", "1") != "0"}

# Optional timing hook (bench.py): an object with begin(name) / end(name) that records CUDA events
# on the current stream around selected C-ABI calls.  None (default) costs nothing.
profile_hook = None


def _call(name, *args, tag=None):
    """lib().call with the optional profiling span."""
    hook = profile_hook
    if hook is None or not hook.wants(tag or name):
        return _lib.lib().call(name, *args)
    hook.begin(tag or name)
    try:
        return _lib.lib().call(name, *args)
    finally:
        hook.end(tag or name)


def _require_cuda(*tensors):
    for t in tensors:
        if t is not None and not t.is_cuda:
            raise DdfaError("deepdfa_b200 runs on CUDA (sm_90a) only: got a CPU tensor; there is no CPU fallback")


# ------------------------------------------------------------------------------------------
# Graph structure on the device
# ------------------------------------------------------------------------------------------
@dataclass
class DeviceGraph:
    """CSR (by destination) + transposed CSR + graph segment pointers, all int32 on the device."""
    num_nodes: int
    num_edges: int
    batch_size: int
    indptr: torch.Tensor
    indices: torch.Tensor
    indptr_t: torch.Tensor
    indices_t: torch.Tensor
    graph_ptr: torch.Tensor
    device: torch.device


def per_node_view(g, dg: DeviceGraph) -> DeviceGraph:
    """The same batch with every node as its own one-node graph (graph_ptr = 0..N): what label_style="node" hands to the readout /
    label kernels (ggnn.py:101-107 without the pooling, base_module.py:84-85).  Cached on the graph object."""
    key = f"devgraph_nodes:{dg.device}"
    view = g._cache.get(key)
    if view is None or view.indptr is not dg.indptr:
        with torch.cuda.device(dg.device):
            ptr = torch.arange(dg.num_nodes + 1, dtype=torch.int32, device=dg.device)
        view = DeviceGraph(dg.num_nodes, dg.num_edges, dg.num_nodes, dg.indptr, dg.indices, dg.indptr_t, dg.indices_t, ptr, dg.device)
        view._csr_ws = getattr(dg, "_csr_ws", None)
        g._cache[key] = view
    return view


def prepare_graph(g, device=None, need_transpose: bool = True) -> DeviceGraph:
    """COO (as handed over by DGL / BatchedCFG) -> DeviceGraph, entirely on the device, no host sync.
    Cached on the graph object."""
    g = as_batched_cfg(g)
    device = torch.device(device) if device is not None else g.device
    if device.type != "cuda":
        raise DdfaError("prepare_graph: target device must be CUDA; deepdfa_b200 has no CPU path")
    key = f"devgraph:{device}:{int(need_transpose)}"
    cached = g._cache.get(key) or g._cache.get(f"devgraph:{device}:1")
    if cached is not None:
        return cached
    src, dst = g.edges()
    src = src.to(device, non_blocking=True)
    dst = dst.to(device, non_blocking=True)
    bnn = g.batch_num_nodes().to(device=device, dtype=torch.int64, non_blocking=True)
    if src.dtype not in (torch.int64, torch.int32) or dst.dtype != src.dtype:
        src, dst = src.to(torch.int64), dst.to(torch.int64)
    src, dst = src.contiguous(), dst.contiguous()
    N, E, B = g.num_nodes(), g.num_edges(), g.batch_size
    L = _lib.lib()
    with torch.cuda.device(device):
        indptr = torch.empty(N + 1, dtype=torch.int32, device=device)
        indices = torch.empty(max(E, 1), dtype=torch.int32, device=device)
        if need_transpose:
            indptr_t = torch.empty(N + 1, dtype=torch.int32, device=device)
            indices_t = torch.empty(max(E, 1), dtype=torch.int32, device=device)
        else:
            indptr_t = indices_t = None
        graph_ptr = torch.empty(B + 1, dtype=torch.int32, device=device)
        ws_bytes = L.call("ddfa_build_csr_workspace_bytes", E, N)
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device=device)
        st = _stream_ptr()
        L.call("ddfa_build_csr", _p(src), _p(dst), src.element_size(), E, N, _p(indptr), _p(indices),
               _p(indptr_t), _p(indices_t), _p(ws), ws_bytes, st)
        L.call("ddfa_graph_ptr", _p(bnn), B, _p(graph_ptr), st)
    dg = DeviceGraph(N, E, B, indptr, indices, indptr_t, indices_t, graph_ptr, device)
    dg._csr_ws = ws  # keep the error counter alive (ws[0:4] = dropped-edge count)
    g._cache[key] = dg
    return dg


# ------------------------------------------------------------------------------------------
# Parameters
# ------------------------------------------------------------------------------------------
@dataclass
class ParamPack:
    """Tensors of one FlowGNNGGNNModule, in the reference's state_dict naming (SURVEY.md §5):
    tables: all_embeddings.{api,datatype,literal,operator}.weight (or [embedding.weight]);
    w_msg/b_msg: ggnn.linears.0.{weight,bias}; w_ih/w_hh/b_ih/b_hh: ggnn.gru.*;
    w_gate/b_gate: pooling.gate_nn.{weight,bias}; mlp_w/mlp_b: output_layer.{0,2,..}.{weight,bias}."""
    tables: List[torch.Tensor]
    w_msg: torch.Tensor
    b_msg: torch.Tensor
    w_ih: torch.Tensor
    w_hh: torch.Tensor
    b_ih: torch.Tensor
    b_hh: torch.Tensor
    w_gate: torch.Tensor
    b_gate: torch.Tensor
    mlp_w: List[torch.Tensor] = field(default_factory=list)
    mlp_b: List[torch.Tensor] = field(default_factory=list)

    def flat_list(self) -> List[torch.Tensor]:
        return [*self.tables, self.w_msg, self.b_msg, self.w_ih, self.w_hh, self.b_ih, self.b_hh,
                self.w_gate, self.b_gate, *self.mlp_w, *self.mlp_b]

    @staticmethod
    def from_flat_list(ts, num_tables: int, num_layers: int) -> "ParamPack":
        ts = list(ts)
        k = num_tables
        return ParamPack(ts[:k], *ts[k:k + 8], mlp_w=ts[k + 8:k + 8 + num_layers],
                         mlp_b=ts[k + 8 + num_layers:k + 8 + 2 * num_layers])

    def zeros_like(self) -> "ParamPack":
        return ParamPack.from_flat_list([torch.zeros_like(t) for t in self.flat_list()], len(self.tables), len(self.mlp_w))


@dataclass
class Saved:
    """Activations kept between forward and backward."""
    T: int
    D: int
    x: torch.Tensor
    h: List[Optional[torch.Tensor]]  # h[0..T] fp32; tcgen05 engine: only h[0] = x and h[T], the others live as images (None here)
    s: List[torch.Tensor]            # s[0..T-1] (tcgen05: activation images)
    gates: List[torch.Tensor]        # per step: [4,N,D] fp32 planes (simt) or packed 64-bit words (tcgen05)
    w_fold: torch.Tensor
    b_fold: torch.Tensor
    pooled: torch.Tensor
    gate_logit: torch.Tensor
    seg_max: torch.Tensor
    seg_sum: torch.Tensor
    mlp_act: Optional[torch.Tensor]
    idx: List[torch.Tensor]
    h_img: Optional[List[torch.Tensor]] = None   # tcgen05 engine: activation images of h[0..T-1]


class Workspace:
    """Grow-only named device buffers (used by the fused trainer to avoid per-step allocation).

    A captured CUDA graph bakes in the raw pointers of the buffers it was captured with.  When a larger batch shape makes a
    buffer grow, the old block is therefore RETIRED, not freed: it stays alive (``_retired``) for as long as the workspace
    does, so a graph captured earlier keeps replaying over memory that is still its own (a step produces every intermediate
    it reads, so the retired block needs no content).  Growth is geometric (x1.25) to bound the number of retired blocks;
    ``generation`` counts reallocations (tests)."""

    def __init__(self, device, scrub_image_tails: bool = False):
        """``scrub_image_tails``: clear, on every request, the last tile of each image whose producer leaves padding rows
        unwritten (``get_image(..., tail_unwritten=True)``).  A trainer that skips non-finite steps and carries on needs this: a
        skipped step can leave NaN in rows that a later, smaller batch treats as padding."""
        self.device = device
        self.scrub_image_tails = bool(scrub_image_tails)
        self._bufs = {}
        self._retired = []
        self.generation = 0

    def _get(self, name, shape, dtype, zeroed):
        numel = 1
        for s in shape:
            numel *= int(s)
        buf = self._bufs.get(name)
        if buf is None or buf.numel() < numel or buf.dtype != dtype:
            grow = max(numel, 1)
            if buf is not None:
                self._retired.append(buf)
                self.generation += 1
                if buf.dtype == dtype:
                    grow = max(grow, int(buf.numel() * 1.25))
            # images rely on never containing non-finite garbage in their padding rows -> zero-filled on (re)allocation
            buf = (torch.zeros if zeroed else torch.empty)(grow, dtype=dtype, device=self.device)
            self._bufs[name] = buf
        return buf[:numel].view(*shape)

    def get(self, name, shape, dtype=torch.float32):
        return self._get(name, shape, dtype, False)

    def get_zeroed(self, name, shape, dtype=torch.float32):
        """Like get(), but the backing store is zero-filled when it is (re)allocated."""
        return self._get(name, shape, dtype, True)

    def get_image(self, name, nbytes, tail_unwritten: bool = False):
        """An activation image (tile-major, 64 KB per 128-node tile).  Only the padding rows of the last tile may be left
        unwritten by the producing kernel (``tail_unwritten``: ddfa_embed_concat_fwd_image; the gathers and the forward GRU step
        write zeros there); they are multiplied by zeros in the weight-gradient GEMM, so they must be finite — here the
        backing store is zero-filled when it is (re)allocated, and holds only finite values afterwards as long as every step
        is finite.  With ``scrub_image_tails`` the last tile of a ``tail_unwritten`` image is also cleared on every request."""
        buf = self._get(name, (nbytes,), torch.uint8, True)
        if tail_unwritten and self.scrub_image_tails and nbytes > 0:
            buf[max(0, nbytes - 65536):].zero_()
        return buf

    def retired_bytes(self) -> int:
        return sum(b.numel() * b.element_size() for b in self._retired)


class _FreshAlloc:
    """Allocation policy of the autograd path: every buffer is a fresh tensor (caching allocator)."""

    def __init__(self, device):
        self.device = device

    def get(self, name, shape, dtype=torch.float32):
        return torch.empty(*shape, dtype=dtype, device=self.device)

    def get_zeroed(self, name, shape, dtype=torch.float32):
        return torch.zeros(*shape, dtype=dtype, device=self.device)

    def get_image(self, name, nbytes, tail_unwritten: bool = False):
        """A fresh activation image: every row below N is written by the producing kernel, so only the last 64 KB tile (the one
        that can hold padding rows) is cleared — not the whole image (16 images x 78.6 MB per C1 train step otherwise)."""
        buf = torch.empty(nbytes, dtype=torch.uint8, device=self.device)
        buf[max(0, nbytes - 65536):].zero_()
        return buf


def node_indices(g: BatchedCFG, concat_all_absdf: bool, feature_key: str, device) -> List[torch.Tensor]:
    """ggnn.py:84-92: which ndata vectors feed the embedding(s)."""
    if concat_all_absdf:
        keys = [f"_ABS_DATAFLOW_{k}" for k in ABS_DATAFLOW_SUBKEYS]
    else:
        keys = [feature_key]
    out = []
    for k in keys:
        t = g.ndata[k]
        if t.dtype != torch.int64:
            t = t.to(torch.int64)
        out.append(t.to(device, non_blocking=True).contiguous())
    return out


# ------------------------------------------------------------------------------------------
# Forward / backward
# ------------------------------------------------------------------------------------------
def forward(params: ParamPack, dg: DeviceGraph, idx: List[torch.Tensor], n_steps: int, *, training: bool,
            engine: int = ENGINE_SIMT, alloc=None, oob_counter: Optional[torch.Tensor] = None, head: bool = True,
            grad_ggnn: bool = True, x_in: Optional[torch.Tensor] = None, x_scale: float = 1.0,
            attention: Optional[torch.Tensor] = None, x_fill=None):
    """Returns (pooled [B,2D], logits [B] or None, Saved or None).  ``head=False`` stops before the readout and returns
    (x [N,D], h_T [N,D], Saved or None) instead: the label_style="node" trainer runs its own head over a row list
    (``node_head_fwd``); Saved then holds no readout state.
    ``training=True, grad_ggnn=False`` (frozen embedding tables and GGNN): the GGNN runs in its inference form — no per-step
    h / s images or gates are kept — and Saved holds only x, h_T and the readout state, enough for
    ``backward(..., grad_ggnn=False)``.
    ``x_in`` ([N, D] fp32, e.g. the embedding output ``alloc`` holds as "x" after an earlier forward): the pass starts from
    ``x_scale * x_in`` instead of the embedding lookup — h_0 and the readout's concat half both see the scaled rows, which are
    written to the buffer "x_scaled" (and, for the tcgen05 engine, to h_0's activation image) by ``ddfa_stmt_scale_input``.
    ``attention`` ([N] fp32): receives the readout's per-node softmax gate α_n (``ddfa_stmt_attention``).
    ``x_fill`` (instead of ``x_in``): ``x_fill(out, image)`` writes the pass's h_0 rows into ``out`` (the buffer "x_scaled", [N, D])
    and, when ``image`` is not None (tcgen05 engine at D = 128), their activation image — ``ddfa_stmt_shap_input`` does both."""
    _require_cuda(*params.flat_list(), dg.indptr, *idx)
    L = _lib.lib()
    _lib.apply_deterministic_mode()
    dev = dg.device
    alloc = alloc or _FreshAlloc(dev)
    K = len(params.tables)
    V, H = params.tables[0].shape
    D = K * H
    N, B, T = dg.num_nodes, dg.batch_size, n_steps
    nl = len(params.mlp_w)
    st = _stream_ptr()

    # activations travel as MMA-ready bf16 hi/lo images (include/ddfa_b200.h); at the other tcgen05 widths the step follows the
    # SIMT call sequence and ddfa_gru_step_fwd runs its GEMMs on the tensor cores (csrc/gru_tc_wide.cu)
    use_images = engine == ENGINE_TCGEN05 and D == 128
    ggnn_train = training and grad_ggnn       # keep the per-step state the GGNN backward reads
    if x_in is not None and tuple(x_in.shape) != (N, D):
        raise DdfaError(f"forward: x_in of shape {tuple(x_in.shape)}, need ({N}, {D})")
    if x_in is not None and x_fill is not None:
        raise DdfaError("forward: x_in and x_fill are alternatives")
    x = alloc.get("x" if x_in is None and x_fill is None else "x_scaled", (N, D))
    h_imgs = None
    img_bytes = L.call("ddfa_act_image_bytes", N) if use_images else 0
    if x_in is not None or x_fill is not None:
        img = None
        if use_images and OPTIONS["packed_state"]:
            n_img = T if ggnn_train else 2
            h_imgs = [alloc.get_image(f"h_img{i}", img_bytes) for i in range(max(n_img, 1))]
            img = h_imgs[0]
        if x_fill is not None:
            x_fill(x, img)
        else:
            _call("ddfa_stmt_scale_input", _p(x_in), float(x_scale), N, D, _p(x), _p(img), st)
    elif use_images and OPTIONS["packed_state"]:
        # the embedding kernel writes h_0 = x as fp32 rows AND as its activation image (one pass instead of embed + ddfa_act_to_image)
        n_img = T if ggnn_train else 2        # training keeps the image of every h_t (the weight-gradient GEMM reads it)
        h_imgs = [alloc.get_image(f"h_img{i}", img_bytes, tail_unwritten=i == 0) for i in range(max(n_img, 1))]
        _call("ddfa_embed_concat_fwd_image", ptr_array([_p(t) for t in idx]), ptr_array([_p(t) for t in params.tables]),
              K, V, H, N, _p(x), _p(h_imgs[0]), _p(oob_counter), st)
    else:
        _call("ddfa_embed_concat_fwd", ptr_array([_p(t) for t in idx]), ptr_array([_p(t) for t in params.tables]),
              K, V, H, N, _p(x), _p(oob_counter), st)
    w_fold = alloc.get("w_fold", (3 * D, D))
    b_fold = alloc.get("b_fold", (3 * D,))
    L.call("ddfa_fold_weights_fwd", _p(params.w_msg), _p(params.b_msg), _p(params.w_ih), D, _p(w_fold), _p(b_fold), st)

    ws_bytes = L.call("ddfa_gru_step_workspace_bytes", 0 if use_images else N, D, engine)
    ws = alloc.get("gru_ws", (max(ws_bytes, 16),), torch.uint8)
    L.call("ddfa_gru_step_prepare", _p(w_fold), _p(b_fold), _p(params.b_ih), _p(params.w_hh), _p(params.b_hh), D, engine,
           _p(ws), ws_bytes, st)
    hs, ss, gs = [x], [], []
    h_cur = x
    if use_images and not OPTIONS["packed_state"]:
        # round-1 form (A/B only): fp32 copy of every h_t next to its image, four fp32 gate planes per step
        img_bytes = L.call("ddfa_act_image_bytes", N)
        n_img = T if ggnn_train else 2
        h_imgs = [alloc.get_zeroed(f"h_img{i}", (img_bytes,), torch.uint8) for i in range(max(n_img, 1))]
        L.call("ddfa_act_to_image", _p(x), N, D, _p(h_imgs[0]), st)
        for t in range(T):
            s_t = alloc.get_zeroed(f"s_img{t}" if ggnn_train else "s_img", (img_bytes,), torch.uint8)
            h_next = alloc.get(f"h{t + 1}" if ggnn_train else f"hpp{t % 2}", (N, D))
            g_t = alloc.get(f"gates{t}", (4, N, D)) if ggnn_train else None
            _call("ddfa_gather_sum_image", _p(dg.indptr), _p(dg.indices), _p(h_cur), N, D, _p(s_t), None, st, tag="gather_fwd")
            _call("ddfa_gru_step_fwd_image", _p(s_t), _p(h_imgs[t % n_img]), _p(h_cur), _p(dg.indptr), N, D, _p(h_next),
                  _p(h_imgs[(t + 1) % n_img]) if t + 1 < T else None, _p(g_t), _p(ws), ws_bytes, st, tag="ddfa_gru_step_fwd")
            if ggnn_train:
                hs.append(h_next); ss.append(s_t); gs.append(g_t)
            h_cur = h_next
    elif use_images:
        # tcgen05 engine: between steps h_t exists ONLY as its activation image (the GEMM operand; h = hi + lo to 2^-17) — the
        # gather, the z*h term and the backward pass read that; fp32 copies exist of h_0 = x and of h_T (for the readout).  The
        # four saved gate values of an element travel as one 8-byte word (14/14/16-bit fixed point + a 20-bit float, <= 3.1e-5).
        gate_bytes = L.call("ddfa_gru_gates_packed_bytes", N, D)
        for t in range(T):
            last = t == T - 1
            s_t = alloc.get_image(f"s_img{t}" if ggnn_train else "s_img", img_bytes)
            g_t = alloc.get(f"gates_pk{t}", (gate_bytes,), torch.uint8) if ggnn_train else None
            h_in_img = h_imgs[t % n_img]
            if t == 0:
                _call("ddfa_gather_sum_image", _p(dg.indptr), _p(dg.indices), _p(x), N, D, _p(s_t), None, st, tag="gather_fwd")
            else:
                _call("ddfa_gather_sum_image_src", _p(dg.indptr), _p(dg.indices), _p(h_in_img), N, D, _p(s_t), st, tag="gather_fwd")
            h_next = alloc.get("h_final", (N, D)) if last else None
            _call("ddfa_gru_step_fwd_image_v2", _p(s_t), _p(h_in_img), _p(x) if t == 0 else None, _p(dg.indptr), N, D, _p(h_next),
                  None if last else _p(h_imgs[(t + 1) % n_img]), _p(g_t), _p(ws), ws_bytes, st, tag="ddfa_gru_step_fwd")
            if ggnn_train:
                hs.append(h_next); ss.append(s_t); gs.append(g_t)
            if last:
                h_cur = h_next
    else:
        for t in range(T):
            if ggnn_train:
                s_t = alloc.get(f"s{t}", (N, D))
                h_next = alloc.get(f"h{t + 1}", (N, D))
                g_t = alloc.get(f"gates{t}", (4, N, D))
            else:
                s_t = alloc.get("s", (N, D))
                h_next = alloc.get(f"hpp{t % 2}", (N, D))
                g_t = None
            _call("ddfa_gather_sum", _p(dg.indptr), _p(dg.indices), _p(h_cur), N, D, _p(s_t), 0, st, tag="gather_fwd")
            _call("ddfa_gru_step_fwd", _p(s_t), _p(h_cur), _p(dg.indptr), _p(w_fold), _p(b_fold), _p(params.b_ih),
                  _p(params.w_hh), _p(params.b_hh), N, D, _p(h_next), _p(g_t), _p(ws), ws_bytes, engine, st)
            if ggnn_train:
                hs.append(h_next); ss.append(s_t); gs.append(g_t)
            h_cur = h_next

    if training and not grad_ggnn:
        hs, ss, gs, h_imgs = [x] + [None] * (T - 1) + [h_cur], [], [], None     # h[T] = h_T for the readout backward
    if not head:
        if attention is not None:
            raise DdfaError("forward: attention needs the readout (head=True)")
        saved = None
        if training:
            saved = Saved(T, D, x, hs, ss, gs, w_fold, b_fold, None, None, None, None, None, idx,
                          h_img=h_imgs if use_images else None)
        return x, h_cur, saved
    pooled, logits, gate_logit, seg_max, seg_sum, mlp_act = _readout(params, dg, x, h_cur, training, alloc, attention)
    saved = None
    if training:
        saved = Saved(T, D, x, hs, ss, gs, w_fold, b_fold, pooled, gate_logit, seg_max, seg_sum, mlp_act, idx,
                      h_img=h_imgs if use_images else None)
    return pooled, logits, saved


def _readout(params: ParamPack, dg: DeviceGraph, x: torch.Tensor, h_final: torch.Tensor, training: bool, alloc, attention):
    """The readout + MLP head over the rows ``x`` / ``h_final`` ([N, D]) of the batch ``dg`` (its graph_ptr only):
    ``(pooled, logits, gate_logit, seg_max, seg_sum, mlp_act)``, the last four kept for the backward when ``training``."""
    N, D = x.shape
    B = dg.batch_size
    nl = len(params.mlp_w)
    pooled = alloc.get("pooled", (B, 2 * D))
    logits = alloc.get("logits", (B,)) if nl > 0 else None
    keep_gate = training or attention is not None
    gate_logit = alloc.get("gate_logit", (N,)) if keep_gate else None
    seg_max = alloc.get("seg_max", (B,)) if keep_gate else None
    seg_sum = alloc.get("seg_sum", (B,)) if keep_gate else None
    mlp_act = alloc.get("mlp_act", (max(nl - 1, 1), B, 2 * D)) if (training and nl > 1) else None
    st = _stream_ptr()
    _call("ddfa_readout_mlp_fwd", _p(h_final), _p(x), _p(dg.graph_ptr), B, D, _p(params.w_gate), _p(params.b_gate),
           ptr_array([_p(t) for t in params.mlp_w]) if nl else None,
           ptr_array([_p(t) for t in params.mlp_b]) if nl else None,
           nl, _p(pooled), _p(logits), _p(gate_logit), _p(seg_max), _p(seg_sum), _p(mlp_act), st)
    if attention is not None:
        _call("ddfa_stmt_attention", _p(gate_logit), _p(seg_max), _p(seg_sum), _p(dg.graph_ptr), B, _p(attention), st)
    return pooled, logits, gate_logit, seg_max, seg_sum, mlp_act


def readout_forward(params: ParamPack, dg: DeviceGraph, x: torch.Tensor, h_final: torch.Tensor, n_steps: int, *, training: bool,
                    alloc=None, attention: Optional[torch.Tensor] = None):
    """The readout + MLP head of :func:`forward` over given GGNN outputs — the rows an encoder cache gathered (``x`` the
    embedding rows, ``h_final`` h_T, [N, D] each) — with no embedding and no GGNN launch: ``(pooled, logits, Saved or None)``,
    the Saved holding x, h_T and the readout state, what ``backward(..., grad_ggnn=False)`` reads.  ``dg`` needs graph_ptr
    only."""
    _require_cuda(*params.flat_list(), x, h_final, dg.graph_ptr)
    _lib.apply_deterministic_mode()
    alloc = alloc or _FreshAlloc(dg.device)
    T, D = n_steps, x.shape[1]
    pooled, logits, gate_logit, seg_max, seg_sum, mlp_act = _readout(params, dg, x, h_final, training, alloc, attention)
    if not training:
        return pooled, logits, None
    hs = [None] * (T + 1)
    hs[0], hs[T] = x, h_final
    return pooled, logits, Saved(T, D, x, hs, [], [], None, None, pooled, gate_logit, seg_max, seg_sum, mlp_act, [])


def backward(params: ParamPack, dg: DeviceGraph, saved: Saved, grads: ParamPack, *, dlogits: Optional[torch.Tensor] = None,
             dpooled: Optional[torch.Tensor] = None, engine: int = ENGINE_SIMT, alloc=None, on_small_grads_ready=None,
             dh_final: Optional[torch.Tensor] = None, dx_direct: Optional[torch.Tensor] = None, grad_ggnn: bool = True,
             grad_tables: bool = True, grad_weights: bool = True, mlp_ref: Optional[tuple] = None):
    """Accumulates (+=) parameter gradients into ``grads``.  Exactly one of dlogits / dpooled / (dh_final, dx_direct) is given.
    ``dh_final`` / ``dx_direct`` ([N, D] each, from ``node_head_bwd``): the gradients of h_T and of the direct use of x; the
    GGNN backward starts from them and the MLP / readout backward is skipped (their gradients are left alone).  ``dh_final``
    is used as scratch afterwards.
    ``on_small_grads_ready``: called once every gradient EXCEPT those of ggnn.linears[0] and the GRU weight matrices (w_msg,
    b_msg, w_ih, w_hh) is final — with the tcgen05 engine that is before the batched weight-gradient launch, so a data-parallel
    trainer can start reducing them while that launch runs.
    ``grad_ggnn=False`` (frozen embedding tables and GGNN; ``saved`` may come from ``forward(..., grad_ggnn=False)``): stops after
    the readout — the gate gradients only, no GGNN gradient, no transposed gather, no embedding backward.
    ``grad_tables=False`` (frozen embedding tables): the full GGNN backward without the embedding backward.
    ``grad_weights=False`` (input attribution): the dgrad chain only, returning ``(dh_0, dx_direct)``, whose sum is the gradient
    of the logits (or of h_T / pooled) with respect to the embedding output x.  No weight-gradient GEMM (the tcgen05 step kernels
    still keep their operands, but ``ddfa_gru_bwd_wgrad_batched`` / ``_finish`` are not launched), no ``ddfa_fold_weights_bwd``,
    no embedding backward.  The gradients the MLP, readout and step kernels compute inline (the SIMT step kernel's weight
    gradient among them) still go to ``grads``, which the caller then passes as scratch."""
    L = _lib.lib()
    det = _lib.apply_deterministic_mode()
    dev = dg.device
    alloc = alloc or _FreshAlloc(dev)
    K = len(params.tables)
    V, H = params.tables[0].shape
    D, T = saved.D, saved.T
    N, B = dg.num_nodes, dg.batch_size
    nl = len(params.mlp_w)
    st = _stream_ptr()
    if dg.indptr_t is None and grad_ggnn:
        raise DdfaError("backward needs the transposed CSR (prepare_graph(need_transpose=True))")
    if not grad_weights and not grad_ggnn:
        raise DdfaError("backward: grad_weights=False needs the GGNN backward (grad_ggnn=True)")

    if mlp_ref is not None and dlogits is None:
        raise DdfaError("backward: mlp_ref goes with dlogits")
    if dh_final is not None or dx_direct is not None:
        if dh_final is None or dx_direct is None or dlogits is not None or dpooled is not None:
            raise DdfaError("backward: dh_final and dx_direct go together, without dlogits / dpooled")
    elif dlogits is not None and mlp_ref is not None:
        if nl == 0 or grad_weights:
            raise DdfaError("backward: mlp_ref needs an MLP head and grad_weights=False (the rescaled pass computes no weight gradient)")
        dpooled = alloc.get("dpooled", (B, 2 * D))
        scratch = alloc.get("mlp_rescale_scratch", (4, B, 2 * D))
        _call("ddfa_mlp_dgrad_rescale", _p(dlogits), _p(saved.pooled), _p(saved.mlp_act), _p(mlp_ref[0]), _p(mlp_ref[1]),
              ptr_array([_p(t) for t in params.mlp_w]), ptr_array([_p(t) for t in params.mlp_b]), B, D, nl, _p(dpooled), _p(scratch), st)
    elif dlogits is not None:
        if nl == 0:
            raise DdfaError("dlogits given but the module has no MLP head")
        dpooled_buf = alloc.get("dpooled", (B, 2 * D))
        scratch = alloc.get("mlp_scratch", (2, B, 2 * D))
        L.call("ddfa_mlp_bwd", _p(dlogits), _p(saved.pooled), _p(saved.mlp_act), ptr_array([_p(t) for t in params.mlp_w]),
               B, D, nl, _p(dpooled_buf), ptr_array([_p(t) for t in grads.mlp_w]), ptr_array([_p(t) for t in grads.mlp_b]),
               _p(scratch), st)
        dpooled = dpooled_buf
    elif dpooled is None:
        raise DdfaError("backward: neither dlogits nor dpooled given")

    if not grad_ggnn:
        if dh_final is not None:
            raise DdfaError("backward: grad_ggnn=False starts from dlogits / dpooled")
        ro_bytes = L.call("ddfa_readout_bwd_workspace_bytes", B, D)
        ro_ws = alloc.get("readout_bwd_ws", (max(ro_bytes, 16),), torch.uint8)
        _call("ddfa_readout_bwd_ws", _p(dpooled), _p(saved.pooled), _p(saved.h[T]), _p(saved.x), _p(dg.graph_ptr), B, D,
              _p(params.w_gate), _p(saved.gate_logit), _p(saved.seg_max), _p(saved.seg_sum), None, None,
              _p(grads.w_gate), _p(grads.b_gate), _p(ro_ws), ro_bytes, st, tag="ddfa_readout_bwd")
        if on_small_grads_ready is not None:
            on_small_grads_ready()
        return
    dh_alt = alloc.get("dh_b", (N, D))
    if dh_final is not None:
        dh = dh_final
    else:
        dh = alloc.get("dh_a", (N, D))
        dx_direct = alloc.get("dx_direct", (N, D))
        ro_bytes = L.call("ddfa_readout_bwd_workspace_bytes", B, D)
        ro_ws = alloc.get("readout_bwd_ws", (max(ro_bytes, 16),), torch.uint8)
        _call("ddfa_readout_bwd_ws", _p(dpooled), _p(saved.pooled), _p(saved.h[T]), _p(saved.x), _p(dg.graph_ptr), B, D,
               _p(params.w_gate), _p(saved.gate_logit), _p(saved.seg_max), _p(saved.seg_sum), _p(dh), _p(dx_direct),
               _p(grads.w_gate), _p(grads.b_gate), _p(ro_ws), ro_bytes, st, tag="ddfa_readout_bwd")

    dw_fold = alloc.get("dw_fold", (3 * D, D))
    db_fold = alloc.get("db_fold", (3 * D,))
    dw_fold.zero_()
    db_fold.zero_()
    ds = alloc.get("ds", (N, D))
    # the D == 128 tensor-core path (images, packed state, fused backward); at the wider tcgen05 widths the SIMT call sequence
    images = engine == ENGINE_TCGEN05 and D == 128
    ds_prev = None                     # tcgen05 engine: ds of the step after t, folded into step t's call (dh' = dh + A^T ds)
    ds_alt = alloc.get("ds_b", (N, D)) if images else None
    fuse_gather = OPTIONS["fuse_gather_bwd"]
    # tcgen05: keep the q images of every step and run the weight-gradient GEMM of the whole pass as ONE launch at the end
    batched_wgrad = images and bool(saved.h_img) and 0 < T <= 16 and OPTIONS["batched_wgrad"]
    ws_bytes = L.call("ddfa_gru_step_bwd_workspace_bytes_steps", N, D, engine, T if batched_wgrad else 1)
    ws = alloc.get("gru_ws_bwd", (max(ws_bytes, 16),), torch.uint8)
    L.call("ddfa_gru_step_prepare_bwd", _p(saved.w_fold), _p(params.w_hh), D, engine, _p(ws), ws_bytes, st)
    for t in range(T - 1, -1, -1):
        if images:     # saved.s[t] is the activation image of s_t
            _call("ddfa_gru_step_bwd_image_v2" if saved.gates[t].dtype == torch.uint8 else "ddfa_gru_step_bwd_image",
                  _p(dh), _p(ds_prev), _p(dg.indptr_t), _p(dg.indices_t), _p(saved.h[t]),
                  _p(saved.h_img[t]), _p(saved.s[t]), _p(saved.gates[t]), _p(dg.indptr), N, D,
                  _p(ds), _p(dh_alt), _p(dw_fold), _p(db_fold), _p(grads.b_ih), _p(grads.w_hh), _p(grads.b_hh), _p(ws), ws_bytes,
                  (16 + t) if batched_wgrad else (1 if t == T - 1 else 2), st, tag="ddfa_gru_step_bwd")   # deferred weight gradient
            if fuse_gather:
                ds_prev, ds, ds_alt = ds, ds_alt, ds
                dh, dh_alt = dh_alt, dh
                continue
        else:
            _call("ddfa_gru_step_bwd", _p(dh), _p(saved.h[t]), _p(saved.s[t]), _p(saved.gates[t]), _p(dg.indptr),
                  _p(saved.w_fold), _p(params.w_hh), N, D, _p(ds), _p(dh_alt), _p(dw_fold), _p(db_fold), _p(grads.b_ih),
                  _p(grads.w_hh), _p(grads.b_hh), _p(ws), ws_bytes, engine, st)
        # dh_t += A^T ds   (gather over the transposed graph)
        _call("ddfa_gather_sum", _p(dg.indptr_t), _p(dg.indices_t), _p(ds), N, D, _p(dh_alt), 1, st, tag="gather_bwd")
        dh, dh_alt = dh_alt, dh
    if images and T > 0 and fuse_gather:     # the gather of the last ds (step 0) has no following step to ride on
        _call("ddfa_gather_sum", _p(dg.indptr_t), _p(dg.indices_t), _p(ds_prev), N, D, _p(dh), 1, st, tag="gather_bwd")
    if not grad_weights:
        return dh, dx_direct
    # the deterministic form's scratch (sort keys and partial sums): allocated only in that mode, the default form does not read it
    if grad_tables:
        emb_bytes = L.call("ddfa_embed_concat_bwd_workspace_bytes", K, V, H, N) if det else 0
        emb_ws = alloc.get("embed_bwd_ws", (emb_bytes,), torch.uint8) if emb_bytes else None
        _call("ddfa_embed_concat_bwd_ws", ptr_array([_p(t) for t in saved.idx]), _p(dh), _p(dx_direct), K, V, H, N,
              ptr_array([_p(t) for t in grads.tables]), _p(emb_ws), emb_bytes, st, tag="ddfa_embed_concat_bwd")
    if on_small_grads_ready is not None:
        on_small_grads_ready()
    if images and T > 0:
        if batched_wgrad:
            _call("ddfa_gru_bwd_wgrad_batched", ptr_array([_p(saved.s[t]) for t in range(T)]), ptr_array([_p(saved.h_img[t]) for t in range(T)]),
                  T, N, D, _p(dw_fold), _p(grads.w_hh), _p(ws), ws_bytes, st, tag="wgrad_batched")
        else:
            L.call("ddfa_gru_step_bwd_finish", N, D, _p(dw_fold), _p(grads.w_hh), _p(ws), ws_bytes, st)
    L.call("ddfa_fold_weights_bwd", _p(params.w_msg), _p(params.b_msg), _p(params.w_ih), _p(dw_fold), _p(db_fold), D,
           _p(grads.w_msg), _p(grads.b_msg), _p(grads.w_ih), st)


def graph_label_bce(dg: DeviceGraph, vuln: torch.Tensor, logits: Optional[torch.Tensor], pos_weight: float,
                    loss_scale: float, grad_scale: float, want_grad: bool, alloc=None, loss_out=None, num_valid: Optional[int] = None):
    """Labels (segment max of _VULN) + BCE-with-logits sum (+ dlogits). Returns (labels, loss[1], dlogits).
    ``num_valid``: graphs [num_valid, B) are bucket padding (no loss term, zero gradient)."""
    L = _lib.lib()
    _lib.apply_deterministic_mode()
    alloc = alloc or _FreshAlloc(dg.device)
    B = dg.batch_size
    labels = alloc.get("labels", (B,))
    loss = None
    if logits is not None:
        loss = loss_out if loss_out is not None else alloc.get("loss", (1,))
    dlogits = alloc.get("dlogits", (B,)) if (want_grad and logits is not None) else None
    if vuln.dtype != torch.int32:
        vuln = vuln.to(torch.int32)
    L.call("ddfa_graph_label_bce_valid", _p(logits), _p(vuln.contiguous()), _p(dg.graph_ptr), B, B if num_valid is None else int(num_valid),
           float(pos_weight), float(loss_scale), float(grad_scale), _p(labels), _p(loss), _p(dlogits), _stream_ptr())
    return labels, loss, dlogits


# ------------------------------------------------------------------------------------------
# label_style="node": the loss rows drawn on the device, the head and the loss over them (csrc/node_loss.cu)
# ------------------------------------------------------------------------------------------
def undersample_count(n_vuln: int, factor: float) -> int:
    """How many non-vulnerable rows an undersampled node-style loss draws: ``round(n_vuln * factor)`` (base_module.py:96-137),
    Python's round-half-to-even of the fp64 product — what ``ddfa_node_sample`` computes on the device with ``rint``."""
    return round(n_vuln * float(factor))


def node_sample(vuln: torch.Tensor, num_valid: torch.Tensor, factor: Optional[float], seed: int, draw: torch.Tensor,
                rows: torch.Tensor, num_rows: torch.Tensor, status: torch.Tensor, alloc=None):
    """``ddfa_node_sample``: writes the loss rows of the batch (ascending) into ``rows`` (int32 [N]) and their count into
    ``num_rows`` (int32 [1]), on the device.  ``factor=None``: every valid node.  ``draw`` (int64 [1]) is advanced by the call;
    ``status`` (int32 [1]) is set to 1 when the draw asks for more non-vulnerable nodes than there are."""
    N = rows.numel()
    f = -1.0 if factor is None else float(factor)
    ws_bytes = _lib.lib().call("ddfa_node_sample_workspace_bytes", N) if factor is not None else 0
    alloc = alloc or _FreshAlloc(rows.device)
    ws = alloc.get("node_sample_ws", (max(ws_bytes, 16),), torch.uint8) if factor is not None else None
    _call("ddfa_node_sample", _p(vuln), _p(num_valid), N, f, int(seed), _p(draw), _p(rows), _p(num_rows), _p(status), _p(ws),
          ws_bytes, _stream_ptr())


class NodeDrawDP:
    """The phases of the node-row draw over the global batch of ``world`` ranks (``ddfa_node_dp_*``, include/ddfa_b200.h), for
    the rank ``rank`` whose shard has ``rows.numel()`` nodes (capacity).  Between the phases the caller SUM-all-reduces one
    region of ``exchange`` over the ranks: :meth:`counts` after :meth:`count`, :meth:`hist` after each :meth:`radix_hist`,
    :meth:`ties` after :meth:`tie_count`.  :meth:`run` sequences them with a given all-reduce; a test can call the phases of
    several emulated ranks in lockstep.  ``node_offset`` / ``num_rows_global`` (int32 [1]) receive this shard's first node in
    the global batch and the global row count S."""

    def __init__(self, vuln, num_valid, factor, seed: int, draw, rows, num_rows, status, num_rows_global, node_offset, rank: int,
                 world: int, alloc=None):
        self.vuln, self.num_valid, self.seed, self.draw, self.rows, self.num_rows, self.status = vuln, num_valid, int(seed), draw, rows, num_rows, status
        self.factor = -1.0 if factor is None else float(factor)
        self.num_rows_global, self.node_offset, self.rank, self.world = num_rows_global, node_offset, int(rank), int(world)
        self.N = rows.numel()
        L = _lib.lib()
        alloc = alloc or _FreshAlloc(rows.device)
        self.ws_bytes = L.call("ddfa_node_sample_workspace_bytes", self.N)
        self.ws = alloc.get("node_sample_ws", (max(self.ws_bytes, 16),), torch.uint8)
        self.exchange = alloc.get("node_dp_exchange", (L.call("ddfa_node_dp_exchange_words", self.world),), torch.int32)

    @property
    def undersampled(self) -> bool:
        return self.factor >= 0.0

    def counts(self) -> torch.Tensor:
        return self.exchange[256:256 + 2 * self.world]

    def hist(self) -> torch.Tensor:
        return self.exchange[:256]

    def ties(self) -> torch.Tensor:
        return self.exchange[256 + 2 * self.world:]

    def count(self):
        _call("ddfa_node_dp_count", _p(self.vuln), _p(self.num_valid), self.N, self.factor, self.rank, self.world, _p(self.rows),
              _p(self.num_rows), _p(self.ws), self.ws_bytes, _p(self.exchange), _stream_ptr())

    def plan(self):
        _call("ddfa_node_dp_plan", self.N, self.factor, self.rank, self.world, _p(self.draw), _p(self.status), _p(self.num_rows_global),
              _p(self.node_offset), _p(self.ws), self.ws_bytes, _p(self.exchange), _stream_ptr())

    def radix_hist(self, p: int):
        _call("ddfa_node_dp_radix_hist", _p(self.vuln), _p(self.num_valid), self.N, self.seed, p, _p(self.ws), self.ws_bytes,
              _p(self.exchange), _stream_ptr())

    def radix_pick(self, p: int):
        _call("ddfa_node_dp_radix_pick", self.N, p, _p(self.ws), self.ws_bytes, _p(self.exchange), _stream_ptr())

    def tie_count(self):
        _call("ddfa_node_dp_ties", _p(self.vuln), _p(self.num_valid), self.N, self.seed, self.rank, self.world, _p(self.ws),
              self.ws_bytes, _p(self.exchange), _stream_ptr())

    def finish(self):
        _call("ddfa_node_dp_rows", _p(self.vuln), _p(self.num_valid), self.N, self.seed, self.rank, self.world, _p(self.rows),
              _p(self.num_rows), _p(self.ws), self.ws_bytes, _p(self.exchange), _stream_ptr())

    def run(self, all_reduce):
        """The whole draw on the current stream; ``all_reduce(t)`` sums the int32 tensor ``t`` over the ranks in place (one call
        without undersampling, six with it)."""
        self.count()
        all_reduce(self.counts())
        self.plan()
        if not self.undersampled:
            return
        for p in range(4):
            self.radix_hist(p)
            all_reduce(self.hist())
            self.radix_pick(p)
        self.tie_count()
        all_reduce(self.ties())
        self.finish()


def node_bce_global(logits: torch.Tensor, vuln: torch.Tensor, rows: torch.Tensor, num_rows: torch.Tensor, num_rows_global: torch.Tensor,
                    pos_weight: float, loss_out: torch.Tensor, grad_scale: float = 1.0, alloc=None):
    """``ddfa_node_bce_global``: this rank's share of the global mean BCE (the sum over its S rows / S_global) into ``loss_out``
    and dlogits scaled by ``grad_scale / S_global`` (fp32 [N] capacity), returned."""
    N = logits.numel()
    alloc = alloc or _FreshAlloc(logits.device)
    dlogits = alloc.get("node_dlogits", (N,))
    _call("ddfa_node_bce_global", _p(logits), _p(vuln), _p(rows), _p(num_rows), _p(num_rows_global), N, float(pos_weight),
          float(grad_scale), _p(loss_out), _p(dlogits), _stream_ptr())
    return dlogits


def node_head_fwd(params: ParamPack, x: torch.Tensor, h_final: torch.Tensor, rows: torch.Tensor, num_rows: torch.Tensor, alloc=None):
    """``ddfa_node_head_fwd``: logits (fp32 [N] capacity; the first S are valid) and the hidden activations
    ([L-1, N, 2D] capacity, or None for one layer) of the MLP head over the listed rows of ``[h_final | x]``."""
    N, D = x.shape
    nl = len(params.mlp_w)
    alloc = alloc or _FreshAlloc(x.device)
    logits = alloc.get("node_logits", (N,))
    act = alloc.get("node_mlp_act", (nl - 1, N, 2 * D)) if nl > 1 else None
    _call("ddfa_node_head_fwd", _p(h_final), _p(x), _p(rows), _p(num_rows), N, D, ptr_array([_p(t) for t in params.mlp_w]),
          ptr_array([_p(t) for t in params.mlp_b]), nl, _p(act), _p(logits), _stream_ptr())
    return logits, act


def node_bce(logits: torch.Tensor, vuln: torch.Tensor, rows: torch.Tensor, num_rows: torch.Tensor, pos_weight: float,
             loss_out: torch.Tensor, alloc=None, grad_scale: Optional[float] = None):
    """``ddfa_node_bce``: the mean BCE over the S rows into ``loss_out`` and dlogits (fp32 [N] capacity), returned.
    ``grad_scale``: ``ddfa_node_bce_scaled`` instead, dlogits scaled by it (the loss is not); None: the unscaled entry point."""
    N = logits.numel()
    alloc = alloc or _FreshAlloc(logits.device)
    dlogits = alloc.get("node_dlogits", (N,))
    if grad_scale is None:
        _call("ddfa_node_bce", _p(logits), _p(vuln), _p(rows), _p(num_rows), N, float(pos_weight), _p(loss_out), _p(dlogits), _stream_ptr())
    else:
        _call("ddfa_node_bce_scaled", _p(logits), _p(vuln), _p(rows), _p(num_rows), N, float(pos_weight), float(grad_scale), _p(loss_out),
              _p(dlogits), _stream_ptr())
    return dlogits


def grad_accumulate(acc: torch.Tensor, grads: torch.Tensor, begin: int, end: int, mode: int) -> None:
    """``ddfa_grad_accumulate`` over the elements ``[begin, end)`` of two flat fp32 buffers: ``mode`` is
    ``_lib.GRAD_ACC_SET`` (acc = grads), ``GRAD_ACC_ADD`` (acc += grads) or ``GRAD_ACC_APPLY`` (grads += acc)."""
    _require_cuda(acc, grads)
    if acc.dtype != torch.float32 or grads.dtype != torch.float32 or acc.numel() < end or grads.numel() < end:
        raise DdfaError(f"grad_accumulate: fp32 buffers of at least {end} elements needed")
    _call("ddfa_grad_accumulate", _p(acc), _p(grads), int(begin), int(end), int(mode), _stream_ptr())


def node_head_bwd(params: ParamPack, grads: ParamPack, dlogits: torch.Tensor, x: torch.Tensor, h_final: torch.Tensor,
                  rows: torch.Tensor, num_rows: torch.Tensor, act: Optional[torch.Tensor], alloc=None, input_grads: bool = True):
    """``ddfa_node_head_bwd``: accumulates the head's weight / bias gradients into ``grads`` and returns (dh_final, dx_direct),
    [N, D] each, zero outside the listed rows — the starting point of ``backward(..., dh_final=, dx_direct=)``.
    ``input_grads=False`` (frozen encoder): the weight / bias gradients only; returns (None, None)."""
    N, D = x.shape
    nl = len(params.mlp_w)
    L = _lib.lib()
    alloc = alloc or _FreshAlloc(x.device)
    dh = alloc.get("dh_a", (N, D)) if input_grads else None
    dx = alloc.get("dx_direct", (N, D)) if input_grads else None
    ws_bytes = L.call("ddfa_node_head_bwd_workspace_bytes", N, D)
    ws = alloc.get("node_head_bwd_ws", (max(ws_bytes, 16),), torch.uint8)
    _call("ddfa_node_head_bwd", _p(dlogits), _p(h_final), _p(x), _p(rows), _p(num_rows), N, D,
          ptr_array([_p(t) for t in params.mlp_w]), nl, _p(act), _p(dh), _p(dx), ptr_array([_p(t) for t in grads.mlp_w]),
          ptr_array([_p(t) for t in grads.mlp_b]), _p(ws), ws_bytes, _stream_ptr())
    return dh, dx
