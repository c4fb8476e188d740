"""GPU: NaN and +-inf propagate through the kernels the way they do through the fp32 oracle (tests/nonfinite_sites.py).

FusedTrainer(skip_nonfinite=True) skips a step whose gradients are not finite (GradScaler's rule), which matches the reference
only if a non-finite value reaches the same logits, loss and gradients as in torch.  Checked, at one site at a time (a one-node
embedding row as NaN / +inf / -inf, one element of every other parameter as NaN), on the SIMT engine, the D = 128 tensor-core
engine and the wide tensor-core engine at W = 192 and 256, in both label styles, at B = 255 and 256 (the per-graph and the
batched MLP head):
  (a) the module's training forward and backward against the fp32 oracle: the non-finite logits, the loss's finiteness, which
      parameters get a non-finite gradient, the elementwise non-finite masks of the embedding tables and the head parameters,
      and every untouched logit finite and close to the oracle's;
  (b) the readout, MLP head and their backward through the C ABI, with one graph's node rows NaN (first row, last row, the rows
      of one warp, a 40 000-node graph);
  (c) FusedTrainer: the step is skipped exactly when the oracle's gradients are not finite, and a run that skipped it is
      bit-identical to one that never saw it (eager, captured, and through a GraphArena);
  (d) FusedEvaluator: one poisoned graph or node row counts as "not >= 0.5", the loss word is NaN, and every other stored
      probability is bit-identical to the clean run's.
Every test prints its site, engine and the masks it compared."""
import contextlib
import math
import os

import numpy as np
import pytest
import torch

import deepdfa_b200 as D
from deepdfa_b200 import _lib, synth
from deepdfa_b200._lib import lib, ptr_array
from deepdfa_b200.engine import _p, _stream_ptr
from head_batches import HUGE_GRAPH, graph_ptr, segment_ids
from nonfinite_sites import (EMBED, ENGINES, FEAT, GATE, HEAD, INF, INPUT_DIM, LAYERS, NAN, POS_WEIGHT, STEPS, case_id, element,
                             grad_flags, model_state, nonfinite, oracle_step, poison, poison_batch, site_id, sites)

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
ENGINE_IDS = [case_id(*e) for e in ENGINES]


@contextlib.contextmanager
def det_mode():
    prev = os.environ.get("DDFA_DETERMINISTIC")
    os.environ["DDFA_DETERMINISTIC"] = "1"
    _lib.apply_deterministic_mode()
    try:
        yield
    finally:
        if prev is None:
            os.environ.pop("DDFA_DETERMINISTIC")
        else:
            os.environ["DDFA_DETERMINISTIC"] = prev
        _lib.apply_deterministic_mode()


def make_module(engine, hidden, style, state, factor=None):
    m = D.FlowGNNGGNNModule(FEAT, INPUT_DIM, hidden, STEPS, LAYERS, label_style=style, concat_all_absdf=True,
                            positive_weight=POS_WEIGHT, undersample_node_on_loss_factor=factor, engine=engine)
    m.load_state_dict(state)
    return m.to(DEV)


def logit_tol(hidden):
    """The module-level logit bound of the smoke test (1e-3 at W = 128), grown like a dot product's error with the width."""
    return 1e-3 * max(1.0, (4 * hidden / 128) ** 0.5)


def mask_str(t):
    bad = nonfinite(t)
    return f"{int(bad.sum())}/{bad.numel()}"


# ---- (a) the module against the fp32 oracle, per site ---------------------------------------------------------------------------
def loss_rows(rows, where, N):
    """Node style: the loss rows — every node ("all"), or every other node with the poisoned node in ("inside") or with the
    poisoned node's whole graph out ("outside"), as the module's undersampling would pass them to its loss."""
    if rows == "all":
        return None
    offs, gi = where["offs"], where["graph"]
    keep = np.zeros(N, dtype=bool)
    keep[::2] = True
    if rows == "inside":
        keep[where["node"]] = True
    else:
        keep[offs[gi]:offs[gi + 1]] = False
    return torch.from_numpy(np.nonzero(keep)[0])


MODULE_CASES = [("graph", "all"), ("node", "all"), ("node", "inside"), ("node", "outside")]


@pytest.mark.parametrize("B", [255, 256])
@pytest.mark.parametrize("style,rows", MODULE_CASES, ids=[f"{s}-{r}" for s, r in MODULE_CASES])
@pytest.mark.parametrize("engine,hidden", ENGINES, ids=ENGINE_IDS)
def test_module_nonfinite_sets_match_the_fp32_oracle(engine, hidden, style, rows, B):
    g, where = poison_batch(style, B)
    gd = g.to(DEV)
    sel = loss_rows(rows, where, g.num_nodes())
    state = model_state(hidden, style, seed=3)
    m = make_module(engine, hidden, style, state)
    tol = logit_tol(hidden)
    failures = []
    for site in sites(style):
        tag = f"{case_id(engine, hidden)} {style} rows={rows} B={B} {site_id(site)}"
        psd = poison(state, site, where)
        ref = oracle_step(psd, g, style, sel)
        m.load_state_dict(psd)
        for p in m.parameters():
            p.grad = None
        out = m(gd)
        if sel is None:
            loss, _ = m.loss_and_labels(gd, out)
        else:       # the module's undersampled loss (training_step with undersample_node_on_loss_factor) over these rows
            sd = sel.to(DEV)
            loss = m.loss_fn(out[sd], m.get_label(gd)[sd])
        loss.backward()
        torch.cuda.synchronize()
        logits = out.detach().cpu()
        grads = {k: p.grad.cpu() for k, p in m.named_parameters()}
        bad, rbad = nonfinite(logits), nonfinite(ref["logits"])
        msgs = []
        if not torch.equal(bad, rbad):
            msgs.append(f"non-finite logits {torch.nonzero(bad).flatten().tolist()[:8]} vs oracle "
                        f"{torch.nonzero(rbad).flatten().tolist()[:8]}")
        if math.isfinite(float(loss)) != math.isfinite(float(ref["loss"])):
            msgs.append(f"loss {float(loss)} vs oracle {float(ref['loss'])}")
        flags, rflags = grad_flags(grads), grad_flags(ref["grads"])
        diff = sorted(k for k in rflags if flags[k] != rflags[k])
        if diff:
            msgs.append("gradient finiteness differs: " + ", ".join(f"{k} ({flags[k]} vs oracle {rflags[k]})" for k in diff))
        for k in ref["grads"]:
            # Known difference, not compared elementwise: the module runs node rows through the readout as one-node graphs with a
            # zero gate, whose logit 0 . o is NaN for a partly NaN row, so that row's pooled copy is NaN in every column where torch
            # keeps its finite columns.  Only a row outside the loss rows shows it (its zero logit gradient times the NaN columns in
            # output_layer.0.weight's gradient); whether that gradient is finite is still compared above.
            if rows == "outside" and k == "output_layer.0.weight":
                continue
            if k.startswith("all_embeddings.") or k in GATE + HEAD:
                if not torch.equal(nonfinite(grads[k]), nonfinite(ref["grads"][k])):
                    msgs.append(f"{k}: non-finite mask {mask_str(grads[k])} vs oracle {mask_str(ref['grads'][k])}")
        keep = ~rbad & ~bad
        if keep.any():
            err = float(((logits[keep] - ref["logits"][keep]).abs() / ref["logits"][keep].abs().clamp_min(1.0)).max())
            if not err <= tol:
                msgs.append(f"untouched logits off by {err:.2e} > {tol:.1e}")
        ggnn = ", ".join(f"{k.split('.', 1)[1]} {mask_str(grads[k])}|{mask_str(ref['grads'][k])}" for k in grads if k.startswith("ggnn."))
        print(f"{tag}: logits {mask_str(logits)} (oracle {mask_str(ref['logits'])}), loss {float(loss):.4g} "
              f"(oracle {float(ref['loss']):.4g}), non-finite grads {sum(flags.values())}/{len(flags)}; ggnn kernel|oracle: {ggnn}"
              + (" -- " + "; ".join(msgs) if msgs else ""))
        if msgs:
            failures.append(f"{tag}: " + "; ".join(msgs))
    assert not failures, "\n".join(failures)


# ---- (b) the readout, MLP head and their backward through the ABI -----------------------------------------------------------------
def readout_sizes(B, huge):
    rng = np.random.default_rng(B)
    sizes = rng.integers(20, 60, size=B)
    if huge:
        sizes[B // 2] = HUGE_GRAPH
    return sizes


def torch_head(h, x, w, b, ws, bs, sizes, dl):
    """fp32 torch autograd of the readout + MLP head, with loss = sum(logits * dl): logits and every gradient."""
    seg = segment_ids(sizes)
    B = len(sizes)
    h, x, w, b = (t.clone().requires_grad_(True) for t in (h, x, w, b))
    ws = [t.clone().requires_grad_(True) for t in ws]
    bs = [t.clone().requires_grad_(True) for t in bs]
    o = torch.cat([h, x], 1)
    g = o @ w + b
    gmax = torch.full((B,), -math.inf).scatter_reduce(0, seg, g, "amax", include_self=True)
    e = torch.exp(g - gmax[seg])
    den = torch.zeros(B).index_add(0, seg, e)
    pooled = torch.zeros(B, o.shape[1]).index_add(0, seg, o * (e / den[seg])[:, None])
    y = pooled
    for i in range(len(ws)):
        y = y @ ws[i].t() + bs[i]
        if i + 1 < len(ws):
            y = torch.relu(y)
    logits = y.squeeze(1)
    (logits * dl).sum().backward()
    return dict(pooled=pooled.detach(), logits=logits.detach(), dh=h.grad, dx=x.grad, dw=w.grad, db=b.grad,
                dW=[t.grad for t in ws], dB=[t.grad for t in bs])


def kernel_head(h, x, w, b, ws, bs, sizes, dl):
    B, N, D = len(sizes), h.shape[0], h.shape[1]
    L, D2 = len(ws), 2 * D
    hd, xd, wd, bd, gp = (t.to(DEV) for t in (h, x, w, b, graph_ptr(sizes)))
    wsd, bsd = [t.to(DEV) for t in ws], [t.to(DEV) for t in bs]
    pooled, logits = torch.empty(B, D2, device=DEV), torch.empty(B, device=DEV)
    gl, smax, ssum = torch.empty(N, device=DEV), torch.empty(B, device=DEV), torch.empty(B, device=DEV)
    act = torch.empty(L - 1, B, D2, device=DEV)
    L_ = lib()
    L_.call("ddfa_readout_mlp_fwd", _p(hd), _p(xd), _p(gp), B, D, _p(wd), _p(bd), ptr_array([_p(t) for t in wsd]),
            ptr_array([_p(t) for t in bsd]), L, _p(pooled), _p(logits), _p(gl), _p(smax), _p(ssum), _p(act), _stream_ptr())
    dpooled = torch.empty(B, D2, device=DEV)
    dW, dB = [torch.zeros_like(t) for t in wsd], [torch.zeros_like(t) for t in bsd]
    scratch = torch.empty(2 * B * D2, device=DEV)
    L_.call("ddfa_mlp_bwd", _p(dl.to(DEV)), _p(pooled), _p(act), ptr_array([_p(t) for t in wsd]), B, D, L, _p(dpooled),
            ptr_array([_p(t) for t in dW]), ptr_array([_p(t) for t in dB]), _p(scratch), _stream_ptr())
    dh, dx = torch.empty(N, D, device=DEV), torch.empty(N, D, device=DEV)
    dw, db = torch.zeros(D2, device=DEV), torch.zeros(1, device=DEV)
    wsb = L_.call("ddfa_readout_bwd_workspace_bytes", B, D)
    wsp = torch.empty(wsb, dtype=torch.uint8, device=DEV)
    L_.call("ddfa_readout_bwd_ws", _p(dpooled), _p(pooled), _p(hd), _p(xd), _p(gp), B, D, _p(wd), _p(gl), _p(smax), _p(ssum),
            _p(dh), _p(dx), _p(dw), _p(db), _p(wsp), wsb, _stream_ptr())
    torch.cuda.synchronize()
    return dict(pooled=pooled.cpu(), logits=logits.cpu(), dh=dh.cpu(), dx=dx.cpu(), dw=dw.cpu(), db=db.cpu(),
                dW=[t.cpu() for t in dW], dB=[t.cpu() for t in dB])


@pytest.mark.parametrize("B", [255, 256])
@pytest.mark.parametrize("rows", ["first", "last", "warp", "huge"])
def test_readout_and_head_propagate_a_nan_graph_like_torch(rows, B):
    D, L = 128, 3
    sizes = readout_sizes(B, rows == "huge")
    gen = torch.Generator().manual_seed(B)
    N = int(sizes.sum())
    h, x = torch.randn(N, D, generator=gen), torch.randn(N, D, generator=gen)
    w, b = torch.randn(2 * D, generator=gen) / (2 * D) ** 0.5, torch.randn(1, generator=gen)
    ws = [torch.randn(1 if i == L - 1 else 2 * D, 2 * D, generator=gen) * (2.0 / (2 * D)) ** 0.5 for i in range(L)]
    bs = [0.1 * torch.randn(1 if i == L - 1 else 2 * D, generator=gen) for i in range(L)]
    dl = torch.randn(B, generator=gen)
    gp = graph_ptr(sizes).long()
    j = B // 2 if rows == "huge" else B // 3
    n0, n1 = int(gp[j]), int(gp[j + 1])
    sel = {"first": [n0], "last": [n1 - 1], "warp": list(range(n0 + 3, n1, 8)), "huge": [n0 + 12345]}[rows]
    h[sel] = NAN
    ref = torch_head(h, x, w, b, ws, bs, sizes, dl)
    got = kernel_head(h, x, w, b, ws, bs, sizes, dl)
    pairs = [(k, got[k], ref[k]) for k in ("pooled", "logits", "dh", "dx", "dw", "db")]
    pairs += [(f"dW{i}", got["dW"][i], ref["dW"][i]) for i in range(L)] + [(f"dB{i}", got["dB"][i], ref["dB"][i]) for i in range(L)]
    print(f"readout B={B} NaN rows={rows} ({len(sel)} of graph {j}, {n1 - n0} nodes): "
          + ", ".join(f"{k} {mask_str(a)}|{mask_str(r)}" for k, a, r in pairs))
    assert torch.isnan(got["logits"][j]) and int(nonfinite(got["logits"]).sum()) == 1
    for k, a, r in pairs:
        assert torch.equal(nonfinite(a), nonfinite(r)), k


def test_node_head_propagates_a_nan_row_like_torch():
    """ddfa_node_head_fwd / _bwd over a row list: a NaN node row inside the rows makes its logit NaN and reaches dh / dx of that
    row and every weight gradient; a NaN row outside the rows changes nothing."""
    from test_node_trainer_gpu import head_case, ref_head, run_head
    N, D, L = 1000, 128, 3
    rows = np.sort(np.random.default_rng(0).choice(N, size=300, replace=False))
    inside, outside = int(rows[100]), int(np.setdiff1d(np.arange(N), rows)[50])
    h, x, ws, bs, rows_t = head_case(N, D, L, rows)
    h[inside, 7] = NAN
    x[outside, 3] = NAN
    dl = torch.randn(rows_t.numel(), generator=torch.Generator().manual_seed(1)) / rows_t.numel()
    got = run_head(h, x, ws, bs, rows_t, dl)
    ref = ref_head(h, x, ws, bs, rows_t, dl)
    names = ["logits", "dh", "dx"] + [f"dW{i}" for i in range(L)] + [f"dB{i}" for i in range(L)]
    pairs = list(zip(names, [got[0], got[1], got[2], *got[3], *got[4]], [ref[0], ref[1], ref[2], *ref[3], *ref[4]]))
    print("node head, NaN row inside and outside the rows: " + ", ".join(f"{k} {mask_str(a)}|{mask_str(r)}" for k, a, r in pairs))
    assert int(nonfinite(got[0]).sum()) == 1
    for k, a, r in pairs:
        assert torch.equal(nonfinite(a), nonfinite(r)), k


# One D = 128 tensor-core GRU step through the image entries, forward (ddfa_gru_step_fwd_image_v2) and the fused backward
# (ddfa_gru_step_bwd_image_v2), against fp32 torch autograd of the same step.  NaN in one element of a row of s or h, and +-inf in the
# n-gate half of b_hh (gh_n infinite in every row: torch's gate backward takes 0 * inf = NaN where n saturates), must give the same
# elementwise non-finite masks: they exercise the packed saved gates, which must carry NaN and inf into the backward.  +-inf in s or h
# is different: the bf16x3 GEMMs split an infinite operand into hi = inf, lo = NaN, so the kernel's row turns NaN where torch's
# saturating gates can keep it finite.  There only the other rows (finite) and whether any gradient is non-finite (the step guard's
# decision) must agree.
GRU_CASES = [("s", NAN), ("h", NAN), ("bhh_n", INF), ("bhh_n", -INF), ("s", INF), ("s", -INF), ("h", INF), ("h", -INF)]


@pytest.mark.parametrize("where,value", GRU_CASES, ids=[f"{w}={v}" for w, v in GRU_CASES])
def test_tc_gru_step_carries_nonfinite_values_like_torch(where, value):
    from deepdfa_b200._lib import ENGINE_TCGEN05
    from deepdfa_b200.engine import prepare_graph
    from test_scale_gpu import _gru_reference
    D = 128
    g = synth.make_batch(24, 60, seed=2, variable=True)
    dg = prepare_graph(g, DEV)
    N = g.num_nodes()
    gen = torch.Generator().manual_seed(9)
    k = 1.0 / D ** 0.5
    mk = lambda *sh: (torch.rand(*sh, generator=gen) * 2 - 1) * k
    wf, bf, bih, whh, bhh = mk(3 * D, D) * 1.5, mk(3 * D), mk(3 * D), mk(3 * D, D), mk(3 * D)
    s = torch.randn(N, D, generator=gen) * 2
    h = torch.tanh(torch.randn(N, D, generator=gen))
    dh_out = torch.randn(N, D, generator=gen)
    row, col = N // 3, 5
    if where == "s":
        s[row, col] = value
    elif where == "h":
        h[row, col] = value
    else:
        bhh[2 * D + col] = value
    deg = torch.bincount(g.edges()[1], minlength=N).float()
    leaves = [t.clone().requires_grad_(True) for t in (s, h, wf, bf, bih, whh, bhh)]
    h_ref = _gru_reference(*leaves[:2], deg, *leaves[2:])[0]
    (h_ref * dh_out).sum().backward()
    ref = {"h'": h_ref.detach(), "ds": leaves[0].grad, "dh": leaves[1].grad, "dwf": leaves[2].grad, "dbf": leaves[3].grad,
           "dbih": leaves[4].grad, "dwhh": leaves[5].grad, "dbhh": leaves[6].grad}

    L, st = lib(), _stream_ptr()
    ib = L.call("ddfa_act_image_bytes", N)
    sd, hd, wfd, bfd, bihd, whhd, bhhd, dd = (t.to(DEV).contiguous() for t in (s, h, wf, bf, bih, whh, bhh, dh_out))
    s_img, h_img, o_img = (torch.zeros(ib, dtype=torch.uint8, device=DEV) for _ in range(3))
    L.call("ddfa_act_to_image", _p(sd), N, D, _p(s_img), st)
    L.call("ddfa_act_to_image", _p(hd), N, D, _p(h_img), st)
    wsb = L.call("ddfa_gru_step_workspace_bytes", 0, D, ENGINE_TCGEN05)
    ws = torch.empty(wsb, dtype=torch.uint8, device=DEV)
    L.call("ddfa_gru_step_prepare", _p(wfd), _p(bfd), _p(bihd), _p(whhd), _p(bhhd), D, ENGINE_TCGEN05, _p(ws), wsb, st)
    gates = torch.empty(L.call("ddfa_gru_gates_packed_bytes", N, D), dtype=torch.uint8, device=DEV)
    h_out = torch.empty(N, D, device=DEV)
    L.call("ddfa_gru_step_fwd_image_v2", _p(s_img), _p(h_img), None, _p(dg.indptr), N, D, None, _p(o_img), _p(gates), _p(ws), wsb, st)
    L.call("ddfa_gru_step_fwd_image_v2", _p(s_img), _p(h_img), None, _p(dg.indptr), N, D, _p(h_out), None, None, _p(ws), wsb, st)
    wsb_b = L.call("ddfa_gru_step_bwd_workspace_bytes", N, D, ENGINE_TCGEN05)
    ws_b = torch.empty(wsb_b, dtype=torch.uint8, device=DEV)
    L.call("ddfa_gru_step_prepare_bwd", _p(wfd), _p(whhd), D, ENGINE_TCGEN05, _p(ws_b), wsb_b, st)
    ds, dh = torch.empty(N, D, device=DEV), torch.empty(N, D, device=DEV)
    acc = {n_: torch.zeros(sh, device=DEV) for n_, sh in (("dwf", (3 * D, D)), ("dbf", (3 * D,)), ("dbih", (3 * D,)),
                                                          ("dwhh", (3 * D, D)), ("dbhh", (3 * D,)))}
    ds_prev = torch.zeros(N, D, device=DEV)           # no transposed-gather term: dh' is dh_out
    L.call("ddfa_gru_step_bwd_image_v2", _p(dd), _p(ds_prev), _p(dg.indptr_t), _p(dg.indices_t), None, _p(h_img), _p(s_img),
           _p(gates), _p(dg.indptr), N, D, _p(ds), _p(dh), _p(acc["dwf"]), _p(acc["dbf"]), _p(acc["dbih"]), _p(acc["dwhh"]),
           _p(acc["dbhh"]), _p(ws_b), wsb_b, 0, st)
    torch.cuda.synchronize()
    got = {"h'": h_out.cpu(), "ds": ds.cpu(), "dh": dh.cpu(), **{k_: v.cpu() for k_, v in acc.items()}}
    print(f"tc GRU step {where}={value} (row {row}): " + ", ".join(f"{k_} {mask_str(got[k_])}|{mask_str(ref[k_])}" for k_ in ref))
    if where == "bhh_n" or value != value:
        for k_ in ref:
            assert torch.equal(nonfinite(got[k_]), nonfinite(ref[k_])), k_
    else:
        other = torch.ones(N, dtype=torch.bool)
        other[row] = False
        for k_ in ("h'", "ds", "dh"):
            assert torch.equal(nonfinite(got[k_])[other], nonfinite(ref[k_])[other]), k_
            assert bool(nonfinite(got[k_][row]).any()) or not bool(nonfinite(ref[k_][row]).any()), k_
        grads = ("dwf", "dbf", "dbih", "dwhh", "dbhh")
        assert any(bool(nonfinite(got[k_]).any()) for k_ in grads) == any(bool(nonfinite(ref[k_]).any()) for k_ in grads)


@pytest.mark.parametrize("W", [192, 256])
@pytest.mark.parametrize("value", [NAN, INF, -INF])
def test_wide_gemm_keeps_a_nonfinite_operand_nonfinite(W, value):
    """ddfa_gru_tc_wide_gemm, all four call forms, with one non-finite element in the A operand: the non-finite elements of the
    result are where fp32 torch's are (NaN or inf may differ: bf16x3 splits inf into hi = inf, lo = NaN)."""
    N = 1000
    L, st = lib(), _stream_ptr()
    gen = torch.Generator(device=DEV).manual_seed(W)
    a_gi = torch.randn(N, W, device=DEV, generator=gen)
    a_dg = torch.randn(N, 3 * W, device=DEV, generator=gen) * 0.1
    wmat = torch.randn(3 * W, W, device=DEV, generator=gen) * W ** -0.5
    calls = [("gi", 0, a_gi, wmat), ("ds", 1, a_dg, wmat), ("dh", 2, a_dg, wmat), ("dW", 3, a_dg, a_gi)]
    for name, call, a, b in calls:
        a = a.clone()
        a[N // 2, 7] = value
        wsb = L.call("ddfa_gru_tc_wide_gemm_workspace_bytes", call, N, W)
        ws = torch.empty(max(wsb, 16), dtype=torch.uint8, device=DEV)
        if call == 0:
            ref, c = a @ b.t(), torch.empty(N, 3 * W, device=DEV)
        elif call == 3:
            ref, c = a.t() @ b, torch.zeros(3 * W, W, device=DEV)
        else:
            ref, c = a @ b, torch.zeros(N, W, device=DEV)
        L.call("ddfa_gru_tc_wide_gemm", call, _p(a), _p(b), N, W, _p(c), _p(ws), wsb, st)
        torch.cuda.synchronize()
        print(f"wide gemm W={W} {name} operand={value}: non-finite {mask_str(c)} (torch {mask_str(ref)})")
        assert torch.equal(nonfinite(c), nonfinite(ref)), name


# ---- (c) the trainer: skip exactly when the oracle's gradients are not finite, and leave nothing behind ---------------------------
def trainer_batches(style):
    """(the poisoned batch, its poison place, two smaller ragged batches with N % 128 != 0 and N below the poisoned batch's)."""
    big, where = poison_batch(style, 256)
    if style == "graph":
        small = [synth.make_batch(40, 11, seed=60 + i, variable=True, vuln_rate=0.3) for i in range(2)]
    else:
        small = [synth.make_batch(sizes=[13, 7, 30, 20 + 9 * i], seed=60 + i, vuln_rate=0.6) for i in range(2)]
        for i, s in enumerate(small):
            s.ndata["_VULN"] = torch.from_numpy((np.random.default_rng(i).random(s.num_nodes()) < 0.3).astype(np.int32))
    for s in small:
        assert s.num_nodes() % 128 and s.num_nodes() < big.num_nodes()
    return big, where, small


def snapshot(tr):
    torch.cuda.synchronize()
    return [t.detach().clone() for t in (tr.flat_p, tr.exp_avg, tr.exp_avg_sq, tr.step_count)]


def run_trainer(engine, hidden, style, state, graph_mode, big, small, site=None, where=None, arena=None, factor=None):
    """Clean step on `big`, then (with a site) the poisoned step on `big` with the poison removed after it, then the small
    batches.  Returns (final state, losses, skipped count, the poisoned step's grad norm and loss rows)."""
    m = make_module(engine, hidden, style, state, factor)
    tr = D.FusedTrainer(m, skip_nonfinite=True, max_grad_norm=1.0, use_cuda_graph=graph_mode, node_sample_seed=11)

    def step(i):
        if arena is None:
            return tr.step(([big] + small)[i])
        return tr.step_ids(arena[0], arena[1][i])

    losses = [float(step(0))]
    info = {}
    if site is not None:
        params = dict(m.named_parameters())
        name, value = site
        idx = (where["row"],) if name == EMBED else element(name, params[name].shape)
        torch.cuda.synchronize()
        info["state"] = {k: v.detach().cpu().clone() for k, v in m.state_dict().items()}
        draws = tr.node_sample_draws if style == "node" else None
        keep = params[name].data[idx].clone()
        with torch.no_grad():
            params[name].data[idx] = value
        step(0)
        torch.cuda.synchronize()
        info["norm"] = float(tr.grad_norm)
        info["rows"] = tr.last_loss_rows().cpu().long() if style == "node" else None
        with torch.no_grad():
            params[name].data[idx] = keep
        if style == "node":
            tr.node_sample_draws = draws             # a run that never saw the step has not made its draw either
    for i in (1, 2):
        losses.append(float(step(i)))
    return snapshot(tr), losses, tr.skipped_steps, info


@pytest.mark.parametrize("graph_mode", [False, True], ids=["eager", "captured"])
@pytest.mark.parametrize("style", ["graph", "node"])
@pytest.mark.parametrize("engine,hidden", ENGINES, ids=ENGINE_IDS)
def test_trainer_skips_exactly_the_nonfinite_steps_and_recovers_bit_exactly(engine, hidden, style, graph_mode):
    big, where, small = trainer_batches(style)
    state = model_state(hidden, style, seed=5)
    variants = [("", None, None)]
    if style == "node":
        # the poisoned node inside the sampled loss rows (vulnerable: always drawn; one non-vulnerable node drawn per vulnerable
        # one), and outside them: its graph has no vulnerable node and no other node is drawn (factor 0)
        offs = where["offs"]
        v_in = big.ndata["_VULN"].clone()
        v_in[where["node"]] = 1
        v_out = big.ndata["_VULN"].clone()
        v_out[offs[where["graph"]]:offs[where["graph"] + 1]] = 0
        variants = [("inside", v_in, 1.0), ("outside", v_out, 0.0)]
    failures = []
    with det_mode():
        for vname, v, factor in variants:
            if style == "node":
                big, where, small = trainer_batches(style)     # a fresh object: a batch keeps device copies of its node data
                big.ndata["_VULN"] = v
            clean, clean_losses, skipped, _ = run_trainer(engine, hidden, style, state, graph_mode, big, small, factor=factor)
            assert skipped == 0 and all(math.isfinite(x) for x in clean_losses)
            for site in sites(style):
                tag = f"{case_id(engine, hidden)} {style}{' ' + vname if vname else ''} {'captured' if graph_mode else 'eager'} {site_id(site)}"
                got, losses, skipped, info = run_trainer(engine, hidden, style, state, graph_mode, big, small, site, where,
                                                         factor=factor)
                ref = oracle_step(poison(info["state"], site, where), big, style, info["rows"])
                want_skip = any(grad_flags(ref["grads"]).values())
                inside_rows = None
                if info["rows"] is not None:
                    offs = where["offs"]
                    touched = set(range(offs[where["graph"]], offs[where["graph"] + 1]))
                    inside_rows = (where["node"] in set(info["rows"].tolist()), len(touched & set(info["rows"].tolist())))
                    assert inside_rows[0] == (vname == "inside") and (inside_rows[1] == 0) == (vname == "outside"), (tag, inside_rows)
                print(f"{tag}: norm {info['norm']:.4g}, skipped {skipped}, oracle grads non-finite {want_skip}"
                      + (f", poisoned node in loss rows {inside_rows[0]} ({inside_rows[1]} rows of its graph)" if inside_rows else ""))
                if skipped != int(want_skip) or math.isfinite(info["norm"]) == want_skip:
                    failures.append(f"{tag}: skipped {skipped}, norm {info['norm']}, oracle non-finite {want_skip}")
                    continue
                if want_skip:
                    if losses != clean_losses or not all(torch.equal(a, b) for a, b in zip(got, clean)):
                        failures.append(f"{tag}: the run after the skipped step differs from the clean run")
    assert not failures, "\n".join(failures)


def test_trainer_skip_and_recovery_through_a_graph_arena():
    engine, hidden = "tcgen05", 32
    big, where, small = trainer_batches("graph")
    arena = D.GraphArena.from_graphs([big] + small, DEV)
    offs = np.cumsum([0] + [b.batch_size for b in [big] + small])
    ids = [np.arange(offs[i], offs[i + 1]) for i in range(3)]
    state = model_state(hidden, "graph", seed=5)
    with det_mode():
        clean, clean_losses, _, _ = run_trainer(engine, hidden, "graph", state, True, big, small, arena=(arena, ids))
        for site in [(EMBED, NAN), ("output_layer.0.bias", NAN), (f"{HEAD[2]}", NAN)]:
            got, losses, skipped, info = run_trainer(engine, hidden, "graph", state, True, big, small, site, where, arena=(arena, ids))
            print(f"arena {site_id(site)}: norm {info['norm']}, skipped {skipped}")
            assert skipped == 1 and not math.isfinite(info["norm"])
            assert losses == clean_losses and all(torch.equal(a, b) for a, b in zip(got, clean))


# ---- (d) the evaluator -------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("style", ["graph", "node"])
@pytest.mark.parametrize("engine,hidden", ENGINES, ids=ENGINE_IDS)
def test_evaluator_counts_a_nan_prediction_as_negative(engine, hidden, style):
    g, where = poison_batch(style, 256)
    state = model_state(hidden, style, seed=4)
    site = (EMBED, NAN)
    psd = poison(state, site, where)
    ref = oracle_step(psd, g, style)
    probs_ref = torch.sigmoid(ref["logits"])
    vuln = g.ndata["_VULN"]
    if style == "graph":
        y = torch.zeros(g.batch_size, dtype=torch.int32).scatter_reduce(0, segment_ids(g.batch_num_nodes().numpy()), vuln, "amax",
                                                                          include_self=False)
    else:
        y = vuln.clone()
    pred, t = probs_ref >= 0.5, y != 0               # NaN >= 0.5 is False
    want = [int((pred & t).sum()), int((pred & ~t).sum()), int((~pred & ~t).sum()), int((~pred & t).sum())]
    out = {}
    for tag, sd in (("clean", state), ("poisoned", psd)):
        m = make_module(engine, hidden, style, sd)
        ev = D.FusedEvaluator(m, use_cuda_graph=True, max_predictions=len(probs_ref))
        ev.update(g)
        res = ev.compute("val_")
        probs, _ = ev.predictions()
        out[tag] = (res, probs.cpu())
    res, probs = out["poisoned"]
    tn, fp = res["val_confusion"][0]
    fn, tp = res["val_confusion"][1]
    bad = nonfinite(ref["logits"])
    print(f"evaluator {case_id(engine, hidden)} {style}: non-finite probs {mask_str(probs)} (oracle {mask_str(ref['logits'])}), "
          f"TP FP TN FN {[tp, fp, tn, fn]} (oracle rule {want}), loss {res['val_loss']}")
    assert [tp, fp, tn, fn] == want
    assert math.isnan(res["val_loss"])
    assert torch.equal(nonfinite(probs), bad)
    assert torch.equal(probs[~bad], out["clean"][1][~bad])
