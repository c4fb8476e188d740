"""GPU: everything after the GatedGraphConv — the readout and MLP head forward (csrc/readout.cu), the readout and MLP backward,
the graph loss with bucket padding (csrc/loss_adam.cu) and the node-row sampler (csrc/node_loss.cu) — at training sizes and edge
shapes, against fp64 host references with per-element a-priori bounds and against an exact host sampler (tests/head_batches.py;
tests/test_head_premises.py checks the references and that the shapes reach their edges).  Every test prints its worst error
as a fraction of its bound."""
import numpy as np
import pytest
import torch

import head_batches as H
from deepdfa_b200 import engine as E
from deepdfa_b200._lib import TUNE_DETERMINISTIC, DdfaError, lib, ptr_array
from deepdfa_b200.engine import _p, _stream_ptr

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
NAN = float("nan")


class _Mode:
    """DDFA_TUNE_DETERMINISTIC set for the block, restored after it."""

    def __init__(self, det: bool):
        self.det = det

    def __enter__(self):
        self.old = lib().call("ddfa_tuning_get", TUNE_DETERMINISTIC)
        lib().call("ddfa_tuning_set", TUNE_DETERMINISTIC, int(self.det))

    def __exit__(self, *exc):
        lib().call("ddfa_tuning_set", TUNE_DETERMINISTIC, self.old)


def _report(what, worst):
    print(f"{what}: worst |err| / bound: " + ", ".join(f"{k}={v:.3g}" for k, v in worst.items()))
    assert all(v <= 1.0 for v in worst.values()), worst      # also fails on nan


def _readout_fwd(hd, xd, gp, sizes, D, wd, bd, mw, mb, L, with_act=True):
    """One ddfa_readout_mlp_fwd call with every output pre-filled with NaN."""
    B, N = len(sizes), hd.shape[0]
    out = dict(pooled=torch.full((B, 2 * D), NAN, device=DEV), logits=torch.full((B,), NAN, device=DEV),
               gl=torch.full((N,), NAN, device=DEV), smax=torch.full((B,), NAN, device=DEV), ssum=torch.full((B,), NAN, device=DEV),
               act=torch.full((max(L - 1, 1), B, 2 * D), NAN, device=DEV))
    lib().call("ddfa_readout_mlp_fwd", _p(hd), _p(xd), _p(gp), B, D, _p(wd), _p(bd), ptr_array([_p(t) for t in mw]) if L else None,
               ptr_array([_p(t) for t in mb]) if L else None, L, _p(out["pooled"]), _p(out["logits"]) if L else None, _p(out["gl"]),
               _p(out["smax"]), _p(out["ssum"]), _p(out["act"]) if with_act else None, _stream_ptr())
    torch.cuda.synchronize()
    return {k: v.cpu() for k, v in out.items()}


def _check_fwd(sizes, h, x, w, b, ws, bs, L, out, D):
    """worst / bound of every forward output; the MLP stages from the kernel's own input to each stage."""
    worst = {}
    r = H.pool_ref(h, x, w, b, sizes)
    seg = H.segment_ids(sizes)
    B = len(sizes)
    worst["gate_logit"] = H.ratio((out["gl"].double() - r["g"]).abs(), r["g_bound"])
    gl_max = torch.full((B,), -np.inf).scatter_reduce(0, seg, out["gl"], "amax")
    assert torch.equal(out["smax"], gl_max)                                         # -inf for an empty graph
    S, S_b = H.seg_sum_ref(out["gl"], out["smax"], sizes)
    worst["seg_sum"] = H.ratio((out["ssum"].double() - S).abs(), S_b)
    worst["pooled"] = H.ratio((out["pooled"].double() - r["pooled"]).abs(), r["pooled_bound"])
    empty = torch.from_numpy(np.asarray(sizes) == 0)
    assert (out["pooled"][empty] == 0).all() and (out["ssum"][empty] == 0).all()
    a = out["pooled"]
    for i in range(L):
        ref, bound = H.linear_ref(a, ws[i], bs[i], relu=i < L - 1)
        got = out["act"][i] if i < L - 1 else out["logits"][:, None]
        worst[f"layer{i}"] = H.ratio((got.double() - ref).abs(), bound)
        a = got
    return worst


def _put(ws, bs):
    return [w.to(DEV) for w in ws], [b.to(DEV) for b in bs]


# ---- readout forward ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("shape,D,L,extreme", [
    ("c1", 128, 3, False), ("big", 128, 3, False), ("big", 512, 1, False), ("mixed", 256, 16, False), ("mixed", 384, 3, False),
    ("mixed", 512, 0, False), ("big", 128, 3, True), ("c1", 128, 1, True)])
def test_readout_fwd_matches_fp64(shape, D, L, extreme):
    """Gate logits, segment max / sum, pooling and every MLP stage against fp64 with a-priori bounds.  B >= 256 (c1) takes the
    batched MLP, the others the in-CTA one; D = 384 runs the 4-chunk kernel with its masked fourth chunk.  extreme: b_gate = +85
    (no softmax without the running max survives it) and one graph whose logits span 200."""
    sizes = H.READOUT_SHAPES[shape]()
    h, x, w, b = H.readout_inputs(sizes, D, seed=D + L, extreme=extreme)
    ws, bs = H.mlp_params(D, L, D)
    mw, mb = _put(ws, bs)
    gp = H.graph_ptr(sizes).to(DEV)
    out = _readout_fwd(h.to(DEV), x.to(DEV), gp, sizes, D, w.to(DEV), b.to(DEV), mw, mb, L)
    worst = _check_fwd(sizes, h, x, w, b, ws, bs, L, out, D)
    _report(f"readout fwd {shape} D={D} L={L}{' extreme' if extreme else ''} N={h.shape[0]} B={len(sizes)}", worst)


@pytest.mark.parametrize("L", [1, 3, 16])
def test_readout_fwd_both_sides_of_the_batched_mlp_switch(L):
    """B = 255 (in-CTA MLP) and B = 256 (batched MLP) over the same first 255 graphs: each side within its bound, the same pooling
    bits, and the first MLP layer's output (same input on both sides) of the shared graphs within the sum of the two bounds."""
    D = 128
    sizes = H.switch_sizes()
    h, x, w, b = H.readout_inputs(sizes, D, seed=L)
    ws, bs = H.mlp_params(D, L, L)
    mw, mb = _put(ws, bs)
    worst, outs = {}, {}
    for B in (255, 256):
        s = sizes[:B]
        n = int(s.sum())
        out = _readout_fwd(h[:n].to(DEV), x[:n].to(DEV), H.graph_ptr(s).to(DEV), s, D, w.to(DEV), b.to(DEV), mw, mb, L)
        for k, v in _check_fwd(s, h[:n], x[:n], w, b, ws, bs, L, out, D).items():
            worst[f"B={B},{k}"] = v
        outs[B] = out
    assert torch.equal(outs[255]["pooled"], outs[256]["pooled"][:255])
    _, bound = H.linear_ref(outs[255]["pooled"], ws[0], bs[0], relu=L > 1)
    first = [(outs[B]["act"][0] if L > 1 else outs[B]["logits"][:, None])[:255].double() for B in (255, 256)]
    worst["B=255 vs 256 layer0"] = H.ratio((first[1] - first[0]).abs(), 2 * bound)
    _report(f"readout fwd switch L={L}", worst)


def test_readout_fwd_rejects_17_layers():
    D, B = 128, 2
    with pytest.raises(DdfaError, match="num_layers=17 out of range"):
        lib().call("ddfa_readout_mlp_fwd", 256, 256, 256, B, D, 256, 256, ptr_array([256] * 17), ptr_array([256] * 17), 17, 256, 256,
                   None, None, None, None, _stream_ptr())


# ---- readout backward ---------------------------------------------------------------------------------------------------------
PAD = 5            # sentinel rows after N in the dh / dx views
SENTINEL = 12345.0


@pytest.mark.parametrize("shape,D,extreme", [("c1", 128, False), ("big", 128, True), ("mixed", 384, False), ("big", 512, False)])
def test_readout_bwd_matches_fp64(shape, D, extreme):
    """ddfa_readout_bwd_ws (default and deterministic mode, full and gate-only) and ddfa_readout_bwd against the fp64 gradient fed
    the kernel's own saved gate logits, segment max and sum.  dh / dx are views into buffers with sentinel rows after N: those
    must come back untouched, every row below N written; dw_gate / db_gate accumulate onto a nonzero start."""
    sizes = H.READOUT_SHAPES[shape]()
    B, D2 = len(sizes), 2 * D
    h, x, w, b = H.readout_inputs(sizes, D, seed=7 + D, extreme=extreme)
    N = h.shape[0]
    hd, xd, wd, gp = h.to(DEV), x.to(DEV), w.to(DEV), H.graph_ptr(sizes).to(DEV)
    out = _readout_fwd(hd, xd, gp, sizes, D, wd, b.to(DEV), [], [], 0)
    gen = torch.Generator().manual_seed(D)
    dp = torch.randn(B, D2, generator=gen)
    dw0, db0 = torch.randn(D2, generator=gen), torch.randn(1, generator=gen)
    r = H.readout_bwd_ref(h, x, w, sizes, dp, out["pooled"], out["gl"], out["smax"], out["ssum"], dw0, db0)
    dpd, pd = dp.to(DEV), out["pooled"].to(DEV)
    gld, smd, ssd = out["gl"].to(DEV), out["smax"].to(DEV), out["ssum"].to(DEV)
    ws_bytes = lib().call("ddfa_readout_bwd_workspace_bytes", B, D)
    wsp = torch.empty(ws_bytes, dtype=torch.uint8, device=DEV)

    def run(name, planes=True):
        bufs = [torch.full((N + PAD, D), NAN, device=DEV) for _ in range(2)]
        for t in bufs:
            t[N:] = SENTINEL
        dh, dx = (bufs[0][:N], bufs[1][:N]) if planes else (None, None)
        dwg, dbg = dw0.to(DEV), db0.to(DEV)
        args = [_p(dpd), _p(pd), _p(hd), _p(xd), _p(gp), B, D, _p(wd), _p(gld), _p(smd), _p(ssd), _p(dh), _p(dx), _p(dwg), _p(dbg)]
        if name == "ws":
            lib().call("ddfa_readout_bwd_ws", *args, _p(wsp), ws_bytes, _stream_ptr())
        else:
            lib().call("ddfa_readout_bwd", *args, _stream_ptr())
        torch.cuda.synchronize()
        if planes:
            for t in bufs:
                assert (t[N:] == SENTINEL).all()                 # rows past N untouched
        return [t[:N].cpu() for t in bufs] if planes else None, dwg.cpu(), dbg.cpu()

    def check(tag, res):
        planes, dwg, dbg = res
        if planes is not None:
            worst[f"{tag} dh"] = H.ratio((planes[0].double() - r["dh"]).abs(), r["dh_bound"])
            worst[f"{tag} dx"] = H.ratio((planes[1].double() - r["dx"]).abs(), r["dx_bound"])
        worst[f"{tag} dw_gate"] = H.ratio((dwg.double() - r["dw"]).abs(), r["dw_bound"])
        worst[f"{tag} db_gate"] = H.ratio((dbg.double() - r["db"]).abs(), r["db_bound"])

    worst = {}
    with _Mode(False):
        check("ws", run("ws"))
        check("atomic", run("plain"))
        check("ws gate-only", run("ws", planes=False))
    with _Mode(True):
        first, again, gate = run("ws"), run("ws"), run("ws", planes=False)
        check("det", first)
        check("det gate-only", gate)
        assert all(torch.equal(p, q) for p, q in zip(first[0], again[0]))
        assert torch.equal(first[1], again[1]) and torch.equal(first[2], again[2])
        assert torch.equal(gate[1], first[1]) and torch.equal(gate[2], first[2])
    _report(f"readout bwd {shape} D={D}{' extreme' if extreme else ''} N={N} B={B}", worst)


# ---- MLP backward ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B", [1000, 1024, 255])
@pytest.mark.parametrize("L", [1, 3, 16])
def test_mlp_bwd_matches_fp64(B, L):
    """ddfa_mlp_bwd at the batch sizes of the bias-gradient row slices (1000: ragged slices, 1024: even, 255: one slice), in both
    modes: dpooled, and dW / db accumulated onto a nonzero start, within bounds propagated through the layers; the
    deterministic mode bit-identical over two calls."""
    D = 128
    D2 = 2 * D
    ws, _ = H.mlp_params(D, L, B + L)
    gen = torch.Generator().manual_seed(B * L)
    pooled = torch.randn(B, D2, generator=gen)
    acts = [torch.relu(torch.randn(B, D2, generator=gen)) for _ in range(L - 1)]
    dl = (torch.randn(B, generator=gen) + 0.5) / B          # mostly one sign, like a batch whose predictions lean one way
    dw0 = [0.01 * torch.randn(w.shape, generator=gen) for w in ws]
    db0 = [0.01 * torch.randn(w.shape[0], generator=gen) for w in ws]
    r = H.mlp_bwd_ref(dl, pooled, acts, ws, dw0, db0)
    mw = [w.to(DEV) for w in ws]
    pd, dld = pooled.to(DEV), dl.to(DEV)
    actd = torch.stack(acts).to(DEV) if L > 1 else torch.zeros(1, B, D2, device=DEV)

    def run():
        gw, gb = [t.to(DEV) for t in dw0], [t.to(DEV) for t in db0]
        dpo = torch.full((B, D2), NAN, device=DEV)
        scratch = torch.full((2, B, D2), NAN, device=DEV)
        lib().call("ddfa_mlp_bwd", _p(dld), _p(pd), _p(actd), ptr_array([_p(t) for t in mw]), B, D, L, _p(dpo),
                   ptr_array([_p(t) for t in gw]), ptr_array([_p(t) for t in gb]), _p(scratch), _stream_ptr())
        torch.cuda.synchronize()
        return dpo.cpu(), [t.cpu() for t in gw], [t.cpu() for t in gb]

    worst = {}
    for det in (False, True):
        with _Mode(det):
            dpo, gw, gb = run()
            if det:
                again = run()
                assert torch.equal(again[0], dpo) and all(torch.equal(p, q) for p, q in zip(again[1] + again[2], gw + gb))
        m = "det" if det else "default"
        worst[f"{m} dpooled"] = H.ratio((dpo.double() - r["dpooled"][0]).abs(), r["dpooled"][1])
        for i in range(L):
            dW, dW_b, db, db_b = r[i]
            worst[f"{m} dW{i}"] = H.ratio((gw[i].double() - dW).abs(), dW_b)
            worst[f"{m} db{i}"] = H.ratio((gb[i].double() - db).abs(), db_b)
    top = {k: v for k, v in worst.items() if k.endswith(f"W{L - 1}") or k.endswith(f"b{L - 1}") or k.endswith("dpooled")}
    print(f"mlp bwd B={B} L={L} (last layer and dpooled shown, all {len(worst)} checked): "
          + ", ".join(f"{k}={v:.3g}" for k, v in top.items()))
    _report(f"mlp bwd B={B} L={L} all", {"max": max(worst.values())})


# ---- graph loss with bucket padding --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B,num_valid", H.BCE_CASES)
@pytest.mark.parametrize("pw", [1.0, 4.0])
def test_graph_label_bce_valid_matches_fp64(B, num_valid, pw):
    """ddfa_graph_label_bce_valid against torch.nn.BCEWithLogitsLoss in fp64 over the valid graphs, both modes.  Padding graphs
    get their label and a dlogit of exactly 0 and add nothing to the loss; the deterministic loss is bit-identical over repeats."""
    sizes = H.bce_sizes(B, B + num_valid)
    gp = H.graph_ptr(sizes)
    seg = H.segment_ids(sizes)
    N = int(sizes.sum())
    vuln = (torch.rand(N, generator=torch.Generator().manual_seed(B)) < 0.05).to(torch.int32)
    labels_ref = torch.zeros(B, dtype=torch.int32).scatter_reduce(0, seg, vuln, "amax").double()
    z = H.bce_logits(B, B)
    ls, gs = 1.0 / max(num_valid, 1), 1.0 / max(num_valid, 1)
    zv = z[:num_valid].double().requires_grad_(True)
    crit = torch.nn.BCEWithLogitsLoss(reduction="sum", pos_weight=torch.tensor([pw], dtype=torch.float64))
    loss_ref = crit(zv, labels_ref[:num_valid]) * ls
    loss_ref.backward()
    loss_ref = float(loss_ref.detach())
    dl_ref = torch.zeros(B, dtype=torch.float64)
    if num_valid:
        dl_ref[:num_valid] = zv.grad / ls * gs
    y = labels_ref[:num_valid]
    lw = 1 + (pw - 1) * y
    zz = z[:num_valid].double()
    terms = (1 - y) * zz.abs() + lw * (torch.log1p(torch.exp(-zz.abs())) + torch.clamp(-zz, min=0))
    # each term to a few ulps, then the longest summation chain: 8 warp terms per CTA plus the CTA atomics (default mode), or
    # B / 256 terms per thread plus the 256-way tree (deterministic mode)
    loss_bound = 2 * H.U * (B // 8 + 16) * float(terms.sum()) * ls
    dl_bound = torch.zeros(B, dtype=torch.float64)
    dl_bound[:num_valid] = 4 * H.U * gs * ((1 - y) + 2 * lw)
    vd, gpd, zd = vuln.to(DEV), gp.to(DEV), z.to(DEV)
    worst = {}
    for det in (False, True):
        with _Mode(det):
            losses = []
            for _ in range(2 if det else 1):
                labels, loss, dl = torch.full((B,), NAN, device=DEV), torch.full((1,), NAN, device=DEV), torch.full((B,), NAN, device=DEV)
                lib().call("ddfa_graph_label_bce_valid", _p(zd), _p(vd), _p(gpd), B, num_valid, pw, ls, gs, _p(labels), _p(loss), _p(dl),
                           _stream_ptr())
                torch.cuda.synchronize()
                losses.append(loss.cpu())
            if det:
                assert torch.equal(losses[0], losses[1])
            labels, loss, dl = labels.cpu(), losses[0], dl.cpu()
        m = "det" if det else "default"
        assert torch.equal(labels.double(), labels_ref)                      # padding graphs get their label too
        assert (dl[num_valid:] == 0).all() and not torch.signbit(dl[num_valid:]).any()
        worst[f"{m} loss"] = H.ratio(abs(float(loss) - float(loss_ref)), loss_bound)
        worst[f"{m} dlogits"] = H.ratio((dl.double() - dl_ref).abs(), dl_bound)
    if num_valid == 0:
        assert float(loss) == 0.0
    _report(f"graph bce B={B} valid={num_valid} pw={pw}", worst)


# ---- node-row sampler -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", H.sampler_cases(), ids=lambda c: c[0])
def test_node_sample_is_the_exact_host_draw(case):
    """ddfa_node_sample's row list, row count, status and draw counter equal the host reference's (the k smallest (Philox key,
    node) pairs, ties in node order) — among them a C1 draw whose k-th key is shared by two nodes in different sampler CTAs, once
    with only the first taken and once with both."""
    name, vuln, num_valid, factor, seed, draw = case
    rows_ref, S_ref, over, draw_next = H.sample_ref(vuln, num_valid, factor, seed, draw)
    N = len(vuln)
    rows = torch.full((N,), -7, dtype=torch.int32, device=DEV)
    num_rows = torch.full((1,), -1, dtype=torch.int32, device=DEV)
    status = torch.zeros(1, dtype=torch.int32, device=DEV)
    drawd = torch.tensor([draw], dtype=torch.int64, device=DEV)
    E.node_sample(torch.from_numpy(vuln).to(DEV), torch.tensor([num_valid], dtype=torch.int32, device=DEV), None if factor < 0 else factor,
                  seed, drawd, rows, num_rows, status)
    torch.cuda.synchronize()
    S = int(num_rows)
    assert S == S_ref, (name, S, S_ref)
    assert np.array_equal(rows[:S].cpu().numpy(), rows_ref), name
    assert int(status) == int(over) and int(drawd) == draw_next, name
    if name.startswith("c1_tie"):
        t = H.tie_case()
        got = set(rows[:S].cpu().numpy().tolist())
        assert t["a"] in got and (t["b"] in got) == (name == "c1_tie_ab")
    print(f"node sample {name}: N={N} rows={S} exact")
