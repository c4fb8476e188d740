"""GPU: the node-style head (csrc/node_loss.cu: ddfa_node_head_fwd, ddfa_node_head_bwd, ddfa_node_bce and ddfa_node_bce_scaled)
at every hidden width the engines train, D = 20 .. 512 (K = 2D inputs up to 1024), at the C1 node count with a trainer-like row
list, at the 40 001-node hub count with 0 to N rows, and 16 layers deep, against float64 on the GPU.

The reference is tests/head_batches.py::node_head_ref: each stage from the kernel's own fp32 inputs, each hidden ReLU on the side
of its kink the kernel's forward took, and a per-element bound |got - ref| <= tau * mag from the accumulation depth of that stage
(the forward GEMM's K, the weight-gradient chunk of ceil(S / 32) rows plus the 32-way chunk reduction, the bias partials).  A
proportional bias got = (1 + beta) ref is bounded on its own (see _beta_bound).  Also pinned: the weight and bias gradients are
accumulated onto their start values; dh / dx are exactly 0 outside the listed rows; logits and activations past S keep their
sentinel; the rows past S are never read (they hold valid, wrong node ids); the frozen-encoder call (no dh / dx) gives the same
gradients bit for bit; two runs are bit-identical in both tuning modes.  Every case prints its worst error / bound."""
import contextlib
import math

import pytest
import torch

import head_batches as H
from deepdfa_b200 import engine as E
from deepdfa_b200._lib import TUNE_DETERMINISTIC, lib
from scale_batches import HUB_SHAPES
from width_batches import C1_NODES

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
SENTINEL = 7.0
BETA_TOL = 1e-5             # tests/test_wide_tc_gpu.py::BETA_TOL
HUB_NODES = HUB_SHAPES["mid"][2]


@contextlib.contextmanager
def _mode(det):
    L = lib()
    prev = L.call("ddfa_tuning_get", TUNE_DETERMINISTIC)
    L.call("ddfa_tuning_set", TUNE_DETERMINISTIC, int(det))
    try:
        yield
    finally:
        L.call("ddfa_tuning_set", TUNE_DETERMINISTIC, prev)


@pytest.fixture(autouse=True)
def _free_memory():
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    yield
    torch.cuda.empty_cache()


class _Filled:
    """engine's allocator interface with every buffer pre-filled: outputs with SENTINEL, the backward workspace with NaN bytes
    (a partial or plane read before it is written shows up as NaN)."""

    def get(self, name, shape, dtype=torch.float32):
        if dtype == torch.uint8:
            return torch.full(shape, 0xFF, dtype=dtype, device=DEV)
        return torch.full(shape, SENTINEL, dtype=dtype, device=DEV)


def _beta(got, ref):
    return float(((got - ref) * ref).sum() / (ref * ref).sum().clamp_min(1e-300))


def _beta_bound(ref, bound):
    """|beta| <= max(BETA_TOL, 4 sqrt(sum (bound ref)^2) / sum ref^2): errors of random sign within the per-element bound give a
    beta below a quarter of the second term; a shrink of the whole result by a fraction of the element bound does not."""
    return max(BETA_TOL, 4 * float((bound * ref).square().sum().sqrt() / (ref * ref).sum().clamp_min(1e-300)))


def _case(N, D, L, rows, seed):
    """Inputs on the device: h, x [N, D]; He-scaled layers (head_batches.mlp_params); dlogits [N] (the first S used); the
    gradients' start values; rows [N] with the listed rows first and valid but wrong node ids after S."""
    gen = torch.Generator(device=DEV).manual_seed(seed)
    h = torch.randn(N, D, device=DEV, generator=gen)
    x = torch.randn(N, D, device=DEV, generator=gen)
    ws, bs = H.mlp_params(D, L, seed)
    ws, bs = [w.to(DEV) for w in ws], [b.to(DEV) for b in bs]
    dl = torch.randn(N, device=DEV, generator=gen)
    dw0 = [torch.randn(w.shape, device=DEV, generator=gen) for w in ws]
    db0 = [torch.randn(b.shape, device=DEV, generator=gen) for b in bs]
    S = len(rows)
    rows_d = torch.empty(N, dtype=torch.int32, device=DEV)
    rows_d[:S] = torch.as_tensor(rows, dtype=torch.int32).to(DEV)
    rows_d[S:] = torch.randperm(N, device=DEV, generator=gen)[: N - S].to(torch.int32)
    return h, x, ws, bs, dl, dw0, db0, rows_d, S


def _run(h, x, ws, bs, dl, dw0, db0, rows_d, S, input_grads=True):
    params = E.ParamPack([], None, None, None, None, None, None, None, None, ws, bs)
    grads = E.ParamPack([], None, None, None, None, None, None, None, None, [t.clone() for t in dw0], [t.clone() for t in db0])
    num_rows = torch.tensor([S], dtype=torch.int32, device=DEV)
    alloc = _Filled()
    logits, act = E.node_head_fwd(params, x, h, rows_d, num_rows, alloc=alloc)
    dh, dx = E.node_head_bwd(params, grads, dl, x, h, rows_d, num_rows, act, alloc=alloc, input_grads=input_grads)
    torch.cuda.synchronize()
    return dict(logits=logits, act=act, dh=dh, dx=dx, dw=grads.mlp_w, db=grads.mlp_b)


def _check(N, D, L, rows, seed, repeats=True):
    """One case: the kernel against node_head_ref, the exact semantics, and (repeats) the bit-identical repeats."""
    h, x, ws, bs, dl, dw0, db0, rows_d, S = _case(N, D, L, rows, seed)
    got = _run(h, x, ws, bs, dl, dw0, db0, rows_d, S)
    K = 2 * D
    # past S: logits and activations untouched; dh / dx exactly zero outside the listed rows
    assert bool((got["logits"][S:] == SENTINEL).all()), "a logit past S was written"
    if L > 1:
        assert bool((got["act"][:, S:] == SENTINEL).all()), "an activation row past S was written"
    listed = torch.zeros(N, dtype=torch.bool, device=DEV)
    r = rows_d[:S].long()
    listed[r] = True
    for t in (got["dh"], got["dx"]):
        assert not bool(t[~listed].any()), "dh / dx not zero outside the listed rows"
    worst, betas = {}, {}

    def put(name, g, ref, mag, tau, beta=True):
        g = g.double()
        bound = tau * mag
        worst[name] = H.ratio((g - ref).abs(), bound)
        if beta and ref.numel():
            worst[f"{name} beta"] = abs(_beta(g, ref)) / _beta_bound(ref, bound)
        elif ref.numel():
            betas[name] = _beta(g, ref)

    if S:
        ins0 = torch.cat([h[r], x[r]], 1)
        acts = [got["act"][i][:S] for i in range(L - 1)]
        ref = H.node_head_ref(ins0, acts, ws, bs, dl[:S], dw0, db0)
        del ins0
        for i in range(L - 1):
            put(f"act{i}", acts[i], *ref.pop(f"act{i}"))
        put("logits", got["logits"][:S], *ref.pop("logits"))
        din, dmag, dtau = ref.pop("din")
        put("dh", got["dh"][r], din[:, :D], dmag[:, :D], dtau)
        put("dx", got["dx"][r], din[:, D:], dmag[:, D:], dtau)
        del din, dmag
        for i in range(L):
            put(f"dw{i}", got["dw"][i], *ref.pop(f"dw{i}"))
            put(f"db{i}", got["db"][i], *ref.pop(f"db{i}"), beta=False)
        del ref
    else:       # no rows: nothing but the start values
        for i in range(L):
            assert torch.equal(got["dw"][i], dw0[i]) and torch.equal(got["db"][i], db0[i])
    chunk = -(-S // H.NODE_HEAD_CHUNKS)
    print(f"node head D={D} K={K} L={L} N={N} S={S} (weight-gradient chunks of {chunk} rows): worst |err| / bound: "
          + ", ".join(f"{k}={v:.3g}" for k, v in worst.items())
          + ("; bias-vector beta (reported): " + ", ".join(f"{k}={v:+.1e}" for k, v in betas.items()) if betas else ""))
    bad = {k: v for k, v in worst.items() if not v <= 1.0}
    assert not bad, bad
    if not repeats:
        return
    # other wrong ids past S, the other tuning mode, and the frozen-encoder call: the same bits
    rows_b = rows_d.clone()
    rows_b[S:] = torch.flip(rows_d[S:], [0])
    for det, rows_ in ((False, rows_b), (True, rows_d)):
        with _mode(det):
            again = _run(h, x, ws, bs, dl, dw0, db0, rows_, S)
        for k in ("logits", "dh", "dx"):
            assert torch.equal(again[k], got[k]), (k, det)
        if L > 1:
            assert torch.equal(again["act"], got["act"]), det
        assert all(torch.equal(a, b) for a, b in zip(again["dw"] + again["db"], got["dw"] + got["db"])), det
        del again
    frozen = _run(h, x, ws, bs, dl, dw0, db0, rows_d, S, input_grads=False)
    assert frozen["dh"] is None and frozen["dx"] is None
    assert all(torch.equal(a, b) for a, b in zip(frozen["dw"] + frozen["db"], got["dw"] + got["db"])), "frozen-encoder call differs"


# ---- C1: 157 381 nodes, the trainer's row list ---------------------------------------------------------------------------------
@pytest.mark.parametrize("D", H.NODE_HEAD_WIDTHS)
def test_head_at_c1_every_width(D):
    """Three layers at the C1 node count over a trainer-like row list (about 30 % of the nodes, S % 64 != 0, nodes 0 and N - 1
    listed): both hidden GEMM forms (gathered and compact), the masked and the scattering dgrad, chunks of about 1 500 rows."""
    _check(C1_NODES, D, 3, H.node_rows_trainer(C1_NODES, seed=D + 1), seed=D)


@pytest.mark.parametrize("D", [20, 192, 512])
@pytest.mark.parametrize("L", [1, 2])
def test_head_at_c1_every_row(D, L):
    """One and two layers at C1 with every node listed: the gathered last layer (L = 1) and the dgrad straight from the last
    layer into the planes (L = 2); weight-gradient chunks of 4 919 rows; at D = 512 a workspace of 1.4 GB."""
    _check(C1_NODES, D, L, H.node_rows(C1_NODES, -1, 0), seed=100 + D + L, repeats=(D == 512))


# ---- the hub node count: few rows, empty chunks, every row ----------------------------------------------------------------------
@pytest.mark.parametrize("D", [20, 448])
@pytest.mark.parametrize("S", H.NODE_SMALL_S)
def test_head_row_counts_at_hub_size(D, S):
    """Three layers at the 40 001-node hub count with S = 0, 1, 5, 31, 32, 33 and N rows: below 32 rows most of the 32 chunks are
    empty; S = 0 leaves everything but the zeroed dh / dx untouched."""
    _check(HUB_NODES, D, 3, H.node_rows(HUB_NODES, S, S + D), seed=S + D, repeats=S in (5, 33))


@pytest.mark.parametrize("D", [20, 64])
def test_head_sixteen_layers(D):
    """The deepest head (kMaxLayers = 16) at a small N: the bound grows with each layer's tau."""
    N = 613
    _check(N, D, 16, H.node_rows(N, 245, D), seed=D)


# ---- the loss -----------------------------------------------------------------------------------------------------------------
def _bce_ref(z, y, pw):
    """float64 BCEWithLogits(pos_weight) per row and its derivative: (1 - y) z + lw softplus(-z), (1 - y) - lw sigmoid(-z)."""
    z, y = z.double(), y.double()
    lw = 1 + (pw - 1) * y
    loss = (1 - y) * z + lw * torch.nn.functional.softplus(-z)
    grad = (1 - y) - lw * torch.sigmoid(-z)
    mag = (1 - y) * z.abs() + lw * (torch.log1p(torch.exp(-z.abs())) + torch.relu(-z))     # the kernel's terms before they cancel
    return loss, grad, lw, mag


@pytest.mark.parametrize("pw,grad_scale", [(1.0, None), (4.0, None), (4.0, 0.25), (1.0, 3.0)])
def test_node_bce_at_c1(pw, grad_scale):
    """ddfa_node_bce (grad_scale None) and ddfa_node_bce_scaled over the C1 trainer row list, with logits 0, +-1e-8, +-30 and
    +-100 among the rows, against float64 BCEWithLogits(pos_weight) and its gradient; dlogits past S keep their sentinel; S = 0
    gives a NaN loss.  Bounds: each row's term within a few ulps of the magnitudes it cancels (expf / log1pf are not correctly
    rounded), then a ceil(S / 1024)-term strided sum and a 10-level tree; each dlogit 8 u of (|1 - y| + 2 lw) / S x the scale."""
    N = C1_NODES
    rows = H.node_rows_trainer(N, seed=3)
    S = len(rows)
    gen = torch.Generator(device=DEV).manual_seed(5)
    vuln = (torch.rand(N, device=DEV, generator=gen) < 0.3).to(torch.int32)
    logits = torch.randn(N, device=DEV, generator=gen) * 4
    special = torch.tensor([0.0, 1e-8, -1e-8, 30.0, -30.0, 100.0, -100.0], device=DEV)
    for j, v in enumerate(special.tolist()):
        logits[j * 997 % S: S: 4111] = v           # each value spread over the row positions
    rows_d = torch.as_tensor(rows, dtype=torch.int32).to(DEV)
    rows_d = torch.cat([rows_d, torch.zeros(N - S, dtype=torch.int32, device=DEV)])
    num_rows = torch.tensor([S], dtype=torch.int32, device=DEV)
    loss = torch.full((1,), SENTINEL, device=DEV)
    dl = E.node_bce(logits, vuln, rows_d, num_rows, pw, loss, alloc=_Filled(), grad_scale=grad_scale)
    torch.cuda.synchronize()
    assert bool((dl[S:] == SENTINEL).all()), "a dlogit past S was written"
    y = vuln[rows_d[:S].long()]
    terms, grad, lw, mag = _bce_ref(logits[:S], y, pw)
    for v in special.tolist():
        assert bool((logits[:S] == v).any())
    scale = (1.0 if grad_scale is None else grad_scale) / S
    ref_loss = float(terms.sum()) / S
    loss_bound = 2 * H.U * (-(-S // 1024) + 10 + 8) * float(mag.sum()) / S
    dl_bound = 8 * H.U * scale * ((1 - y.double()) + 2 * lw)
    worst = dict(loss=abs(float(loss) - ref_loss) / loss_bound, dlogits=H.ratio((dl[:S].double() - scale * grad).abs(), dl_bound))
    print(f"node bce pw={pw} grad_scale={grad_scale} S={S}: worst |err| / bound: " + ", ".join(f"{k}={v:.3g}" for k, v in worst.items()))
    assert all(v <= 1.0 for v in worst.values()), worst
    num_rows.zero_()
    E.node_bce(logits, vuln, rows_d, num_rows, pw, loss, alloc=_Filled(), grad_scale=grad_scale)
    torch.cuda.synchronize()
    assert math.isnan(float(loss)), "a mean over no rows is NaN"
