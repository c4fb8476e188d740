"""GPU: the SIMT engine, the embedding and the weight fold at every hidden width the module accepts, at training sizes, against
float64 references of the same operations.

Widths other than 128 train on the fp32 SIMT engine (csrc/gru_step.cu + csrc/sgemm.cu).  Here each of its kernels runs at the
benchmark's C1 size (about 157 000 nodes) for W = 20 .. 512, chosen so that every dispatch path runs: both sgemm kernels with and
without their K splits, the ordered split-K of deterministic mode, every gather instance, both team forms of the deterministic
embedding backward (tests/width_batches.py; tests/test_width_premises.py checks on the CPU that the shapes still reach them).
References are float64 on the GPU (cuBLAS DGEMM, index_add_); the kernels are always called through the C ABI.  Every test
prints its worst error divided by its bound.

Bounds.  A sum of n fp32 terms evaluated with n - 1 roundings (in any order) is within (n - 1) u sum |terms| of the exact sum, u =
2^-24.  The kernels' sums are chains of known length: an sgemm output element is one FMA chain over a K slice, then the slices
added into C (sgemm_plan's "depth"), an embedding-gradient element one chain over a CTA's or a chunk's rows, then one partial per
CTA or chunk (embed_depth).  The bounds below are depth * u * (sum of the magnitudes), plus one rounding each for alpha, beta and
the store.  The GRU step, GatedGraphConv and module tests keep the bounds of tests/test_kernels_gpu.py and tests/test_scale_gpu.py,
which were set at widths up to 128; a length-W dot product's rounding errors grow like sqrt(W), so above 128 they are scaled by
sqrt(W / 128)."""
import contextlib

import pytest
import torch

import deepdfa_b200 as D
from deepdfa_b200 import synth
from deepdfa_b200._lib import ENGINE_SIMT, TUNE_DETERMINISTIC, DdfaError, lib, ptr_array
from deepdfa_b200.engine import _p, _stream_ptr, prepare_graph
from oracle import ggnn_oracle as O
from scale_batches import MODULE_C1, hub_batch
from test_scale_gpu import _gru_reference
from width_batches import C1_NODES, EMBED_V, SGEMM_EDGES, WIDTHS, embed_depth, engine_sgemm_calls, gather_instance, sgemm_plan

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
FEAT = "_ABS_DATAFLOW_api_all_limitall_1000_limitsubkeys_1000"
U = 2.0 ** -24


def _ratio(err, bound):
    """Largest err / bound (0 where both are 0, inf where only the bound is)."""
    return float(torch.where(bound > 0, err / bound.clamp_min(1e-300), torch.where(err > 0, float("inf"), 0.0)).max())


def _wf(W):
    """Growth of the bounds set at W <= 128 with the dot-product length."""
    return max(1.0, (W / 128) ** 0.5)


@contextlib.contextmanager
def _mode(deterministic):
    L = lib()
    prev = L.call("ddfa_tuning_get", TUNE_DETERMINISTIC)
    L.call("ddfa_tuning_set", TUNE_DETERMINISTIC, int(deterministic))
    try:
        yield
    finally:
        L.call("ddfa_tuning_set", TUNE_DETERMINISTIC, prev)


def _report(title, worst):
    peak = torch.cuda.max_memory_allocated() / 2 ** 30
    print(f"{title}: worst |err| / bound: " + ", ".join(f"{k}={v:.3f}" for k, v in worst.items()) + f"; peak {peak:.1f} GiB")


def _assert_within(worst):
    bad = {k: v for k, v in worst.items() if not v <= 1.0}          # NaN fails too
    assert not bad, bad


@pytest.fixture(autouse=True)
def _peak_memory():
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    yield


# ---- sgemm --------------------------------------------------------------------------------------------------------------
def _operand(rows, cols, gen, pad=0, offset=0):
    """A [rows x cols] fp32 operand with leading dimension cols + pad, starting `offset` floats into its allocation."""
    buf = torch.randn(offset + rows * (cols + pad), device=DEV, generator=gen)
    return buf[offset:].view(rows, cols + pad)[:, :cols], cols + pad


class _Sgemm:
    """One ddfa_sgemm problem: seeded operands, the fp64 reference and the magnitude sum |alpha| |A||B| + |beta| |C0|."""

    def __init__(self, ta, tb, M, N, K, alpha, beta, seed, pad_a=0, off_a=0, off_b=0):
        gen = torch.Generator(device=DEV).manual_seed(seed)
        self.A, self.lda = _operand(*((K, M) if ta else (M, K)), gen, pad_a, off_a)
        self.B, self.ldb = _operand(*((N, K) if tb else (K, N)), gen, 0, off_b)
        self.C0 = torch.randn(M, N, device=DEV, generator=gen)
        self.args = (ta, tb, M, N, K, alpha, beta)
        opA = (self.A.t() if ta else self.A).double()
        opB = (self.B.t() if tb else self.B).double()
        self.ref = alpha * (opA @ opB) + beta * self.C0.double()
        self.mag = abs(alpha) * (opA.abs() @ opB.abs()) + abs(beta) * self.C0.double().abs()

    def run(self, split=1):
        ta, tb, M, N, K, alpha, beta = self.args
        C = self.C0.clone()
        lib().call("ddfa_sgemm", ta, tb, M, N, K, alpha, _p(self.A), self.lda, _p(self.B), self.ldb, beta, _p(C), N, split, _stream_ptr())
        return C

    def ratio(self, C, plan):
        return _ratio((C.double() - self.ref).abs(), (plan["depth"] + 3) * U * self.mag)


def _check_sgemm(case, split, worst, key, repeats):
    """Default mode: within the bound of its plan.  Deterministic mode: refused with split_k > 1, else bit-repeatable and within
    the bound of its (unsplit) plan."""
    ta, tb, M, N, K, alpha, beta = case.args
    worst[key] = case.ratio(case.run(split), sgemm_plan(M, N, K, beta, split))
    with _mode(True):
        plan = sgemm_plan(M, N, K, beta, split, deterministic=True)
        if plan["kernel"] == "refused":
            with pytest.raises(DdfaError, match="deterministic"):
                case.run(split)
            return
        outs = [case.run(split) for _ in range(repeats)]
    assert all(torch.equal(o, outs[0]) for o in outs[1:]), key
    worst[key + " det"] = case.ratio(outs[0], plan)


@pytest.mark.parametrize("W", list(WIDTHS))
def test_sgemm_engine_calls_at_c1(W):
    """The exact sgemm calls of the SIMT GRU step (N = 157 381: forward, dgrad with beta 0 and 1, the split-K weight gradient),
    the weight fold and the batched MLP head (1024 graphs), default and deterministic mode."""
    worst = {}
    for i, (name, (ta, tb, M, N, K, beta, split)) in enumerate(engine_sgemm_calls(W, C1_NODES).items()):
        case = _Sgemm(ta, tb, M, N, K, 1.0, beta, seed=W * 100 + i)
        _check_sgemm(case, split, worst, name, repeats=2)
        del case
    _report(f"sgemm engine calls W={W}", worst)
    _assert_within(worst)


def test_sgemm_dispatch_edges():
    """Either side of each dispatch boundary of sgemm(): M N = 512^2, K = 4096, the small kernel's K split at K = 256 and at 132
    output tiles; alpha != 1 and beta 0, 0.5, 1 on both kernels; a leading dimension that is not a multiple of 4 and operands one
    float off 16-byte alignment (the scalar load paths)."""
    worst = {}
    for i, (name, (ta, tb, M, N, K, alpha, beta)) in enumerate(SGEMM_EDGES.items()):
        _check_sgemm(_Sgemm(ta, tb, M, N, K, alpha, beta, seed=i), 1, worst, name, repeats=3)
    for name in ("small,alpha,beta=0.5", "big,alpha,beta=0.5", "k=256,beta=1"):
        ta, tb, M, N, K, alpha, beta = SGEMM_EDGES[name]
        _check_sgemm(_Sgemm(ta, tb, M, N, K, alpha, beta, seed=7, pad_a=1), 1, worst, name + ",lda%4=1", repeats=2)
        _check_sgemm(_Sgemm(ta, tb, M, N, K, alpha, beta, seed=8, off_a=1, off_b=1), 1, worst, name + ",+1 float", repeats=2)
    # the 128x128 kernel's atomic split-K (beta == 1) on a ragged K
    c = _Sgemm(1, 0, 200, 72, 10_001, 1.0, 1.0, seed=9)
    _check_sgemm(c, 7, worst, "big split 7", repeats=2)
    _report("sgemm dispatch edges", worst)
    _assert_within(worst)


# ---- embedding ----------------------------------------------------------------------------------------------------------
EMBED_CASES = {          # name -> (V, index kind)
    "V=1002": (EMBED_V, "synth"),
    "V=1": (1, "synth"),
    "V=2": (2, "synth"),
    "all zero": (EMBED_V, "zeros"),
    "no hot row": (EMBED_V, "cold"),
    "out of range": (EMBED_V, "oob"),
}


def _indices(kind, N, V, K, gen):
    """synth's distribution (index 0 on ~75 % of the nodes, 1 on ~3 %, the rest uniform), all zeros, none in {0, 1}, or synth's
    with 10 % negative and 10 % >= V."""
    out = []
    for _ in range(K):
        if kind == "zeros":
            out.append(torch.zeros(N, dtype=torch.int64, device=DEV))
            continue
        if kind == "cold":
            out.append(torch.randint(2, V, (N,), device=DEV, generator=gen))
            continue
        v = torch.randint(0, V, (N,), device=DEV, generator=gen)
        r = torch.rand(N, device=DEV, generator=gen)
        v[r < 0.75] = 0
        v[(r >= 0.75) & (r < 0.78)] = min(1, V - 1)
        if kind == "oob":
            v[r >= 0.9] = V + torch.randint(0, 1000, (int((r >= 0.9).sum()),), device=DEV, generator=gen)
            v[(r >= 0.8) & (r < 0.9)] = -1 - torch.randint(0, 1000, (int(((r >= 0.8) & (r < 0.9)).sum()),), device=DEV, generator=gen)
        out.append(v)
    return out


@pytest.mark.parametrize("W", list(WIDTHS))
def test_embedding_at_c1(W):
    """ddfa_embed_concat_fwd / _bwd / _bwd_ws at N = 157 381: the forward is the table lookup bit for bit (and, for one 128-wide
    table, the image entry equals ddfa_act_to_image of the rows); the default backward (hot rows 0 and 1 privatised) and the
    deterministic one (segmented sums over the sorted indices, bit-repeatable over a garbage workspace) against fp64 index_add_,
    with and without dx2.  Out-of-range indices are clamped in the backward exactly as the forward reads them: negative ones to
    the hot row 0, those >= V to V - 1."""
    K, H = WIDTHS[W]
    N = C1_NODES
    L, st = lib(), _stream_ptr()
    gen = torch.Generator(device=DEV).manual_seed(W)
    dx = torch.randn(N, W, device=DEV, generator=gen)
    dx2 = torch.randn(N, W, device=DEV, generator=gen)
    worst = {}
    for case, (V, kind) in EMBED_CASES.items():
        idx = _indices(kind, N, V, K, gen)
        clamped = [i.clamp(0, V - 1) for i in idx]
        tables = [torch.randn(V, H, device=DEV, generator=gen) for _ in range(K)]
        ip, tp = ptr_array([_p(i) for i in idx]), ptr_array([_p(t) for t in tables])
        x = torch.full((N, W), float("nan"), device=DEV)
        oob = torch.zeros(1, dtype=torch.int32, device=DEV)
        L.call("ddfa_embed_concat_fwd", ip, tp, K, V, H, N, _p(x), _p(oob), st)
        assert torch.equal(x, torch.cat([t[i] for t, i in zip(tables, clamped)], 1)), case
        assert int(oob) == sum(int(((i < 0) | (i >= V)).sum()) for i in idx), case
        if W == 128 and case == "V=1002":
            ib = L.call("ddfa_act_image_bytes", N)
            img, img_ref = torch.full((ib,), 0x55, dtype=torch.uint8, device=DEV), torch.zeros(ib, dtype=torch.uint8, device=DEV)
            x2 = torch.empty_like(x)
            L.call("ddfa_embed_concat_fwd_image", ip, tp, K, V, H, N, _p(x2), _p(img), None, st)
            L.call("ddfa_act_to_image", _p(x), N, W, _p(img_ref), st)
            # rows N .. 128 ceil(N / 128) - 1 of the last tile are not written (include/ddfa_b200.h): compare rows < N there, and
            # check that the padding rows still hold what the buffer held
            tail = N % 128
            assert tail and torch.equal(x2, x) and torch.equal(img[:-65536], img_ref[:-65536])
            b = torch.arange(65536, device=DEV)
            row = (b % 16384) // 1024 * 8 + (b % 1024) // 128        # 4 planes of 128 rows x 128 B, rows in groups of 8
            last, last_ref = img[-65536:], img_ref[-65536:]
            assert torch.equal(last[row < tail], last_ref[row < tail]) and bool((last[row >= tail] == 0x55).all())
        init = [torch.randn(V, H, device=DEV, generator=gen) for _ in range(K)]
        # rows other than the two hot ones take one RED.ADD per node in the default backward: their chains are as long as their
        # node count
        depth = [embed_depth(N) + torch.bincount(c, minlength=V).double().index_fill_(0, torch.arange(min(2, V), device=DEV), 0)[:, None]
                 for c in clamped]
        for second in (None, dx2):
            g = dx if second is None else dx + second
            mag_rows = dx.abs() if second is None else dx.abs() + second.abs()
            refs = [init[k].double().index_add_(0, clamped[k], g[:, k * H:(k + 1) * H].double()) for k in range(K)]
            mags = [init[k].double().abs().index_add_(0, clamped[k], mag_rows[:, k * H:(k + 1) * H].double()) for k in range(K)]

            def ratio(gd):
                return max(_ratio((a.double() - r).abs(), d * U * m) for a, r, m, d in zip(gd, refs, mags, depth))

            tag = f"{case},dx2={'no' if second is None else 'yes'}"
            gd = [t.clone() for t in init]
            L.call("ddfa_embed_concat_bwd", ip, _p(dx), _p(second), K, V, H, N, ptr_array([_p(t) for t in gd]), st)
            worst[tag] = ratio(gd)
            nbytes = L.call("ddfa_embed_concat_bwd_workspace_bytes", K, V, H, N)
            ws = torch.empty(nbytes, dtype=torch.uint8, device=DEV)
            outs = []
            with _mode(True):
                for _ in range(2):
                    gd = [t.clone() for t in init]
                    ws.fill_(0xAB)                        # stale scratch must not matter
                    L.call("ddfa_embed_concat_bwd_ws", ip, _p(dx), _p(second), K, V, H, N, ptr_array([_p(t) for t in gd]), _p(ws),
                           nbytes, st)
                    outs.append(gd)
                torch.cuda.synchronize()
            assert all(torch.equal(a, b) for a, b in zip(*outs)), tag
            worst[tag + " det"] = ratio(outs[0])
            del outs, refs, mags, ws
    _report(f"embedding W={W} (K={K}, H={H}) N={N}", worst)
    _assert_within(worst)


# ---- weight folding ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("W", list(WIDTHS))
def test_fold_weights(W):
    """ddfa_fold_weights_fwd (w_fold = W_ih W, b_fold = W_ih b) and _bwd (+= into dW, db, dW_ih) against fp64."""
    gen = torch.Generator(device=DEV).manual_seed(W)
    k = W ** -0.5
    Wm, b, Wih = [(torch.rand(*sh, device=DEV, generator=gen) * 2 - 1) * k for sh in ((W, W), (W,), (3 * W, W))]
    dwf, dbf = torch.randn(3 * W, W, device=DEV, generator=gen), torch.randn(3 * W, device=DEV, generator=gen)
    gW0, gb0, gWih0 = torch.randn(W, W, device=DEV, generator=gen), torch.randn(W, device=DEV, generator=gen), torch.randn(3 * W, W, device=DEV, generator=gen)
    Wd, bd, Wihd, dwfd, dbfd = [t.double() for t in (Wm, b, Wih, dwf, dbf)]
    L, st = lib(), _stream_ptr()
    wf, bf = torch.full((3 * W, W), float("nan"), device=DEV), torch.full((3 * W,), float("nan"), device=DEV)
    L.call("ddfa_fold_weights_fwd", _p(Wm), _p(b), _p(Wih), W, _p(wf), _p(bf), st)
    worst = {}
    plan = sgemm_plan(3 * W, W, W)
    worst["w_fold"] = _ratio((wf.double() - Wihd @ Wd).abs(), (plan["depth"] + 2) * U * (Wihd.abs() @ Wd.abs()))
    worst["b_fold"] = _ratio((bf.double() - Wihd @ bd).abs(), (W + 2) * U * (Wihd.abs() @ bd.abs()))
    gW, gb, gWih = gW0.clone(), gb0.clone(), gWih0.clone()
    L.call("ddfa_fold_weights_bwd", _p(Wm), _p(b), _p(Wih), _p(dwf), _p(dbf), W, _p(gW), _p(gb), _p(gWih), st)
    p_ih, p_w = sgemm_plan(3 * W, W, W, 1.0), sgemm_plan(W, W, 3 * W, 1.0)
    ref = gWih0.double() + dwfd @ Wd.t() + torch.outer(dbfd, bd)
    mag = gWih0.double().abs() + dwfd.abs() @ Wd.abs().t() + torch.outer(dbfd.abs(), bd.abs())
    worst["dW_ih"] = _ratio((gWih.double() - ref).abs(), (p_ih["depth"] + 4) * U * mag)
    worst["dW"] = _ratio((gW.double() - gW0.double() - Wihd.t() @ dwfd).abs(),
                         (p_w["depth"] + 3) * U * (gW0.double().abs() + Wihd.abs().t() @ dwfd.abs()))
    worst["db"] = _ratio((gb.double() - gb0.double() - Wihd.t() @ dbfd).abs(),
                         (3 * W // 8 + 11) * U * (gb0.double().abs() + Wihd.abs().t() @ dbfd.abs()))
    _report(f"fold W={W}", worst)
    _assert_within(worst)


# ---- SIMT GRU step -------------------------------------------------------------------------------------------------------
GRAD_NAMES = ("dwf", "dbf", "dbih", "dwhh", "dbhh")


@pytest.mark.parametrize("W", list(WIDTHS))
def test_simt_gru_step_at_c1(W):
    """ddfa_gru_step_fwd / _bwd on the SIMT engine over the C1 hub batch (157 381 nodes, hub rows of in-degree up to 1100): h',
    the four gate planes, ds, dh and the five weight / bias gradients against fp64 autograd of the same math, in default and
    deterministic mode (bit-repeatable over a garbage workspace; the forward is the same in both).  Bounds of
    test_kernels_gpu.py::test_gru_step_fwd_bwd."""
    g = hub_batch("c1")
    dg = prepare_graph(g, DEV)
    N = g.num_nodes()
    L, st = lib(), _stream_ptr()
    gen = torch.Generator(device=DEV).manual_seed(W)
    k = W ** -0.5
    mk = lambda *sh: ((torch.rand(*sh, device=DEV, generator=gen) * 2 - 1) * k)
    wf, bf, bih, whh, bhh = mk(3 * W, W) * 1.5, mk(3 * W), mk(3 * W), mk(3 * W, W), mk(3 * W)
    h32 = torch.tanh(torch.randn(N, W, device=DEV, generator=gen))
    s32 = torch.empty(N, W, device=DEV)
    L.call("ddfa_gather_sum", _p(dg.indptr), _p(dg.indices), _p(h32), N, W, _p(s32), 0, st)
    dh_out = torch.randn(N, W, device=DEV, generator=gen)
    deg = torch.bincount(g.edges()[1].to(DEV), minlength=N).double()
    leaves = [t.double().requires_grad_(True) for t in (s32, h32, wf, bf, bih, whh, bhh)]
    h_ref, *gate_refs = _gru_reference(leaves[0], leaves[1], deg, *leaves[2:])
    (h_ref * dh_out.double()).sum().backward()
    h_ref = h_ref.detach()
    gate_refs = [t.detach() for t in gate_refs]
    refs = dict(ds=leaves[0].grad, dh=leaves[1].grad, dwf=leaves[2].grad, dbf=leaves[3].grad, dbih=leaves[4].grad,
                dwhh=leaves[5].grad, dbhh=leaves[6].grad)
    del leaves
    wfac = _wf(W)
    tol = dict(h=2e-5 * wfac, gate=5e-5 * wfac, grad=2e-4 * wfac)
    wsb = L.call("ddfa_gru_step_workspace_bytes", N, W, ENGINE_SIMT)
    ws = torch.empty(wsb, dtype=torch.uint8, device=DEV)
    wsb_b = L.call("ddfa_gru_step_bwd_workspace_bytes", N, W, ENGINE_SIMT)
    ws_b = torch.empty(wsb_b, dtype=torch.uint8, device=DEV)
    worst, results = {}, {}
    for det in (False, True):
        mode = "det" if det else "default"
        with _mode(det):
            h_out = torch.full((N, W), float("nan"), device=DEV)
            gates = torch.full((4, N, W), float("nan"), device=DEV)
            L.call("ddfa_gru_step_fwd", _p(s32), _p(h32), _p(dg.indptr), _p(wf), _p(bf), _p(bih), _p(whh), _p(bhh), N, W, _p(h_out),
                   _p(gates), _p(ws), wsb, ENGINE_SIMT, st)
            runs = []
            for rep in range(2 if det else 1):
                ws_b.fill_(0xAB)
                got = dict(ds=torch.full((N, W), float("nan"), device=DEV), dh=torch.full((N, W), float("nan"), device=DEV))
                got.update({n_: torch.zeros_like(refs[n_], dtype=torch.float32) for n_ in GRAD_NAMES})
                L.call("ddfa_gru_step_bwd", _p(dh_out), _p(h32), _p(s32), _p(gates), _p(dg.indptr), _p(wf), _p(whh), N, W, _p(got["ds"]),
                       _p(got["dh"]), *[_p(got[n_]) for n_ in GRAD_NAMES], _p(ws_b), wsb_b, ENGINE_SIMT, st)
                runs.append(got)
            torch.cuda.synchronize()
        if det:
            assert torch.equal(h_out, results["default"][0]) and torch.equal(gates, results["default"][1])
            assert all(torch.equal(runs[1][n_], runs[0][n_]) for n_ in refs), "deterministic backward not repeatable"
        else:
            worst["h'"] = float((h_out.double() - h_ref).abs().max()) / tol["h"]
            for name, got_, ref in zip(("r", "z", "n", "gh_n"), gates, gate_refs):
                scale = max(1.0, float(ref.abs().max())) if name == "gh_n" else 1.0
                worst[name] = float((got_.double() - ref).abs().max()) / (tol["gate"] * scale)
        for n_, ref in refs.items():
            worst[f"{n_} {mode}"] = float((runs[0][n_].double() - ref).abs().max()) / (tol["grad"] * max(1.0, float(ref.abs().max())))
        results[mode] = (h_out, gates)
        del runs
    _report(f"simt gru step W={W} N={N}", worst)
    _assert_within(worst)


# ---- edge gather -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("W", [W for W in WIDTHS if W != 128])
def test_gather_at_hub_degrees(W):
    """ddfa_gather_sum at every width other than 128 (gather_sum_kernel instances G = 8, 16, 32 with CH = 1, 2, 4) on the C1 hub
    batch, plain and accumulating, over the CSR and the transposed CSR.  Bound of
    test_scale_gpu.py::test_gather_variants_at_hub_degrees: |err| <= 2 (deg + acc) u (sum |h_src| + acc |out_0|)."""
    g = hub_batch("c1")
    dg = prepare_graph(g, DEV)
    N = g.num_nodes()
    gen = torch.Generator(device=DEV).manual_seed(W)
    h, base = torch.randn(N, W, device=DEV, generator=gen), torch.randn(N, W, device=DEV, generator=gen)
    L, st = lib(), _stream_ptr()
    src, dst = [t.to(DEV) for t in g.edges()]
    worst = {}
    for orient, ip, ix, s_, d_ in (("csr", dg.indptr, dg.indices, src, dst), ("transposed", dg.indptr_t, dg.indices_t, dst, src)):
        ref = torch.zeros(N, W, dtype=torch.float64, device=DEV).index_add_(0, d_, h.double()[s_])
        mag = torch.zeros(N, W, dtype=torch.float64, device=DEV).index_add_(0, d_, h.double().abs()[s_])
        deg = torch.bincount(d_, minlength=N).double()[:, None]
        for acc in (0, 1):
            out = base.clone() if acc else torch.full((N, W), float("nan"), device=DEV)
            L.call("ddfa_gather_sum", _p(ip), _p(ix), _p(h), N, W, _p(out), acc, st)
            r = ref + base.double() if acc else ref
            bound = 2 * (deg + acc) * U * (mag + base.double().abs() if acc else mag)
            worst[f"{orient},acc={acc}"] = _ratio((out.double() - r).abs(), bound)
    _report(f"gather W={W} instance {gather_instance(W)} N={N}", worst)
    _assert_within(worst)


# ---- whole GatedGraphConv -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("W", [32, 256, 512])
def test_ggnn_simt_drivers_at_width(W):
    """ddfa_ggnn_fwd / ddfa_ggnn_bwd on the SIMT engine, T = 8, on the 40 001-node hub batch, against fp64 autograd of the
    oracle's GatedGraphConv restatement.  Bounds of test_scale_gpu.py::test_ggnn_fused_drivers_at_scale."""
    T = 8
    g = hub_batch("mid")
    dg = prepare_graph(g, DEV)
    N = g.num_nodes()
    torch.manual_seed(W)
    conv = O.GatedGraphConvRestated(W, W, T).double().to(DEV)
    with torch.no_grad():
        conv.linears[0].bias.uniform_(-0.2, 0.2)
        for p in conv.parameters():
            p.copy_(p.float().double())                 # the kernels run on the fp32 values
    x = (torch.randn(N, W, device=DEV) * 0.5).double().requires_grad_(True)
    h_ref = conv(g.to(DEV), x)
    dh_T = torch.randn(N, W, device=DEV)
    (h_ref * dh_T.double()).sum().backward()
    par = dict(w_msg=conv.linears[0].weight, b_msg=conv.linears[0].bias, w_ih=conv.gru.weight_ih, w_hh=conv.gru.weight_hh,
               b_ih=conv.gru.bias_ih, b_hh=conv.gru.bias_hh)
    pd = {k: v.detach().float() for k, v in par.items()}
    xd = x.detach().float()
    amp = (torch.bincount(g.edges()[1].to(DEV), minlength=N).double() / 16).sqrt().clamp_min(1.0)[:, None]
    L, st = lib(), _stream_ptr()
    wsb = L.call("ddfa_ggnn_workspace_bytes", N, W, T, ENGINE_SIMT, 1)
    ws = torch.empty(wsb, dtype=torch.uint8, device=DEV)
    h_out = torch.full((N, W), float("nan"), device=DEV)
    L.call("ddfa_ggnn_fwd", _p(dg.indptr), _p(dg.indices), _p(xd), N, W, T, _p(pd["w_msg"]), _p(pd["b_msg"]), _p(pd["w_ih"]),
           _p(pd["w_hh"]), _p(pd["b_ih"]), _p(pd["b_hh"]), _p(h_out), _p(ws), wsb, 1, ENGINE_SIMT, st)
    worst = {"h_T": float(((h_out.double() - h_ref.detach()).abs() / amp).max()) / (3e-5 * T * _wf(W))}
    dx = torch.full((N, W), float("nan"), device=DEV)
    gr = {k: torch.zeros_like(v) for k, v in pd.items()}
    L.call("ddfa_ggnn_bwd", _p(dg.indptr), _p(dg.indptr_t), _p(dg.indices_t), _p(xd), N, W, T, _p(pd["w_msg"]), _p(pd["b_msg"]),
           _p(pd["w_ih"]), _p(pd["w_hh"]), _p(dh_T), _p(dx), _p(gr["w_msg"]), _p(gr["b_msg"]), _p(gr["w_ih"]), _p(gr["w_hh"]),
           _p(gr["b_ih"]), _p(gr["b_hh"]), _p(ws), wsb, ENGINE_SIMT, st)
    gtol = 1e-4 * T ** 0.5 * _wf(W)
    for k, got, ref in [("dx", dx, x.grad)] + [(k, gr[k], par[k].grad) for k in par]:
        worst[k] = float((got.double() - ref).abs().max()) / (gtol * max(1.0, float(ref.abs().max())))
    _report(f"ggnn simt drivers W={W} N={N} T={T}", worst)
    _assert_within(worst)


# ---- the module end to end ------------------------------------------------------------------------------------------------
GRAD_TOL = 1e-5         # test_scale_gpu.py::GRAD_TOL["simt"], per parameter, relative to its largest reference entry
BETA_TOL = 1e-5         # test_scale_gpu.py::BETA_TOL: proportional bias of the GGNN weight gradients
MODULE_WIDTHS = {       # W -> (hidden_dim, concat_all_absdf, batch)
    32: (32, False, "c1"),
    64: (16, True, "c1"),
    256: (64, True, "c1"),
    512: (512, False, "mid"),
}


def _module_batch(name):
    return synth.make_batch(**MODULE_C1) if name == "c1" else hub_batch("mid")


@pytest.mark.parametrize("W", list(MODULE_WIDTHS))
def test_module_gradients_at_width(W):
    """The SIMT training step's loss and every parameter gradient against OracleFlowGNNGGNN in float64 (run on the GPU), T = 8,
    three output layers: on the C1 batch (1024 graphs) for W = 32 (one table), 64 and 256, on the 40 001-node hub batch for
    W = 512.  At W = 256 also one FusedTrainer step against torch.optim.Adam on the oracle's gradients."""
    hidden, concat, batch = MODULE_WIDTHS[W]
    g = _module_batch(batch)
    gd = g.to(DEV)
    torch.manual_seed(1)
    o = O.OracleFlowGNNGGNN(FEAT, 1002, hidden, 8, 3, concat_all_absdf=concat, positive_weight=4.0).double().to(DEV)
    with torch.no_grad():
        for p in o.parameters():
            p.copy_(p.float().double())
    state = {k: v.float().cpu() for k, v in o.state_dict().items()}
    loss_ref, _ = o.training_loss(gd)
    loss_ref.backward()
    loss_ref = float(loss_ref)
    m = D.FlowGNNGGNNModule(FEAT, 1002, hidden, 8, 3, concat_all_absdf=concat, positive_weight=4.0)
    assert m.engine == "simt" and m._D == W
    m.load_state_dict(state)
    m.to(DEV)
    loss_t = m.training_step((gd, {}), 0)
    loss_t.backward()
    loss = float(loss_t)
    tol = GRAD_TOL * _wf(W)
    worst, shrink, delta = {}, {}, {}
    for (name, p), (_, q) in zip(m.named_parameters(), o.named_parameters()):
        ref, got = q.grad, p.grad.double()
        scale = max(float(ref.abs().max()), 1e-3)       # pooling.gate_nn.bias: true gradient 0 (softmax shift invariance)
        worst[name] = float((got - ref).abs().max()) / (tol * scale)
        shrink[name] = float(((got - ref) * ref).sum() / (ref * ref).sum().clamp_min(1e-300))
        delta[name] = tol * scale
    print(f"module W={W} (hidden_dim={hidden}, concat={concat}) N={g.num_nodes()}: |dloss|={abs(loss - loss_ref):.1e}; beta: "
          + ", ".join(f"{k}={v:+.1e}" for k, v in shrink.items() if k.startswith("ggnn.")))
    assert abs(loss - loss_ref) < 1e-4
    biased = {k: v for k, v in shrink.items() if k.startswith("ggnn.") and abs(v) >= BETA_TOL}
    assert not biased, biased
    if W == 256:
        # Adam's first step is lr * g' / (|g'| + eps), g' = g + wd p: a gradient error delta moves it by at most
        # lr * 2 delta / |g'| where |g'| > 2 delta, and by at most 2 lr anywhere; plus the fp32 roundings of the update and of p
        m2 = D.FlowGNNGGNNModule(FEAT, 1002, hidden, 8, 3, concat_all_absdf=concat, positive_weight=4.0)
        m2.load_state_dict(state)
        m2.to(DEV)
        tr = D.FusedTrainer(m2)
        lr, wd = 1e-3, 1e-2
        assert tr.lr == lr and tr.weight_decay == wd
        loss_tr = float(tr.step(gd))
        p0 = {k: q.detach().clone() for k, q in o.named_parameters()}
        opt = torch.optim.Adam(o.parameters(), lr=lr, weight_decay=wd)
        opt.step()
        for (name, p), (_, q) in zip(m2.named_parameters(), o.named_parameters()):
            gp = (q.grad + wd * p0[name]).abs()
            dl = delta[name]
            allowed = lr * torch.where(gp > 2 * dl, 2 * dl / gp.clamp_min(1e-300), torch.full_like(gp, 2.0)) + 2 * U * p0[name].abs() + 8 * U * lr
            worst[f"adam {name}"] = _ratio((p.detach().double() - q.detach()).abs(), allowed)
        assert abs(loss_tr - loss_ref) < 1e-4
    _report(f"module gradients W={W}", worst)
    _assert_within(worst)
