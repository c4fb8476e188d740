"""Host restatements for the statement-level localisation tests (not a test module).

``host_state`` restates ddfa_stmt_metric (csrc/statements.cu) with numpy: per function the first-ranked vulnerable statement
(maximum score, lowest node id among equal scores) and the number of statements ranked ahead of it, summed into the
DDFA_STMT_STATE_WORDS layout.  ``rank_by_sort`` is the same number computed the reference's way, with Python's stable sort.
The ``oracle_*`` functions restate the per-node scores on the fp64 oracle with torch.autograd.
"""
import numpy as np
import torch

WORDS = 16
FUNCTIONS, VULN, HIT1, RANK_SUM, CLEAN, NAN, BATCHES = 0, 1, 2, 12, 13, 14, 15


def ranks(scores, vuln, bnn):
    """Per function: (vulnerable, rank or None, has a score > 0.5, has a NaN score)."""
    scores = np.asarray(scores, dtype=np.float32)
    vuln = np.asarray(vuln)
    out = []
    n0 = 0
    for n in np.asarray(bnn).tolist():
        s, v = scores[n0:n0 + n], vuln[n0:n0 + n]
        ids = np.arange(n)
        nan = bool(np.isnan(s).any())
        vul = bool((v != 0).any())
        rank = None
        if vul and not nan:
            vs = s[v != 0]
            best = vs.max()
            bid = ids[(v != 0) & (s == best)].min()
            rank = int(((s > best) | ((s == best) & (ids < bid))).sum())
        out.append((vul, rank, bool((s > np.float32(0.5)).any()), nan))
        n0 += n
    return out


def rank_by_sort(scores, vuln):
    """evaluate.py's way: sorted(zip(probs, labels), key=prob, reverse=True), the position of the first label 1."""
    z = sorted(zip([float(s) for s in scores], [int(v) for v in vuln]), key=lambda t: t[0], reverse=True)
    return next(i for i, (_, y) in enumerate(z) if y != 0)


def host_state(scores, vuln, bnn, full: bool, batches: int = 1):
    st = np.zeros(WORDS, dtype=np.float64)
    for vul, rank, above, nan in ranks(scores, vuln, bnn):
        st[FUNCTIONS] += 1
        if nan:
            st[NAN] += 1
        elif vul:
            st[VULN] += 1
            st[RANK_SUM] += rank
            for k in range(1, 11):
                st[HIT1 + k - 1] += rank < k
        elif full and not above:
            st[CLEAN] += 1
    st[BATCHES] = batches
    return st


# ---- the per-node scores on the fp64 oracle --------------------------------------------------------------------------------
def oracle_logits_from_x(o, g, x):
    """The oracle's forward (ggnn.py:95-107) from a given embedding output x."""
    out = torch.cat([o.ggnn(g, x), x], -1)
    return o.output_layer(o.pooling(g, out)).reshape(-1)


def oracle_attention(o, g):
    with torch.no_grad():
        x = o.embed(g)
        out = torch.cat([o.ggnn(g, x), x], -1)
        _, alpha = o.pooling(g, out, get_attention=True)
    return alpha.reshape(-1)


def oracle_input_grad(o, g, x):
    """∂(Σ_b logit_b)/∂x at x: row n holds ∂logit_{b(n)}/∂x_n, functions being independent."""
    x = x.detach().clone().requires_grad_(True)
    oracle_logits_from_x(o, g, x).sum().backward()
    return x.grad.detach()


def oracle_saliency(o, g):
    with torch.no_grad():
        x = o.embed(g)
    return oracle_input_grad(o, g, x).abs().sum(1)


def oracle_integrated_gradients(o, g, m: int):
    """captum IntegratedGradients(method="riemann_middle"), zero baseline: x · (1/m) Σ_k grad at ((k + ½)/m)·x, summed over d."""
    with torch.no_grad():
        x = o.embed(g)
    acc = torch.zeros_like(x)
    for k in range(m):
        acc += oracle_input_grad(o, g, ((k + 0.5) / m) * x)
    return (x * acc / m).sum(1)


# ---- launch shapes of csrc/statements.cu (H100: kNumSMs = 132) -------------------------------------------------------------
STMT_THREADS = 128                 # stmt_metric_kernel / attention_kernel: one CTA of 4 warps per function
STMT_MAX_CTAS = 2 * 132            # kMaxCtas: above it the metric kernel strides over functions
SHAP_MAX_CTAS = 8 * 132            # ddfa_stmt_shap_input's grid: above it shap_input_kernel strides over functions
SCORE_WARP_ROWS = 8                # input_grad_score_kernel: a warp per node, 8 nodes per CTA
SCORE_WIDTHS = (4, 20, 80, 128, 192, 512)
SHAP_WIDTHS = (4, 20, 128, 512)
SHAP_COUNTER = (1 << 32) + 7       # a batch counter past 2^32: the kernel uses its low word
SHAP_SIZES_B = 3000


def shap_sizes(seed: int = 0) -> np.ndarray:
    """SHAP_SIZES_B functions of 0 to 19 nodes, every 7th empty (the last one too)."""
    s = np.random.default_rng(seed).integers(1, 20, SHAP_SIZES_B)
    s[::7] = 0
    s[-1] = 0
    return s.astype(np.int64)


def metric_case():
    """Scores, labels and sizes of the exact metric test: 600 functions (more than STMT_MAX_CTAS) of up to 20 000 nodes, with
    the ties and special values the ranking has to get right (see the comments)."""
    rng = np.random.default_rng(2024)
    fns = []

    def grid(n):          # scores on a 4-value grid: ties everywhere
        return (rng.integers(0, 4, n) / 4).astype(np.float32), np.zeros(n, np.int32)

    # 20 000 nodes: the top score 0.75 held by vulnerable nodes in different warps and loop iterations, non-vulnerable ones ahead
    s, v = grid(20_000)
    s = np.minimum(s, np.float32(0.5))
    for j in (19_999, 13_001, 5_070, 129, 97):
        s[j], v[j] = 0.75, 1
    s[[3, 40, 4_000]] = 0.75
    fns.append((s, v))
    # 1 000 nodes: the unique first-ranked vulnerable node in the last warp (lane offset 96..127 of the CTA), late iteration
    s, v = grid(1_000)
    s[:] = np.minimum(s, np.float32(0.25))
    v[rng.choice(1_000, 30, replace=False)] = 1
    s[3 * 128 + 100], v[3 * 128 + 100] = 0.9, 1
    s[[7, 500, 999]] = 0.95
    fns.append((s, v))
    # +0.0 tied with -0.0: a vulnerable -0.0 with +0.0 non-vulnerable nodes before and after it, and a lower vulnerable +0.0
    s = np.full(300, -1.0, np.float32)
    v = np.zeros(300, np.int32)
    s[[10, 150, 290]] = 0.0
    s[[200, 260]] = -0.0
    v[[200, 260]] = 1
    fns.append((s, v))
    s2, v2 = s.copy(), v.copy()
    v2[150] = 1            # +0.0 at a lower id than the -0.0 ones: it ranks first
    fns.append((s2, v2))
    # +inf ties, a vulnerable -inf below everything, a NaN on a non-vulnerable node (the function counts as NaN)
    s = rng.standard_normal(700).astype(np.float32)
    v = np.zeros(700, np.int32)
    s[[5, 333, 600]] = np.inf
    v[[333, 600]] = 1
    fns.append((s, v))
    s = rng.standard_normal(257).astype(np.float32)
    v = np.zeros(257, np.int32)
    s[256], v[256] = -np.inf, 1
    fns.append((s, v))
    s = rng.standard_normal(129).astype(np.float32)
    v = np.zeros(129, np.int32)
    v[100] = 1
    s[128] = np.nan
    fns.append((s, v))
    # small functions, half of them clean, up to num_graphs = 600
    while len(fns) < 600:
        n = int(rng.integers(1, 150))
        s, v = grid(n)
        if rng.random() < 0.5:
            v[rng.integers(0, n)] = 1
        fns.append((s, v))
    order = rng.permutation(len(fns) - 7) + 7       # the special functions first (in the first CTAs), the rest shuffled
    fns = fns[:7] + [fns[i] for i in order]
    return (np.concatenate([f[0] for f in fns]), np.concatenate([f[1] for f in fns]), np.array([len(f[0]) for f in fns]))
