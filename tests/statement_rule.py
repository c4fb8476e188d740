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
