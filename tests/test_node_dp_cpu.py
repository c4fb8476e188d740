"""CPU: label_style="node" over several ranks — the constructor's backend rule, and the premise of the sharded draw: the k smallest
(key, global node) pairs of the whole batch are the union of what each rank selects from its shard with the global threshold
and the ties of the ranks before it (restated in numpy with the Philox keys of head_batches.py, whose known answers
test_head_premises.py checks)."""
import numpy as np
import pytest
import torch

import head_batches as H
from head_batches import node_keys, sample_ref
from test_node_trainer_cpu import _accepts, node_module


@pytest.mark.skipif(torch.cuda.is_available(), reason="the CPU form of this check fakes the device")
def test_node_style_accepts_a_two_rank_nccl_group(monkeypatch):
    import deepdfa_b200.trainer as T
    monkeypatch.setattr(T.dist, "is_initialized", lambda: True)
    monkeypatch.setattr(T.dist, "get_world_size", lambda group=None: 2)
    monkeypatch.setattr(T.dist, "get_backend", lambda group=None: "nccl")
    assert _accepts(node_module())
    assert _accepts(node_module(undersample_node_on_loss_factor=1.0), node_sample_seed=3)


def sharded_draw(vuln, cuts, factor, seed, draw):
    """The phases of ddfa_node_dp_* in numpy: per-rank counts summed; k from the global counts; the global k-th smallest key by
    a 4 x 8-bit radix select over summed per-rank histograms; per-rank ties, each rank taking its ties after those of the ranks
    before it.  Returns the global ids of every rank's rows, concatenated in rank order, and the overflow flag."""
    R = len(cuts) - 1
    shards = [np.asarray(vuln[cuts[r]:cuts[r + 1]]) for r in range(R)]
    n_vuln = sum(int(np.count_nonzero(s)) for s in shards)
    pop = sum(int(np.count_nonzero(s == 0)) for s in shards)
    want = np.rint(float(n_vuln) * factor)
    over = not (want <= pop)
    k = pop if over else int(want)
    # this rank's keys: those of nodes cuts[r] + n of the global batch
    keys = [node_keys(cuts[r + 1], seed, draw)[cuts[r]:][s == 0] for r, s in enumerate(shards)]
    prefix, k_rem = 0, k
    if k > 0:
        for p in range(4):
            shift = 24 - 8 * p
            hist = np.zeros(256, np.int64)
            for kk in keys:
                cand = kk if p == 0 else kk[(kk >> np.uint64(shift + 8)) == (np.uint64(prefix) >> np.uint64(shift + 8))]
                hist += np.bincount(((cand >> np.uint64(shift)) & np.uint64(255)).astype(np.int64), minlength=256)
            cum = np.cumsum(hist)
            b = int(np.searchsorted(cum, k_rem))
            k_rem -= int(cum[b - 1]) if b else 0
            prefix |= b << shift
    out, tie_before = [], 0
    for r, s in enumerate(shards):
        nodes = np.nonzero(s == 0)[0]
        kk = keys[r]
        sure = nodes[kk < prefix] if k > 0 else nodes[:0]
        ties = nodes[kk == prefix] if k > 0 else nodes[:0]
        take = ties[:max(0, min(len(ties), k_rem - tie_before))]
        tie_before += len(ties)
        rows = np.sort(np.concatenate([np.nonzero(s != 0)[0], sure, take]))
        out.append(rows + cuts[r])
    return np.concatenate(out), over


@pytest.mark.parametrize("trial", range(12))
def test_sharded_selection_is_the_global_k_smallest(trial):
    rng = np.random.default_rng(1000 + trial)
    N = int(rng.integers(1, 6000))
    vuln = (rng.random(N) < rng.choice([0.0, 0.02, 0.2, 0.6])).astype(np.int32)
    R = int(rng.integers(1, 6))
    cuts = np.sort(np.concatenate([[0, N], rng.integers(0, N + 1, R - 1)])).tolist()     # empty shards included
    factor = float(rng.choice([0.0, 0.5, 1.0, 3.0, 1e9]))
    seed, draw = int(rng.integers(0, 2 ** 63)), int(rng.integers(0, 2 ** 40))
    rows, over = sharded_draw(vuln, cuts, factor, seed, draw)
    ref_rows, _, ref_over, _ = sample_ref(vuln, N, factor, seed, draw)
    assert over == ref_over
    np.testing.assert_array_equal(rows, ref_rows)


def test_sharded_selection_splits_threshold_ties_in_global_node_order():
    """head_batches.tie_case: at C1 size two nodes a < b share the k-th smallest key; factor_a takes a alone, factor_ab both.
    Cut between them, and with a last on rank 0 and b first on rank 2, the sharded draw still takes them in global node order."""
    t = H.tie_case()
    a, b, vuln = t["a"], t["b"], t["vuln"]
    N = len(vuln)
    for factor in (t["factor_a"], t["factor_ab"]):
        ref_rows, *_ = sample_ref(vuln, N, factor, t["seed"], 0)
        for cuts in ([0, (a + b) // 2 + 1, N], [0, a + 1, b, N], [0, a, b + 1, N]):
            rows, _ = sharded_draw(vuln, cuts, factor, t["seed"], 0)
            np.testing.assert_array_equal(rows, ref_rows)
