"""CPU: FusedTrainer.optimizer's conversion between torch.optim.Adam's state_dict format and the trainer's flat buffers.

FusedAdam keeps no state of its own: the moments live in flat buffers laid out in ``module.param_list()`` order, while
torch's format (and a reference Lightning checkpoint's ``optimizer_states[0]``) indexes parameters in
``module.parameters()`` order.  The buffers may be CPU tensors, so everything here runs without a GPU."""
import copy
import os
import warnings

import pytest
import torch

import deepdfa_b200 as D
from deepdfa_b200.trainer import FusedAdam, flat_offsets, owned_range

FEAT = "_ABS_DATAFLOW_api_all_limitall_1000_limitsubkeys_1000"
GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "reference_optimizer_golden.pt")


def cpu_module(L=2, concat=True, seed=0):
    torch.manual_seed(seed)
    return D.FlowGNNGGNNModule(FEAT, 40, 4 if concat else 12, 2, L, concat_all_absdf=concat)


def fused_for(module, **kw):
    _, total = flat_offsets(module.param_list())
    kw = dict(dict(lr=1e-3, weight_decay=1e-2), **kw)
    return FusedAdam(module, torch.zeros(total), torch.zeros(total), torch.zeros(1, dtype=torch.int32), torch.zeros(5), **kw)


def torch_adam_after(module, steps=3, seed=1):
    opt = torch.optim.Adam(module.parameters(), lr=1e-3, weight_decay=1e-2)
    gen = torch.Generator().manual_seed(seed)
    for i in range(steps):
        for p in module.parameters():
            p.grad = torch.randn(p.shape, generator=gen) * (0.1 if i % 2 else 3.0)
        opt.step()
    return opt


def assert_same_state(a, b):
    assert a["param_groups"] == b["param_groups"]
    assert sorted(a["state"]) == sorted(b["state"])
    for i, sa in a["state"].items():
        sb = b["state"][i]
        assert float(sa["step"]) == float(sb["step"]), i
        for k in ("exp_avg", "exp_avg_sq"):
            assert sa[k].dtype == sb[k].dtype and sa[k].shape == sb[k].shape, (i, k)
            assert torch.equal(sa[k], sb[k]), (i, k)      # bit-equal: the conversion only moves values


@pytest.mark.parametrize("L,concat", [(1, True), (2, True), (3, True), (3, False)])
def test_torch_adam_state_round_trips_through_the_flat_buffers(L, concat):
    m = cpu_module(L, concat)
    if L >= 2:     # the two orders really differ: param_list() puts every MLP weight before every MLP bias
        assert [id(p) for p in m.parameters()] != [id(p) for p in m.param_list()]
    opt = torch_adam_after(m)
    sd = opt.state_dict()
    fa = fused_for(m)
    fa.load_state_dict(copy.deepcopy(sd))
    assert_same_state(fa.state_dict(), sd)
    exp_avg, exp_avg_sq, step_count, hyper = fa._flat
    assert int(step_count) == 3
    assert torch.equal(hyper, torch.tensor([1e-3, 0.9, 0.999, 1e-8, 1e-2], dtype=torch.float32))
    # the index mapping: every parameter's moments sit at ITS slot of the param_list() layout
    offs, _ = flat_offsets(m.param_list())
    for p, o in zip(m.param_list(), offs):
        n = p.numel()
        assert torch.equal(exp_avg[o:o + n], opt.state[p]["exp_avg"].reshape(-1))
        assert torch.equal(exp_avg_sq[o:o + n], opt.state[p]["exp_avg_sq"].reshape(-1))
    # padding between slots stays zero
    used = torch.zeros(exp_avg.numel(), dtype=torch.bool)
    for p, o in zip(m.param_list(), offs):
        used[o:o + p.numel()] = True
    assert not exp_avg[~used].any() and not exp_avg_sq[~used].any()


def test_fresh_optimizer_matches_fresh_torch_adam():
    m = cpu_module(3)
    ours = fused_for(m).state_dict()
    ref = torch.optim.Adam(m.parameters(), lr=1e-3, weight_decay=1e-2).state_dict()
    assert ours == ref and ours["state"] == {}


def test_legacy_checkpoint_forms_load():
    m = cpu_module(3)
    sd = torch_adam_after(m).state_dict()
    old = copy.deepcopy(sd)
    for st in old["state"].values():
        st["step"] = 3                                  # torch <= 1.12 kept the step as a Python int
    for k in ("foreach", "capturable", "differentiable", "fused", "decoupled_weight_decay"):
        old["param_groups"][0].pop(k)                   # keys older versions never wrote
    fa = fused_for(m)
    fa.load_state_dict(old)
    assert_same_state(fa.state_dict(), sd)
    # an empty state (saved before the first step) is step 0 and zero moments, whatever the buffers held
    empty = {"state": {}, "param_groups": copy.deepcopy(old["param_groups"])}
    fa.load_state_dict(empty)
    exp_avg, exp_avg_sq, step_count, _ = fa._flat
    assert int(step_count) == 0 and not exp_avg.any() and not exp_avg_sq.any()
    assert fa.state_dict()["state"] == {}


def _mutations():
    def two_groups(sd):
        sd["param_groups"].append(dict(sd["param_groups"][0], params=[]))

    def fewer_params(sd):
        sd["param_groups"][0]["params"].pop()
        sd["state"].pop(max(sd["state"]))

    def wrong_shape(sd):
        sd["state"][6]["exp_avg"] = sd["state"][6]["exp_avg"].t().contiguous()     # gru.weight_ih [3D, D]

    def flag(key):
        def f(sd):
            sd["param_groups"][0][key] = True
        return f

    def steps_differ(sd):
        sd["state"][2]["step"] = torch.tensor(2.0)

    def partial_state(sd):
        sd["state"].pop(0)                      # a parameter without state is at step 0, the others at step 3

    return {"two_groups": two_groups, "fewer_params": fewer_params, "wrong_shape": wrong_shape, "amsgrad": flag("amsgrad"),
            "maximize": flag("maximize"), "adamw": flag("decoupled_weight_decay"), "steps_differ": steps_differ,
            "partial_state": partial_state}


@pytest.mark.parametrize("case", sorted(_mutations()))
def test_unsupported_checkpoints_are_rejected_untouched(case):
    m = cpu_module(2)
    sd = torch_adam_after(m).state_dict()
    fa = fused_for(m)
    fa.load_state_dict(copy.deepcopy(sd))
    before = [t.clone() for t in fa._flat]
    bad = copy.deepcopy(sd)
    _mutations()[case](bad)
    with pytest.raises(ValueError):
        fa.load_state_dict(bad)
    assert all(torch.equal(a, b) for a, b in zip(before, fa._flat))       # nothing written
    assert fa.param_groups[0]["amsgrad"] is False


def test_hyperparameters_reach_the_device_word_and_schedulers_see_step():
    m = cpu_module(2)
    fa = fused_for(m)
    hyper = fa._flat[3]
    fa.param_groups[0]["lr"] = 0.25
    fa.param_groups[0]["betas"] = (0.5, 0.75)
    assert float(hyper[0]) == pytest.approx(1e-3)          # written by step(), not by the assignment
    fa.step()
    assert torch.equal(hyper, torch.tensor([0.25, 0.5, 0.75, 1e-8, 1e-2], dtype=torch.float32))
    fa.param_groups[0]["lr"] = 1e-3
    sched = torch.optim.lr_scheduler.StepLR(fa, step_size=2, gamma=0.5)
    seen = []
    with warnings.catch_warnings():
        warnings.simplefilter("error")                     # no "lr_scheduler.step() before optimizer.step()" warning
        for _ in range(5):
            fa.step()
            seen.append(float(hyper[0]))
            sched.step()
    assert seen == [pytest.approx(x) for x in (1e-3, 1e-3, 5e-4, 5e-4, 2.5e-4)]
    fa.add_param_group({"params": [torch.nn.Parameter(torch.zeros(2))]})
    with pytest.raises(ValueError):
        fa.step()


@pytest.mark.parametrize("world", [1, 2, 3, 4, 7, 8])
def test_owned_ranges_partition_the_flat_buffer(world):
    for numel in (64, 64 * 97, 375_936):
        ranges = [owned_range(numel, r, world) for r in range(world)]
        assert ranges[0][0] == 0 and ranges[-1][1] == numel
        for (a, b), (c, d) in zip(ranges, ranges[1:]):
            assert b == c and a <= b
        per = -(-(numel // 4) // world)
        assert all(hi - lo <= 4 * per and lo % 4 == 0 for lo, hi in ranges)


def test_reference_checkpoint_order_and_state_round_trip():
    """tests/golden/reference_optimizer_golden.pt (make_reference_optimizer_golden.py): the reference's own module under
    torch.optim.Adam.  Its parameter order is this module's, its optimizer state loads and comes back unchanged."""
    fx = torch.load(GOLDEN, weights_only=False)
    m = D.FlowGNNGGNNModule(**fx["ctor"])
    assert fx["names"] == [n for n, _ in m.named_parameters()]
    m.load_state_dict(fx["state_dict"])
    fa = fused_for(m)
    fa.load_state_dict(copy.deepcopy(fx["optimizer"]))
    assert_same_state(fa.state_dict(), fx["optimizer"])
    assert float(fx["optimizer"]["state"][0]["step"]) == len(fx["losses"])


def test_hyperparameter_entry_points_are_exported_and_validate_without_a_gpu():
    from deepdfa_b200 import _lib, build
    build.build()
    L = _lib.lib()
    assert {"ddfa_adam_flat_hp", "ddfa_allreduce_adam_p2p_hp"} <= set(_lib.declared_symbols())
    assert L.raw("ddfa_adam_flat_hp")(None, None, None, None, None, 0, None, None) == -1
    assert "ddfa_adam_flat_hp: NULL pointer" in L.last_error()
    assert L.raw("ddfa_allreduce_adam_p2p_hp")(None, None, None, 0, 1, None, None, None, 0, 0, None, None, None, None) == -1
    assert "NULL hyperparameter pointer" in L.last_error()
