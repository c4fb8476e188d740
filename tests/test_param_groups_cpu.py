"""CPU: parameter groups and AdamW in FusedTrainer's optimizer — group resolution and its errors, the [begin, end, group]
range table, the group table rows, the optimizer state in torch.optim.AdamW's format on CPU buffers, loading torch Adam / AdamW
checkpoints with several groups, per-group LambdaLR reaching the table, and the new C ABI symbols."""
import copy
import ctypes
import re

import pytest
import torch

import deepdfa_b200 as D
from deepdfa_b200 import _lib, build
from deepdfa_b200.trainer import (FusedAdam, _ALIGN, flat_offsets, flat_param_list, group_ranges, group_row,
                                  resolve_param_groups)

FEAT = "_ABS_DATAFLOW_api_all_limitall_1000_limitsubkeys_1000"


def module(style="graph", L=2, seed=0):
    torch.manual_seed(seed)
    return D.FlowGNNGGNNModule(FEAT, 40, 4, 2, L, label_style=style, concat_all_absdf=True, engine="simt")


def decay_split(m, wd=0.1):
    """linevul_main.py's grouping: biases without weight decay."""
    return [{"params": [p for n, p in m.named_parameters() if "bias" not in n], "weight_decay": wd},
            {"params": [p for n, p in m.named_parameters() if "bias" in n], "weight_decay": 0.0}]


def fused_for(m, groups=None, decoupled=True, **kw):
    _, total = flat_offsets(flat_param_list(m))
    G = len(groups) if groups is not None else 1
    return FusedAdam(m, torch.zeros(total), torch.zeros(total), torch.zeros(1, dtype=torch.int32), torch.zeros(G, _lib.ADAM_GROUP_WORDS),
                     lr=1e-3, weight_decay=1e-2, param_groups=groups, decoupled_weight_decay=decoupled, **kw)


def torch_after(opt, params, steps=3, seed=1):
    gen = torch.Generator().manual_seed(seed)
    for _ in range(steps):
        for p in params:
            p.grad = torch.randn(p.shape, generator=gen) if p.requires_grad else None
        opt.step()
    return opt


# ---- group resolution --------------------------------------------------------------------------------------------------------
def test_resolution_keeps_torch_groups():
    m = module()
    groups = resolve_param_groups(m, decay_split(m))
    assert [len(g["params"]) for g in groups] == [len(g["params"]) for g in decay_split(m)]
    assert groups[0]["weight_decay"] == 0.1 and groups[1]["weight_decay"] == 0.0
    single = resolve_param_groups(m, [{"params": m.ggnn.gru.weight_ih}, {"params": [p for n, p in m.named_parameters()
                                                                                    if n != "ggnn.gru.weight_ih"]}])
    assert single[0]["params"] == [m.ggnn.gru.weight_ih]          # a bare tensor, as torch allows


def _errors(m):
    ps = list(m.named_parameters())
    rest = [p for n, p in ps[1:]]
    return {
        "missing": ([{"params": rest}], re.escape(ps[0][0])),
        "duplicated": ([{"params": [p for _, p in ps]}, {"params": [ps[2][1]]}], re.escape(ps[2][0])),
        "unknown_key": ([{"params": [p for _, p in ps], "momentum": 0.9}], "momentum"),
        "amsgrad": ([{"params": [p for _, p in ps], "amsgrad": True}], "amsgrad"),
        "maximize": ([{"params": [p for _, p in ps], "maximize": True}], "maximize"),
        "too_many": ([{"params": [p]} for _, p in ps] + [{"params": []}] * 64, "at most 64"),
        "foreign_tensor": ([{"params": [p for _, p in ps] + [torch.nn.Parameter(torch.zeros(3))]}], "not a parameter"),
        "empty": ([], "non-empty"),
        "no_params_key": ([{"lr": 1e-3}], "'params'"),
    }


@pytest.mark.parametrize("case", sorted(_errors(module())))
def test_resolution_errors(case):
    m = module()
    groups, match = _errors(m)[case]
    with pytest.raises(ValueError, match=match):
        resolve_param_groups(m, groups)


def test_frozen_parameters_may_be_left_out_or_listed():
    m = module()
    for n, p in m.named_parameters():
        if "embedding" in n:
            p.requires_grad_(False)
    trainable = [p for p in m.parameters() if p.requires_grad]
    assert len(resolve_param_groups(m, [{"params": trainable}])[0]["params"]) == len(trainable)
    assert len(resolve_param_groups(m, [{"params": list(m.parameters())}])[0]["params"]) == len(list(m.parameters()))


@pytest.mark.skipif(torch.cuda.is_available(), reason="the CPU form of this check fakes the device")
def test_trainer_refuses_bad_groups_before_any_device_work():
    m = module()
    orig = type(m).device
    try:
        type(m).device = property(lambda self: torch.device("cuda", 0))
        with pytest.raises(ValueError, match=re.escape(next(iter(m.named_parameters()))[0])):
            D.FusedTrainer(m, param_groups=[{"params": list(m.parameters())[1:]}])
    finally:
        type(m).device = orig


# ---- range and group tables ----------------------------------------------------------------------------------------------------
def test_adjacent_slots_of_one_group_merge_and_groups_split():
    m = module(L=3)
    flat = flat_param_list(m)
    offs, total = flat_offsets(flat)
    assert group_ranges(flat, {id(p): 0 for p in flat}) == [(0, total, 0)]
    ends = offs[1:] + [total]
    gof = {id(p): (1 if i % 3 == 2 else 0) for i, p in enumerate(flat)}
    r = group_ranges(flat, gof)
    for a, b, g in r:
        assert a % _ALIGN == 0 and b % _ALIGN == 0
    for (a, b, g), (c, d, h) in zip(r, r[1:]):
        assert b <= c and (b < c or g != h)                 # adjacent ranges of one group are merged
    covered = [(offs[i], ends[i], gof[id(p)]) for i, p in enumerate(flat)]
    for lo, hi, g in covered:
        assert any(a <= lo and hi <= b and g == h for a, b, h in r)


def test_frozen_slots_are_excluded():
    m = module(L=3)
    flat = flat_param_list(m)
    offs, total = flat_offsets(flat)
    ends = offs[1:] + [total]
    k = len(m._tables())
    flat[k + 3].requires_grad_(False)                        # gru.weight_hh, listed in the group all the same
    r = group_ranges(flat, {id(p): 0 for p in flat})
    assert r == [(0, offs[k + 3], 0), (ends[k + 3], total, 0)]
    r = group_ranges(flat, {id(p): 0 for p in flat if p is not flat[-1]})     # a tensor in no group: left out as well
    assert r[-1][1] == offs[-1]


def test_group_row_rounds_the_decay_once_from_double():
    lr, wd = 3e-4, 0.1
    r = group_row(dict(lr=lr, betas=(0.9, 0.98), eps=1e-6, weight_decay=wd, decoupled_weight_decay=True))
    t = torch.tensor(r, dtype=torch.float32)
    assert float(t[6]) == float(torch.tensor(1.0 - lr * wd, dtype=torch.float32))
    assert r[5] == 1.0 and r[:5] == (lr, 0.9, 0.98, 1e-6, wd)
    assert group_row(dict(lr=lr, betas=(0.9, 0.98), eps=1e-6, weight_decay=wd))[5:7] == (0.0, 1.0)


# ---- state in torch's format ---------------------------------------------------------------------------------------------------
def test_fresh_state_dict_is_torch_adamw_groups():
    m = module()
    ours = fused_for(m, decay_split(m)).state_dict()
    ref = torch.optim.AdamW(decay_split(m), lr=1e-3, weight_decay=1e-2).state_dict()
    assert ours == ref and ours["state"] == {}
    mixed = decay_split(m)
    mixed[1]["decoupled_weight_decay"] = False                # a coupled group among AdamW groups
    assert fused_for(m, mixed).state_dict()["param_groups"][1]["decoupled_weight_decay"] is False


@pytest.mark.parametrize("kind", ["adamw", "adam"])
def test_multi_group_checkpoints_round_trip(kind):
    m = module()
    ref = (torch.optim.AdamW if kind == "adamw" else torch.optim.Adam)(decay_split(m), lr=1e-3, weight_decay=1e-2)
    sd = torch_after(ref, list(m.parameters())).state_dict()
    fa = fused_for(m, decay_split(m), decoupled=True)
    fa.load_state_dict(copy.deepcopy(sd))
    back = fa.state_dict()
    assert back["param_groups"] == sd["param_groups"]
    assert sorted(back["state"]) == sorted(sd["state"])
    for i, s in sd["state"].items():
        assert float(back["state"][i]["step"]) == 3.0
        for key in ("exp_avg", "exp_avg_sq"):
            assert torch.equal(back["state"][i][key], s[key])
    table = fa._flat[3]
    assert [float(x) for x in table[:, 5]] == ([1.0, 1.0] if kind == "adamw" else [0.0, 0.0])
    # indices are in group order: the first index of group 1 follows the last of group 0
    assert sd["param_groups"][1]["params"][0] == len(sd["param_groups"][0]["params"])


def _bad(sd):
    return {"more_groups": lambda s: s["param_groups"].append(dict(s["param_groups"][0], params=[])),
            "fewer_groups": lambda s: s["param_groups"].pop(),
            "group_size": lambda s: (s["param_groups"][0]["params"].pop(), s["param_groups"][1]["params"].append(10 ** 6)),
            "amsgrad": lambda s: s["param_groups"][1].__setitem__("amsgrad", True)}


@pytest.mark.parametrize("case", sorted(_bad(None)))
def test_mismatched_checkpoints_raise_untouched(case):
    m = module()
    sd = torch_after(torch.optim.AdamW(decay_split(m)), list(m.parameters())).state_dict()
    fa = fused_for(m, decay_split(m))
    fa.load_state_dict(copy.deepcopy(sd))
    before = [t.clone() for t in fa._flat]
    bad = copy.deepcopy(sd)
    _bad(sd)[case](bad)
    with pytest.raises(ValueError):
        fa.load_state_dict(bad)
    assert all(torch.equal(a, b) for a, b in zip(before, fa._flat))


def test_single_word_form_refuses_adamw_and_groups():
    m = module()
    _, total = flat_offsets(flat_param_list(m))
    with pytest.raises(ValueError, match="group table"):
        FusedAdam(m, torch.zeros(total), torch.zeros(total), torch.zeros(1, dtype=torch.int32), torch.zeros(5), decoupled_weight_decay=True)


def test_add_param_group_after_construction_raises():
    m = module()
    fa = fused_for(m, decay_split(m))
    with pytest.raises(ValueError, match="add_param_group"):
        fa.add_param_group({"params": [torch.nn.Parameter(torch.zeros(2))]})


# ---- schedulers ------------------------------------------------------------------------------------------------------------
def test_lambdalr_per_group_changes_the_pushed_table():
    m = module()
    groups = decay_split(m)
    groups[0]["lr"], groups[1]["lr"] = 2e-3, 1e-3
    fa = fused_for(m, groups)
    table = fa._flat[3]
    warm = 2
    sched = torch.optim.lr_scheduler.LambdaLR(fa, [lambda s: min(1.0, (s + 1) / warm), lambda s: 0.5 ** s])
    seen = []
    for _ in range(4):
        fa.step()
        seen.append((float(table[0, 0]), float(table[1, 0]), float(table[0, 6]), float(table[1, 6])))
        sched.step()
    f32 = lambda x: float(torch.tensor(x, dtype=torch.float32))
    for s, (a, b, da, db) in enumerate(seen):
        lr0 = 2e-3 * min(1.0, (s + 1) / warm)
        assert a == f32(lr0) and b == f32(1e-3 * 0.5 ** s)
        assert da == f32(1.0 - lr0 * 0.1) and db == 1.0              # no-decay group: wd = 0, decay 1
    assert seen[0][0] != seen[1][0]


# ---- C ABI -----------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def L():
    build.build()
    return _lib.lib()


NEW = {"ddfa_adam_flat_groups": 13, "ddfa_allreduce_adam_p2p_groups": 17, "ddfa_allreduce_adam_p2p_groups_guarded": 20}


def test_new_symbols_are_exported_with_their_declared_arity(L):
    text = re.sub(r"/\*.*?\*/", "", _lib.HEADER.read_text(), flags=re.S)
    dll = ctypes.CDLL(str(L.path))
    for name, n in NEW.items():
        assert hasattr(dll, name) and name in _lib.declared_symbols()
        args = re.search(r"\b" + name + r"\s*\(([^;]*?)\)\s*;", text, flags=re.S).group(1)
        assert len([a for a in args.split(",") if a.strip()]) == n == len(_lib._SIGNATURES[name][1])
    assert re.search(r"#define DDFA_ADAM_GROUP_WORDS %d\b" % _lib.ADAM_GROUP_WORDS, text)
    assert re.search(r"#define DDFA_ADAM_MAX_GROUPS %d\b" % _lib.ADAM_MAX_GROUPS, text)


def test_grouped_entry_points_check_their_arguments(L):
    F = 256                                                  # a fake device pointer: the checks reject before any launch
    with pytest.raises(_lib.DdfaError, match="num_groups"):
        L.call("ddfa_adam_flat_groups", F, F, F, F, F, 64, F, 1, F, 65, None, None, None)
    with pytest.raises(_lib.DdfaError, match="num_groups"):
        L.call("ddfa_adam_flat_groups", F, F, F, F, F, 64, F, 1, F, 0, None, None, None)
    with pytest.raises(_lib.DdfaError, match="NULL pointer"):
        L.call("ddfa_adam_flat_groups", F, F, F, F, F, 64, F, 1, None, 1, None, None, None)
    with pytest.raises(_lib.DdfaError, match="skipped given without gstate"):
        L.call("ddfa_adam_flat_groups", F, F, F, F, F, 64, F, 1, F, 1, None, F, None)
    w = _lib.ptr_array([F])
    with pytest.raises(_lib.DdfaError, match="num_groups"):
        L.call("ddfa_allreduce_adam_p2p_groups", w, w, w, 0, 1, F, F, F, 64, 64, None, F, F, 1, F, 99, None)
    with pytest.raises(_lib.DdfaError, match="NULL pointer"):
        L.call("ddfa_allreduce_adam_p2p_groups_guarded", w, w, w, 0, 1, F, F, F, 64, 64, None, F, 1, None, 1, None, F, None, F, None)
