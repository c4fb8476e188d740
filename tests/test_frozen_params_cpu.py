"""CPU: frozen parameters in FusedTrainer — the trainable ranges of the flat buffers, the exchange rule, the optimizer state in
torch.optim.Adam's format, the constructor's refusals and the C ABI's NULL rules of the pruned backward (nothing is launched)."""
import copy

import pytest
import torch

import deepdfa_b200 as D
from deepdfa_b200 import _lib, build
from deepdfa_b200.trainer import FusedAdam, _ALIGN, exchange_for_frozen, flat_offsets, flat_param_list, trainable_ranges

FEAT = "_ABS_DATAFLOW_api_all_limitall_1000_limitsubkeys_1000"


def module(style="graph", L=2, seed=0):
    torch.manual_seed(seed)
    return D.FlowGNNGGNNModule(FEAT, 40, 4, 2, L, label_style=style, concat_all_absdf=True, engine="simt")


def freeze_encoder(m):
    """main_cli.py:136-144's split: everything but output_layer.* and pooling.* is frozen."""
    for name, p in m.named_parameters():
        if not name.startswith(("output_layer.", "pooling.")):
            p.requires_grad_(False)
    return m


# ---- trainable ranges ----------------------------------------------------------------------------------------------------------
def test_all_trainable_is_one_range_over_the_buffer():
    m = module()
    _, total = flat_offsets(flat_param_list(m))
    assert trainable_ranges(flat_param_list(m)) == [(0, total)]


@pytest.mark.parametrize("style", ["graph", "node"])
def test_frozen_encoder_leaves_the_head_as_one_tail_range(style):
    m = freeze_encoder(module(style))
    flat = flat_param_list(m)
    offs, total = flat_offsets(flat)
    k = len(m._tables()) + 6                   # tables + the six GatedGraphConv tensors
    assert trainable_ranges(flat) == [(offs[k], total)]


def test_ranges_merge_adjacent_slots_and_keep_gaps():
    m = module(L=3)
    flat = flat_param_list(m)
    offs, total = flat_offsets(flat)
    ends = offs[1:] + [total]
    k = len(m._tables())
    flat[k + 3].requires_grad_(False)                        # gru.weight_hh
    flat[-1].requires_grad_(False)                           # the last MLP bias
    r = trainable_ranges(flat)
    assert r == [(0, offs[k + 3]), (ends[k + 3], offs[-1])]
    assert all(a % _ALIGN == 0 and b % _ALIGN == 0 for a, b in r)


def test_nothing_trainable_is_refused():
    m = module()
    for p in m.parameters():
        p.requires_grad_(False)
    with pytest.raises(ValueError, match="nothing to train"):
        trainable_ranges(flat_param_list(m))


# ---- exchange ----------------------------------------------------------------------------------------------------------------
def test_exchange_rule():
    assert exchange_for_frozen("p2p", 2, False) == ("p2p", None)
    assert exchange_for_frozen("auto", 8, False) == ("auto", None)
    assert exchange_for_frozen("p2p", 1, True) == ("p2p", None)          # one rank: no exchange at all
    assert exchange_for_frozen("nccl", 4, True) == ("nccl", None)
    ex, note = exchange_for_frozen("auto", 2, True)
    assert ex == "nccl" and "frozen" in note
    with pytest.raises(NotImplementedError, match="p2p"):
        exchange_for_frozen("p2p", 2, True)


# ---- the constructor's refusals (the device is faked: they come before any device work) --------------------------------------
def _construct(m, **kw):
    orig = type(m).device
    try:
        type(m).device = property(lambda self: torch.device("cuda", 0))
        try:
            D.FusedTrainer(m, **kw)
        except (NotImplementedError, ValueError):
            raise
        except Exception:
            pass
        return True
    finally:
        type(m).device = orig


@pytest.mark.skipif(torch.cuda.is_available(), reason="the CPU form of this check fakes the device")
def test_constructor_refusals(monkeypatch):
    m = module()
    for p in m.parameters():
        p.requires_grad_(False)
    with pytest.raises(ValueError, match="nothing to train"):
        _construct(m)
    import deepdfa_b200.trainer as T
    monkeypatch.setattr(T.dist, "is_initialized", lambda: True)
    monkeypatch.setattr(T.dist, "get_world_size", lambda group=None: 2)
    monkeypatch.setattr(T.dist, "get_backend", lambda group=None: "nccl")
    with pytest.raises(NotImplementedError, match="p2p"):
        _construct(freeze_encoder(module()), exchange="p2p")
    assert _construct(freeze_encoder(module()), exchange="nccl")


# ---- optimizer state -----------------------------------------------------------------------------------------------------------
def fused_for(m):
    _, total = flat_offsets(m.param_list())
    return FusedAdam(m, torch.zeros(total), torch.zeros(total), torch.zeros(1, dtype=torch.int32), torch.zeros(5),
                     lr=1e-3, weight_decay=1e-2)


def torch_adam_after(m, steps=3):
    opt = torch.optim.Adam(m.parameters(), lr=1e-3, weight_decay=1e-2)
    gen = torch.Generator().manual_seed(1)
    for _ in range(steps):
        for p in m.parameters():
            p.grad = torch.randn(p.shape, generator=gen) if p.requires_grad else None
        opt.step()
    return opt


def test_state_dict_has_torch_keys_without_frozen_entries():
    m = freeze_encoder(module())
    sd = torch_adam_after(m).state_dict()
    frozen = {i for i, p in enumerate(m.parameters()) if not p.requires_grad}
    assert frozen and not frozen & set(sd["state"])
    fa = fused_for(m)
    fa.load_state_dict(copy.deepcopy(sd))
    back = fa.state_dict()
    assert back["param_groups"] == sd["param_groups"]
    assert sorted(back["state"]) == sorted(sd["state"])
    for i, s in sd["state"].items():
        assert float(back["state"][i]["step"]) == float(s["step"]) == 3.0
        for k in ("exp_avg", "exp_avg_sq"):
            assert torch.equal(back["state"][i][k], s[k])


def test_load_ignores_entries_of_frozen_parameters():
    """A checkpoint of an all-trainable run (other step counts on the encoder) loads into a frozen-encoder optimizer: the
    frozen entries are ignored, the step count is the head's."""
    full = module()
    opt = torch_adam_after(full, steps=5)
    sd = copy.deepcopy(opt.state_dict())
    m = freeze_encoder(module())
    frozen = [i for i, p in enumerate(m.parameters()) if not p.requires_grad]
    for i in frozen:
        sd["state"][i]["step"] = torch.tensor(2.0)          # would be "per-parameter steps differ" if they counted
        sd["state"][i]["exp_avg"] = torch.zeros(7)           # ... or a shape mismatch
    fa = fused_for(m)
    fa.load_state_dict(sd)
    assert int(fa._flat[2]) == 5
    back = fa.state_dict()
    assert sorted(back["state"]) == [i for i, p in enumerate(m.parameters()) if p.requires_grad]
    exp_avg = fa._flat[0]
    offs, _ = flat_offsets(m.param_list())
    where = {id(p): o for p, o in zip(m.param_list(), offs)}
    for i, p in enumerate(m.parameters()):
        if not p.requires_grad:
            assert not exp_avg[where[id(p)]:where[id(p)] + p.numel()].any()


# ---- C ABI: the NULL rules of the pruned backward -----------------------------------------------------------------------------
@pytest.fixture(scope="module")
def L():
    build.build()
    return _lib.lib()


def test_readout_gate_only_needs_both_planes_null(L):
    F = 256                                                  # a fake device pointer: the checks reject before any launch
    args = lambda dh, dx: (F, F, F, F, F, 1, 32, F, F, F, F, dh, dx, F, F)
    with pytest.raises(_lib.DdfaError, match="dh_final and dx are both NULL"):
        L.call("ddfa_readout_bwd_ws", *args(F, None), F, 1 << 20, None)
    with pytest.raises(_lib.DdfaError, match="dh_final and dx are both NULL"):
        L.call("ddfa_readout_bwd_ws", *args(None, F), F, 1 << 20, None)
    with pytest.raises(_lib.DdfaError, match="gate-only form is ddfa_readout_bwd_ws"):
        L.call("ddfa_readout_bwd", *args(None, None), None)


def test_node_head_without_input_grads_needs_both_planes_null(L):
    F = 256
    w = _lib.ptr_array([F])
    for dh, dx in ((F, None), (None, F)):
        with pytest.raises(_lib.DdfaError, match="dh_final and dx are both NULL"):
            L.call("ddfa_node_head_bwd", F, F, F, F, F, 8, 32, w, 1, None, dh, dx, w, w, F, 1 << 20, None)


def test_adam_flat_ranges_argument_checks(L):
    F = 256
    with pytest.raises(_lib.DdfaError, match="ddfa_adam_flat_ranges: NULL pointer"):
        L.call("ddfa_adam_flat_ranges", F, F, F, F, F, 64, None, 1, F, None, None, None)
    with pytest.raises(_lib.DdfaError, match="ddfa_adam_flat_ranges: negative"):
        L.call("ddfa_adam_flat_ranges", F, F, F, F, F, 64, F, -1, F, None, None, None)
    with pytest.raises(_lib.DdfaError, match="skipped given without gstate"):
        L.call("ddfa_adam_flat_ranges", F, F, F, F, F, 64, F, 1, F, None, F, None)
