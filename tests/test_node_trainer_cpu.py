"""CPU: FusedTrainer's label_style="node" constructor contract and the undersampling count rule (no GPU needed)."""
import pytest
import torch

import deepdfa_b200 as D
from deepdfa_b200 import engine as E

FEAT = "_ABS_DATAFLOW_api_all_limitall_1000_limitsubkeys_1000"


def node_module(**kw):
    return D.FlowGNNGGNNModule(FEAT, 1002, 8, 2, 2, label_style="node", concat_all_absdf=True, engine="simt", **kw)


@pytest.mark.parametrize("product,want", [(0.5, 0), (1.5, 2), (2.5, 2), (3.5, 4), (4.5, 4), (0.49999999999999994, 0), (7.0, 7)])
def test_undersample_count_rounds_half_to_even_like_python_round(product, want):
    assert E.undersample_count(1, product) == want == round(product)


@pytest.mark.parametrize("n_vuln,factor", [(3, 0.5), (5, 0.5), (7, 0.5), (10, 0.25), (6, 0.75), (153, 1.0 / 3.0), (1000, 0.1)])
def test_undersample_count_is_round_of_the_fp64_product(n_vuln, factor):
    assert E.undersample_count(n_vuln, factor) == round(n_vuln * factor)


def test_constructor_needs_a_cuda_module_before_anything_else():
    with pytest.raises(D.DdfaError, match="CUDA"):
        D.FusedTrainer(node_module())


def _accepts(m, **kw):
    """The constructor's style checks run before anything touches a device: fake the device so they can be reached on CPU.
    Returns True once construction got past them (the first device allocation then fails without a GPU)."""
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
def test_node_style_passes_the_style_checks():
    assert _accepts(node_module())
    assert _accepts(node_module(undersample_node_on_loss_factor=1.0), node_sample_seed=2 ** 64 - 1)


@pytest.mark.skipif(torch.cuda.is_available(), reason="the CPU form of this check fakes the device")
def test_refusals():
    with pytest.raises(NotImplementedError, match="encoder_mode"):
        _accepts(D.FlowGNNGGNNModule(FEAT, 1002, 8, 2, 2, label_style="node", concat_all_absdf=True, encoder_mode=True))
    with pytest.raises(ValueError, match="node_sample_seed"):
        _accepts(node_module(), node_sample_seed=-1)
    with pytest.raises(ValueError, match="node_sample_seed"):
        _accepts(node_module(), node_sample_seed=2 ** 64)


@pytest.mark.skipif(torch.cuda.is_available(), reason="the CPU form of this check fakes the device")
def test_node_style_refuses_more_than_one_rank(monkeypatch):
    import deepdfa_b200.trainer as T
    monkeypatch.setattr(T.dist, "is_initialized", lambda: True)
    monkeypatch.setattr(T.dist, "get_world_size", lambda group=None: 2)
    monkeypatch.setattr(T.dist, "get_backend", lambda group=None: "gloo")
    with pytest.raises(NotImplementedError, match="one rank"):
        _accepts(node_module())
    assert _accepts(node_module(), distributed=False)


def test_flat_parameter_list_leaves_the_node_gate_buffers_out():
    from deepdfa_b200.trainer import flat_param_list
    m = node_module()
    flat = flat_param_list(m)
    assert len(flat) == len(list(m.parameters()))
    assert {id(p) for p in flat} == {id(p) for p in m.parameters()}
    g = D.FlowGNNGGNNModule(FEAT, 1002, 8, 2, 2, concat_all_absdf=True, engine="simt")
    assert flat_param_list(g) == g.param_list()
