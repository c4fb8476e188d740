"""CPU: gradient accumulation's host logic — the argument check, the micro-batch phases and graph keys — and the argument checks
of its entry point (no GPU needed: nothing is launched)."""
import pytest

import deepdfa_b200 as D
from deepdfa_b200 import _lib, build
from deepdfa_b200.trainer import FusedTrainer

FEAT = "_ABS_DATAFLOW_api_all_limitall_1000_limitsubkeys_1000"


@pytest.fixture(scope="module")
def L():
    build.build()
    return _lib.lib()


def cpu_module():
    return D.FlowGNNGGNNModule(FEAT, 1002, 32, 2, 2, concat_all_absdf=True, engine="simt")


@pytest.mark.parametrize("k", [0, -1, 2.0, 1.5, "2", True, None])
def test_accumulate_grad_batches_must_be_a_positive_integer(k):
    with pytest.raises(ValueError, match="accumulate_grad_batches"):
        FusedTrainer(cpu_module(), accumulate_grad_batches=k)


def test_a_valid_k_gets_as_far_as_the_device_check():
    with pytest.raises(_lib.DdfaError, match="CUDA device"):
        FusedTrainer(cpu_module(), accumulate_grad_batches=4)


def bare_trainer(k):
    """The phase logic alone: a FusedTrainer shell with no buffers (building one needs a GPU)."""
    tr = object.__new__(FusedTrainer)
    tr._k, tr._accumulated = k, 0
    return tr


@pytest.mark.parametrize("k,want", [(1, ["apply"] * 4),
                                    (2, ["first", "apply"] * 3),
                                    (3, ["first", "add", "apply"] * 2),
                                    (4, ["first", "add", "add", "apply"] * 2)])
def test_micro_batch_phases(k, want):
    tr = bare_trainer(k)
    got = []
    for _ in want:
        phase = tr._phase()
        got.append(phase)
        tr._accumulated = 0 if phase == "apply" else tr._accumulated + 1     # what _end does
        assert tr.accumulated == tr._accumulated < k
    assert got == want


def test_graph_keys_gain_the_phase_only_with_accumulation():
    assert bare_trainer(1)._phase_key("apply") == ()
    assert bare_trainer(3)._phase_key("add") == ("add",)


def test_grad_accumulate_argument_checks(L):
    assert (_lib.GRAD_ACC_SET, _lib.GRAD_ACC_ADD, _lib.GRAD_ACC_APPLY) == (0, 1, 2)
    with pytest.raises(_lib.DdfaError, match="mode=3"):
        L.call("ddfa_grad_accumulate", 256, 256, 0, 4, 3, None)
    for begin, end in ((2, 8), (0, 6), (8, 4), (-4, 4)):
        with pytest.raises(_lib.DdfaError, match="multiples of 4"):
            L.call("ddfa_grad_accumulate", 256, 256, begin, end, _lib.GRAD_ACC_ADD, None)
    with pytest.raises(_lib.DdfaError, match="NULL pointer"):
        L.call("ddfa_grad_accumulate", None, 256, 0, 4, _lib.GRAD_ACC_SET, None)
    with pytest.raises(_lib.DdfaError, match="16-byte alignment"):
        L.call("ddfa_grad_accumulate", 256 + 4, 256, 0, 4, _lib.GRAD_ACC_APPLY, None)
    assert L.call("ddfa_grad_accumulate", None, None, 8, 8, _lib.GRAD_ACC_ADD, None) == 0     # an empty range launches nothing


def test_node_bce_scaled_argument_checks(L):
    with pytest.raises(_lib.DdfaError, match="ddfa_node_bce_scaled: num_nodes=-1"):
        L.call("ddfa_node_bce_scaled", None, None, None, None, -1, 1.0, 0.5, None, None, None)
    with pytest.raises(_lib.DdfaError, match="ddfa_node_bce_scaled: NULL pointer"):
        L.call("ddfa_node_bce_scaled", None, None, None, None, 4, 1.0, 0.5, None, None, None)
