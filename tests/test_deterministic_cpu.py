"""CPU: the deterministic-mode tuning key and how the Python layer picks the mode (no compute calls)."""
import pytest
import torch

from deepdfa_b200 import _lib, build


@pytest.fixture(scope="module")
def L():
    build.build()
    return _lib.lib()


def test_tuning_key_sets_reads_back_and_rejects_bad_values(L):
    assert L.call("ddfa_tuning_get", _lib.TUNE_DETERMINISTIC) == 0           # default mode
    try:
        L.call("ddfa_tuning_set", _lib.TUNE_DETERMINISTIC, 1)
        assert L.call("ddfa_tuning_get", _lib.TUNE_DETERMINISTIC) == 1
        for bad in (2, -1):
            assert L.raw("ddfa_tuning_set")(_lib.TUNE_DETERMINISTIC, bad) == -1
            assert "DDFA_TUNE_DETERMINISTIC" in L.last_error()
            assert L.call("ddfa_tuning_get", _lib.TUNE_DETERMINISTIC) == 1
    finally:
        L.call("ddfa_tuning_set", _lib.TUNE_DETERMINISTIC, 0)
    assert L.call("ddfa_tuning_get", 7) == -1                                 # DDFA_TUNE__COUNT = 7


def test_old_entry_points_name_their_replacement_in_deterministic_mode(L):
    try:
        L.call("ddfa_tuning_set", _lib.TUNE_DETERMINISTIC, 1)
        rc = L.raw("ddfa_embed_concat_bwd")(None, None, None, 4, 1002, 32, 10, None, None)
        assert rc == -1 and "ddfa_embed_concat_bwd_ws" in L.last_error()
        rc = L.raw("ddfa_readout_bwd")(None, None, None, None, None, 4, 128, None, None, None, None, None, None, None, None, None)
        assert rc == -1 and "ddfa_readout_bwd_ws" in L.last_error()
        rc = L.raw("ddfa_sgemm")(0, 0, 0, 4, 64, 1.0, None, 4, None, 4, 1.0, None, 4, 2, None)     # m = 0: nothing to launch either way
        assert rc == -1 and "split_k = 1" in L.last_error()
    finally:
        L.call("ddfa_tuning_set", _lib.TUNE_DETERMINISTIC, 0)


def test_mode_comes_from_the_environment_then_from_torch(monkeypatch, L):
    prev = torch.are_deterministic_algorithms_enabled()
    try:
        monkeypatch.delenv("DDFA_DETERMINISTIC", raising=False)
        torch.use_deterministic_algorithms(True)
        assert _lib.deterministic_requested()
        torch.use_deterministic_algorithms(False)
        assert not _lib.deterministic_requested()
        monkeypatch.setenv("DDFA_DETERMINISTIC", "1")
        assert _lib.deterministic_requested()
        assert _lib.apply_deterministic_mode() and L.call("ddfa_tuning_get", _lib.TUNE_DETERMINISTIC) == 1
        torch.use_deterministic_algorithms(True)
        monkeypatch.setenv("DDFA_DETERMINISTIC", "0")
        assert not _lib.apply_deterministic_mode() and L.call("ddfa_tuning_get", _lib.TUNE_DETERMINISTIC) == 0
        monkeypatch.setenv("DDFA_DETERMINISTIC", "yes")
        with pytest.raises(_lib.DdfaError, match="DDFA_DETERMINISTIC"):
            _lib.deterministic_requested()
    finally:
        torch.use_deterministic_algorithms(prev)
        L.call("ddfa_tuning_set", _lib.TUNE_DETERMINISTIC, 0)


def test_workspace_queries():
    assert _lib.lib().call("ddfa_readout_bwd_workspace_bytes", 1024, 128) == 4 * 1024 * 257
    small = _lib.lib().call("ddfa_embed_concat_bwd_workspace_bytes", 4, 1002, 32, 1000)
    big = _lib.lib().call("ddfa_embed_concat_bwd_workspace_bytes", 4, 1002, 32, 157_381)
    assert 0 < small < big < 64 << 20
