"""CPU: the gradient-guard entry points' size queries and argument checks (no GPU needed: nothing is launched)."""
import pytest

from deepdfa_b200 import _lib, build


@pytest.fixture(scope="module")
def L():
    build.build()
    return _lib.lib()


def test_size_queries(L):
    ws = L.call("ddfa_grad_norm_workspace_bytes", 375_938)
    assert ws > 0 and ws % 8 == 0 and ws == L.call("ddfa_grad_norm_workspace_bytes", 2 ** 24 + 4)    # a fixed grid of fp64 partials
    st = L.call("ddfa_p2p_guard_state_bytes")
    assert 16 < st <= 1024 and st % 16 == 0
    assert _lib.P2P_GUARD_FLAG_WORDS == 96


def test_argument_checks(L):
    with pytest.raises(_lib.DdfaError, match="ddfa_grad_norm: negative numel"):
        L.call("ddfa_grad_norm", None, -1, None, None, None, 0, None)
    with pytest.raises(_lib.DdfaError, match="ddfa_grad_norm: NULL pointer"):
        L.call("ddfa_grad_norm", None, 4, None, None, None, 0, None)
    with pytest.raises(_lib.DdfaError, match="workspace of 8 bytes"):
        L.call("ddfa_grad_norm", 256, 4, None, 256, 256, 8, None)
    with pytest.raises(_lib.DdfaError, match="ddfa_adam_flat_guarded: NULL pointer"):
        L.call("ddfa_adam_flat_guarded", 256, 256, 256, 256, 256, 4, 256, None, None, None)
    with pytest.raises(_lib.DdfaError, match="rank 2 / world 2"):
        L.call("ddfa_allreduce_adam_p2p_guarded", None, None, None, 2, 2, None, None, None, 4, 4, None, None, None, None, None, None, None)
    with pytest.raises(_lib.DdfaError, match="multiple of 4"):
        L.call("ddfa_allreduce_adam_p2p_guarded", None, None, None, 0, 1, None, None, None, 6, 6, None, None, None, None, None, None, None)
