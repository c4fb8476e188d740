"""CPU: ddfa_gru_step_bwd_image_v2 rejects pointers the fused backward step cannot move with TMA (bulk and tensor-map copies
address 16-byte units).  The checks run before any device work, so no GPU is needed: the pointers are never dereferenced."""
import pytest

from deepdfa_b200 import _lib, build

BASE = 1 << 20                 # a 16-byte-aligned stand-in address for every pointer argument
N, D_, KEEP0 = 256, 128, 16


@pytest.fixture(scope="module")
def L():
    build.build()
    return _lib.lib()


def _call(L, **override):
    p = {n: BASE for n in ("dh_out", "indptr_t", "indices_t", "h_image", "s_image", "gates", "indptr", "ds", "dw_fold",
                           "db_fold", "db_ih", "dw_hh", "db_hh", "workspace")}
    p["dh"] = BASE + 4096      # dh must not alias dh_out
    p.update(override)
    return L.raw("ddfa_gru_step_bwd_image_v2")(p["dh_out"], None, p["indptr_t"], p["indices_t"], p.get("h"), p["h_image"],
                                               p["s_image"], p["gates"], p["indptr"], N, D_, p["ds"], p["dh"], p["dw_fold"],
                                               p["db_fold"], p["db_ih"], p["dw_hh"], p["db_hh"], p["workspace"], 0, KEEP0, None)


def test_bwd_image_v2_rejects_unaligned_tma_operands(L):
    # aligned pointers pass the argument checks and stop at the (empty) workspace
    assert _call(L) == -4
    for name in ("ds", "dh", "dh_out", "gates", "h"):
        rc = _call(L, **{name: BASE + 8192 + 8})
        assert rc == -1 and "16-byte aligned" in L.last_error(), (name, rc, L.last_error())
