"""CPU: the encoder cache's C-ABI entry points (exported, declared, bound, argument checks before any launch, a C99 host), and the
refusals that come before any device work — a trainer over a trainable encoder, the gradient statement modes, a fingerprint that
no longer matches the module, a cache of another module.  The caches here hold no planes: only the fingerprint ``check`` reads."""
import os
import shutil
import subprocess

import pytest
import torch

import deepdfa_b200 as D
from deepdfa_b200 import _lib, build
from deepdfa_b200.encoder_cache import EncoderCache, encoder_names
from deepdfa_b200.evaluator import FusedEvaluator
from deepdfa_b200.predictor import FusedPredictor
from deepdfa_b200.trainer import FusedTrainer, flat_param_list

FEAT = "_ABS_DATAFLOW_api_all_limitall_1000_limitsubkeys_1000"
ENTRY_POINTS = ("ddfa_cache_batch", "ddfa_cache_batch_workspace_bytes")


@pytest.fixture(scope="module")
def lib():
    build.build()
    return _lib.lib()


def module(style="graph", seed=0, **kw):
    torch.manual_seed(seed)
    return D.FlowGNNGGNNModule(FEAT, 40, 4, 2, 2, label_style=style, concat_all_absdf=True, engine="simt", **kw)


def freeze_encoder(m):
    for name, p in m.named_parameters():
        if not name.startswith(("output_layer.", "pooling.")):
            p.requires_grad_(False)
    return m


def fingerprint_of(m) -> EncoderCache:
    """A cache object that holds only the fingerprint of ``m`` (what EncoderCache.__init__ records before its pass)."""
    c = EncoderCache.__new__(EncoderCache)
    c._record(m)
    return c


# ---- the C ABI ---------------------------------------------------------------------------------------------------------------
def test_entry_points_are_declared_exported_and_bound(lib):
    declared = _lib.declared_symbols()
    for name in ENTRY_POINTS:
        assert name in declared and name in _lib._SIGNATURES and hasattr(lib._dll, name)
    assert len(_lib._SIGNATURES["ddfa_cache_batch"][1]) == 17


def test_workspace_bytes(lib):
    for B in (1, 1023, 1024, 4097, 190_000):
        assert lib.call("ddfa_cache_batch_workspace_bytes", B) == 4 * (2 * B + 3)      # counter, node_ptr and chunk_ptr [B + 1]


def _args(**over):
    """ddfa_cache_batch with valid arguments (fake 16-byte-aligned pointers: a launch would fault) and ``over`` replaced."""
    a = dict(ids=256, B=4, G=10, node_off=512, vuln_all=768, h_all=1024, x_all=2048, N_all=100, D=128, N=40, graph_ptr=3072,
             vuln=3328, h=4096, x=8192, ws=12288, ws_bytes=4 * 11, stream=None)
    a.update(over)
    return list(a.values())


@pytest.mark.parametrize("over,msg", [
    (dict(B=0), "bad sizes"), (dict(G=0), "bad sizes"), (dict(D=130), "D=130"), (dict(D=0), "bad sizes"), (dict(N=-1), "bad sizes"),
    (dict(N_all=-1), "bad sizes"), (dict(ids=None), "NULL"), (dict(node_off=None), "NULL"), (dict(graph_ptr=None), "NULL"),
    (dict(h_all=None), "NULL cache plane"), (dict(vuln=None), "NULL output"), (dict(x=None), "NULL output"),
    (dict(h_all=1028), "16-byte"), (dict(x=8196), "16-byte"),
])
def test_argument_checks_come_before_any_launch(lib, over, msg):
    rc = lib.raw("ddfa_cache_batch")(*_args(**over))
    assert rc == -1 and msg in lib.last_error(), lib.last_error()


def test_short_workspace_is_refused_before_any_launch(lib):
    assert lib.raw("ddfa_cache_batch")(*_args(ws_bytes=4 * 10)) == -4 and "workspace too small" in lib.last_error()
    assert lib.raw("ddfa_cache_batch")(*_args(ws=None)) == -4


def test_empty_batch_may_pass_null_rows(lib):
    """N = 0 (only 0-node graphs) needs no output rows: the NULL checks pass and only the fake-pointer launch remains, which is
    not made here — a short workspace stops the call right after the checks."""
    rc = lib.raw("ddfa_cache_batch")(*_args(N=0, vuln=None, h=None, x=None, ws_bytes=0))
    assert rc == -4                    # DDFA_ERR_WORKSPACE


def test_a_c99_host_calls_the_entry_points(lib, tmp_path):
    cc = shutil.which("gcc") or shutil.which("cc")
    if cc is None:
        pytest.skip("no C compiler")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    src = tmp_path / "host.c"
    src.write_text(r'''
#include <stdio.h>
#include <string.h>
#include "ddfa_b200.h"
int main(void) {
  if (ddfa_cache_batch_workspace_bytes(1024) != sizeof(int32_t) * 2051) return 1;
  if (ddfa_cache_batch(NULL, 4, 10, NULL, NULL, NULL, NULL, 0, 130, 0, NULL, NULL, NULL, NULL, NULL, 0, NULL) != DDFA_ERR_INVALID_ARG) return 2;
  if (strstr(ddfa_last_error(), "D=130") == NULL) return 3;
  printf("ok\n");
  return 0;
}
''')
    exe = tmp_path / "host"
    libdir = os.path.dirname(str(build.LIB))
    r = subprocess.run([cc, "-std=c99", "-Wall", "-Werror", "-pedantic", "-I", os.path.join(root, "include"), str(src), "-o", str(exe),
                        "-L", libdir, "-lddfa_b200", f"-Wl,-rpath,{libdir}"], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    run = subprocess.run([str(exe)], capture_output=True, text=True)
    assert run.returncode == 0 and run.stdout.strip() == "ok", (run.returncode, run.stdout, run.stderr)


# ---- fingerprint -------------------------------------------------------------------------------------------------------------
def test_an_unchanged_module_matches():
    m = freeze_encoder(module())
    c = fingerprint_of(m)
    c.check(m)
    with torch.no_grad():                      # head parameters are not part of the fingerprint
        m.output_layer[0].weight.add_(1.0)
    c.check(m)


@pytest.mark.parametrize("which", ["all_embeddings.api.weight", "ggnn.gru.weight_ih", "ggnn.linears.0.bias"])
def test_load_state_dict_into_the_encoder_is_seen(which):
    m = module()
    c = fingerprint_of(m)
    sd = {k: v.clone() for k, v in m.state_dict().items()}
    sd[which].add_(0.5)
    ptrs = [p.data_ptr() for p in m.parameters()]
    m.load_state_dict(sd)                                        # in place: same storage, a new _version
    assert [p.data_ptr() for p in m.parameters()] == ptrs
    with pytest.raises(ValueError, match="rebuild the cache") as e:
        c.check(m)
    assert which in str(e.value)


def test_new_storage_is_seen():
    m = module()
    c = fingerprint_of(m)
    m.ggnn.gru.weight_hh.data = m.ggnn.gru.weight_hh.data.clone()     # what FusedTrainer does when it builds its flat buffer
    with pytest.raises(ValueError, match="ggnn.gru.weight_hh"):
        c.check(m)


def test_a_cache_of_another_module_raises():
    a, b = module(seed=0), module(seed=0)
    c = fingerprint_of(a)
    with pytest.raises(ValueError, match="another module"):
        c.check(b)


def test_engine_and_deterministic_mode_are_part_of_it(monkeypatch):
    m = module()
    monkeypatch.setenv("DDFA_DETERMINISTIC", "0")
    c = fingerprint_of(m)
    monkeypatch.setenv("DDFA_DETERMINISTIC", "1")
    with pytest.raises(ValueError, match="deterministic mode off.*now on"):
        c.check(m)
    monkeypatch.setenv("DDFA_DETERMINISTIC", "0")
    c.check(m)
    c.engine = "tcgen05"
    with pytest.raises(ValueError, match="engine"):
        c.check(m)


def test_encoder_names_cover_tables_and_ggnn():
    m = module()
    names = encoder_names(m)
    assert names[:4] == [f"all_embeddings.{k}.weight" for k in D.allfeats]
    assert names[4:] == ["ggnn.linears.0.weight", "ggnn.linears.0.bias", "ggnn.gru.weight_ih", "ggnn.gru.weight_hh",
                         "ggnn.gru.bias_ih", "ggnn.gru.bias_hh"]


# ---- the owners' refusals (they come before any device work) -----------------------------------------------------------------
def _trainer_stub(m):
    """The state ``FusedTrainer._run_ids`` reads before it touches the device, without the device work of the constructor."""
    tr = FusedTrainer.__new__(FusedTrainer)
    tr.module = m
    tr._stream_slots = {}
    tr._trainable = tuple(bool(p.requires_grad) for p in flat_param_list(m))
    ntab = len(m._tables())
    tr._grad_ggnn = any(tr._trainable[:ntab + 6])
    return tr


@pytest.mark.parametrize("style", ["graph", "node"])
def test_a_trainer_over_a_trainable_encoder_rejects_a_cache(style):
    m = module(style)
    m.all_embeddings["api"].weight.requires_grad_(False)            # tables partly frozen, the GGNN trainable
    c = fingerprint_of(m)
    with pytest.raises(ValueError, match="frozen graph encoder") as e:
        _trainer_stub(m)._run_ids(c, [0], (None, "apply"), "step_ids")
    assert "ggnn.gru.weight_ih" in str(e.value) and "all_embeddings.api.weight" not in str(e.value)


def test_a_frozen_trainer_gets_past_the_refusal_to_the_fingerprint():
    m = freeze_encoder(module())
    c = fingerprint_of(module(seed=1))
    with pytest.raises(ValueError, match="another module"):
        _trainer_stub(m)._run_ids(c, [0], (None, "apply"), "step_ids")


@pytest.mark.parametrize("owner", [FusedEvaluator, FusedPredictor])
@pytest.mark.parametrize("mode", ["saliency", "integrated_gradients", "deeplift", "deeplift_shap", "gradient_shap"])
def test_gradient_statement_modes_reject_a_cache(owner, mode):
    m = module()
    ev = owner.__new__(owner)
    ev.module, ev.statements, ev._stream_slots = m, mode, {}
    with pytest.raises(ValueError, match="differentiates through the GGNN"):
        ev._run_ids(fingerprint_of(m), [0], None, "update_ids")


@pytest.mark.parametrize("mode", [None, "attention"])
def test_other_statement_modes_get_past_the_refusal(mode):
    m = module()
    ev = FusedEvaluator.__new__(FusedEvaluator)
    ev.module, ev.statements, ev._stream_slots = m, mode, {}
    with pytest.raises(ValueError, match="another module"):
        ev._run_ids(fingerprint_of(module(seed=2)), [0], None, "update_ids")


def test_matches_is_check_without_raising():
    m = module()
    c = fingerprint_of(m)
    assert c.matches(m) and not c.matches(module(seed=1))
    with torch.no_grad():
        m.ggnn.gru.bias_hh.add_(1.0)
    assert not c.matches(m)


def test_a_stale_cache_loses_its_slots():
    """A cache that fails the check loses the slots an owner keeps for it (and with them the owner's reference to it); making a
    slot for a new cache drops those of every other cache that no longer matches.  The slots here hold no captured graph."""
    m = module()
    ev = FusedEvaluator.__new__(FusedEvaluator)
    ev.module, ev.statements = m, None
    old, other = fingerprint_of(m), fingerprint_of(m)
    ev._stream_slots = {("cache", id(old), 10, 2, False): {"arena": old, "graph": None},
                        ("cache", id(other), 10, 2, False): {"arena": other, "graph": None},
                        ("arena", 123, 10, 5, 2, False): {"arena": None, "graph": None}}
    ev._drop_cache_slots(lambda c: c is not other and not c.matches(m))     # every cache matches: nothing goes
    assert len(ev._stream_slots) == 3
    with torch.no_grad():
        m.ggnn.gru.weight_hh.mul_(0.5)
    with pytest.raises(ValueError, match="rebuild the cache"):
        ev._run_ids(old, [0], None, "update_ids")
    assert [k[0] for k in ev._stream_slots] == ["cache", "arena"] and id(other) in [k[1] for k in ev._stream_slots]
    ev._drop_cache_slots(lambda c: not c.matches(m))
    assert [k[0] for k in ev._stream_slots] == ["arena"]
