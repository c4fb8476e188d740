"""CPU: the C-ABI shared library builds for sm_90a, loads, and exports every symbol that
include/ddfa_b200.h declares.  No compute calls (there is no GPU here)."""
import ctypes
import re
import subprocess

import pytest

from deepdfa_b200 import _lib, build


@pytest.fixture(scope="module")
def libpath():
    return build.build()


def test_library_builds_and_loads(libpath):
    assert libpath.exists()
    L = _lib.lib()
    assert L.call("ddfa_abi_version") == 1
    assert isinstance(L.last_error(), str)


def test_every_declared_symbol_is_exported_and_bound(libpath):
    declared = _lib.declared_symbols()
    assert len(declared) >= 20
    dll = ctypes.CDLL(str(libpath))
    for name in declared:
        assert hasattr(dll, name), f"{name} declared in include/ddfa_b200.h but not exported"
    assert sorted(_lib._SIGNATURES) == declared, "ctypes binding and header disagree"


def test_binding_arity_matches_header():
    text = re.sub(r"/\*.*?\*/", "", _lib.HEADER.read_text(), flags=re.S)
    for name, (_, argtypes) in _lib._SIGNATURES.items():
        m = re.search(r"\b" + name + r"\s*\(([^;]*?)\)\s*;", text, flags=re.S)
        assert m, name
        args = m.group(1).strip()
        n = 0 if args in ("", "void") else len([a for a in args.split(",") if a.strip()])
        assert n == len(argtypes), f"{name}: header has {n} parameters, binding has {len(argtypes)}"


def test_library_is_sm90a_and_torch_free(libpath):
    out = subprocess.run([str(build.cuda_tool("cuobjdump")), "-lelf", str(libpath)], capture_output=True, text=True).stdout
    assert "sm_90a" in out and "sm_100" not in out
    ldd = subprocess.run(["ldd", str(libpath)], capture_output=True, text=True).stdout
    assert "libtorch" not in ldd and "libc10" not in ldd and "libpython" not in ldd     # C ABI only: no torch / Python types behind the boundary


def test_argument_validation_is_reported_without_a_gpu(libpath):
    L = _lib.lib()
    rc = L.raw("ddfa_gather_sum")(None, None, None, 10, 130, None, 0, None)   # D % 4 != 0
    assert rc == -1 and "D=130" in L.last_error()
    rc = L.raw("ddfa_build_csr")(None, None, 3, 0, 0, None, None, None, None, None, 0, None)
    assert rc == -1 and "idx_bytes" in L.last_error()
    with pytest.raises(_lib.DdfaError, match="ddfa_sgemm"):
        L.call("ddfa_sgemm", 0, 0, -1, 1, 1, 1.0, None, 1, None, 1, 0.0, None, 1, 1, None)
    assert L.call("ddfa_gru_step_workspace_bytes", 100, 128, 0) == 4 * 2 * 100 * 384
    rc = L.raw("ddfa_tuning_set")(_lib.TUNE_FWD_PAIR, 1)      # reserved key: the CTA-pair forward form does not exist on sm_90a
    assert rc == -1 and "FWD_PAIR" in L.last_error() and L.call("ddfa_tuning_get", _lib.TUNE_FWD_PAIR) == 0


@pytest.mark.parametrize("name", ["ddfa_readout_bwd", "ddfa_readout_bwd_ws"])
@pytest.mark.parametrize("arg", ["dpooled", "pooled", "h_final", "x", "w_gate", "dh_final", "dx"])
def test_readout_bwd_rejects_unaligned_rows_without_a_gpu(libpath, name, arg):
    """The readout backward reads and writes its [., D] rows with 16-byte vector accesses: each of those pointers 4 bytes off is
    refused before any launch (fake pointers: a launch would fault)."""
    L = _lib.lib()
    F = 256
    names = ["dpooled", "pooled", "h_final", "x", "graph_ptr", "B", "D", "w_gate", "gate_logit", "seg_max", "seg_sum", "dh_final",
             "dx", "dw_gate", "db_gate"]
    args = [F] * len(names)
    args[names.index("B")], args[names.index("D")] = 4, 128
    args[names.index(arg)] = F + 4
    extra = (F, 1 << 20, None) if name.endswith("_ws") else (None,)
    rc = L.raw(name)(*args, *extra)
    assert rc == -1 and "16-byte alignment" in L.last_error()


def test_header_is_plain_c_and_a_c_host_links_the_library(libpath, tmp_path):
    """The boundary is a C ABI: include/ddfa_b200.h must compile as C99 (no C++, no torch / CUDA headers) and a C host must link
    against libddfa_b200.so and call the entry points that need no GPU (version, error string, size queries, argument validation)."""
    import os
    import shutil
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
  if (ddfa_abi_version() != 1) return 1;
  if (ddfa_act_image_bytes(129) != 2 * 65536) return 2;                       /* two 128-node tiles of 64 KB */
  if (ddfa_build_csr_workspace_bytes(10, 4) != sizeof(int32_t) * (4 + 2 * 4 + 2 * 10)) return 3;
  if (ddfa_gather_sum(NULL, NULL, NULL, 10, 130, NULL, 0, NULL) != DDFA_ERR_INVALID_ARG) return 4;   /* D % 4 != 0 */
  if (strstr(ddfa_last_error(), "D=130") == NULL) return 5;
  if (ddfa_tuning_get(DDFA_TUNE_GATE_BWD_TMA) != 2 || ddfa_tuning_get(DDFA_TUNE__COUNT) != -1) return 6;
  printf("ok\n");
  return 0;
}
''')
    exe = tmp_path / "host"
    libdir = os.path.dirname(str(libpath))
    r = subprocess.run([cc, "-std=c99", "-Wall", "-Werror", "-pedantic", "-I", os.path.join(root, "include"), str(src), "-o", str(exe),
                        "-L", libdir, "-lddfa_b200", f"-Wl,-rpath,{libdir}"], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    run = subprocess.run([str(exe)], capture_output=True, text=True)
    assert run.returncode == 0 and run.stdout.strip() == "ok", (run.returncode, run.stdout, run.stderr)
