"""CPU: the C-ABI library builds, loads, and exports every symbol include/*.h declares;
host-side argument validation fails loudly (no compute calls - there is no GPU here)."""
import ctypes
import os
import re

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def header_symbols():
    names = set()
    for fn in sorted(os.listdir(os.path.join(ROOT, "include"))):
        if fn.endswith(".h"):
            text = open(os.path.join(ROOT, "include", fn)).read()
            text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
            names.update(re.findall(r"\b(tb_[a-z0-9_]+)\s*\(", text))
    return sorted(names)


def test_library_exports_every_declared_symbol():
    from torchbeast_b200 import _lib
    h = ctypes.CDLL(_lib.LIB_PATH)
    syms = header_symbols()
    assert len(syms) >= 10
    for s in syms:
        assert hasattr(h, s), "libtorchbeast_b200.so lacks %s" % s
    # the ctypes binding table covers exactly the header
    assert sorted(_lib.declared_symbols()) == syms
    assert _lib.lib().tb_abi_version() == 1
    assert _lib.lib().tb_workspace_bytes() > 64


_CTYPES_OF = {"float": ctypes.c_float, "double": ctypes.c_double, "int": ctypes.c_int, "int64_t": ctypes.c_int64,
              "uint64_t": ctypes.c_uint64, "size_t": ctypes.c_size_t}


def _ctype_of(decl):
    """The ctypes type a binding must use for one C parameter or return type (`decl` without its name)."""
    if "*" in decl:
        return (ctypes.c_char_p,) if decl.replace(" ", "") == "constchar*" else (ctypes.c_void_p, ctypes.c_char_p)
    return (_CTYPES_OF[decl.strip()],)


def test_binding_matches_every_header_signature():
    # a ctypes call with a stale argument list passes whatever its arguments happen to be: check count and kind
    from torchbeast_b200 import _lib
    text = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "torchbeast_b200.h")).read(), flags=re.S)
    decls = re.findall(r"([A-Za-z_][\w ]*?[\s*]+)(tb_[a-z0-9_]+)\s*\(([^()]*)\)\s*;", text)
    assert sorted(name for _, name, _ in decls) == header_symbols()
    for ret, name, params in decls:
        params = [p.strip() for p in params.split(",") if p.strip() not in ("", "void")]
        argtypes, restype = _lib._SIGNATURES[name]
        assert len(argtypes) == len(params), "%s: %d argtypes for %d parameters" % (name, len(argtypes), len(params))
        for i, (param, argtype) in enumerate(zip(params, argtypes)):
            kind = re.sub(r"\s*\b\w+$", "", param)  # drop the parameter name
            assert argtype in _ctype_of(kind), "%s: parameter %d (%s) bound as %s" % (name, i, param, argtype.__name__)
        assert restype in _ctype_of(ret), "%s: returns %s, bound as %s" % (name, ret.strip(), restype.__name__)


def test_cpu_tensors_fail_loudly():
    from torchbeast_b200 import _lib
    from torchbeast_b200.core import vtrace
    from torchbeast_b200 import losses
    z = torch.zeros
    with pytest.raises(_lib.TorchBeastB200Error, match="CUDA tensors only"):
        vtrace.from_importance_weights(z(3, 2), z(3, 2), z(3, 2), z(3, 2), z(2))
    with pytest.raises(_lib.TorchBeastB200Error, match="CUDA tensors only"):
        vtrace.action_log_probs(z(3, 2, 4), z(3, 2, dtype=torch.int64))
    with pytest.raises(_lib.TorchBeastB200Error, match="CUDA tensors only"):
        losses.compute_baseline_loss(z(4))


def test_null_pointer_and_size_validation_host_side():
    from torchbeast_b200 import _lib
    h = _lib.lib()
    rc = h.tb_vtrace_from_importance_weights_f32(None, None, None, None, None, 4, 4, 1.0, 1.0, None, None, None)
    assert rc != 0 and b"null pointer" in h.tb_last_error()
    rc = h.tb_vtrace_from_importance_weights_f32(None, None, None, None, None, -1, 4, 1.0, 1.0, None, None, None)
    assert rc != 0 and b"negative size" in h.tb_last_error()
    # empty problems are a no-op success
    assert h.tb_vtrace_from_importance_weights_f32(None, None, None, None, None, 0, 4, 1.0, 1.0, None, None, None) == 0
    assert h.tb_action_log_probs_f32(None, None, 0, 6, None, None) == 0


def test_cuda_sources_read_no_environment():
    # the library chooses kernels from shapes alone: an environment switch would add a path no test runs, and could
    # pair a forward with a backward (or a workspace size) chosen under a different setting
    csrc = os.path.join(ROOT, "torchbeast_b200", "csrc")
    sources = sorted(fn for fn in os.listdir(csrc) if fn.endswith((".cu", ".cuh")))
    assert sources
    offenders = [fn for fn in sources if "getenv" in open(os.path.join(csrc, fn)).read()]
    assert not offenders, "getenv in %s" % ", ".join(offenders)
