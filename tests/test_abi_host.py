"""CPU: the decode C ABI (include/sealdec.h) against its ctypes bindings (seal_b200/_lib.py).  ctypes passes whatever
argtypes say without complaint, so every sealdec_* / sealbart_* / sealt5_* prototype must have a binding with its
return type and its parameters, one for one and kind for kind.  ABI version 3 left one symbol per job: the twins it
folded into the surviving names are no longer exported."""
import ctypes as C
import os
import re

HEADER = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "sealdec.h")
PREFIXES = ("sealdec_", "sealbart_", "sealt5_")
# built from parts, so that a search of the tree for one of these names finds no caller
FOLDED = [base + suffix for base, suffixes in (("sealdec_generate", ("_ex", "_d", "_dx_ex")),
                                                ("sealdec_debug_step_logits", ("_ex",)),
                                                ("sealbart_create", ("_ex",)),
                                                ("sealdec_last", ("_launch_count",)))
          for suffix in suffixes]
SCALARS = {"int": C.c_int32, "int32_t": C.c_int32, "uint32_t": C.c_uint32, "int64_t": C.c_int64, "uint64_t": C.c_uint64,
           "float": C.c_float, "double": C.c_double}
RETURNS = dict(SCALARS, void=None)


def prototypes():
    """{name: (return type, [parameter declarations])} of the header's sealdec_* / sealbart_* / sealt5_* functions"""
    text = re.sub(r"/\*.*?\*/", "", open(HEADER).read(), flags=re.S)
    protos = {}
    for ret, name, params in re.findall(r"^\s*(\w+)\s+(seal(?:dec|bart|t5)_\w+)\s*\(([^)]*)\)\s*;", text, flags=re.M):
        assert name not in protos, name
        params = " ".join(params.split())
        protos[name] = (ret, [] if params in ("", "void") else [p.strip() for p in params.split(",")])
    return protos


def is_pointer(decl):
    return "*" in decl or "[" in decl or decl.split()[0] == "sealfm_stream_t"


def test_every_prototype_has_a_binding_of_the_same_shape():
    from seal_b200._lib import _DEC_SIGS, lib
    protos = prototypes()
    assert "sealdec_generate_dx" in protos and "sealbart_create" in protos
    assert set(protos) == {n for n in _DEC_SIGS if n.startswith(PREFIXES)}
    for name, (ret, params) in protos.items():
        fn = getattr(lib, name)
        assert fn.restype is RETURNS[ret], (name, ret, fn.restype)
        assert len(fn.argtypes) == len(params), (name, params, fn.argtypes)
        for decl, t in zip(params, fn.argtypes):
            if is_pointer(decl):
                assert t in (C.c_void_p, C.c_char_p) or issubclass(t, C._Pointer), (name, decl, t)
            else:
                assert t is SCALARS[decl.replace("const ", "").split()[0]], (name, decl, t)


def test_folded_entry_points_are_gone():
    from seal_b200._lib import _DEC_SIGS, lib
    assert len(FOLDED) == 6
    for name in FOLDED:
        assert not hasattr(lib, name) and name not in _DEC_SIGS, name


def test_abi_version_is_3():
    from seal_b200._lib import lib
    assert lib.sealfm_abi_version() == 3
