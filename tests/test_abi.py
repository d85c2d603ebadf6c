"""CPU: the C-ABI library loads and exports every symbol include/cocos_b200.h
declares (no compute calls without a GPU)."""
import os
import re


def test_header_symbols_and_abi_version():
    from cocosnet_b200 import _lib
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    if not os.path.exists(_lib.LIB_PATH):
        _lib.build()
    hdr = open(os.path.join(root, "include", "cocos_b200.h")).read()
    declared = set(re.findall(r"\b(cocos_[a-z0-9_]+)\s*\(", hdr))
    assert declared, "no declarations parsed"
    h = _lib.lib()
    for name in declared:
        assert hasattr(h, name), name
    assert declared == set(_lib.SIGNATURES), (declared ^ set(_lib.SIGNATURES))
    assert h.cocos_abi_version() == 8


def test_ctypes_signatures_match_header_arity_and_kinds():
    """Every ctypes argtypes list in _lib.SIGNATURES has the arity and pointer/int/float kinds of the C prototype."""
    import ctypes
    from cocosnet_b200 import _lib
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    hdr = open(os.path.join(root, "include", "cocos_b200.h")).read()
    hdr = re.sub(r"/\*.*?\*/", "", hdr, flags=re.S)
    protos = dict(re.findall(r"\b(cocos_[a-z0-9_]+)\s*\(([^)]*)\)\s*;", hdr))
    assert set(protos) == set(_lib.SIGNATURES)
    for name, params in protos.items():
        params = [p.strip() for p in params.split(",") if p.strip() and p.strip() != "void"]
        argtypes = _lib.SIGNATURES[name]
        assert len(params) == len(argtypes), (name, len(params), len(argtypes))
        for p, a in zip(params, argtypes):
            if "*" in p:
                assert a is ctypes.c_void_p, (name, p)
            elif p.startswith("long long"):
                assert a in (ctypes.c_longlong, ctypes.c_long) and ctypes.sizeof(a) == 8, (name, p)
            elif p.startswith("float"):
                assert a is ctypes.c_float, (name, p)
            else:
                assert a is ctypes.c_int, (name, p)


def test_bad_arguments_are_errors_not_crashes():
    from cocosnet_b200 import _lib
    if not os.path.exists(_lib.LIB_PATH):
        _lib.build()
    h = _lib.lib()
    # argument validation happens before any CUDA call
    assert h.cocos_corr_warp_fwd(None, None, None, None, None, None, None, 1, 1, 1, 64, 3, 16, 8, 1.0, None) != 0
    assert b"null" in h.cocos_last_error()
    assert h.cocos_pack_rows_f16(None, None, 0, 1, 1, 2, 0, None, None) != 0
    # the attention's position-major V and dO rows hold every value channel in one row: Cvk narrower than Cv is refused
    # (non-null dummy pointers: nothing is dereferenced before the check)
    assert h.cocos_attn_pack_nhwc(16, 3, 384, 1, 8, 8, 64, 256, 0, 16, 16, 16, 256, 16, 16, 128, None, 64, None,
                                  None) != 0
    assert b"bad arguments" in h.cocos_last_error()
    assert h.cocos_attn_do_rows(16, 256, 1, 64, 256, 16, 128, 16, 16, 64, None) != 0
    assert b"bad arguments" in h.cocos_last_error()
