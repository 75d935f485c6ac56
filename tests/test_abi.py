"""CPU-side checks of the C-ABI boundary: the library loads, exports every symbol that
include/ctr_b200.h declares, and rejects bad arguments without touching a GPU."""
import ctypes
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared_symbols():
    text = open(os.path.join(ROOT, "include", "ctr_b200.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(ctr_[a-z0-9_]+)\s*\(", text)))


def test_header_symbols_are_exported_and_bound_at_abi_2():
    from tf_repos_b200 import _lib
    names = _declared_symbols()
    assert "ctr_fm_embed_fwd" in names and len(names) >= 15
    lib = ctypes.CDLL(_lib.LIB_PATH)
    for n in names:
        assert hasattr(lib, n), f"{n} declared in include/ctr_b200.h but not exported"
        assert n in _lib.SIGNATURES, f"{n} has no ctypes signature in tf_repos_b200/_lib.py"
    assert set(_lib.SIGNATURES) <= set(names)
    assert _lib.abi_version() == 2


def test_argument_validation_needs_no_gpu():
    from tf_repos_b200 import _lib
    L = _lib.raw()
    # bad id width / missing buffers are rejected before any CUDA call
    assert L.ctr_fm_embed_fwd(None, 16, None, None, None, 10, 1, 1, 4, 0, None, None, None, None, None, None) == -1
    assert "id_bits" in _lib.last_error()
    assert L.ctr_fm_embed_fwd(None, 32, None, None, None, 10, 1, 1, 4, 0, None, None, None, None, None, None) == -1
    assert L.ctr_unique_segment(None, 10, 0, None, None, None, None, None, None, None, 0, None) == -1
    assert L.ctr_opt_sparse_rows(9, None, None, None, None, None, None, 5, 4, None, None, None) == -1
    assert L.ctr_unique_segment_workspace_bytes(319488, 200_000_000) > 3 * 319488 * 4
    assert L.ctr_launch_count() == 0


def test_missing_library_fails_loudly(tmp_path, monkeypatch):
    import importlib
    from tf_repos_b200 import _lib
    monkeypatch.setattr(_lib, "LIB_PATH", str(tmp_path / "nope.so"))
    try:
        _lib._load()
    except _lib.CtrError as e:
        assert "no CPU/eager fallback" in str(e)
    else:
        raise AssertionError("loading a missing library must raise")


def _c_kind(decl: str):
    """'const float* x' -> 'ptr'; 'int64_t n' -> ctypes.c_int64 ..."""
    decl = decl.strip()
    if "*" in decl or decl.startswith("ctr_stream_t"):
        return "ptr"
    words = decl.replace("const", " ").split()
    base = " ".join(words[:-1]) if len(words) > 1 else words[0]
    return {"int": ctypes.c_int, "int32_t": ctypes.c_int32, "int64_t": ctypes.c_int64, "uint64_t": ctypes.c_uint64,
            "size_t": ctypes.c_size_t, "float": ctypes.c_float, "double": ctypes.c_double, "void": None}[base]


def _py_kind(t):
    if t is None:
        return None
    if t in (ctypes.c_void_p, ctypes.c_char_p) or issubclass(t, ctypes._Pointer):
        return "ptr"
    return t


def test_ctypes_signatures_match_the_header_prototypes():
    """Every prototype of include/ctr_b200.h against tf_repos_b200/_lib.py::SIGNATURES: same number of arguments, same
    width and kind (pointer / int / int64 / size_t / float) in every position, same return type -- a mismatch here would
    pass garbage through the boundary without any error."""
    from tf_repos_b200 import _lib
    text = open(os.path.join(ROOT, "include", "ctr_b200.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    text = re.sub(r"//.*", "", text)
    protos = re.findall(r"([A-Za-z_][A-Za-z0-9_ \*]*?)\b(ctr_[a-z0-9_]+)\s*\(([^)]*)\)\s*;", text)
    assert len(protos) == len(_declared_symbols())
    for ret, name, args in protos:
        res, sig = _lib.SIGNATURES[name]
        want = [] if args.strip() in ("", "void") else [_c_kind(a) for a in args.split(",")]
        got = [_py_kind(t) for t in sig]
        assert got == want, (name, got, want)
        assert _py_kind(res) == _c_kind(ret + " x"), (name, res, ret)


def test_integration_md_binding_snippet_matches_the_header():
    """The reference-side ctypes stub shown in INTEGRATION.md §2 must bind the real prototype (it is documentation a
    maintainer copies): run its binding lines and compare the argtypes with SIGNATURES."""
    from tf_repos_b200 import _lib
    md = open(os.path.join(ROOT, "INTEGRATION.md")).read()
    block = md.split("## 2.")[1].split("```python")[1].split("```")[0]
    binding = block.split("def fm_forward")[0].replace('"tf_repos_b200/libctr_b200.so"', repr(_lib.LIB_PATH))
    ns = {}
    exec(binding, ns)                                   # import ctypes, torch; CDLL; argtypes -- no compute call
    got = [_py_kind(t) for t in ns["L"].ctr_fm_embed_fwd.argtypes]
    assert got == [_py_kind(t) for t in _lib.SIGNATURES["ctr_fm_embed_fwd"][1]]
    call = block.split("L.ctr_fm_embed_fwd(")[1].split(")\n")[0]
    assert len([a for a in re.split(r",(?![^()]*\))", call) if a.strip()]) == len(got)
