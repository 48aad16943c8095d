"""The C-ABI library loads (no GPU needed) and exports every symbol include/*.h declares; the
product fails loudly when the extension is missing; the host C++ layer loads too."""
import ctypes
import glob
import os
import re
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared_symbols(host=False):
    """symbols declared by include/*.h; mrs_b200_host.h belongs to libmrs_b200_host.so, the rest to
    the CUDA library"""
    names = set()
    for h in sorted(glob.glob(os.path.join(ROOT, "include", "*.h"))):
        if h.endswith("_host.h") != host:
            continue
        src = subprocess.run(["gcc", "-E", "-P", h], capture_output=True, text=True, check=True).stdout
        src = re.sub(r"typedef\s+struct\s*\{.*?\}\s*\w+\s*;", "", src, flags=re.S)
        for m in re.finditer(r"\b([A-Za-z_][A-Za-z0-9_]*)\s*\(([^;{}]*)\)\s*;", src):
            names.add(m.group(1))
    return names


def test_every_declared_symbol_is_exported():
    from mistralrs_b200 import LIB_PATH
    assert os.path.exists(LIB_PATH), "run __graft_entry__.build() first"
    lib = ctypes.CDLL(LIB_PATH)
    decl = _declared_symbols()
    assert len(decl) >= 93 + 20, len(decl)
    missing = [n for n in sorted(decl) if not hasattr(lib, n)]
    assert not missing, missing
    assert sum(n.startswith("launch_mmvq_gguf_") for n in decl) == 93


def test_host_library_exports_its_header():
    from mistralrs_b200.kv_index import HOST_LIB_PATH
    assert os.path.exists(HOST_LIB_PATH), "run __graft_entry__.build() first"
    lib = ctypes.CDLL(HOST_LIB_PATH)
    decl = _declared_symbols(host=True)
    assert len(decl) >= 26, len(decl)
    missing = [n for n in sorted(decl) if not hasattr(lib, n)]
    assert not missing, missing


FFI_FILES = ("mistralrs-quant/src/gguf/ffi.rs", "mistralrs-quant/src/rotary/ffi.rs", "mistralrs-quant/src/utils/ffi.rs",
             "mistralrs-quant/src/gptq/marlin_ffi.rs", "mistralrs-paged-attn/src/cuda/ffi.rs", "mistralrs-core/src/cuda/ffi.rs",
             "mistralrs-quant/src/gguf/packed_affine.rs")
# reference symbols that happen to carry the mrs_ prefix themselves (declared in packed_affine.rs:1436-1457)
REF_MRS_NAMES = ("mrs_gguf_affine_repack_f16", "mrs_gguf_affine_repack_bf16")


def _rust_class(t):
    t = t.strip()
    if t.startswith("*"):
        return "ptr"
    t = t.split("::")[-1]
    return {"i32": "i32", "c_int": "i32", "u32": "u32", "c_uint": "u32", "i64": "i64", "c_long": "i64", "c_longlong": "i64",
            "u64": "u64", "usize": "u64", "c_ulong": "u64", "f32": "f32", "c_float": "f32", "f64": "f64", "bool": "bool",
            "u8": "u8", "CUstream": "ptr"}.get(t, "?" + t)


def _c_class(t):
    t = re.sub(r"\b(const|volatile|restrict|__restrict__)\b", "", t).strip()
    t = re.sub(r"\s+[A-Za-z_][A-Za-z0-9_]*$", "", t).strip() if not t.endswith("*") and " " in t else t
    if "*" in t or t in ("cudaStream_t", "mrs_ops_stream_t", "mrs_stream_t", "CUstream"):
        return "ptr"
    return {"int": "i32", "int32_t": "i32", "unsigned int": "u32", "unsigned": "u32", "uint32_t": "u32", "long": "i64",
            "int64_t": "i64", "long long": "i64", "uint64_t": "u64", "size_t": "u64", "uintptr_t": "u64", "float": "f32", "double": "f64",
            "bool": "bool", "_Bool": "bool", "uint8_t": "u8"}.get(t, "?" + t)


def _split_args(text):
    out, depth, cur = [], 0, ""
    for ch in text:
        if ch in "(<[":
            depth += 1
        elif ch in ")>]":
            depth -= 1
        if ch == "," and depth == 0:
            out.append(cur); cur = ""
        else:
            cur += ch
    if cur.strip():
        out.append(cur)
    return [a.strip() for a in out if a.strip()]


def _rust_signatures(text):
    """name -> ([arg classes], returns_value) for plain `pub fn` items and `declare_*!(ident)` macro uses"""
    text = re.sub(r"//[^\n]*", "", text)
    sigs, macros = {}, {}
    for m in re.finditer(r"macro_rules!\s*(\w+)\s*\{\s*\(\s*\$(\w+):ident\s*\)\s*=>\s*\{(.*?)\n\s*\};\s*\n\}", text, flags=re.S):
        body = m.group(3)
        f = re.search(r"fn\s+\$" + m.group(2) + r"\s*\((.*?)\)\s*(->\s*[\w:]+)?\s*;", body, flags=re.S)
        if f:
            macros[m.group(1)] = (f.group(1), f.group(2))
    for m in re.finditer(r"\bfn\s+([A-Za-z_][A-Za-z0-9_]*)\s*\((.*?)\)\s*(->\s*(?:\*(?:mut|const)\s+)?[\w:]+)?\s*;", text, flags=re.S):
        args = [_rust_class(a.split(":", 1)[1]) for a in _split_args(m.group(2))]
        sigs[m.group(1)] = (args, m.group(3) is not None)
    for m in re.finditer(r"\b(\w+)!\s*\(\s*([A-Za-z_][A-Za-z0-9_]*)\s*\)\s*;", text):
        if m.group(1) in macros:
            argtext, ret = macros[m.group(1)]
            sigs[m.group(2)] = ([_rust_class(a.split(":", 1)[1]) for a in _split_args(argtext)], ret is not None)
    return sigs


def _c_signatures(host=False):
    sigs = {}
    for h in sorted(glob.glob(os.path.join(ROOT, "include", "*.h"))):
        if h.endswith("_host.h") != host:
            continue
        src = subprocess.run(["gcc", "-E", "-P", h], capture_output=True, text=True, check=True).stdout
        src = re.sub(r"typedef\s+struct\s*\{.*?\}\s*\w+\s*;", "", src, flags=re.S)
        src = re.sub(r"typedef[^;]*;", "", src)
        for m in re.finditer(r"([A-Za-z_][A-Za-z0-9_ \*]*?)\b([A-Za-z_][A-Za-z0-9_]*)\s*\(([^;{}]*)\)\s*;", src):
            ret, name, args = m.group(1).strip(), m.group(2), m.group(3)
            if args.strip() in ("", "void"):
                cls = []
            else:
                cls = [_c_class(a) for a in _split_args(args)]
            sigs[name] = (cls, ret not in ("void", "extern void"))
    return sigs


def test_reference_signatures_match_ffi_rs():
    """Every symbol we export under a reference name must have the ARGUMENT LIST of the reference's
    `extern "C"` declaration (arity, pointer / i32 / u32 / i64 / f32 / bool class per position, and
    whether it returns a value) — parsed out of the reference's ffi.rs files, macro-declared
    launchers included (tests/golden/reference_ffi_signatures.json).  A wrong argument order or width fails here,
    not at run time."""
    import json
    with open(os.path.join(ROOT, "tests", "golden", "reference_ffi_signatures.json")) as f:   # make_ffi_signatures.py
        rust = {n: (v[0], v[1]) for n, v in json.load(f).items()}
    ours = {n: v for n, v in _c_signatures().items() if not n.startswith("mrs_") or n in REF_MRS_NAMES}
    missing = sorted(n for n in ours if n not in rust)
    assert not missing, missing
    assert sum(n.startswith("launch_mmvq_gguf_") for n in ours) == 93
    bad = []
    for n, (cargs, cret) in sorted(ours.items()):
        rargs, rret = rust[n]
        if any(c.startswith("?") for c in cargs + rargs):
            bad.append((n, "unclassified type", cargs, rargs))
        elif cargs != rargs or cret != rret:
            bad.append((n, cargs, cret, rargs, rret))
    assert not bad, bad[:5]


def test_rust_ffi_source_matches_headers():
    """rust/mrs_b200_ffi.rs (the `extern "C"` block a maintainer adds for the mrs_* entry points) is
    generated from include/*.h; re-parse the committed file with the same parser used on the
    reference's ffi.rs and compare arity / argument classes / return with the headers."""
    rust = _rust_signatures(open(os.path.join(ROOT, "rust", "mrs_b200_ffi.rs")).read())
    ours = {n: v for n, v in _c_signatures().items() if n.startswith("mrs_")}
    assert set(rust) == set(ours), sorted(set(rust) ^ set(ours))
    for n, (cargs, cret) in ours.items():
        rargs, rret = rust[n]
        cargs = ["ptr" if c.startswith("?") else c for c in cargs]     # structs / callbacks cross as opaque pointers
        assert cargs == rargs and cret == rret, (n, cargs, rargs)
    shim = open(os.path.join(ROOT, "rust", "b200_quant_method.rs")).read()
    for name in re.findall(r"ffi::(mrs_[a-z0-9_]+)", shim):
        assert name in ours, name


def test_missing_extension_fails_loudly(monkeypatch, tmp_path):
    import mistralrs_b200 as pkg
    monkeypatch.setattr(pkg, "_lib", None)
    monkeypatch.setattr(pkg, "LIB_PATH", str(tmp_path / "nope.so"))
    with pytest.raises(pkg.ExtensionMissing, match="no CPU fallback"):
        pkg.lib()


def test_product_never_imports_oracle():
    for path in glob.glob(os.path.join(ROOT, "mistral.rs_b200", "**", "*.*"), recursive=True):
        if path.endswith((".py", ".cu", ".cuh", ".cpp", ".hpp", ".h")):
            src = open(path).read()
            assert "import oracle" not in src and "from oracle" not in src and "liboracle" not in src, path


def test_rust_host_ffi_source_matches_header():
    """rust/mrs_b200_host_ffi.rs — generated declarations for libmrs_b200_host (block pool / prefix cache / KV manager,
    slot + CSR builders, sampler tail, file readers) — re-parsed and compared with include/mrs_b200_host.h."""
    rust = _rust_signatures(open(os.path.join(ROOT, "rust", "mrs_b200_host_ffi.rs")).read())
    ours = _c_signatures(host=True)
    assert set(rust) == set(ours), sorted(set(rust) ^ set(ours))
    assert len(ours) >= 60
    for n, (cargs, cret) in ours.items():
        rargs, rret = rust[n]
        cargs = ["ptr" if c.startswith("?") else c for c in cargs]
        assert cargs == rargs and cret == rret, (n, cargs, rargs)
