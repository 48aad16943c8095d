"""Parses the reference's `extern "C"` declarations (its ffi.rs files, macro-declared launchers included) with the
parser of tests/test_abi.py and stores, for every symbol this library exports under a reference name, the argument
classes per position and whether it returns a value:
    python tests/golden/make_ffi_signatures.py REFERENCE_CHECKOUT     (writes tests/golden/reference_ffi_signatures.json)
tests/test_abi.py checks the headers against this table."""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import test_abi as T  # noqa: E402

ref = sys.argv[1]
rust = {}
for f in T.FFI_FILES:
    text = open(os.path.join(ref, f)).read()
    if not f.endswith("ffi.rs"):                       # a full source file: only its trailing `mod ffi { extern "C" { .. } }`
        text = text[text.rindex("mod ffi"):]
    rust.update(T._rust_signatures(text))
ours = [n for n in T._c_signatures() if not n.startswith("mrs_") or n in T.REF_MRS_NAMES]
table = {n: [rust[n][0], rust[n][1]] for n in sorted(ours) if n in rust}   # name: [argument classes, returns a value]
with open(os.path.join(HERE, "reference_ffi_signatures.json"), "w") as f:
    f.write("{\n" + ",\n".join(f"{json.dumps(n)}: {json.dumps(v)}" for n, v in table.items()) + "\n}\n")
print(len(table), "signatures")
