"""The ctypes signature table (api.SIGNATURES) against include/ipcfp.h: one entry per declared function, with one argtype per
parameter. Read from the header's text, so no library and no device is needed."""
import os
import re

from ipc_filecoin_proofs_b200 import api

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared_functions():
    """{name: parameter count} of every function include/ipcfp.h declares"""
    hdr = open(os.path.join(ROOT, "include", "ipcfp.h")).read()
    hdr = re.sub(r"/\*.*?\*/", " ", hdr, flags=re.S)
    hdr = re.sub(r"//[^\n]*", " ", hdr)
    hdr = re.sub(r"^\s*#[^\n]*", " ", hdr, flags=re.M)
    decls = {}
    # a declaration: a return type, the name and a parameter list without parentheses (function-pointer parameters are typedefs)
    for stmt in re.split(r"[;{}]", hdr):
        m = re.fullmatch(r"(?!typedef\b)[A-Za-z_][\w\s*]*?\b(ipcfp_\w+)\s*\(([^()]*)\)", stmt.strip())
        if not m:
            continue
        name, params = m.group(1), m.group(2).strip()
        assert name not in decls, f"{name} is declared twice"
        decls[name] = 0 if params in ("", "void") else len(params.split(","))
    return decls


def test_header_parse_sees_every_declaration():
    decls = _declared_functions()
    assert decls["ipcfp_last_error"] == 0
    assert decls["ipcfp_store_create"] == 9
    assert decls["ipcfp_verify_bundle_json_any"] == 9
    hdr = open(os.path.join(ROOT, "include", "ipcfp.h")).read()
    named = set(re.findall(r"\b(ipcfp_[a-z0-9_]+)\s*\(", hdr)) - {"ipcfp_store", "ipcfp_tipset"}   # as test_abi_layout.py reads it
    assert set(decls) == named, (named - set(decls), set(decls) - named)


def test_signature_table_matches_header():
    decls = _declared_functions()
    assert set(api.SIGNATURES) == set(decls), (set(decls) - set(api.SIGNATURES), set(api.SIGNATURES) - set(decls))
    assert api.EXPORTS == list(api.SIGNATURES)
    wrong = {name: (len(argtypes or ()), decls[name]) for name, (_, argtypes) in api.SIGNATURES.items()
             if len(argtypes or ()) != decls[name]}
    assert not wrong, wrong
