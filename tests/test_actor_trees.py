"""The actor-proof trees and restatement of tests/actor_trees.py without a GPU: every tree's outcome is the one its builder meant, the
ground truth of the main tree, and the ctypes layout of ipcfp_actor_proof / ipcfp_actor_result against include/ipcfp.h."""
import ctypes as C
import os
import subprocess
import tempfile

import pytest

from ipc_filecoin_proofs_b200 import _abi as A
from oracle.pyoracle import keccak256
from tests import actor_trees as AT

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def world(ts3_small):
    return AT.world(ts3_small)


@pytest.mark.parametrize("name", [t.name for t in AT.blocks_and_trees()[1]])
def test_tree_outcome(world, name):
    blocks, trees, _, _ = world
    t = trees[name]
    try:
        proofs, lists, union = AT.prove(blocks, t.child, t.root, t.addrs, AT.EVM_SETS[t.evm], t.with_code)
    except AT.Failure as f:
        assert (f.status, f.index) == (t.status, 1 if t.status != A.ERR_INVALID_ARG else f.index), name
        return
    assert t.status is None, name
    assert set(union) == set().union(*map(set, lists)) if lists else union == []
    for p, lst in zip(proofs, lists):
        assert bytes(t.child) in lst   # the header anchors every proof
        if p["bytecode"] is not None:
            assert keccak256(p["bytecode"]) == p["bytecode_hash"]


def test_main_truth(world):
    blocks, trees, main, _ = world
    t = trees["main-code"]
    proofs, _, _ = AT.prove(blocks, t.child, t.root, t.addrs, AT.EVM_SETS[t.evm], True)
    by_addr = {p["address"]: p for p in proofs}
    for a, aid in main["amap"].items():
        assert by_addr[a]["actor_id"] == aid
    assert by_addr[AT.R.id_addr(104)]["balance"] == -(2 ** 90 + 3)
    assert by_addr[AT.R.id_addr(106)]["balance"] == 0          # minus zero is zero
    assert by_addr[AT.R.id_addr(999)]["status"] == A.ACTOR_NO_ACTOR
    assert sum(p["is_evm"] for p in proofs) == 6 and all(p["bytecode"] for p in proofs if p["is_evm"])


def test_refusals_restated(world):
    blocks, trees, _, _ = world
    t = trees["main"]
    with pytest.raises(AT.Failure) as e:
        AT.prove(blocks, t.child, t.root, [AT.R.id_addr(0), b"\x05" + bytes(20)])
    assert (e.value.status, e.value.index) == (A.ERR_INVALID_ARG, 1)


def test_deepest_path_fits_the_recorder():
    """The deepest accepted two-HAMT path (address_map and actors HAMT chains of 51 nodes) records 107 blocks in the proof's list."""
    import synth
    ts = synth.Tipset(synth.config_params(3, hamt_entries=20000))
    blocks, trees, _, _ = AT.world(ts)
    t = trees["deep"]
    _, lists, _ = AT.prove(blocks, t.child, t.root, t.addrs, AT.EVM_SETS[t.evm], True)
    assert max(len(l) for l in lists) == 107 <= 320


def test_ctypes_layout_matches_c_header():
    structs = {"ipcfp_actor_proof": A.ActorProofC, "ipcfp_actor_result": A.ActorResultC}
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "ipcfp.h"', "int main(void) {"]
    for cname, st in structs.items():
        lines.append(f'printf("{cname} %zu\\n", sizeof({cname}));')
        for fname, _ in st._fields_:
            lines.append(f'printf("{cname}.{fname} %zu\\n", offsetof({cname}, {fname}));')
    lines += ["return 0; }"]
    with tempfile.TemporaryDirectory() as td:
        src, exe = os.path.join(td, "layout.c"), os.path.join(td, "layout")
        open(src, "w").write("\n".join(lines))
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), "-o", exe, src])
        got = dict(l.split() for l in subprocess.check_output([exe], text=True).strip().splitlines())
    assert int(got["ipcfp_actor_proof"]) == C.sizeof(A.ActorProofC) == 400
    for cname, st in structs.items():
        assert int(got[cname]) == C.sizeof(st), cname
        for fname, _ in st._fields_:
            assert int(got[f"{cname}.{fname}"]) == getattr(st, fname).offset, f"{cname}.{fname}"


@pytest.mark.parametrize("name", [t.name for t in AT.blocks_and_trees()[1]])
def test_cpp_oracle_agrees_with_the_restatement(world, name):
    """The two restatements — tests/actor_trees.py and the C++ oracle tests/oracle_actors.cpp on oracle/oracle.cpp's ActorState decoder,
    get_actor_state and hamt_get — give the same proofs, per-proof read sets and union, or the same (status, index), with and without
    code, on every tree."""
    from tests import oracle_actors as O
    blocks, trees, _, _ = world
    t = trees[name]
    oracle = _oracle(O, blocks)
    for with_code in (False, True):
        for evm in AT.EVM_SETS.values():
            try:
                exp = AT.prove(blocks, t.child, t.root, t.addrs, evm, with_code)
            except AT.Failure as f:
                with pytest.raises(AT.Failure) as e:
                    oracle.prove(t.child, t.root, t.addrs, evm, with_code)
                assert (e.value.status, e.value.index) == (f.status, f.index), (name, with_code)
                continue
            assert oracle.prove(t.child, t.root, t.addrs, evm, with_code) == exp, (name, with_code)


_ORACLES = {}


def _oracle(O, blocks):
    if id(blocks) not in _ORACLES:
        _ORACLES.clear()
        _ORACLES[id(blocks)] = (blocks, O.Oracle(blocks))
    return _ORACLES[id(blocks)][1]


def test_rust_sys_structs_match_the_c_layout():
    """integration/rust/ipcfp-sys declares ipcfp_actor_proof / ipcfp_actor_result with the C field order and types: the fields, in order,
    with the size each Rust type has, give the C header's offsets (computed with the C alignment rules)."""
    import re
    src = open(os.path.join(ROOT, "integration", "rust", "ipcfp-sys", "src", "lib.rs")).read()
    size = {"u8": (1, 1), "u32": (4, 4), "u64": (8, 8), "f32": (4, 4), "ipcfp_address": (66, 1), "ipcfp_witness": (48, 8)}
    for rname, st in (("ipcfp_actor_proof", A.ActorProofC), ("ipcfp_actor_result", A.ActorResultC)):
        body = re.search(r"pub struct " + rname + r" \{(.*?)\}", src, re.S).group(1)
        fields = re.findall(r"pub (\w+): ([^,]+?)\s*(?:,|$)", body.strip())
        assert [f for f, _ in fields] == [f for f, _ in st._fields_], rname
        off = 0
        for (fname, ty), (_, cty) in zip(fields, st._fields_):
            ty = ty.strip()
            m = re.fullmatch(r"\[(\w+); (\w+)\]", ty)
            if m:
                n = {"IPCFP_ADDRESS_MAX": 65}.get(m.group(2)) or int(m.group(2))
                sz, al = size[m.group(1)][0] * n, size[m.group(1)][1]
            elif ty.startswith("*"):
                sz, al = 8, 8
            else:
                sz, al = size[ty]
            off = (off + al - 1) // al * al
            assert off == getattr(st, fname).offset and sz == C.sizeof(cty), (rname, fname)
            off += sz
        assert (off + 7) // 8 * 8 == C.sizeof(st), rname
