"""Storage paths on the CPU: the Python restatement of Solidity's layout rules (tests/storage_paths.py) against public vectors and the
reference's own slot helper, the contract catalogue against its ground truth, StoragePath's key encodings and packed decoding, and the
C layout of the new ABI structs. No GPU."""
import ctypes as C
import os
import subprocess
import tempfile

import pytest

from ipc_filecoin_proofs_b200 import _abi as A
from ipc_filecoin_proofs_b200.api import StoragePath, encode_key
from oracle.pyoracle import keccak256
from tests import storage_paths as SP
from tests.test_oracle_cpu import SOLIDITY_ARRAY_VECTORS, SOLIDITY_SLOT_VECTORS

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_one_step_paths_are_compute_mapping_slot(oracle_mod):
    """calculate_storage_slot("calib-subnet-1", 0) (storage/utils.rs:16-19) and the public vectors as one-step MAPPING paths"""
    key = b"calib-subnet-1".ljust(32, b"\0")
    _, values, slot, _ = SP.derive(StoragePath(0, 0).mapping(key, "bytes32"))
    assert slot == values[0] == oracle_mod.compute_mapping_slot(key, 0)
    for key, idx, want in SOLIDITY_SLOT_VECTORS:
        assert SP.derive(StoragePath(0, idx).mapping(key))[2].hex() == want
    # a dynamic array's data starts at keccak256(p): element 0 of an array at p = 0 and p = 1
    for p, want in SOLIDITY_ARRAY_VECTORS:
        lengths, _, slot, _ = SP.derive(StoragePath(0, p).array(0))
        assert slot.hex() == want and lengths == [p]


def test_subnet_member_is_a_mapping_then_a_field():
    """subnets[id].topDownNonce: the path {0, MAPPING id} then the member's slot offset"""
    sid = bytes(range(32))
    base = keccak256(sid + bytes(32))
    for off in range(4):
        assert SP.derive(StoragePath(0, 0).mapping(sid, "bytes32").field(off))[2] == SP.b32(SP.u256(base) + off)


def test_solidity_documentation_worked_example():
    """docs.soliditylang.org: struct S { uint16 a; uint16 b; uint256 c; } uint x; mapping(uint => mapping(uint => S)) data;
    data[4][9].c lives at keccak256(uint256(9) . keccak256(uint256(4) . uint256(1))) + 1."""
    want = SP.b32(SP.u256(keccak256(SP.b32(9) + keccak256(SP.b32(4) + SP.b32(1)))) + 1)
    path = StoragePath(0, 1).mapping(4, "uint256").mapping(9, "uint256").field(1)
    assert SP.derive(path)[2] == want
    # a and b share slot + 0: b sits 2 bytes above the low end
    word = bytes(28) + (0xBBBB).to_bytes(2, "big") + (0xAAAA).to_bytes(2, "big")
    assert StoragePath.decode(word, "uint16", 0) == 0xAAAA and StoragePath.decode(word, "uint16", 2) == 0xBBBB


def test_key_encodings():
    a = bytes(range(20))
    assert encode_key(a, "address") == bytes(12) + a
    assert encode_key("0x" + a.hex(), "address") == bytes(12) + a
    assert encode_key(5, "uint256") == SP.b32(5)
    assert encode_key(-1, "int64") == b"\xff" * 32
    assert encode_key(True, "bool") == SP.b32(1)
    assert encode_key(b"ab", "bytes4") == b"ab" + bytes(30)
    assert encode_key("hello", "string") == b"hello" and encode_key(b"\x00\x01", "bytes") == b"\x00\x01"
    with pytest.raises(ValueError):
        encode_key(bytes(31))
    with pytest.raises(ValueError):
        encode_key(b"abcde", "bytes4")


def test_long_string_expansion_and_statuses():
    slot = SP.b32(12)
    for n in (0, 31, 32, 33, 64, 65, A.PATH_MAX_BYTES):
        s = bytes((i * 7 + 1) % 251 for i in range(n))
        st = SP.encode_string(slot, s)
        specs, status, value, _, _ = SP.expand(StoragePath(1, 12).bytes(), lambda x: st.get(x, SP.ZERO))
        assert status == A.PATH_OK and value == s
        assert len(specs) == 1 + (0 if n <= 31 else (n + 31) // 32)
        assert [x for _, x in specs[1:]] == [SP.b32(SP.u256(keccak256(slot)) + j) for j in range(len(specs) - 1)]
    for word, status in ((SP.b32(2 * (A.PATH_MAX_BYTES + 1) + 1), A.PATH_TOO_LONG), (SP.b32(80), A.PATH_BAD_BYTES), (SP.b32(11), A.PATH_BAD_BYTES),
                         (b"\xff" * 32, A.PATH_TOO_LONG)):
        specs, got, value, _, _ = SP.expand(StoragePath(1, 12).bytes(), lambda x: word if x == slot else SP.ZERO)
        assert got == status and value == b"" and len(specs) == 1


def test_contract_catalogue_matches_its_ground_truth():
    c = SP.Contract()
    by = dict(c.paths)
    for i, sid in enumerate(c.subnet_ids):
        _, st, val, _, _ = c.expected(by[f"subnet{i}.name"])
        assert st == A.PATH_OK and val == f"calib-subnet-{i}".encode() * (i * 3 + 1)
        _, st, val, _, off = c.expected(by[f"subnet{i}.owner+nonce"])
        assert StoragePath.decode(val, "uint64", 20) == 1000 + i
    for i in (0, 31, 32, 69):
        specs, st, val, _, off = c.expected(by[f"small[{i}]"])
        assert st == A.PATH_OK and off == i % 32 and StoragePath.decode(val, "uint8", off) == c.small[i] and len(specs) == 2
    assert c.expected(by["small[70]"])[1] == A.PATH_INDEX_OUT_OF_RANGE
    assert c.expected(by[f"nums[{2 ** 40}]"])[1] == A.PATH_INDEX_OUT_OF_RANGE
    assert c.expected(by["nums[4]"])[2] == SP.b32(c.nums[4])
    assert c.expected(by["owners[3]"])[1] == A.PATH_INDEX_OUT_OF_RANGE
    assert c.expected(by["triples[1].2"])[2] == SP.b32(103) and c.expected(by["triples[2]"])[1] == A.PATH_INDEX_OUT_OF_RANGE
    assert c.expected(by["fixed3"])[2] == SP.b32(7) + SP.b32(8) + SP.b32(9)
    for k, s in c.texts.items():
        _, st, val, _, _ = c.expected(by[f"texts[{k}]"])
        assert (st, val) == ((A.PATH_OK, s) if len(s) <= A.PATH_MAX_BYTES else (A.PATH_TOO_LONG, b""))
    assert c.expected(by["texts[100]"])[1] == c.expected(by["texts[101]"])[1] == A.PATH_BAD_BYTES
    assert c.expected(by["empty.bytes"])[1:3] == (A.PATH_OK, b"")


def test_path_structs_have_the_c_layout():
    structs = {"ipcfp_path_step": A.PathStepC, "ipcfp_storage_path": A.StoragePathC, "ipcfp_path_value": A.PathValueC,
               "ipcfp_path_result": A.PathResultC}
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "ipcfp.h"', "int main(void) {"]
    for cname, st in structs.items():
        lines.append(f'printf("{cname} %zu\\n", sizeof({cname}));')
        lines += [f'printf("{cname}.{f} %zu\\n", offsetof({cname}, {f}));' for f, _ in st._fields_]
    consts = ["IPCFP_PATH_MAX_PATHS", "IPCFP_PATH_MAX_STEPS", "IPCFP_PATH_MAX_KEY", "IPCFP_PATH_MAX_WORDS", "IPCFP_PATH_MAX_BYTES"]
    lines += [f'printf("{k} %u\\n", (unsigned){k});' for k in consts] + ["return 0; }"]
    with tempfile.TemporaryDirectory() as td:
        src, exe = os.path.join(td, "l.c"), os.path.join(td, "l")
        open(src, "w").write("\n".join(lines))
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), "-o", exe, src])
        got = dict(l.split() for l in subprocess.check_output([exe], text=True).split("\n") if l)
    for cname, st in structs.items():
        assert int(got[cname]) == C.sizeof(st), cname
        for f, _ in st._fields_:
            assert int(got[f"{cname}.{f}"]) == getattr(st, f).offset, f"{cname}.{f}"
    for k in consts:
        assert int(got[k]) == getattr(A, k[len("IPCFP_"):])
