"""Address resolution on the CPU: the host address codecs (ipcfp_address_parse, ipcfp_address_from_eth), the reference's Ethereum-address
validation, the ctypes layout of the new structs, and the Python restatement of tests/address_trees.py on its own catalogue."""
import ctypes as C
import hashlib
import os
import random
import struct
import subprocess
import tempfile

import pytest

from ipc_filecoin_proofs_b200 import _abi as A
from ipc_filecoin_proofs_b200 import api
from tests import address_trees as T
from tests import oracle_resolve as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# The Filecoin documentation's example of an f410 address and the Ethereum address it wraps
DOC_F410 = "f410f2oekwcmo2pueydmaq53eic2i62crtbeyuzx2gmy"
DOC_ETH = "0xd388ab098ed3e84c0d808776440b48f685198498"


def test_documentation_example_round_trips():
    b = api.address_parse(DOC_F410)
    assert b == bytes.fromhex("040a") + bytes.fromhex(DOC_ETH[2:])
    assert api.address_from_eth(DOC_ETH) == b
    assert api.address_from_eth(bytes.fromhex(DOC_ETH[2:])) == b
    assert T.address_text(b) == DOC_F410


def test_id_addresses_and_networks():
    assert api.address_parse("f01") == b"\x00\x01"
    assert api.address_parse("t01") == b"\x00\x01"
    assert api.address_parse("t" + DOC_F410[1:]) == api.address_parse(DOC_F410)
    for v in T.VALUES + (127, 128, 16383, 16384):
        assert api.address_parse(f"f0{v}") == T.id_addr(v)
    assert api.address_parse("f0+5") == T.id_addr(5)        # Rust's u64::from_str takes a leading '+'
    assert api.address_parse("f0007") == T.id_addr(7)


@pytest.mark.parametrize("kind", T.KINDS)
def test_text_round_trip_of_every_protocol(kind):
    rng = random.Random(str(kind))
    for _ in range(200):
        a = T.random_address(rng, kind)
        assert api.address_parse(T.address_text(a)) == a
        assert api.address_parse(T.address_text(a, "t")) == a


def _refused(text):
    with pytest.raises(A.IpcfpError) as e:
        api.address_parse(text)
    assert e.value.status == A.ERR_INVALID_ARG


def test_malformed_text_is_refused():
    good = T.address_text(b"\x01" + bytes(range(20)))
    flip = good[:5] + ("a" if good[5] != "a" else "b") + good[6:]
    for t in ("", "f", "f0", "x01", "F01", "f5abc", "f9abc", "f0-1", "f0x", "f018446744073709551616", "f0" + "1" * 21,
              flip, good.upper(), good + "=", good[:-1] + "1", good[:-1],
              "f1" + T.b32(bytes(19) + bytes(4)),
              "f3" + T.b32(bytes(47) + bytes(4)), "f2" + T.b32(bytes(21) + bytes(4)), "f1" + T.b32(bytes(3)),
              "f410" + T.b32(bytes(24)), "f4f" + T.b32(bytes(24)), "f418446744073709551616f" + T.b32(bytes(24)),
              "f410f" + T.b32(bytes(55) + _checksum(b"\x04\x0a" + bytes(55)))):
        _refused(t)
    # the 54-byte subaddress is the longest accepted
    a = T.delegated(10, bytes(range(54)))
    assert api.address_parse(T.address_text(a)) == a


def _checksum(b):
    return hashlib.blake2b(b, digest_size=4).digest()


def test_trailing_base32_bits_must_be_zero():
    a = b"\x01" + bytes(range(20))
    t = T.address_text(a)          # 24 bytes = 192 bits → 39 characters, the last carrying 3 padding bits
    last = T.B32.index(t[-1])
    assert last & 7 == 0
    _refused(t[:-1] + T.B32[last | 1])


def test_eth_conversion_and_masked_ids():
    for v in T.VALUES:
        assert api.address_from_eth(T.eth_masked_id(v)) == T.id_addr(v)
    near = b"\xff" + bytes(10) + b"\x01" + bytes(8)          # not masked: byte 11 is not zero
    assert api.address_from_eth(near) == T.delegated(10, near)
    assert api.address_from_eth(b"\xfe" + bytes(19)) == T.delegated(10, b"\xfe" + bytes(19))


def test_reference_eth_hex_validation():
    h = DOC_ETH[2:]
    assert api.address_from_eth("0x0x" + h) == api.address_from_eth(h)      # trim_start_matches strips every leading "0x"
    with pytest.raises(ValueError, match=r"^Invalid hex in Ethereum address: Odd number of digits$"):
        api.address_from_eth("0x" + h[:-1])
    with pytest.raises(ValueError, match=r"^Invalid hex in Ethereum address: Invalid character 'z' at position 4$"):
        api.address_from_eth("0x" + h[:4] + "z" + h[5:])
    with pytest.raises(ValueError, match=r"^Invalid Ethereum address length: expected 20 bytes, got 19$"):
        api.address_from_eth("0x" + h[:-2])
    with pytest.raises(ValueError, match=r"^Invalid Ethereum address length: expected 20 bytes, got 0$"):
        api.address_from_eth("0x")


def test_new_structs_match_the_c_header():
    structs = {"ipcfp_address": A.AddressC, "ipcfp_resolve_result": A.ResolveResultC}
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
    for cname, st in structs.items():
        assert int(got[cname]) == C.sizeof(st), cname
        for fname, _ in st._fields_:
            assert int(got[f"{cname}.{fname}"]) == getattr(st, fname).offset, f"{cname}.{fname}"


def test_restatement_on_its_catalogue():
    """The builder's ground truth holds under the restatement, and every case lands where it was built to land."""
    blocks, cases, _ = T.world()
    assert len(cases) == 28
    by = {c.name: c for c in cases}
    for c in cases:
        ids, st, init, missing, read = T.resolve(blocks, c.root, c.addrs)
        assert missing == []
        for a, i, s in zip(c.addrs, ids, st):
            if c.truth is not None and a in c.truth:
                assert (s, i) == (A.OK, c.truth[a]), c.name
            elif a[:1] == b"\x00" and T.address_valid(a):
                assert (s, i) == (A.OK, T._leb_read(a[1:])[0]), c.name
    assert T.resolve(blocks, by["init-absent"].root, [])[2] == A.ERR_ACTOR_NOT_FOUND
    for n in ("init-4-tuple", "init-2-tuple", "init-trailing", "init-map-not-link", "init-next-id-negative", "init-name-bytes",
              "init-not-array", "state-root-version-6", "state-root-4-tuple"):
        assert T.resolve(blocks, by[n].root, [])[2] == A.ERR_DECODE, n
    assert T.resolve(blocks, by["chain-52"].root, by["chain-52"].addrs)[1][0] == A.ERR_DECODE
    assert T.resolve(blocks, by["chain-51"].root, by["chain-51"].addrs)[:2] == ([2 ** 64 - 1, 0], [A.OK, A.ERR_ACTOR_NOT_FOUND])
    for n in ("value-negative", "value-bytes", "value-nonminimal", "value-u64-nonminimal", "value-text", "value-null"):
        assert T.resolve(blocks, by[n].root, by[n].addrs)[1] == [A.ERR_DECODE] * 2, n
    st = T.resolve(blocks, by["ids-and-invalid"].root, by["ids-and-invalid"].addrs)[1]
    assert st.count(A.ERR_INVALID_ARG) == 11
    # a dropped block is reported missing, once, by every walk that needs it
    c = by["map-200"]
    _, _, _, _, read = T.resolve(blocks, c.root, c.addrs)
    for cid in read:
        part = {k: v for k, v in blocks.items() if k != cid}
        _, st, init, missing, _ = T.resolve(part, c.root, c.addrs)
        assert missing == [cid]
        assert A.ERR_MISSING_BLOCK in st or init == A.ERR_MISSING_BLOCK


def _walks(addrs):
    """The addresses the call leaves to the device: valid and not protocol 0."""
    return [a for a in addrs if T.address_valid(a) and a[0] != 0]


@pytest.mark.parametrize("sanitize", [False, True])
def test_per_item_code_on_the_cpu_matches_the_restatement(tmp_path, sanitize):
    """csrc/resolve_items.cuh compiled for the host and driven as csrc/resolve.cu drives it (tests/host_fuzz/emu_resolve.cu), with the
    fast and the strict HAMT node decoder: every case of the catalogue but the 100 000-entry map, every block of three paths dropped in
    turn, and 64 seeded truncations and bit flips give the C++ oracle's (tests/oracle_resolve.cpp) init status, statuses, IDs, missing
    CIDs and read set, which equal the restatement's. Under
    AddressSanitizer + UBSan (sanitize=True) the walks stay inside the padded block buffers."""
    from tests.test_host_fuzz import _harness
    blocks, cases, _ = T.world()
    by = {c.name: c for c in cases}
    order = list(blocks)
    index = {c: i for i, c in enumerate(order)}
    runs = []   # (root, addrs, drop, {cid: new bytes})
    for c in cases:
        if c.name != "map-100000":
            runs.append((c.root, _walks(c.addrs), None, {}))
    for name in ("map-200", "chain-51", "bucket-3"):
        c = by[name]
        for cid in T.resolve(blocks, c.root, c.addrs)[4]:
            runs.append((c.root, _walks(c.addrs), cid, {}))
    c = by["map-200"]
    for _, repl in T.mutations(blocks, c.root, random.Random(31), 64):
        runs.append((c.root, _walks(c.addrs), None, repl))
    out = [struct.pack("<Q", len(order))]
    for cid in order:
        out += [cid, struct.pack("<I", len(blocks[cid])), blocks[cid]]
    out.append(struct.pack("<I", 2 * len(runs)))
    for strict in (0, 1):
        for root, addrs, drop, repl in runs:
            out += [root, struct.pack("<BI", strict, len(addrs))] + [bytes([len(a)]) + a for a in addrs]
            out.append(struct.pack("<I", 0 if drop is None else 1) + (b"" if drop is None else struct.pack("<Q", index[drop])))
            out.append(struct.pack("<I", len(repl)))
            for cid, b in repl.items():
                out += [struct.pack("<QI", index[cid], len(b)), b]
    path = tmp_path / "cases.bin"
    path.write_bytes(b"".join(out))
    exe, env = _harness("emu_resolve", with_synth=False, sanitize=sanitize)
    res = subprocess.run([exe, str(path)], capture_output=True, text=True, env=env, timeout=1800)
    assert res.returncode == 0, res.stderr[-3000:]
    got = res.stdout.split("end\n")
    assert len(got) == 2 * len(runs) + 1 and got[-1] == ""
    oracle = O.Oracle(blocks)
    expected = []
    for root, addrs, drop, repl in runs:
        part = {c: repl.get(c, b) for c, b in blocks.items() if c != drop}
        exp = (oracle if drop is None and not repl else O.Oracle(part)).resolve(root, addrs)
        assert exp == T.resolve(part, root, addrs)
        expected.append(exp)
    for k, (ids, st, init, missing, read) in enumerate(expected * 2):
        addrs = runs[k % len(runs)][1]
        if init != A.OK:
            st, ids = [init] * len(addrs), [0] * len(addrs)
        want = [f"case {k} init {init}"] + [f"addr {s} {i}" for s, i in zip(st, ids)]
        want += [f"missing {m.hex()}" for m in missing] + [f"witness {r.hex()}" for r in read]
        assert got[k].splitlines() == want, k


@pytest.mark.parametrize("sanitize", [False, True])
def test_address_map_nodes_fast_strict_and_oracle_agree(sanitize):
    """tests/host_fuzz/fuzz_hamt_u64.cu: random address_map nodes (values at every head size, some not minimal unsigned integers, half of
    the nodes edited) through the strict and the fast HAMT node decoder with HV_U64 and through the C++ oracle's node decoder: the fast
    decoder accepts only what the strict one accepts, with the same hit, and takes every unedited node of minimal values; strict and
    oracle agree on every node. Built with tests/oracle_resolve.cpp, which includes oracle/oracle.cpp (so that file is not linked again)."""
    import shutil
    from tests.test_host_fuzz import SAN_ENV, SANITIZE
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    build = os.path.join(ROOT, "tests", "host_fuzz", "_build")
    os.makedirs(build, exist_ok=True)
    exe = os.path.join(build, "fuzz_hamt_u64" + ("_san" if sanitize else ""))
    cmd = [nvcc, "-std=c++17", "-O1" if sanitize else "-O2", "-Wno-deprecated-gpu-targets", "-diag-suppress", "20091", "-o", exe,
           os.path.join(ROOT, "tests", "host_fuzz", "fuzz_hamt_u64.cu"), os.path.join(ROOT, "tests", "oracle_resolve.cpp")]
    cc = subprocess.run(cmd + (SANITIZE if sanitize else []) + ["-lpthread"], cwd=ROOT, capture_output=True, text=True)
    if cc.returncode != 0 and sanitize and "sanitize" in cc.stderr:
        pytest.skip("this host compiler has no sanitizer runtime")
    assert cc.returncode == 0, cc.stderr[-3000:]
    for seed in ("7", "20261017"):
        out = subprocess.run([exe, "100000" if sanitize else "300000", seed], capture_output=True, text=True,
                             env=dict(os.environ, **SAN_ENV) if sanitize else None, timeout=1200)
        assert out.returncode == 0, out.stderr[-2000:]
        line = out.stdout.strip()
        assert line.startswith("ok: "), line
        decoded, fast = int(line.split("(")[1].split()[0]), int(line.split("; ")[-1].split()[0])
        found = int(line.split("decoded: ")[1].split()[0])
        assert decoded > int(line.split()[1]) // 4 and fast == decoded and found > decoded // 20, line
