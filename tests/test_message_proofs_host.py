"""Message proofs without a GPU: the ctypes and Rust layouts of ipcfp_message_proof / ipcfp_message_result against include/ipcfp.h, the
worlds and decode rules of tests/message_receipts.py, and the per-request code (csrc/message_proof_items.cuh) compiled for the host
(tests/host_fuzz/emu_message_proofs.cu, also under AddressSanitizer + UBSan with `make sanitize`) against that module's restatement: every
world with and without the body, every block of the read sets dropped in turn, and seeded truncations and bit flips of receipts-AMT
nodes and message blocks."""
import ctypes as C
import functools
import os
import random
import re
import struct
import subprocess
import tempfile

import pytest

from ipc_filecoin_proofs_b200 import _abi as A
from tests import message_amts as MA
from tests import message_receipts as MR
from tests.storage_trees import cbytes, head

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WORLDS = {"min": dict(seed=1), "tall": dict(seed=2, height=21), "h0": dict(seed=3, short=25, height=0),
          "no_events": dict(seed=4, short=3, empty_events=True)}


@functools.lru_cache(maxsize=None)
def _world(name):
    return MR.world(MA.base_tipset(), **WORLDS[name])


def test_layouts_match_the_c_header():
    structs = {"ipcfp_message_proof": A.MessageProofC, "ipcfp_message_result": A.MessageResultC}
    cname_of = {"from_": "from"}
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "ipcfp.h"', "int main(void) {"]
    for cname, st in structs.items():
        lines.append(f'printf("{cname} %zu\\n", sizeof({cname}));')
        for fname, _ in st._fields_:
            f = cname_of.get(fname, fname)
            lines.append(f'printf("{cname}.{fname} %zu\\n", offsetof({cname}, {f}));')
    lines += ["return 0; }"]
    with tempfile.TemporaryDirectory() as td:
        src, exe = os.path.join(td, "layout.c"), os.path.join(td, "layout")
        open(src, "w").write("\n".join(lines))
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), "-o", exe, src])
        got = dict(l.split() for l in subprocess.check_output([exe], text=True).strip().splitlines())
    assert int(got["ipcfp_message_proof"]) == C.sizeof(A.MessageProofC) == 400
    for cname, st in structs.items():
        assert int(got[cname]) == C.sizeof(st), cname
        for fname, _ in st._fields_:
            assert int(got[f"{cname}.{fname}"]) == getattr(st, fname).offset, f"{cname}.{fname}"
    # the offsets the header's comment documents
    hdr = open(os.path.join(ROOT, "include", "ipcfp.h")).read()
    doc = hdr[hdr.index("400 bytes, 8-byte aligned; every byte not named by a field is zero. Offsets: exec_index"):]
    doc = doc[:doc.index("*/")]
    for name, off in re.findall(r"(\w+) (\d+)[,.]", doc.replace("\n *", " ")):
        if name != "bytes":
            assert getattr(A.MessageProofC, cname_of.get(name, name) if name != "from" else "from_").offset == int(off), name
    rs = open(os.path.join(ROOT, "integration", "rust", "ipcfp-sys", "src", "lib.rs")).read()
    for cname, st in structs.items():
        body = re.search(r"pub struct " + cname + r" \{(.*?)\}", rs, re.S).group(1)
        rust = re.findall(r"pub (\w+):", body)
        assert rust == [cname_of.get(f, f) for f, _ in st._fields_], cname


@pytest.mark.parametrize("name", list(WORLDS))
def test_worlds_restate_their_own_truth(name):
    w = _world(name)
    proofs, wit = MR.prove(w.blocks, w.ts, w.requests(), True)
    for p in proofs:
        if p["message_cid"] in w.never:
            assert p["status"] == MR.NOT_EXECUTED and p["exec_index"] is None
            continue
        e = p["exec_index"]
        assert w.exec[e] == p["message_cid"]
        if e in w.receipts:
            assert p["status"] == MR.EXECUTED
            assert (p["exit_code"], p["return_data"], p["gas_used"], p["events_root"]) == w.receipts[e]
        else:
            assert p["status"] == MR.NO_RECEIPT
        assert p["has_body"] and p["message_cid"] in wit
    assert w.ramt.height == WORLDS[name].get("height", w.ramt.height)
    ret_lens = {len(r[1]) for r in w.receipts.values()}
    assert name == "h0" or set(MR.EDGE_LENGTHS) <= ret_lens | {len(p.get("params", b"")) for p in proofs}


def test_message_decode_rules():
    rng = random.Random(3)
    to, frm = MR.address(1, rng), MR.address(4, rng)
    ok = MR.message(0, to, frm, 1, -5, 2, 3, 4, 5, b"xy")
    assert MR.decode_message(ok)["value"] == -5
    for k in (1, 2, 3):
        assert MR.decode_message(MR.signed(ok, bytes([k]) + b"s"))["sig_type"] == k
    bad = [MR.signed(ok, b""), MR.signed(ok, b"\x00s"), MR.signed(ok, b"\x04s"), ok + b"\x00", head(4, 3) + ok + cbytes(b"\x01") + b"\xf6",
           ok.replace(head(0, 1) + cbytes(MR.token(-5)), head(1, 0) + cbytes(MR.token(-5)), 1),                 # negative sequence
           MR.message(0, b"\x05" + bytes(20), frm, 1, 0, 2, 3, 4, 5, b""),                                       # unknown protocol
           MR.message(0, to, frm, 1, 0, 2, 3, 4, 5, b"").replace(cbytes(b""), cbytes(b"\x02\x01"), 1)]          # sign byte 2
    for b in bad:
        with pytest.raises(Exception):
            MR.decode_message(b)


# ------------------------------------------------------------------ the per-request code on the CPU
def _runs():
    """(world, with_body, requests, drop CID or None, {cid: new bytes}) per case"""
    runs = []
    for name in WORLDS:
        w = _world(name)
        runs += [(w, False, w.requests(), None, {}), (w, True, w.requests(), None, {})]
    for name in ("min", "tall"):
        w = _world(name)
        base = MR.read_set(w.blocks, w.ts, [])
        for c in sorted(MR.read_set(w.blocks, w.ts, w.requests(), True) - base):
            runs.append((w, True, list(reversed(w.requests())), c, {}))
    rng = random.Random(29)
    for name in ("min", "tall", "h0"):
        w = _world(name)
        targets = sorted(set(w.ramt.nodes.values()) | set(w.exec))
        for i in range(60):
            c = targets[rng.randrange(len(targets))]
            b = bytearray(w.blocks[c])
            if i % 2:
                b[rng.randrange(len(b))] ^= 1 << rng.randrange(8)
            else:
                b = b[:rng.randrange(len(b))]
            runs.append((w, True, w.requests(), None, {c: bytes(b)}))
    return runs


def _expected(w, with_body, reqs, drop, repl):
    """(generator outcome, plan or None where it is not restated)"""
    part = {c: repl.get(c, b) for c, b in w.blocks.items() if c != drop}
    plan = None
    if not repl:   # dropped from a complete read set: every path that reaches it names it, and nothing else is missing
        plan = [drop] if drop is not None and drop in MR.read_set(w.blocks, w.ts, reqs, with_body) else []
    try:
        proofs, wit = MR.prove(part, w.ts, reqs, with_body)
    except MR.Fault as f:
        return ("fail", f.status, f.index), plan
    return ("ok", proofs, wit - MR.read_set(part, w.ts, [])), plan


def _case_file(path, runs):
    blocks = {}
    for w, *_ in runs:
        for c, b in w.blocks.items():
            blocks.setdefault(c, b)
    index = {c: i for i, c in enumerate(blocks)}
    with open(path, "wb") as f:
        f.write(struct.pack("<Q", len(blocks)))
        for c, b in blocks.items():
            f.write(c + struct.pack("<I", len(b)) + b)
        f.write(struct.pack("<I", len(runs)))
        for w, with_body, reqs, drop, repl in runs:
            pos = {c: i for i, c in enumerate(w.exec)}
            f.write(bytes(w.ts.receipts_root) + bytes([with_body]) + struct.pack("<I", len(reqs)))
            for c in reqs:
                f.write(bytes(c) + struct.pack("<Q", pos.get(bytes(c), MR.U64)))
            # blocks of other worlds are dropped too: each case sees its own world's store
            own = set(w.blocks)
            dropped = [index[c] for c in blocks if c not in own or c == drop]
            f.write(struct.pack("<I", len(dropped)) + b"".join(struct.pack("<Q", i) for i in dropped))
            f.write(struct.pack("<I", len(repl)))
            for c, b in repl.items():
                f.write(struct.pack("<QI", index[c], len(b)) + b)


def _parse(out):
    cases, cur = [], []
    for line in out.splitlines():
        if line == "end":
            cases.append(cur)
            cur = []
        else:
            cur.append(line)
    return cases


def _proof_of(line):
    _, rec, ret, par = line.split(" ")
    q = A.MessageProofC.from_buffer_copy(bytes.fromhex(rec))
    p = MR.proof_dict(A.message_proof_from_c(q))
    got_ret = b"" if ret == "-" else bytes.fromhex(ret[:-1])
    got_par = b"" if par == "-" else bytes.fromhex(par[:-1])
    p["return_data"] = got_ret
    if p["has_body"]:
        p["params"] = got_par
    return p


@pytest.mark.parametrize("sanitize", [False, True])
def test_per_request_code_on_the_cpu_matches_the_restatement(tmp_path, sanitize):
    from tests.test_host_fuzz import _harness
    if sanitize and not os.environ.get("IPCFP_HOST_FUZZ_SANITIZE"):
        pytest.skip("AddressSanitizer + UBSan run with `make sanitize`")
    exe, env = _harness("emu_message_proofs", with_synth=False, sanitize=sanitize)
    runs = _runs()
    cf = tmp_path / "cases.bin"
    _case_file(cf, runs)
    out = subprocess.run([exe, str(cf)], capture_output=True, text=True, env=env)
    assert out.returncode == 0, out.stderr[-3000:]
    got = _parse(out.stdout)
    assert len(got) == len(runs)
    n_fail = n_plan = 0
    for k, (run, lines) in enumerate(zip(runs, got)):
        exp, plan = _expected(*run)
        got_plan = [bytes.fromhex(x) for x in [l for l in lines if l.startswith("plan")][0].split()[1:]]
        if plan is not None:
            assert got_plan == sorted(plan), k
            n_plan += bool(plan)
        if exp[0] == "fail":
            n_fail += 1
            assert lines[0] == f"fail {exp[1]} {exp[2]}" and not any(l.startswith(("proof", "verify")) for l in lines), (k, lines, exp)
            continue
        proofs = [_proof_of(l) for l in lines if l.startswith("proof ")]
        assert proofs == exp[1], k
        marked = [l for l in lines if l.startswith("marked")][0].split()[1:]
        assert {bytes.fromhex(x) for x in marked} == exp[2], k
        assert [l for l in lines if l.startswith("verify")] == ["verify" + " 1" * len(proofs)], k
    assert n_fail >= 60 and n_plan >= 20


def test_the_two_restatements_agree_on_every_world_and_fault_case():
    """tests/message_receipts.py and tests/oracle_receipts.cpp: the same proofs, witness and data blob, or the same (status, index), on
    every run of the CPU campaign above."""
    n_fail = 0
    for w, with_body, reqs, drop, repl in _runs():
        part = {c: repl.get(c, b) for c, b in w.blocks.items() if c != drop}
        try:
            proofs, wit = MR.prove(part, w.ts, reqs, with_body)
        except MR.Fault as f:
            with pytest.raises(MR.Fault) as e:
                MR.cpp_prove(part, w.ts, reqs, with_body)
            assert (e.value.status, e.value.index) == (f.status, f.index)
            n_fail += 1
            continue
        got, got_wit, blob = MR.cpp_prove(part, w.ts, reqs, with_body)
        assert got == proofs and got_wit == wit
        assert blob == b"".join(p["return_data"] + p.get("params", b"") for p in proofs)
    assert n_fail >= 60
