"""The per-proof code of actor proofs (csrc/actor_items.cuh) with its planner and verifier items, compiled for the host
(tests/host_fuzz/emu_actor.cu) and run against the restatement of tests/actor_trees.py, also under AddressSanitizer + UBSan (`make
sanitize`): every tree, with and without code; every block of two proofs' read sets dropped in turn; seeded truncations and bit flips of
the blocks the walks read."""
import random
import struct
import subprocess

import pytest

from ipc_filecoin_proofs_b200 import _abi as A
from oracle.pyoracle import cid_sort_key
from tests import actor_trees as AT

SKIP_LARGE = {"actors-100000"}   # the 100 000-actor tree runs on the GPU; its walks are those of actors-1000, one level deeper


def _runs(blocks, trees):
    """(tree, with_code, drop CID or None, {cid: new bytes}) per case"""
    runs = []
    for t in trees.values():
        if t.name not in SKIP_LARGE:
            runs += [(t, False, None, {}), (t, True, None, {})]
    for name in ("main-code", "deep-init"):
        t = trees[name]
        for cid in AT.read_set(blocks, t.child, t.root, t.addrs, AT.EVM_SETS[t.evm], True):
            if cid != t.child:
                runs.append((t, True, cid, {}))
    rng = random.Random(41)
    for name in ("main-code", "actors-1000", "deep"):
        t = trees[name]
        read = [c for c in AT.read_set(blocks, t.child, t.root, t.addrs, AT.EVM_SETS[t.evm], True) if c != t.child]
        for i in range(48):
            c = read[rng.randrange(len(read))]
            b = bytearray(blocks[c])
            if i % 2:
                b[rng.randrange(len(b))] ^= 1 << rng.randrange(8)
            else:
                b = b[:rng.randrange(len(b))]
            runs.append((t, True, None, {c: bytes(b)}))
    return runs


def _expected(blocks, t, with_code, drop, repl):
    part = {c: repl.get(c, b) for c, b in blocks.items() if c != drop}
    evm = AT.EVM_SETS[t.evm]
    try:
        proofs, lists, _ = AT.prove(part, t.child, t.root, t.addrs, evm, with_code)
        gen = ("ok", list(zip(proofs, lists)))
    except AT.Failure as f:
        gen = ("fail", (f.status, f.index))
    plan = []
    if drop is not None:   # dropped from a complete read set: every walk that reaches it names it, and nothing else is missing
        plan = [drop] if drop in AT.prove(blocks, t.child, t.root, t.addrs, evm, with_code)[2] else []
    return gen, plan


@pytest.mark.parametrize("sanitize", [False, True])
def test_per_proof_code_on_the_cpu_matches_the_restatement(tmp_path, ts3_small, sanitize):
    from tests.test_host_fuzz import _harness
    blocks, trees, _, _ = AT.world(ts3_small)
    runs = _runs(blocks, trees)
    order = list(blocks)
    index = {c: i for i, c in enumerate(order)}
    out = [struct.pack("<Q", len(order))]
    for cid in order:
        out += [cid, struct.pack("<I", len(blocks[cid])), blocks[cid]]
    out.append(struct.pack("<I", len(runs)))
    for t, with_code, drop, repl in runs:
        evm = AT.EVM_SETS[t.evm]
        out += [t.child, t.root, struct.pack("<BBI", int(with_code), 0, len(evm))] + list(evm)
        out.append(struct.pack("<I", len(t.addrs)))
        out += [bytes([len(a)]) + a for a in t.addrs]
        out.append(struct.pack("<I", 0 if drop is None else 1) + (b"" if drop is None else struct.pack("<Q", index[drop])))
        out.append(struct.pack("<I", len(repl)))
        for cid, b in repl.items():
            out += [struct.pack("<QI", index[cid], len(b)), b]
    path = tmp_path / "cases.bin"
    path.write_bytes(b"".join(out))
    exe, env = _harness("emu_actor", with_synth=False, sanitize=sanitize)
    res = subprocess.run([exe, str(path)], capture_output=True, text=True, env=env, timeout=1800)
    assert res.returncode == 0, res.stderr[-3000:]
    got = res.stdout.split("end\n")
    assert len(got) == len(runs) + 1 and got[-1] == ""
    n_fail = 0
    for k, (t, with_code, drop, repl) in enumerate(runs):
        (kind, exp), plan = _expected(blocks, t, with_code, drop, repl)
        lines = got[k].splitlines()
        what = (k, t.name, with_code, drop and drop.hex(), [c.hex() for c in repl])
        if kind == "fail":
            n_fail += 1
            assert lines[0] == f"fail {exp[0]} {exp[1]}", what
            rest = lines[1:]
        else:
            body = lines[:2 * len(exp)]
            for (p, lst), (pl, ll) in zip(exp, zip(body[0::2], body[1::2])):
                _, rec_hex, code_hex = pl.split(" ")
                rec = A.ActorProofC.from_buffer_copy(bytes.fromhex(rec_hex))
                code = b"" if code_hex == "-" else bytes.fromhex(code_hex)
                rec.code_off = 0
                assert vars(A.actor_proof_from_c(rec, code)) == p, what
                assert sorted((bytes.fromhex(x) for x in ll.split()[1:]), key=cid_sort_key) == lst, what
            rest = lines[2 * len(exp):]
        assert rest[0].split()[0] == "plan", what
        if not repl and (drop is not None or kind == "ok"):
            assert [bytes.fromhex(x) for x in rest[0].split()[1:]] == plan, what
        if kind == "ok" and t.addrs:
            assert rest[1] == "verify" + " 1" * len(t.addrs), what
    assert n_fail >= 20
