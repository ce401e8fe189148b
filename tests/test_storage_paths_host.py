"""The per-path code of the storage-path calls (csrc/storage_path_items.cuh) compiled for the host (tests/host_fuzz/emu_storage_paths.cu)
against the Python restatement of Solidity's layout rules (tests/storage_paths.py): slot derivation, expansion, statuses and values on
thousands of seeded random paths and on every edge — u256 carries out of the top byte, indices and offsets at 2^64 - 1, elem_slots up
to 2^32 - 1, every packed element size, mapping keys of every length around the 136-byte Keccak block edges up to IPCFP_PATH_MAX_KEY,
and bytes / string headers of every form (short, long, BAD_BYTES both ways, TOO_LONG, lengths at the cap and one past it). The program
also checks keccak_key_slot against hashes.cuh's keccak256 at every key length. Under `make sanitize` it runs with ASan + UBSan."""
import os
import random
import subprocess
import tempfile

import pytest

from ipc_filecoin_proofs_b200 import _abi as A
from ipc_filecoin_proofs_b200.api import StoragePath
from tests import storage_paths as SP
from tests.test_host_fuzz import _harness

KEY_EDGES = (0, 1, 31, 32, 33, 103, 104, 105, 135, 136, 137, 239, 240, 241, 375, 376, 377, A.PATH_MAX_KEY - 1, A.PATH_MAX_KEY)
U64_EDGES = (0, 1, 2, 31, 32, 33, 2 ** 32 - 1, 2 ** 32, 2 ** 63, 2 ** 64 - 1)


def _u256(rng):
    return rng.choice([rng.randrange(16), SP.M - 1 - rng.randrange(16), rng.randrange(SP.M), (1 << rng.randrange(256)) - rng.randrange(3)]) % SP.M


def _step(rng):
    op = rng.choice((A.PATH_MAPPING, A.PATH_MAPPING, A.PATH_ARRAY, A.PATH_STATIC, A.PATH_FIELD))
    if op == A.PATH_MAPPING:
        n = rng.choice(KEY_EDGES + (32, 32, 20, rng.randrange(A.PATH_MAX_KEY + 1)))
        return (op, rng.randbytes(n), 0, 0, 0)
    index = rng.choice(U64_EDGES + (rng.randrange(100), rng.randrange(2 ** 64)))
    if op == A.PATH_FIELD:
        return (op, b"", index, 0, 0)
    es = rng.choice((1, 1, 1, 2, 3, 7, 2 ** 32 - 1))
    eb = rng.choice((0, 0, 1, 2, 3, 8, 16, 20, 31, 32))
    return (op, b"", index, es, eb)


def _header(rng):
    """a bytes / string header word of every form"""
    kind = rng.randrange(7)
    if kind == 0:
        return bytes(31) + bytes([2 * rng.randrange(32)])                        # short
    if kind == 1:
        return rng.randbytes(31) + bytes([2 * rng.randrange(32, 128)])           # short, BAD_BYTES
    if kind == 2:
        return SP.b32(2 * rng.choice((32, 33, 63, 64, 65, rng.randrange(32, A.PATH_MAX_BYTES + 1), A.PATH_MAX_BYTES)) + 1)   # long
    if kind == 3:
        return SP.b32(2 * rng.randrange(32) + 1)                                 # long, BAD_BYTES
    if kind == 4:
        return SP.b32(2 * rng.choice((A.PATH_MAX_BYTES + 1, rng.randrange(A.PATH_MAX_BYTES + 1, 2 ** 64), rng.randrange(SP.M // 2))) + 1)   # TOO_LONG
    if kind == 5:
        return rng.randbytes(32)
    return bytes(32)


def _case(rng, storage):
    """one random path; its words go into storage"""
    steps = tuple(_step(rng) for _ in range(rng.choice((0, 1, 2, 3, 4, 6, A.PATH_MAX_STEPS))))
    if rng.random() < 0.5:
        p = StoragePath(rng.randrange(2 ** 64), _u256(rng), steps, A.PATH_BYTES, 0)
    else:
        p = StoragePath(rng.randrange(2 ** 64), _u256(rng), steps, A.PATH_WORDS, rng.choice((1, 1, 2, 3, A.PATH_MAX_WORDS)))
    lengths, values, slot, _ = SP.derive(p)
    arrays = [s for s in steps if s[0] == A.PATH_ARRAY]
    for ls, st in zip(lengths, arrays):
        if rng.random() < 0.8:
            storage[ls] = rng.choice((SP.b32(st[2] + 1 + rng.randrange(5)), SP.b32(st[2]), SP.b32(max(st[2] - 1, 0)), rng.randbytes(32)))
    if p.kind == A.PATH_WORDS:
        for v in values:
            if rng.random() < 0.7:
                storage[v] = rng.randbytes(32)
    else:
        storage[slot] = _header(rng)
        base = SP.u256(SP.keccak256(slot))
        for j in range(A.PATH_MAX_BYTES // 32 + 1):
            if rng.random() < 0.9:
                storage[SP.b32(base + j)] = rng.randbytes(32)
    return p


def _run(exe, env, paths, storage):
    lines = [str(len(storage))] + [f"{s.hex()} {w.hex()}" for s, w in storage.items()] + [str(len(paths))]
    for p in paths:
        lines.append(f"{p.actor_id} {p.base_slot.hex()} {p.kind} {p.n_words} {len(p.steps)}")
        lines += [f"{op} {len(k)} {k.hex() or '-'} {i} {es} {eb}" for op, k, i, es, eb in p.steps]
    with tempfile.TemporaryDirectory() as td:
        path = os.path.join(td, "in.txt")
        open(path, "w").write("\n".join(lines) + "\n")
        out = subprocess.run([exe, path], capture_output=True, text=True, env=env)
    assert out.returncode == 0, out.stderr[-3000:]
    assert "runtime error" not in out.stderr and "AddressSanitizer" not in out.stderr, out.stderr[-3000:]
    return out.stdout.splitlines()


def _compare(paths, storage, got):
    read = lambda s: storage.get(bytes(s), SP.ZERO)
    assert len(got) == len(paths)
    statuses = set()
    for p, line in zip(paths, got):
        f = line.split()
        specs, status, value, slot, off = SP.expand(p, read)
        n = int(f[3])
        want = [str(status), slot.hex(), str(off), str(len(specs))] + [s.hex() for _, s in specs] + [value.hex() or "-"]
        assert f == want, (p.steps, p.kind, p.n_words)
        assert n == len(specs)
        statuses.add(status)
    return statuses


def _edges():
    """hand-picked paths: carries out of the top byte, the caps, every header form on one slot each"""
    top = SP.M - 1
    P = lambda base, *steps, kind=A.PATH_WORDS, n=1: StoragePath(7, base, steps, kind, n)
    paths = [P(top, (A.PATH_FIELD, b"", 1, 0, 0)), P(top, (A.PATH_FIELD, b"", 2 ** 64 - 1, 0, 0), n=A.PATH_MAX_WORDS),
             P(top - 5, (A.PATH_STATIC, b"", 2 ** 64 - 1, 2 ** 32 - 1, 0)), P(0, (A.PATH_STATIC, b"", 2 ** 64 - 1, 1, 1)),
             P(3, (A.PATH_ARRAY, b"", 2 ** 64 - 1, 2 ** 32 - 1, 0), (A.PATH_FIELD, b"", 2 ** 64 - 1, 0, 0))]
    paths += [P(5, (A.PATH_MAPPING, (bytes(range(256)) * 4)[:n], 0, 0, 0)) for n in KEY_EDGES]
    paths += [P(k, (A.PATH_ARRAY, b"", i, 1, eb)) for k, (i, eb) in enumerate((i, eb) for eb in range(1, 33) for i in (0, 31, 32, 63))]
    paths += [P(9000 + k, kind=A.PATH_BYTES) for k in range(12)]
    return paths


def _edge_storage(paths):
    storage = {}
    hdr = [bytes(32), bytes(31) + b"\x3e", bytes(31) + b"\x40", SP.b32(2 * 32 + 1), SP.b32(2 * 31 + 1), SP.b32(1),
           SP.b32(2 * A.PATH_MAX_BYTES + 1), SP.b32(2 * (A.PATH_MAX_BYTES + 1) + 1), b"\xff" * 32, SP.b32(2 * 33 + 1),
           SP.b32(2 * 65 + 1), b"\xff" * 31 + b"\xfe"]
    for k, p in enumerate(paths[-12:]):
        storage[p.base_slot] = hdr[k]
        base = SP.u256(SP.keccak256(p.base_slot))
        for j in range(A.PATH_MAX_BYTES // 32 + 1):
            storage[SP.b32(base + j)] = bytes([j % 256]) * 32
    for p in paths[:-12]:
        for ls in SP.derive(p)[0]:
            storage[ls] = SP.b32(2 ** 64 - 1)
    return storage


def _check(sanitize, n, seed):
    exe, env = _harness("emu_storage_paths", with_synth=False, sanitize=sanitize)
    rng = random.Random(seed)
    storage = {}
    paths = [_case(rng, storage) for _ in range(n)]
    statuses = _compare(paths, storage, _run(exe, env, paths, storage))
    assert statuses == {A.PATH_OK, A.PATH_INDEX_OUT_OF_RANGE, A.PATH_BAD_BYTES, A.PATH_TOO_LONG}, statuses
    edges = _edges()
    es = _edge_storage(edges)
    statuses = _compare(edges, es, _run(exe, env, edges, es))
    assert statuses == {A.PATH_OK, A.PATH_INDEX_OUT_OF_RANGE, A.PATH_BAD_BYTES, A.PATH_TOO_LONG}, statuses


def test_per_path_code_on_the_cpu_matches_the_restatement():
    _check(None, 2000, 20261018)


def test_per_path_code_under_sanitizers():
    _check(True, 300, 7)
