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
from tests import storage_paths as SP
from tests.test_host_fuzz import _harness


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


def _check(sanitize, n, seed):
    exe, env = _harness("emu_storage_paths", with_synth=False, sanitize=sanitize)
    rng = random.Random(seed)
    storage = {}
    paths = [SP.case(rng, storage) for _ in range(n)]
    statuses = _compare(paths, storage, _run(exe, env, paths, storage))
    assert statuses == {A.PATH_OK, A.PATH_INDEX_OUT_OF_RANGE, A.PATH_BAD_BYTES, A.PATH_TOO_LONG}, statuses
    edges = SP.edges()
    es = SP.edge_storage(edges)
    statuses = _compare(edges, es, _run(exe, env, edges, es))
    assert statuses == {A.PATH_OK, A.PATH_INDEX_OUT_OF_RANGE, A.PATH_BAD_BYTES, A.PATH_TOO_LONG}, statuses


def test_per_path_code_on_the_cpu_matches_the_restatement():
    _check(None, 2000, 20261018)


def test_per_path_code_under_sanitizers():
    _check(True, 300, 7)
