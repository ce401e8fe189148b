"""The actor-proof functions of include/ipcfp.hpp (generate_actor_proofs, plan_fetch_actor_proofs, verify_actor_proofs), driven by
tests/cpp/actor_proof_test.cpp: the program compiles against the header on the CPU; on the GPU its proofs, per-proof witness lists and
union over the main tree of tests/actor_trees.py (with code) must equal that module's restatement, and the verifier must accept them and
reject a changed balance."""
import os
import shutil
import struct
import subprocess

import pytest

from ipc_filecoin_proofs_b200 import _abi as A
from tests import actor_trees as AT

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def actor_exe(tmp_path_factory):
    """Compiled once per module into a temporary directory: the checkout may be read-only."""
    gxx = shutil.which("g++")
    if not gxx:
        pytest.skip("g++ not available")
    d = os.path.join(ROOT, "ipc_filecoin_proofs_b200")
    if not os.path.exists(os.path.join(d, "libipcfp.so")):
        pytest.skip("libipcfp.so not built (run `make`)")
    exe = str(tmp_path_factory.mktemp("cpp_actor") / "actor_proof_test")
    cmd = [gxx, "-std=c++17", "-O1", "-g", "-Wall", "-Wextra", "-Werror", "-o", exe, os.path.join(ROOT, "tests", "cpp", "actor_proof_test.cpp"),
           "-L" + d, "-lipcfp", "-Wl,-rpath," + d]
    cc = subprocess.run(cmd, capture_output=True, text=True)
    assert cc.returncode == 0, cc.stderr[-3000:]
    return exe


def test_cpp_actor_proof_program_builds(actor_exe):
    out = subprocess.run([actor_exe], capture_output=True, text=True, timeout=60)
    assert out.returncode == 2 and "usage" in out.stderr


@pytest.mark.gpu
def test_cpp_actor_proofs_on_the_gpu(actor_exe, tmp_path, ts3_small):
    blocks, trees, _, _ = AT.world(ts3_small)
    t = trees["main-code"]
    evm = AT.EVM_SETS[t.evm]
    proofs, lists, union = AT.prove(blocks, t.child, t.root, t.addrs, evm, True)
    order = [t.child] + [c for c in blocks if c != t.child]   # the child header first: the program's one-block store
    path = tmp_path / "case.bin"
    with open(path, "wb") as f:
        f.write(t.child + t.root + struct.pack("<Q", len(evm)) + b"".join(evm) + struct.pack("<Q", len(order)))
        for c in order:
            f.write(c + struct.pack("<I", len(blocks[c])) + blocks[c])
        f.write(struct.pack("<Q", len(t.addrs)))
        for a in t.addrs:
            f.write(bytes([len(a)]) + a)
    out = subprocess.run([actor_exe, "gpu", str(path)], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, (out.stdout + out.stderr)[-3000:]
    lines = out.stdout.splitlines()
    got = [l.split() for l in lines if l.startswith("proof ")]
    assert len(got) == len(proofs)
    for g, p, lst in zip(got, proofs, lists):
        rec = A.ActorProofC.from_buffer_copy(bytes.fromhex(g[1]))
        rec.code_off = 0
        assert vars(A.actor_proof_from_c(rec, b"" if g[2] == "-" else bytes.fromhex(g[2]))) == p
        assert [bytes.fromhex(x) for x in g[3:]] == lst
    assert [(bytes.fromhex(l.split()[1]), int(l.split()[2])) for l in lines if l.startswith("witness ")] == [(c, len(blocks[c])) for c in union]
    assert lines[-1].startswith("ok: ")
