"""The address-resolution functions of include/ipcfp.hpp (resolve_addresses, resolve_eth_address_to_actor_id, parse_address), driven
by tests/cpp/resolve_test.cpp: on the CPU the reference's validation and the documentation's f410 example; on the GPU a hand-built state
tree of tests/address_trees.py, whose result must equal the C++ oracle's (tests/oracle_resolve.cpp) and that module's restatement of the
call."""
import os
import random
import shutil
import struct
import subprocess

import pytest

from tests import address_trees as T
from tests import oracle_resolve as O
from tests import storage_trees as S

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def resolve_exe(tmp_path_factory):
    """Compiled once per module into a temporary directory: the checkout may be read-only."""
    gxx = shutil.which("g++")
    if not gxx:
        pytest.skip("g++ not available")
    d = os.path.join(ROOT, "ipc_filecoin_proofs_b200")
    if not os.path.exists(os.path.join(d, "libipcfp.so")):
        pytest.skip("libipcfp.so not built (run `make`)")
    exe = str(tmp_path_factory.mktemp("cpp_resolve") / "resolve_test")
    cmd = [gxx, "-std=c++17", "-O1", "-g", "-Wall", "-Wextra", "-Werror", "-o", exe, os.path.join(ROOT, "tests", "cpp", "resolve_test.cpp"),
           "-L" + d, "-lipcfp", "-Wl,-rpath," + d]
    cc = subprocess.run(cmd, capture_output=True, text=True)
    assert cc.returncode == 0, cc.stderr[-3000:]
    return exe


def test_cpp_resolve_cpu_checks(resolve_exe):
    out = subprocess.run([resolve_exe, "cpu"], capture_output=True, text=True, timeout=120)
    assert out.returncode == 0, (out.stdout + out.stderr)[-3000:]
    assert out.stdout.startswith("ok: cpu checks of the address functions"), out.stdout


@pytest.mark.gpu
def test_cpp_resolve_on_the_gpu(resolve_exe, tmp_path):
    eth = bytes(range(0x40, 0x54))
    blocks = S.Blocks()
    ent = T._entries(random.Random(5), 3000)
    ent[T.delegated(10, eth)] = 4242
    root = T.state_tree(blocks, ent)
    addrs = list(ent)[:200] + [T.delegated(10, bytes(20)), T.id_addr(77), b"\x09"]
    path = tmp_path / "case.bin"
    with open(path, "wb") as f:
        f.write(root + struct.pack("<Q", len(blocks)))
        for c, b in blocks.items():
            f.write(c + struct.pack("<I", len(b)) + b)
        f.write(struct.pack("<Q", len(addrs)))
        for a in addrs:
            f.write(bytes([len(a)]) + a)
    out = subprocess.run([resolve_exe, "gpu", str(path), "0x" + eth.hex()], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, (out.stdout + out.stderr)[-3000:]
    lines = out.stdout.splitlines()
    ids, status, init, missing, read = O.Oracle(blocks).resolve(root, addrs)
    assert (ids, status, init, missing, read) == T.resolve(blocks, root, addrs)
    assert lines[0] == f"init {init}"
    assert lines[1:1 + len(addrs)] == [f"addr {s} {i}" for s, i in zip(status, ids)]
    assert [l for l in lines if l.startswith("missing ")] == []
    assert [l for l in lines if l.startswith("witness ")] == [f"witness {c.hex()} {len(blocks[c])}" for c in read]
    assert "eth 4242" in lines and "unknown -9" in lines
    assert lines[-1].startswith("ok:")
