"""The storage-path functions of include/ipcfp.hpp (StoragePath, generate_storage_path_proofs, plan_fetch_storage_paths,
verify_storage_paths), driven by tests/cpp/storage_path_test.cpp over the contract of tests/storage_paths.py: a nested-mapping struct
member and two long strings, their values against the Python restatement, the proofs verified and a changed one refused."""
import os
import shutil
import struct
import subprocess

import pytest

from tests import storage_paths as SP

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def path_exe(tmp_path_factory):
    """Compiled once per module into a temporary directory: the checkout may be read-only."""
    gxx = shutil.which("g++")
    if not gxx:
        pytest.skip("g++ not available")
    d = os.path.join(ROOT, "ipc_filecoin_proofs_b200")
    if not os.path.exists(os.path.join(d, "libipcfp.so")):
        pytest.skip("libipcfp.so not built (run `make`)")
    exe = str(tmp_path_factory.mktemp("cpp_storage_path") / "storage_path_test")
    cmd = [gxx, "-std=c++17", "-O1", "-g", "-Wall", "-Wextra", "-Werror", "-o", exe, os.path.join(ROOT, "tests", "cpp", "storage_path_test.cpp"),
           "-L" + d, "-lipcfp", "-Wl,-rpath," + d]
    cc = subprocess.run(cmd, capture_output=True, text=True)
    assert cc.returncode == 0, cc.stderr[-3000:]
    return exe


def test_cpp_storage_path_compiles(path_exe):
    assert os.path.exists(path_exe)


@pytest.mark.gpu
def test_cpp_storage_paths_on_the_gpu(path_exe, ts3_small, tmp_path):
    c = SP.Contract()
    flat, tip = c.world(ts3_small)
    text_key = SP.STRING_LENGTHS.index(65)
    path = tmp_path / "case.bin"
    with open(path, "wb") as f:
        f.write(bytes(tip.child_cid) + bytes(tip.parent_state_root) + struct.pack("<Q", len(flat.blocks)))
        for cid, b in flat.blocks.items():
            f.write(cid + struct.pack("<I", len(b)) + b)
        f.write(c.subnet_ids[2] + struct.pack("<Q", text_key))
    out = subprocess.run([path_exe, str(path)], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, (out.stdout + out.stderr)[-3000:]
    subnet = SP.StoragePath(SP.ACTOR, 0).mapping(c.subnet_ids[2], "bytes32")
    paths = [subnet.field(1), subnet.field(2).bytes(), SP.StoragePath(SP.ACTOR, 12).mapping(text_key, "uint256").bytes()]
    want = []
    for p in paths:
        specs, status, value, _, _ = c.expected(p)
        want.append(f"path {status} 0x{value.hex()} {len(specs)}")
    lines = out.stdout.splitlines()
    assert lines[:3] == want
    assert len(c.expected(paths[1])[2]) > 31 and len(c.expected(paths[2])[2]) == 65   # both strings are long
    assert lines[-1].startswith("ok:")
