"""The message-proof functions of include/ipcfp.hpp (generate_message_proofs, plan_fetch_message_proofs, verify_message_proofs), driven by
tests/cpp/message_proofs_test.cpp."""
import os
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def message_exe(tmp_path_factory):
    """Compiled once per module into a temporary directory: the checkout may be read-only."""
    gxx = shutil.which("g++")
    if not gxx:
        pytest.skip("g++ not available")
    libs = [("ipc_filecoin_proofs_b200", "ipcfp"), ("synth", "ipcfp_synth")]
    for d, n in libs:
        if not os.path.exists(os.path.join(ROOT, d, f"lib{n}.so")):
            pytest.skip(f"{d}/lib{n}.so not built (run `make`)")
    exe = str(tmp_path_factory.mktemp("cpp_message_proofs") / "message_proofs_test")
    cmd = [gxx, "-std=c++17", "-O1", "-g", "-Wall", "-Wextra", "-Werror", "-o", exe, os.path.join(ROOT, "tests", "cpp", "message_proofs_test.cpp")]
    for d, n in libs:
        cmd += ["-L" + os.path.join(ROOT, d), "-l" + n, "-Wl,-rpath," + os.path.join(ROOT, d)]
    cc = subprocess.run(cmd, capture_output=True, text=True)
    assert cc.returncode == 0, cc.stderr[-3000:]
    return exe


def test_cpp_message_proofs_cpu_checks(message_exe):
    out = subprocess.run([message_exe, "cpu"], capture_output=True, text=True, timeout=120)
    assert out.returncode == 0, (out.stdout + out.stderr)[-3000:]
    assert out.stdout.startswith("ok: cpu checks of the message-proof functions"), out.stdout


@pytest.mark.gpu
def test_cpp_message_proofs_on_the_gpu(message_exe):
    out = subprocess.run([message_exe, "gpu"], capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, (out.stdout + out.stderr)[-3000:]
    assert out.stdout.startswith("ok: gpu checks of the message-proof functions"), out.stdout
