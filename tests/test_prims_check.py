"""The device-wide primitives of csrc/prims.cu (exclusive scan, bitmap → indices, stable radix sort), called directly by
tests/gpu_prims/prims_check.cu and compared there with plain CPU references at the sizes where their launch shapes change. The
program is compiled with the library's own nvcc flags (the Makefile's NVFLAGS); the compile needs no GPU, running it does."""
import os
import re
import shlex
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "gpu_prims", "prims_check.cu")
PRIMS = os.path.join(ROOT, "ipc_filecoin_proofs_b200", "csrc", "prims.cu")


def _nvflags():
    with open(os.path.join(ROOT, "Makefile")) as f:
        m = re.search(r"^NVFLAGS\s*:=\s*(.*)$", f.read(), re.M)
    assert m, "NVFLAGS not found in the Makefile"
    return shlex.split(m.group(1))


@pytest.fixture(scope="module")
def prims_check_exe(tmp_path_factory):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    # built outside the source tree, which may be read-only
    exe = str(tmp_path_factory.mktemp("prims_check") / "prims_check")
    cc = subprocess.run([nvcc, *_nvflags(), "-o", exe, SRC, PRIMS], cwd=ROOT, capture_output=True, text=True)
    assert cc.returncode == 0, cc.stderr[-3000:]
    return exe


def test_prims_check_compiles(prims_check_exe):
    assert os.access(prims_check_exe, os.X_OK)
    assert "sm_90a" in " ".join(_nvflags())


@pytest.mark.gpu
def test_prims_match_cpu_references(prims_check_exe):
    out = subprocess.run([prims_check_exe], capture_output=True, text=True, timeout=900)
    assert out.returncode == 0, (out.stdout[-2000:], out.stderr[-3000:])
    ok = [line for line in out.stdout.splitlines() if line.startswith("ok:")]
    assert len(ok) == 1, out.stdout
    assert int(ok[0].split(" in ")[1].split()[0]) == 407, ok[0]   # 30 scans, 41 bitmaps, 336 sorts: no case may go missing
