"""The device CAR parser of ipcfp_store_create_car (csrc/car_items.cuh, driven by csrc/car.cu) compiled for the HOST and compared with
ipcfp_blocks_from_car (csrc/car_parse.cpp) (tests/host_fuzz/emu_car.cu): random canonical CARs must be accepted with the host parser's
arrays, CARs with a forged section header inside a block too (the walk steps over it), CARs with a non-minimal length varint must be
deferred, and every mutation of a
canonical CAR must either be deferred or give exactly the host parser's arrays. No GPU involved; the harness is built in a temporary
directory."""
import os
import re
import shutil
import subprocess

import pytest

from tests.test_host_fuzz import ROOT, SAN_ENV, SANITIZE


@pytest.fixture(scope="module")
def harness(tmp_path_factory):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    build = tmp_path_factory.mktemp("emu_car")
    csrc = os.path.join(ROOT, "ipc_filecoin_proofs_b200", "csrc")

    def make(sanitize):
        exe = str(build / ("emu_car" + ("_san" if sanitize else "")))
        cmd = [nvcc, "-std=c++17", "-O1" if sanitize else "-O2", "-Wno-deprecated-gpu-targets", "-diag-suppress", "20091", "-o", exe,
               os.path.join(ROOT, "tests", "host_fuzz", "emu_car.cu"), os.path.join(csrc, "car_parse.cpp"),
               os.path.join(csrc, "rpc_blocks_parse.cpp")]
        cc = subprocess.run(cmd + (SANITIZE if sanitize else []), cwd=ROOT, capture_output=True, text=True)
        if cc.returncode != 0 and sanitize and "sanitize" in cc.stderr:
            pytest.skip("this host compiler has no sanitizer runtime")
        assert cc.returncode == 0, cc.stderr[-3000:]
        return exe, (dict(os.environ, **SAN_ENV) if sanitize else None)
    return make


def _run(harness, sanitize, n_inputs, n_mutants, seed):
    exe, env = harness(sanitize)
    out = subprocess.run([exe, str(n_inputs), str(n_mutants), str(seed)], capture_output=True, text=True, env=env)
    assert out.returncode == 0, (out.stdout + out.stderr)[-3000:]
    assert out.stdout.startswith(f"ok: device CAR parser == ipcfp_blocks_from_car on {n_inputs} inputs"), out.stdout
    assert "runtime error" not in out.stderr and "AddressSanitizer" not in out.stderr, out.stderr[-3000:]
    forged, nonminimal = (int(x) for x in re.search(r"\((\d+) with a forged prefix, all accepted, (\d+) with a non-minimal varint", out.stdout).groups())
    assert forged > n_inputs // 4 and nonminimal > n_inputs // 4, out.stdout
    accepted, host_ok = (int(x) for x in re.search(r"(\d+) accepted by the device items, (\d+) by the host parser\)", out.stdout).groups())
    assert 0 < accepted <= host_ok < n_mutants, out.stdout   # every device accept is a host accept with the same arrays (checked inside)
    return out.stdout


def test_device_car_parser_equals_host_parser(harness):
    """2 × 3 000 inputs and 2 × 60 000 mutations. IPCFP_HOST_FUZZ_SANITIZE=1 builds this one with AddressSanitizer + UBSan as well
    (`make sanitize`)."""
    for seed in (7, 20261018):
        _run(harness, bool(os.environ.get("IPCFP_HOST_FUZZ_SANITIZE")), 3000, 60000, seed)


def test_device_car_parser_under_sanitizers(harness):
    """The same harness with AddressSanitizer + UBSan: the items stay inside the payload and its CAR_PAD zero bytes."""
    _run(harness, True, 900, 20000, 31)
