"""The device JSON renderer of IPCFP_RESULT_JSON (csrc/json_items.cuh, driven by csrc/json.cu) compiled for the HOST and compared byte for
byte with ipcfp_event_result_to_json (csrc/bundle_json.cpp) on random event results (tests/host_fuzz/emu_json.cu): u64 fields 0, 9, 10, 99,
100 and 2^64-1, epochs negative, zero and INT64_MIN, 0 to 3 parent CIDs, blocks of 0 to 300 bytes (every len % 3), 0 to 9 topics, 0 to 200
data bytes, skipped proof slots (the first one included), results without proofs and without blocks. No GPU involved."""
import os
import shutil
import subprocess

import pytest

from tests.test_host_fuzz import ROOT, SAN_ENV, SANITIZE


def _build(sanitize):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    build = os.path.join(ROOT, "tests", "host_fuzz", "_build")
    os.makedirs(build, exist_ok=True)
    exe = os.path.join(build, "emu_json" + ("_san" if sanitize else ""))
    cmd = [nvcc, "-std=c++17", "-O1" if sanitize else "-O2", "-Wno-deprecated-gpu-targets", "-diag-suppress", "20091", "-o", exe,
           os.path.join(ROOT, "tests", "host_fuzz", "emu_json.cu"), os.path.join(ROOT, "ipc_filecoin_proofs_b200", "csrc", "bundle_json.cpp")]
    cc = subprocess.run(cmd + (SANITIZE if sanitize else []), cwd=ROOT, capture_output=True, text=True)
    if cc.returncode != 0 and sanitize and "sanitize" in cc.stderr:
        pytest.skip("this host compiler has no sanitizer runtime")
    assert cc.returncode == 0, cc.stderr[-3000:]
    return exe, (dict(os.environ, **SAN_ENV) if sanitize else None)


def _run(sanitize, n, seed):
    exe, env = _build(sanitize)
    out = subprocess.run([exe, str(n), str(seed)], capture_output=True, text=True, env=env)
    assert out.returncode == 0, (out.stdout + out.stderr)[-3000:]
    assert out.stdout.startswith(f"ok: device JSON renderer == ipcfp_event_result_to_json for {n} results"), out.stdout
    assert "runtime error" not in out.stderr and "AddressSanitizer" not in out.stderr, out.stderr[-3000:]
    return out.stdout


def test_device_json_renderer_equals_host_renderer():
    """IPCFP_HOST_FUZZ_SANITIZE=1 builds this one with AddressSanitizer + UBSan as well (`make sanitize`)."""
    for seed in (7, 20261015):
        _run(bool(os.environ.get("IPCFP_HOST_FUZZ_SANITIZE")), 4000, seed)


def test_device_json_renderer_under_sanitizers():
    """The same harness, always with AddressSanitizer + UBSan: the writers stay inside the exact-size output, and the readers inside the
    padded buffers the engine gives them and the block's own bytes."""
    _run(True, 1500, 31)
