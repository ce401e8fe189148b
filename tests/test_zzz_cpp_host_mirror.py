"""include/ipcfp.hpp — the host side above the C ABI in C++17 with the reference's own names (the reference is a Rust crate; no Rust
toolchain exists in this image) — exercised by tests/cpp/host_mirror_test.cpp, a C++ program that reads like tests of the reference's
crate would: generate_event_proof / generate_storage_proof / generate_proof_bundle / verify_* on a tipset pair, compared with the CPU
oracle (linked as the checker) in the reference's structs. Built with g++ against the in-tree libipcfp.so / liboracle.so /
libipcfp_synth.so. (Last file of the suite on purpose.)"""
import os
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def host_mirror_exe(tmp_path_factory):
    """The harness, compiled once per module into a temporary directory: the checkout may be read-only."""
    gxx = shutil.which("g++")
    if not gxx:
        pytest.skip("g++ not available")
    libs = [("ipc_filecoin_proofs_b200", "ipcfp"), ("synth", "ipcfp_synth"), ("oracle", "oracle")]
    for d, n in libs:
        if not os.path.exists(os.path.join(ROOT, d, f"lib{n}.so")):
            pytest.skip(f"{d}/lib{n}.so not built (run `make`)")
    exe = str(tmp_path_factory.mktemp("cpp_host_mirror") / "host_mirror_test")
    cmd = [gxx, "-std=c++17", "-O1", "-g", "-Wall", "-Wextra", "-Werror", "-o", exe, os.path.join(ROOT, "tests", "cpp", "host_mirror_test.cpp")]
    for d, n in libs:
        cmd += ["-L" + os.path.join(ROOT, d), "-l" + n, "-Wl,-rpath," + os.path.join(ROOT, d)]
    cc = subprocess.run(cmd, capture_output=True, text=True)
    assert cc.returncode == 0, cc.stderr[-3000:]
    return exe


def test_cpp_host_mirror_cpu_checks(host_mirror_exe):
    """Cid <-> string on public Filecoin constants, `Ord` of Cid against the oracle's sort, hex / padding helpers, TipsetDesc packing ==
    the synthetic builder's descriptor, the result → struct conversions on an oracle result; without a device every call that needs
    one throws with IPCFP_ERR_NO_DEVICE."""
    out = subprocess.run([host_mirror_exe, "cpu"], capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, (out.stdout + out.stderr)[-3000:]
    assert out.stdout.startswith("ok: cpu checks of include/ipcfp.hpp"), out.stdout


def test_cpp_header_compiles_standalone_and_as_strict_cxx17():
    """The mirror is header-only over nothing but include/ipcfp.h: it must compile on its own, pedantically."""
    gxx = shutil.which("g++")
    if not gxx:
        pytest.skip("g++ not available")
    cc = subprocess.run([gxx, "-std=c++17", "-Wall", "-Wextra", "-Wpedantic", "-Werror", "-fsyntax-only", "-x", "c++", os.path.join(ROOT, "include", "ipcfp.hpp")],
                        capture_output=True, text=True)
    assert cc.returncode == 0, cc.stderr[-3000:]


@pytest.mark.gpu
def test_cpp_host_mirror_on_the_gpu(host_mirror_exe):
    """generate_event_proof (configs[0], configs[1]) / generate_storage_proof over the six root shapes / read_storage_slot /
    generate_proof_bundle (configs[2], small HAMT) through include/ipcfp.hpp on cuda:0 == the oracle in the reference's structs;
    verify_event_proof / verify_storage_proof / verify_proof_bundle accept them, reject untrusted anchors, forged claims, a foreign
    check_event; a damaged witness block is a CID mismatch; dropping any single witness block never leaves everything accepted; a
    missing store block and a missing actor fail with the oracle's status and index."""
    out = subprocess.run([host_mirror_exe, "gpu"], capture_output=True, text=True, timeout=900)
    assert out.returncode == 0, (out.stdout + out.stderr)[-3000:]
    assert out.stdout.startswith("ok: include/ipcfp.hpp on cuda:0 == the oracle"), out.stdout
    launches = int(out.stdout.split("assertions,")[1].split()[0])
    assert launches > 0   # the product library's own kernels ran in that process
