"""The device bundle parser of ipcfp_verify_bundle_json (csrc/json_parse_items.cuh, driven by csrc/json_parse.cu) compiled for the HOST and
compared with ipcfp_bundle_from_json (csrc/bundle_parse.cpp) (tests/host_fuzz/emu_json_parse.cu): random canonical EventProofBundle and
UnifiedProofBundle texts rendered by csrc/bundle_json.cpp must be accepted with the host parser's PODs field by field, and every byte
mutation of such texts must either be refused by the device items or give exactly the host parser's values. Also the ctypes layout of
ipcfp_bundle_verdict. No GPU involved; the harness is built in a temporary directory."""
import ctypes as C
import os
import re
import shutil
import subprocess

import pytest

from ipc_filecoin_proofs_b200 import _abi as A
from tests.test_host_fuzz import ROOT, SAN_ENV, SANITIZE


@pytest.fixture(scope="module")
def harness(tmp_path_factory):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    build = tmp_path_factory.mktemp("emu_json_parse")
    csrc = os.path.join(ROOT, "ipc_filecoin_proofs_b200", "csrc")

    def make(sanitize):
        exe = str(build / ("emu_json_parse" + ("_san" if sanitize else "")))
        cmd = [nvcc, "-std=c++17", "-O1" if sanitize else "-O2", "-Wno-deprecated-gpu-targets", "-diag-suppress", "20091", "-o", exe,
               os.path.join(ROOT, "tests", "host_fuzz", "emu_json_parse.cu"), os.path.join(csrc, "bundle_json.cpp"), os.path.join(csrc, "bundle_parse.cpp")]
        cc = subprocess.run(cmd + (SANITIZE if sanitize else []), cwd=ROOT, capture_output=True, text=True)
        if cc.returncode != 0 and sanitize and "sanitize" in cc.stderr:
            pytest.skip("this host compiler has no sanitizer runtime")
        assert cc.returncode == 0, cc.stderr[-3000:]
        return exe, (dict(os.environ, **SAN_ENV) if sanitize else None)
    return make


def _run(harness, sanitize, n_bundles, n_mutants, seed):
    exe, env = harness(sanitize)
    out = subprocess.run([exe, str(n_bundles), str(n_mutants), str(seed)], capture_output=True, text=True, env=env)
    assert out.returncode == 0, (out.stdout + out.stderr)[-3000:]
    assert out.stdout.startswith(f"ok: device bundle parser == ipcfp_bundle_from_json on {n_bundles} canonical bundles"), out.stdout
    assert f"and {n_mutants} mutants" in out.stdout, out.stdout
    assert "runtime error" not in out.stderr and "AddressSanitizer" not in out.stderr, out.stderr[-3000:]
    accepted, host_ok = (int(x) for x in re.search(r"\((\d+) accepted by the device items, (\d+) by the host parser\)", out.stdout).groups())
    assert 0 < accepted <= host_ok, out.stdout   # both outcomes occur; every device accept is a host accept (checked value by value inside)
    return out.stdout


def test_device_bundle_parser_equals_host_parser(harness):
    """2 × 2 000 canonical bundles and 2 × 60 000 byte mutations. IPCFP_HOST_FUZZ_SANITIZE=1 builds this one with AddressSanitizer + UBSan
    as well (`make sanitize`)."""
    for seed in (7, 20261015):
        _run(harness, bool(os.environ.get("IPCFP_HOST_FUZZ_SANITIZE")), 2000, 60000, seed)


def test_device_bundle_parser_under_sanitizers(harness):
    """The same harness with AddressSanitizer + UBSan: the items stay inside the text and its JP_PAD zero bytes (the framing and tipset
    items inside the unpadded text), and the writers inside each block's bytes."""
    _run(harness, True, 600, 20000, 31)


def test_bundle_verdict_ctypes_layout_matches_c_header(tmp_path):
    st = A.BundleVerdictC
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "ipcfp.h"', "int main(void) {",
             'printf("size %zu\\n", sizeof(ipcfp_bundle_verdict));']
    lines += [f'printf("{f} %zu\\n", offsetof(ipcfp_bundle_verdict, {f}));' for f, _ in st._fields_]
    lines += ["return 0; }"]
    src, exe = tmp_path / "layout.c", tmp_path / "layout"
    src.write_text("\n".join(lines))
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), "-o", str(exe), str(src)])
    got = dict(l.split() for l in subprocess.check_output([str(exe)], text=True).strip().splitlines())
    assert int(got["size"]) == C.sizeof(st)
    for f, _ in st._fields_:
        assert int(got[f]) == getattr(st, f).offset, f
    assert C.sizeof(st) % 8 == 0
