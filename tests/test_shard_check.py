"""The kernels of the cross-shard protocol (csrc/shard_kernels.cuh: the exchange X, the positions P, the fetch F and the witness union W
of DESIGN.md §6), driven by tests/gpu_prims/shard_check.cu for W simulated ranks on one GPU at world sizes 1 to 255 and compared there
with plain CPU references. The collectives become device copies, so no NCCL and no second GPU is needed. This file also hands the
program the raw message lists of tests/message_amts.py's shared cases and of the 64-parent capacity case; the program rebuilds their
execution order at every world size (select of every exec index, then the fetch), and each must equal `message_amts.exec_order`.
The program is compiled with the library's own nvcc flags (the Makefile's NVFLAGS); the compile needs no GPU, running it does."""
import os
import re
import shlex
import shutil
import struct
import subprocess

import pytest

from tests import message_amts as M

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "gpu_prims", "shard_check.cu")
PRIMS = os.path.join(ROOT, "ipc_filecoin_proofs_b200", "csrc", "prims.cu")
WORLDS = (1, 2, 3, 5, 8, 31, 32, 33, 64, 100, 255)


def _nvflags():
    with open(os.path.join(ROOT, "Makefile")) as f:
        m = re.search(r"^NVFLAGS\s*:=\s*(.*)$", f.read(), re.M)
    assert m, "NVFLAGS not found in the Makefile"
    return shlex.split(m.group(1))


@pytest.fixture(scope="module")
def shard_check_exe(tmp_path_factory):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    # built outside the source tree, which may be read-only
    exe = str(tmp_path_factory.mktemp("shard_check") / "shard_check")
    cc = subprocess.run([nvcc, *_nvflags(), "-o", exe, SRC, PRIMS], cwd=ROOT, capture_output=True, text=True)
    assert cc.returncode == 0, cc.stderr[-3000:]
    return exe


def test_shard_check_compiles(shard_check_exe):
    assert os.access(shard_check_exe, os.X_OK)
    assert "sm_90a" in " ".join(_nvflags())


def test_shard_kernels_header_stands_apart_from_nccl():
    """The harness includes the kernels without the library's NCCL plumbing; the world sizes it runs reach the library's limit."""
    csrc = os.path.join(ROOT, "ipc_filecoin_proofs_b200", "csrc")
    hdr = open(os.path.join(csrc, "shard_kernels.cuh")).read()
    assert not re.search(r"#include\s*[<\"][^>\"]*nccl", hdr) and not re.search(r"\bnccl[A-Z_]", hdr)
    assert '#include "shard_kernels.cuh"' in open(os.path.join(csrc, "parallel.cu")).read()
    assert re.search(r"constexpr uint32_t MAX_WORLD = 255;", open(os.path.join(csrc, "engine.cuh")).read())
    assert max(WORLDS) == 255


def _raw_list(case):
    raw = []
    for bls, secp in case.lists:
        raw += list(bls) + list(secp)
    return raw


@pytest.mark.gpu
def test_shard_kernels_match_cpu_references(shard_check_exe, tmp_path):
    cases = M.shared_cases(M.base_tipset()) + [M.capacity_case(64)]
    assert len(_raw_list(cases[-1])) == 64 * 20000
    src, out_path = tmp_path / "lists.bin", tmp_path / "orders.bin"
    with open(src, "wb") as f:
        f.write(struct.pack("<I", len(cases)))
        for c in cases:
            raw = _raw_list(c)
            assert all(len(x) == 38 for x in raw)
            f.write(struct.pack("<I", len(c.name)) + c.name.encode() + struct.pack("<Q", len(raw)) + b"".join(raw))
    out = subprocess.run([shard_check_exe, str(src), str(out_path)], capture_output=True, text=True, timeout=1800)
    assert out.returncode == 0, (out.stdout[-2000:], out.stderr[-3000:])
    ok = [line for line in out.stdout.splitlines() if line.startswith("ok:")]
    assert len(ok) == 1, out.stdout
    # 598 synthetic cases over the 11 world sizes, then the 10 message lists at each of them: no case may go missing, and the
    # overflow paths (one segment past its capacity at every W > 1; pieces past forced and default slots) must keep being taken
    m = re.search(r" in (\d+) cases \((\d+) exchanges raised their overflow word, (\d+) partitioned unions overflowed a piece\)", ok[0])
    assert m and (int(m.group(1)), int(m.group(2)), int(m.group(3))) == (598 + 10 * len(WORLDS), 10, 72), ok[0]
    data = out_path.read_bytes()
    at = 0
    for c in cases:
        want = M.exec_order(c.lists)
        for w in WORLDS:
            got_w, n = struct.unpack_from("<IQ", data, at)
            at += 12
            got = [data[at + 38 * i:at + 38 * (i + 1)] for i in range(n)]
            at += 38 * n
            assert got_w == w and got == want, (c.name, w, got_w, n, len(want))
    assert at == len(data)
