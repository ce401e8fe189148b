"""The device renderer of the UnifiedProofBundle text (the StorageProof record and the unified framing of csrc/json_items.cuh, with the
EventProof and ProofBlock records, driven as csrc/json.cu::render_unified_json drives them) compiled for the HOST and compared byte for
byte with ipcfp_bundle_to_json (csrc/bundle_json.cpp) on random bundles (tests/host_fuzz/emu_json_unified.cu): 0, 1 or many storage
proofs, event proofs (from 0 to 3 results) and blocks, actor ids 0 and 2^64-1, child epochs INT64_MIN and INT64_MAX. No GPU involved."""
import os
import subprocess

from tests.test_host_fuzz import _harness


def _run(sanitize, n, seed):
    exe, env = _harness("emu_json_unified", with_synth=False, sanitize=sanitize)
    out = subprocess.run([exe, str(n), str(seed)], capture_output=True, text=True, env=env)
    assert out.returncode == 0, (out.stdout + out.stderr)[-3000:]
    assert out.stdout.startswith(f"ok: device UnifiedProofBundle renderer == ipcfp_bundle_to_json for {n} bundles"), out.stdout
    assert "runtime error" not in out.stderr and "AddressSanitizer" not in out.stderr, out.stderr[-3000:]


def test_unified_json_renderer_equals_host_renderer():
    """IPCFP_HOST_FUZZ_SANITIZE=1 builds this one with AddressSanitizer + UBSan as well (`make sanitize`)."""
    for seed in (7, 20261016):
        _run(bool(os.environ.get("IPCFP_HOST_FUZZ_SANITIZE")), 3000, seed)


def test_unified_json_renderer_under_sanitizers():
    """The same harness, always with AddressSanitizer + UBSan."""
    _run(True, 1000, 31)
