"""Differential fuzz of the device decoders, compiled for the HOST from the very same headers (tests/host_fuzz/fuzz_events.cu):
  * register-window fast path `fast_stamped_event` vs the strict decoder `parse_stamped_event` (csrc/ipld.cuh),
  * byte-layout check of the dense message-AMT walk vs `amt_node_begin` / `rd_cid` / `amt_node_finish`,
  * the strict device decoder + extract_evm_log vs the CPU oracle (an independent implementation) on every fuzzed event,
  * pass 1's per-receipt unit (one events-AMT root block: status class and the visited event list) vs the oracle,
  * one receipts-AMT node (the unit of pass 2's path walk: links / receipts / events roots) vs the oracle,
  * one HAMT node (state tree and EVM storage: bitfield, links, buckets, ActorState / Vec<u8> values) vs the oracle.
Whatever a shortcut accepts, the strict decoder must accept with the same meaning — that is what lets the kernels take the
shortcut without changing a result — and the strict decoder must agree with the oracle on well-formed AND malformed input.
No GPU involved (nvcc host pass only); the oracle is linked as the checker."""
import os
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SANITIZE = ["-Xcompiler", "-fsanitize=address", "-Xcompiler", "-fsanitize=undefined", "-Xcompiler", "-fno-omit-frame-pointer", "-g"]
SAN_ENV = dict(ASAN_OPTIONS="detect_leaks=0:halt_on_error=1", UBSAN_OPTIONS="print_stacktrace=1:halt_on_error=1")


def _harness(name, with_synth=True, sanitize=None):
    """Build tests/host_fuzz/<name>.cu for the HOST (nvcc host pass) with the oracle (and the synthetic builder) linked as the checker.
    IPCFP_HOST_FUZZ_SANITIZE=1 (or sanitize=True) builds with AddressSanitizer + UBSan: the harnesses give the device code buffers
    padded exactly as the engine's device buffers are (host_store.h), so an out-of-bounds access of the device code is a report."""
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    if sanitize is None:
        sanitize = bool(os.environ.get("IPCFP_HOST_FUZZ_SANITIZE"))
    build = os.path.join(ROOT, "tests", "host_fuzz", "_build")
    os.makedirs(build, exist_ok=True)
    exe = os.path.join(build, name + ("_san" if sanitize else ""))
    cmd = [nvcc, "-std=c++17", "-O1" if sanitize else "-O2", "-Wno-deprecated-gpu-targets", "-diag-suppress", "20091", "-o", exe,
           os.path.join(ROOT, "tests", "host_fuzz", name + ".cu"), os.path.join(ROOT, "oracle", "oracle.cpp")]
    if with_synth:
        cmd.append(os.path.join(ROOT, "synth", "synth.cpp"))
    cc = subprocess.run(cmd + (SANITIZE if sanitize else []) + ["-lpthread"], cwd=ROOT, capture_output=True, text=True)
    if cc.returncode != 0 and sanitize and "sanitize" in cc.stderr:
        pytest.skip("this host compiler has no sanitizer runtime")
    assert cc.returncode == 0, cc.stderr[-3000:]
    return exe, (dict(os.environ, **SAN_ENV) if sanitize else None)


def test_fast_paths_agree_with_strict_decoders():
    exe, env = _harness("fuzz_events", with_synth=False)
    for seed in ("535", "20260922"):
        out = subprocess.run([exe, "600000", seed], capture_output=True, text=True, env=env)
        assert out.returncode == 0, out.stderr[-2000:]
        lines = [l for l in out.stdout.splitlines() if l.startswith("ok:")]
        assert len(lines) == 5, out.stdout
        # the shortcuts must actually be taken on a large share of the inputs, or the comparison says nothing
        for l in lines:
            if "accepted" in l:
                total, acc = int(l.split()[1]), int(l.split("accepted")[1].split()[0])
                assert acc > total // 4, l
        assert any("compared with the oracle" in l for l in lines) and any("root blocks agree with the oracle" in l for l in lines)
        assert any("receipts-AMT nodes agree with the oracle" in l for l in lines) and any("HAMT nodes agree with the oracle" in l for l in lines)


def test_dense_walk_emulated_on_cpu_matches_oracle():
    """tests/host_fuzz/emu_walk.cu: `amt_item_dense`, `shard_amt_ranges` and `make_dense_plan` (csrc/walk.cuh) compiled for the
    host and run level by level, item by item, lane by lane over a host copy of the block store (arena + BlockRec array + CID
    index laid out as ipcfp_store_create does), for whole tipsets and for every shard at world sizes 1, 2, 3 and 8 — against the
    oracle's raw message list and its recorded block set."""
    exe, env = _harness("emu_walk", with_synth=True)
    out = subprocess.run([exe, "60", "11"], capture_output=True, text=True, env=env)
    assert out.returncode == 0, out.stderr[-3000:]
    assert out.stdout.startswith("ok: dense walk == general walk == oracle on the CPU for 60 tipsets"), out.stdout


def test_storage_path_emulated_on_cpu_matches_oracle():
    """tests/host_fuzz/emu_storage.cu: `storage_proof_one`, `read_storage_slot`, `hamt_get` and the value decoders (csrc/storage.cuh)
    compiled for the host and run spec by spec over a host copy of the store, against `oracle_generate_storage_proofs` — on the
    synthetic state trees (six EVM actors = the six root shapes A1/A2/A3/B1/B2/C, present / absent / special slots, a missing
    actor) and with one block of a proof path replaced by a mutated copy under the same CID: equal values, found flags, CIDs and
    per-proof recorded block sets, or the same status at the same spec index."""
    exe, env = _harness("emu_storage", with_synth=True)
    out = subprocess.run([exe, "8", "250", "77"], capture_output=True, text=True, env=env)
    assert out.returncode == 0, out.stderr[-3000:]
    assert out.stdout.startswith("ok: storage path on the CPU == oracle for 8 state trees"), out.stdout
    runs_ok, runs_err = int(out.stdout.split(":")[2].split()[0]), int(out.stdout.split("equal,")[1].split()[0])
    assert runs_ok > 100 and runs_err > 500, out.stdout


def test_event_path_emulated_on_cpu_matches_oracle():
    """tests/host_fuzz/emu_events.cu: the per-item device code of generate_event_proof — k_setup's sequence, the dense message-AMT
    walk, pass 1's per-receipt decode, `pass2_item` / `receipts_get` / `walk_events` (csrc/events_items.cuh, csrc/walk.cuh) —
    compiled for the host and driven item by item over a host copy of the store, against `oracle_generate_event_proof`: matching
    receipts, every EventProof field (message CID included), n_exec and the witness CID set on tipsets of many shapes (multi-node
    events AMTs, Case A, malformed events, null roots, duplicate messages), and the same status at the same index when ANY block
    the call reads (events blocks, receipts-AMT nodes, message-AMT nodes, TxMeta, headers) is mutated under its CID or missing —
    the dense walk then raises its flag and the general walk (`amt_item_count` / `amt_item_expand`) takes over, as on the GPU."""
    exe, env = _harness("emu_events", with_synth=True)
    out = subprocess.run([exe, "24", "120", "5"], capture_output=True, text=True, env=env)
    assert out.returncode == 0, out.stderr[-3000:]
    assert out.stdout.startswith("ok: event path on the CPU == oracle for 24 tipsets"), out.stdout
    assert "ok: hand-built roots" in out.stdout, out.stdout
    runs_ok, runs_err = int(out.stdout.split(":")[2].split()[0]), int(out.stdout.split("field,")[1].split()[0])
    general = int(out.stdout.split("identically,")[1].split()[0])
    assert runs_ok > 200 and runs_err > 1000 and general > 100, out.stdout


def test_staged_pass1_lane_logic_emulated_on_cpu():
    """tests/host_fuzz/emu_stage.cu: the per-lane logic of the shared-memory-staged pass-1 kernel —
    `StageLane` / `StageWin` / `stage_fill_lane` of csrc/pass1_stage.cuh — under an adversarial model of the asynchronous fills:
    staged decode == arena decode for every node, five ring geometries."""
    exe, env = _harness("emu_stage", with_synth=False)
    out = subprocess.run([exe, "300", "12"], capture_output=True, text=True, env=env)
    assert out.returncode == 0, (out.stdout + out.stderr)[-3000:]
    assert "ok: staged pass 1 == arena pass 1 for 5 geometries x 300 warps" in out.stdout, out.stdout


def test_event_path_emulation_under_sanitizers():
    """The emu_events harness once more, built with AddressSanitizer + UBSan (always, whatever IPCFP_HOST_FUZZ_SANITIZE says): hash
    probes, BlockRec reads, window loads of the decoders, AMT walks and EventProof emission of the device code on intact AND mutated
    tipsets (incl. the empty tipset) stay inside the buffers the engine gives them (arena pads of 16 / 32 bytes, `+ 64` on the CID
    arrays). On the GPU such an access is silent or poisons the context; here it is a report with a stack."""
    exe, env = _harness("emu_events", sanitize=True)
    out = subprocess.run([exe, "10", "60", "31"], capture_output=True, text=True, env=env)
    assert out.returncode == 0, (out.stdout + out.stderr)[-4000:]
    assert out.stdout.startswith("ok: event path on the CPU == oracle for 10 tipsets"), out.stdout
    assert "ok: hand-built roots" in out.stdout, out.stdout   # a root whose height wraps, the 65-frame walk (emu_events.cu)
    assert "runtime error" not in out.stderr and "AddressSanitizer" not in out.stderr, out.stderr[-4000:]


def test_verifiers_emulated_on_cpu_match_oracle():
    """tests/host_fuzz/emu_verify.cu: the per-item device code of the GPU-batched verifiers (csrc/verify_items.cuh — verify_tipset_item,
    verify_txmeta_item, verify_event_item, verify_storage_item, the very functions the kernels of verify.cu call) compiled for the host
    and driven as verify.cu drives the kernels, against the restated verifiers of the oracle on bundles the oracle generated: intact
    (every proof accepted), with forged claims in every proof field, foreign / matching check_event, changed tipset fields, a witness
    block mutated under its CID, a witness block missing — the same Vec<bool>, or the same status at the same proof index."""
    exe, env = _harness("emu_verify")
    out = subprocess.run([exe, "10", "60", "19"], capture_output=True, text=True, env=env)
    assert out.returncode == 0, (out.stdout + out.stderr)[-3000:]
    assert out.stdout.startswith("ok: verifiers on the CPU == oracle for 10 bundles"), out.stdout
    ev_ok, ev_err = int(out.stdout.split("events")[1].split()[0]), int(out.stdout.split("verdicts,")[1].split()[0])
    st_ok, st_err = int(out.stdout.split("storage")[1].split()[0]), int(out.stdout.split("equal,")[1].split()[0])
    accepted, rejected = int(out.stdout.split("identically;")[2].split()[0]), int(out.stdout.split("accepted,")[1].split()[0])
    assert ev_ok > 200 and ev_err > 50 and st_ok > 80 and st_err > 50 and accepted > 1000 and rejected > 1000, out.stdout
