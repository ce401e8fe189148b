"""The fast device decoders against what follows a block (tests/host_fuzz/emu_tail.cu), on the CPU.

Every canonical encoding (StampedEvents, HAMT nodes with ActorState / Vec<u8> / u64 values, the values alone, message-AMT nodes) is
cut at every prefix length k, the block length set to k, and the bytes after the cut replaced by five tails: the encoding's own
remainder, the remainder with one byte changed, the encoding again, zeros, 0xff. Whenever a fast decoder (`fast_stamped_event_t`
over GlobalWin and over the StageWin ring StageLane fills, `hamt_node_lookup_fast`, `skip_u8vec_fast`, `skip_u64_fast`, the dense
walk's layout check in `amt_item_dense`) accepts, its strict twin accepts with the same outputs; and the strict decoder's outcome
does not depend on the tail. A fast decoder whose bound check is off by one accepts a value that ends inside the remainder."""
import subprocess

from tests.test_host_fuzz import _harness

PAIRS = ("StampedEvent (GlobalWin)", "StampedEvent (StageWin)", "HAMT node, ActorState", "HAMT node, Vec<u8>", "HAMT node, u64",
         "Vec<u8> value", "u64 value", "message-AMT node (dense walk)")


def _run(sanitize, n, seed):
    exe, env = _harness("emu_tail", with_synth=False, sanitize=sanitize)
    out = subprocess.run([exe, str(n), str(seed)], capture_output=True, text=True, env=env)
    assert out.returncode == 0, (out.stdout + out.stderr)[-3000:]
    assert "ok: tail bytes:" in out.stdout, out.stdout
    counts = {}
    for line in out.stdout.splitlines():
        for name in PAIRS:
            if line.strip().startswith(name + ":"):
                runs = int(line.split(":")[1].split()[0])
                accepted = int(line.split("accepted")[1].split()[0])
                counts[name] = (runs, accepted)
    assert set(counts) == set(PAIRS), out.stdout
    # every encoding is complete at k == len under all five tails: the fast paths must take (nearly) all of those, or the
    # comparison says nothing (StampedEvents with an 8-byte emitter are left to the strict decoder by design)
    for name, (runs, accepted) in counts.items():
        assert runs >= 5 * n and accepted >= 5 * n // 2, (name, runs, accepted)
    return out


def test_fast_decoders_ignore_the_bytes_after_the_block():
    out = _run(None, 300, 20261017)
    total = int(out.stdout.split("encodings cut at every length under 5 tails,")[1].split()[0])
    assert total > 2_000_000, out.stdout


def test_fast_decoders_ignore_the_bytes_after_the_block_under_sanitizers():
    """The same runs built with AddressSanitizer + UBSan (always): the over-reads of the window loads and the chunk copies stay
    inside the buffers, whatever the tail holds."""
    out = _run(True, 60, 7)
    assert "runtime error" not in out.stderr and "AddressSanitizer" not in out.stderr, out.stderr[-3000:]
