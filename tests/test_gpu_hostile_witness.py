"""The GPU verifiers on hostile witnesses whose every block hashes to its CID (tests/hostile_witness.py). Every case and batch goes
through three routes: api.verify_event_proofs / verify_storage_proofs, and verify_bundle_json on the canonical text (parsed on the
device) and on an indented text (the host parser), the latter two with a trust callback that accepts the re-anchored child and one
that rejects it. Each route returns the case's stated verdicts or (status, first failing proof), which are the C++ oracle's
(tests/test_hostile_witness.py pins them on the CPU and is re-checked here); a rejected child gives false everywhere and no error."""
import json

import pytest

from ipc_filecoin_proofs_b200 import _abi as A
from ipc_filecoin_proofs_b200 import bundle_json as J
from tests import hostile_witness as H
from tests.test_hostile_witness import COUNTS, oracle_outcome

pytestmark = pytest.mark.gpu


def _outcome(fn):
    try:
        return fn()
    except A.IpcfpError as e:
        return (e.status, int(e.index))


def _texts(c):
    """(canonical text, indented text) of the case's bundle."""
    r = c.result()
    blocks = J.proof_blocks(r.witness)
    if c.kind == "event":
        doc = {"proofs": J.event_proofs(c.ts, r), "blocks": blocks}
    else:
        doc = {"storage_proofs": J.storage_proofs(c.ts, r), "event_proofs": [], "blocks": blocks}
    return J.dumps(doc), json.dumps(doc, indent=1)


def _json_outcome(api, text, kind, **kw):
    def run():
        v = api.verify_bundle_json(text, **kw)
        return v.event_results if kind == "event" else v.storage_results, v.parsed_on_device
    return _outcome(run)


def run_case(api, c, json_routes=True):
    want = c.expect
    if c.kind == "event":
        got = _outcome(lambda: api.verify_event_proofs(c.witness(), c.ts, c.result()))
    else:
        got = _outcome(lambda: api.verify_storage_proofs(c.witness(), c.ts, c.result()))
    assert got == want, (c.name, "direct", got if isinstance(got, tuple) else sum(got), want if c.fails else sum(want))
    if not json_routes:
        return
    child = bytes(c.ts.child_cid)
    for text, device in zip(_texts(c), (True, False)):
        for trusted in (True, False):
            out = _json_outcome(api, text, c.kind, trusted_child=lambda e, cid, t=trusted: t and cid == child)
            if trusted:
                if c.fails:
                    assert out == want, (c.name, device, out)
                else:
                    assert out == (want, device), (c.name, device, out[0] if isinstance(out[0], int) else sum(out[0]))
            else:
                assert out == ([False] * len(c.proofs), device), (c.name, device, "untrusted child")


def test_event_cases(api, oracle_mod):
    cases = H.event_cases()
    assert len(cases) == COUNTS["event"]
    for c in cases:
        assert oracle_outcome(oracle_mod, c) == c.expect, c.name
        run_case(api, c)


def test_storage_cases(api, oracle_mod, ts3_small):
    cases = H.storage_cases(ts3_small)
    assert len(cases) == COUNTS["storage"]
    for c in cases:
        assert oracle_outcome(oracle_mod, c) == c.expect, c.name
        run_case(api, c)


@pytest.mark.parametrize("kind", ["event", "storage"])
def test_batches(api, oracle_mod, ts3_small, kind):
    """Faults planted in different proofs of one call, at 1, 4, 5, 128, 129 and 16 385 proofs (one warp per proof, four per CTA):
    the first failing proof in order is the one reported, and a batch without fault gives the oracle's verdicts."""
    batches = H.event_batches() if kind == "event" else H.storage_batches(ts3_small)
    assert len(batches) == COUNTS[f"{kind}_batches"]
    for c in batches:
        assert oracle_outcome(oracle_mod, c) == c.expect, c.name
        run_case(api, c, json_routes=len(c.proofs) <= 129 or c.name.endswith("generated") or "at0" in c.name)
