"""Bundles of log filters on the CPU: the Python composition (pyoracle's storage generator, tests/oracle_logs.py) and the C++ composition
(the C++ oracle's storage generator, tests/oracle_logs.cpp) of tests/log_bundles.py agree on every filter set with 0, 2 and 12 storage
specs, on failures too; and the composition of the filters the specs stand for is the C++ oracle's spec bundle."""
import pytest

import oracle
from tests import log_bundles as LB
from tests import oracle_logs as OL
from tests.util import dict_of

SYNTH_STATE = dict(n_receipts=300, events_per_receipt=3, match_ppm=200000, has_actor_filter=0, n_actors=16, hamt_entries=300,
                   null_root_permille=100)


@pytest.fixture(scope="module")
def state_ts(synth_mod):
    return synth_mod.Tipset(synth_mod.config_params(2, with_state_tree=1, **SYNTH_STATE))


@pytest.mark.parametrize("n_sspecs", [0, 2, 12])
def test_compositions_agree(state_ts, n_sspecs):
    ts = state_ts
    d = dict_of(ts)
    sspecs = LB.storage_specs(ts, n_sspecs)
    ostore, cpp = oracle.Store.from_tipset(ts), OL.CppOracle(ts)
    sets = LB.filter_sets(ts, OL.candidate_logs(d, ts))
    n_events = 0
    for name, filters in sets.items():
        py = LB.py_bundle(d, ts, sspecs, filters)
        cc = LB.cpp_bundle(ts, sspecs, filters, ostore, cpp)
        LB.assert_compositions_agree(py, cc)
        assert cc[0] == "ok", name
        n_events += sum(len(e.proofs) for e in cc[1]["events"])
    assert n_events > 0


def test_failures_agree(state_ts):
    """A storage spec for an actor the state tree lacks fails both compositions before any filter runs."""
    ts = state_ts
    d = dict_of(ts)
    sspecs = LB.storage_specs(ts, 2) + [(1000 + int(ts.params.n_actors) + 7, LB.storage_specs(ts, 1)[0][1])]
    py = LB.py_bundle(d, ts, sspecs, [LB.spec_filter(ts.event_signature, ts.topic1)])
    cc = LB.cpp_bundle(ts, sspecs, [LB.spec_filter(ts.event_signature, ts.topic1)])
    assert py[0] == cc[0] == "err" and cc[2] == 2


def test_spec_filters_compose_the_spec_bundle(state_ts):
    import numpy as np
    from ipc_filecoin_proofs_b200 import _abi as A
    ts = state_ts
    especs = [A.make_event_spec(ts.event_signature, ts.topic1, ts.actor_filter), A.make_event_spec(ts.event_signature, "calib-subnet-2", None),
              A.make_event_spec("NoSuchEvent(bytes32)", "no-such-topic", None)]
    sspecs = LB.storage_specs(ts, 12)
    ref = oracle.Store.from_tipset(ts).generate_proof_bundle(ts, sspecs, especs)
    cc = LB.cpp_bundle(ts, sspecs, [LB.filter_of_cspec(s) for s in especs])
    assert cc[0] == "ok"
    cc = cc[1]
    assert [vars(p) for p in cc["storage"].proofs] == [vars(p) for p in ref.storage.proofs]
    for r, e in zip(cc["events"], ref.events):
        assert r.matching.tolist() == e.matching.tolist() and [p.key() for p in r.proofs] == [p.key() for p in e.proofs]
        assert np.array_equal(r.witness.cids, e.witness.cids)
    assert cc["union"] == [bytes(c) for c in ref.witness.cids]


def test_verify_check_of_a_filter_set_emulated_on_cpu():
    """emu_log_bundle.cu: verify_check(LogFilterAny), the check_event step of verify_event_item<LogFilterAny>, compiled for the host,
    on random filter sets and events, against the Python predicate (LogFilter.matches, OR over the set)."""
    import json
    import subprocess

    from ipc_filecoin_proofs_b200 import api
    from tests.test_host_fuzz import _harness
    exe, env = _harness("emu_log_bundle", with_synth=False)
    out = subprocess.run([exe, "300", "29"], capture_output=True, text=True, env=env)
    assert out.returncode == 0, (out.stdout + out.stderr)[-3000:]
    lines = out.stdout.splitlines()
    assert lines[-1].startswith("ok: 19200 events")
    hits = misses = 0
    for line in lines[:-1]:
        case = json.loads(line)
        filters = [api.LogFilter(emitters=f["emitters"], topics=[None if t is None else [bytes.fromhex(v) for v in t] for t in f["topics"]])
                   for f in case["filters"]]
        for ev in case["events"]:
            topics = [bytes.fromhex(t) for t in ev["topics"]]
            want = bool(ev["some"]) and any(f.matches(ev["emitter"], topics) for f in filters)
            assert bool(ev["got"]) == want, (case["filters"], ev)
            hits += want
            misses += not want
    assert hits > 500 and misses > 500
