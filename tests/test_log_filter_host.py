"""Log filters on the CPU: the device code of the predicate and of the staged pass 1 with it, compiled for the host
(tests/host_fuzz/emu_log_filter.cu, also under AddressSanitizer + UBSan with `make sanitize`); the ctypes layout of ipcfp_log_filter; the
Python LogFilter's parsing and predicate; and the two restated generators (tests/oracle_logs.py, tests/oracle_logs.cpp) against each other
and against the oracles' spec generators for the filter a spec stands for."""
import ctypes as C
import os
import subprocess
import tempfile

import pytest

from ipc_filecoin_proofs_b200 import _abi as A
from ipc_filecoin_proofs_b200 import api
from oracle import pyoracle as P
from tests import oracle_logs as OL
from tests.test_host_fuzz import _harness
from tests.util import dict_of

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_log_filter_layout_matches_the_header():
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "ipcfp.h"', "int main(void) {",
             'printf("size %zu\\n", sizeof(ipcfp_log_filter));',
             'printf("max %u %u\\n", IPCFP_LOG_FILTER_MAX_VALUES, IPCFP_LOG_FILTER_MAX_EMITTERS);']
    for f, _ in A.LogFilterC._fields_:
        lines.append(f'printf("{f} %zu\\n", offsetof(ipcfp_log_filter, {f}));')
    lines.append("return 0; }")
    with tempfile.TemporaryDirectory() as td:
        src, exe = os.path.join(td, "l.c"), os.path.join(td, "l")
        open(src, "w").write("\n".join(lines))
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), "-o", exe, src])
        got = dict(l.split(" ", 1) for l in subprocess.check_output([exe], text=True).strip().splitlines())
    assert int(got["size"]) == C.sizeof(A.LogFilterC)
    assert got["max"].split() == [str(A.LOG_FILTER_MAX_VALUES), str(A.LOG_FILTER_MAX_EMITTERS)]
    for f, _ in A.LogFilterC._fields_:
        assert int(got[f]) == getattr(A.LogFilterC, f).offset, f


def test_log_filter_parsing_and_predicate():
    a, b = bytes(31) + b"\x01", bytes([0xFF] * 32)
    f = api.LogFilter(emitters=[7, 9], topics=[None, "0x" + a.hex(), [a, b]])
    assert f.topics == [None, [a], [a, b]]
    c, keep = f.as_c()
    assert c.n_positions == 3 and c.n_emitters == 2 and list(c.n_values) == [0, 1, 2, 0] and not c.values[0] and not c.values[3]
    assert f.matches(7, [b, a, b]) and f.matches(9, [a, a, a, a, a])
    assert not f.matches(8, [b, a, b]) and not f.matches(7, [b, a]) and not f.matches(7, [b, b, b])
    assert api.LogFilter().matches(1, []) and not api.LogFilter(topics=[None]).matches(1, [])
    assert api.LogFilter(topics=[[], a]).topics == [None, [a]]   # an empty list is a wildcard, in Python as in the C struct
    with pytest.raises(ValueError):
        api.LogFilter(topics=[None] * 5)
    with pytest.raises(ValueError):
        api.LogFilter(topics=[bytes(31)])
    # the restatement's predicate is the same rule
    em, pos = OL.filter_of(f)
    for emitter, topics in [(7, [b, a, b]), (9, [a, a, a, a, a]), (8, [b, a, b]), (7, [b, a]), (7, [b, b, b])]:
        assert OL.log_matches(em, pos, emitter, (topics, b"")) == f.matches(emitter, topics)
    assert not OL.log_matches(set(), [], 1, None)


@pytest.mark.parametrize("which", ["ts1", "ts2"])
def test_restated_generator_equals_the_spec_generator(request, which):
    ts = request.getfixturevalue(which)
    d = dict_of(ts)
    exp = P.generate_event_proof(d, ts, ts.event_signature, ts.topic1, ts.actor_filter)
    emitters = set() if ts.actor_filter is None else {int(ts.actor_filter)}
    got = OL.generate_log_proof(d, ts, emitters, [{P.keccak256(ts.event_signature.encode())}, {P.ascii_to_bytes32(ts.topic1)}])
    assert got["matching"] == exp["matching"] and got["proofs"] == exp["proofs"] and got["witness"] == exp["witness"]
    assert len(got["proofs"]) > 0
    # a wildcard over two topics finds at least as much
    wide = OL.generate_log_proof(d, ts, set(), [None, None])
    assert set(exp["matching"]) <= set(wide["matching"]) and len(wide["proofs"]) >= len(got["proofs"])


def test_log_filter_device_code_emulated_on_cpu():
    """emu_log_filter.cu: the staged pass-1 lane with a LogFilter against the arena path, under the adversarial copy model, and
    event_matches(LogFilter) against the filter evaluated on the C++ oracle's decode, on random filters and events."""
    exe, env = _harness("emu_log_filter", with_synth=False)
    out = subprocess.run([exe, "400", "17"], capture_output=True, text=True, env=env)
    assert out.returncode == 0, (out.stdout + out.stderr)[-3000:]
    assert "ok: log filter staged == arena and per item == oracle, 4 geometries x 400 warps" in out.stdout, out.stdout


@pytest.mark.parametrize("which", ["ts1", "ts2"])
def test_cpp_and_python_restatements_agree(request, which):
    """tests/oracle_logs.cpp against tests/oracle_logs.py on wildcards, every topic position, value and emitter sets; the spec's filter
    against the C++ oracle's spec generator."""
    import numpy as np
    import oracle
    ts = request.getfixturevalue(which)
    d = dict_of(ts)
    cpp = OL.CppOracle(ts)
    logs = OL.candidate_logs(d, ts)
    rng = np.random.default_rng(5)
    pick = lambda k, n: [t[k] for _, t in logs if len(t) > k][:n] + [bytes(rng.integers(0, 256, 32, dtype=np.uint8)) for _ in range(n)]  # noqa: E731
    t0 = P.keccak256(ts.event_signature.encode())
    spec_f = api.LogFilter(None if ts.actor_filter is None else [int(ts.actor_filter)], [t0, P.ascii_to_bytes32(ts.topic1)])
    filters = [spec_f, api.LogFilter(), api.LogFilter(topics=[None] * 3), api.LogFilter(topics=[None, pick(1, 70)]),
               api.LogFilter(topics=[t0, None, pick(2, 3)]), api.LogFilter(topics=[None, None, None, pick(3, 5)]),
               api.LogFilter(emitters=sorted({e for e, _ in logs})[:2] * 3, topics=[pick(0, 2)])]
    for f in filters:
        exp = OL.generate_log_proof(d, ts, *OL.filter_of(f))
        st, got = cpp.generate(ts, f)
        assert st == "ok"
        keys = [(i, j, e, tuple(bytes(t) for t in tp), bytes(dt), bytes(m)) for i, j, e, tp, dt, m in exp["proofs"]]
        assert got.matching.tolist() == exp["matching"] and [p.key() for p in got.proofs] == keys
        assert [bytes(c) for c in got.witness.cids] == exp["witness"]
    spec = A.make_event_spec(ts.event_signature, ts.topic1, ts.actor_filter)
    ref = oracle.Store.from_tipset(ts).generate_event_proof(ts, spec)
    got = cpp.generate(ts, spec_f)[1]
    assert got.matching.tolist() == ref.matching.tolist() and [p.key() for p in got.proofs] == [p.key() for p in ref.proofs]
    assert got.witness.blocks() == ref.witness.blocks() and len(ref.proofs) > 0
