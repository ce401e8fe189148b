"""The message-selected event call on the CPU: the Python restatement (tests/oracle_messages.py) against the restated log-filter generator
(tests/oracle_logs.py) it restricts, and the device code of the selection (csrc/msg_select_items.cuh) compiled for the host
(tests/host_fuzz/emu_message_select.cu, also under AddressSanitizer + UBSan with `make sanitize`) against the Python selection."""
import random
import subprocess

import pytest

from tests import oracle_logs as OL
from tests import oracle_messages as OM
from tests.test_host_fuzz import _harness
from tests.util import dict_of

U64 = OM.NOT_EXECUTED


@pytest.mark.parametrize("which", ["ts1", "ts2", "ts3_small"])
def test_whole_execution_order_restates_the_log_filter_generator(request, which):
    ts = request.getfixturevalue(which)
    d = dict_of(ts)
    order = OM.execution_order(d, ts)
    for emitters, positions in ((set(), []), (set(), [None, None]), ({int(ts.actor_filter)} if ts.actor_filter is not None else set(), [None])):
        a = OL.generate_log_proof(d, ts, emitters, positions)
        b = OM.generate_message_log_proof(d, ts, order, emitters, positions)
        assert b["exec_indices"] == list(range(len(order)))
        assert (a["matching"], a["proofs"], a["witness"]) == (b["matching"], b["proofs"], b["witness"])


def test_subsets_restrict_the_log_filter_generator(ts2):
    ts = ts2
    d = dict_of(ts)
    order = OM.execution_order(d, ts)
    full = OL.generate_log_proof(d, ts, set(), [])
    rng = random.Random(4)
    strangers = [bytes(rng.getrandbits(8) for _ in range(38)) for _ in range(3)]
    for msgs in ([], order[:1], rng.sample(order, 50), order[3:6] * 2, strangers + order[7:9]):
        r = OM.generate_message_log_proof(d, ts, msgs)
        pos = {c: i for i, c in enumerate(order)}
        assert r["exec_indices"] == [pos.get(c, U64) for c in msgs]
        sel = {pos[c] for c in msgs if c in pos}
        assert r["matching"] == [i for i in full["matching"] if i in sel]
        assert r["proofs"] == [p for p in full["proofs"] if p[0] in sel]


def test_read_set_holds_no_unselected_events_amt(ts1):
    ts = ts1
    d = dict_of(ts)
    order = OM.execution_order(d, ts)
    msgs = order[:5]
    sel, _ = OM.select(order, int(ts.n_receipts), msgs)
    reads = OM.read_set(d, ts, msgs)
    others = OM.events_blocks(d, ts, [i for i in range(int(ts.n_receipts)) if i not in sel]) - OM.events_blocks(d, ts, sel)
    assert others and not (reads & others)
    assert OM.events_blocks(d, ts, sel) <= reads


def _emu_input(rng, n_exec, n_req, n_receipts, dup):
    """A random execution order (distinct CIDs of one 6-byte prefix; about a third share the first digest word and differ only in later
    words) and requests drawn from it, from outside it and repeated."""
    order = []
    seen = set()
    head = bytes([1, 0x71, 0xa0, 0xe4, 2, 0x20])
    shared_w0 = bytes(rng.getrandbits(8) for _ in range(8))   # digest bytes 0..7: the first word the sort and the search compare
    while len(order) < n_exec:
        if rng.random() < 0.3:   # the same first word, decided by a later word (often only the last one)
            tail = bytes(23) + bytes([rng.getrandbits(8)]) if rng.random() < 0.5 else bytes(rng.getrandbits(8) for _ in range(24))
            c = head + shared_w0 + tail
        else:
            c = head + bytes(rng.getrandbits(8) for _ in range(32))
        if c not in seen:
            seen.add(c)
            order.append(c)
    req = []
    for _ in range(n_req):
        if order and rng.random() < 0.7:
            req.append(order[rng.randrange(len(order))])
        else:
            req.append(bytes(rng.getrandbits(8) for _ in range(38)))
    if dup and req:
        req += req[: max(1, len(req) // 3)]
    return order, req


def test_emulated_selection_matches_the_python_selection():
    exe, env = _harness("emu_message_select", with_synth=False)
    rng = random.Random(9)
    for case in range(60):
        n_exec = rng.choice([0, 1, 5, 64, 300])
        n_req = rng.choice([0, 1, 3, 40, 200])
        n_receipts = rng.choice([0, n_exec // 2, n_exec, n_exec + 3])
        order, req = _emu_input(rng, n_exec, n_req, n_receipts, case % 2 == 1)
        # the order is handed over as exec_raw in a shuffled layout with exec_idx pointing into it, as the dedup leaves it
        perm = list(range(len(order)))
        rng.shuffle(perm)
        raw = [None] * len(order)
        for i, p in enumerate(perm):
            raw[p] = order[i]
        text = "%d %d %d\n" % (len(order), len(req), n_receipts)
        text += "".join(c.hex() + "\n" for c in raw) + "".join("%d\n" % p for p in perm) + "".join(c.hex() + "\n" for c in req)
        out = subprocess.run([exe], input=text, capture_output=True, text=True, check=True, env=env).stdout.split()
        sel, idx = OM.select(order, n_receipts, req)
        n_sel = int(out[0])
        assert [int(x) for x in out[1:1 + n_sel]] == sel, case
        assert [int(x) for x in out[1 + n_sel:1 + n_sel + len(req)]] == idx, case


def _match_input(path, ts, selected, emitters=()):
    import struct
    n = int(ts.n_blocks)
    with open(path, "wb") as f:
        f.write(struct.pack("<Q", n))
        for k in range(n):
            o, ln = int(ts.offsets[k]), int(ts.lengths[k])
            f.write(bytes(ts.cids[k]) + struct.pack("<I", ln) + bytes(ts.blob[o:o + ln]))
        f.write(struct.pack("<Q", int(ts.n_receipts)))
        for i in range(int(ts.n_receipts)):
            f.write(struct.pack("<B", 1 if ts.has_events_root[i] else 0) + bytes(ts.events_roots[i]))
        f.write(struct.pack("<Q", len(selected)) + b"".join(struct.pack("<I", i) for i in selected))
        f.write(struct.pack("<I", len(emitters)) + b"".join(struct.pack("<Q", e) for e in emitters))


def _expected_match(d, ts, selected, emitters=()):
    """Pass 1's per-receipt result restated on the Python oracle: (first fault (index, code) or None, {i: (matched, events, bytes)})."""
    from ipc_filecoin_proofs_b200 import _abi as A
    from oracle import pyoracle as P
    from tests import event_amts as E
    fault, per = None, {}
    for i in selected:
        per[i] = (0, 0, 0)
        if not ts.has_events_root[i]:
            continue
        acc = [0, 0]

        def f(j, se):
            log = P.extract_evm_log(se[1])
            if log is not None and (not emitters or se[0] in emitters):
                acc[0] += 1
                acc[1] += 32 * len(log[0]) + len(log[1])
        try:
            E.walk(d, bytes(ts.events_roots[i]))   # the AMT's structure, as strictly as the engine reads it
            P.Amt(bytes(ts.events_roots[i]), P.Recorder(d), 3).for_each(f)
        except E.Fault as e:
            fault = fault or (i, 1 if e.status == A.ERR_MISSING_BLOCK else 2)
            continue
        except P.MissingBlock:
            fault = fault or (i, 1)
            continue
        except Exception:
            fault = fault or (i, 2)
            continue
        per[i] = (1 if acc[0] else 0, acc[0], acc[1])
    return fault, per


def test_emulated_match_on_hand_built_events_amts(tmp_path):
    """msg_match_item on the host over every case of tests/event_amts.py (events AMTs at every bit width and height, refused roots and
    nodes, missing blocks, receipts without an events root), selections that include the faulty receipt or leave it out, with and
    without an emitter set: the first fault (pass 1, its receipt, missing or decode) and every selected receipt's match, events and bytes
    equal the Python oracle's."""
    from tests import event_amts as E
    exe, env = _harness("emu_message_select", with_synth=False)
    rng = random.Random(12)
    n_cases = n_faults = 0
    for c in E.catalogue(E.base_tipset()):
        if c.big:
            continue
        ts = c.ts
        d = dict_of(ts)
        nr = int(ts.n_receipts)
        for take_fault in (True, False):
            sel = sorted(set(rng.sample(range(nr), min(nr, 40))) | ({E.FAULT_RECEIPT} if take_fault and nr > E.FAULT_RECEIPT else set()))
            if not take_fault:
                sel = [i for i in sel if i != E.FAULT_RECEIPT]
            emitters = () if rng.random() < 0.5 else tuple({int(x) for x in (1001, 1002)})
            path = str(tmp_path / "in.bin")
            _match_input(path, ts, sel, emitters)
            out = subprocess.run([exe, "match", path], capture_output=True, text=True, check=True, env=env).stdout.splitlines()
            fault, per = _expected_match(d, ts, sel, set(emitters))
            head = out[0].split()
            if fault is None:
                assert head == ["err", "none"], (c.name, out[0])
            else:
                assert head == ["err", "4", str(fault[0]), str(fault[1])], (c.name, out[0], fault)
                n_faults += 1
            got = {int(x.split()[0]): tuple(int(v) for v in x.split()[1:]) for x in out[1:]}
            assert got == per, c.name
            n_cases += 1
    assert n_cases > 20 and n_faults > 5


def _agree(ts, d, cpp, msgs, flt=None):
    """The two restatements on one call: the same result, or both fail. → the C++ one's outcome."""
    ef, pos = (set(), []) if flt is None else OL.filter_of(flt)
    try:
        py = ("ok", OM.generate_message_log_proof(d, ts, msgs, ef, pos))
    except Exception:
        py = ("err",)
    ref = cpp.generate(ts, msgs, flt)
    if ref[0] == "err":
        assert py[0] == "err"
        return ref
    assert py[0] == "ok"
    py, got, idx = py[1], ref[1], ref[2]
    keys = [(i, j, e, tuple(bytes(t) for t in tp), bytes(dt), bytes(m)) for i, j, e, tp, dt, m in py["proofs"]]
    assert idx == py["exec_indices"] and got.matching.tolist() == py["matching"]
    assert [p.key() for p in got.proofs] == keys and [bytes(c) for c in got.witness.cids] == py["witness"]
    return ref


@pytest.mark.parametrize("which", ["ts1", "ts2", "ts3_small"])
def test_cpp_restatement_equals_python_restatement(request, which):
    from ipc_filecoin_proofs_b200 import api
    ts = request.getfixturevalue(which)
    d = dict_of(ts)
    order = OM.execution_order(d, ts)
    cpp = OM.CppOracle(ts)
    rng = random.Random(21)
    strangers = [order[0][:6] + bytes(rng.getrandbits(8) for _ in range(32)) for _ in range(2)]
    lists = [[], order, order[:1], rng.sample(order, min(60, len(order))), order[2:5] * 2, strangers + order[9:11]]
    spec = api.LogFilter([int(ts.actor_filter)] if ts.actor_filter is not None else None, [None])
    for msgs in lists:
        for flt in (None, spec):
            assert _agree(ts, d, cpp, msgs, flt)[0] == "ok"


def test_cpp_restatement_on_hand_built_amts():
    """Rootless receipts, receipts past the execution order and faulty events AMTs: both restatements agree (or both fail)."""
    from tests import event_amts as E
    from tests import message_amts as MA
    n_ok = n_err = 0
    for c in E.catalogue(E.base_tipset()) + MA.shared_cases(MA.base_tipset()):
        if getattr(c, "big", False) or getattr(c, "large", False):
            continue
        ts = c.ts
        d = dict_of(ts)
        try:
            order = OM.execution_order(d, ts)
        except Exception:
            continue
        rng = random.Random(len(order))
        msgs = rng.sample(order, min(len(order), 50)) + order[int(ts.n_receipts):][:3]
        if len(order) > 77:
            msgs.append(order[77])
        r = _agree(ts, d, OM.CppOracle(ts), msgs)
        n_ok += r[0] == "ok"
        n_err += r[0] == "err"
    assert n_ok > 10 and n_err > 3
