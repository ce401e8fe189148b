"""ipcfp_verify_bundle_json (include/ipcfp.h): verify_proof_bundle from the bundle's JSON text. Every case is compared with the composition
the header defines it by — ipcfp_bundle_from_json, the trust callbacks, ipcfp_store_create(IPCFP_STORE_VERIFY_CIDS) and the two batched
verifiers — run here on the same text through ctypes: verdicts, returned proofs, data blob, tipset fields, block count, status and index.
Canonical text must take the device parser (parsed_on_device), any other spelling the host parser, with the same results."""
import base64
import ctypes as C
import json

import numpy as np
import pytest

from ipc_filecoin_proofs_b200 import _abi as A
from ipc_filecoin_proofs_b200 import bundle_json as J
from tests.util import adversarial_tipset, spec_of, synth_tipset

pytestmark = pytest.mark.gpu

NO_INDEX = 2 ** 64 - 1


def compose(api, text, trusted_parent=None, trusted_child=None, filter_spec=None, device=0):
    """The composition of existing calls that defines the call: ("ok", summary) or ("err", status, index)."""
    L = api.lib()
    try:
        pb = api.ParsedBundle(text)
    except A.IpcfpError as e:
        return ("err", e.status, NO_INDEX)
    try:
        c = pb.c
        nS, nE = int(c.n_storage_proofs), int(c.n_event_proofs)
        f = pb.tipset_fields()
        sres, eres = np.zeros(max(nS, 1), np.uint8), np.zeros(max(nE, 1), np.uint8)
        child_ok = parent_ok = False
        if nS + nE:
            child_ok = trusted_child is None or bool(trusted_child(f["child_epoch"], f["child_cid"]))
            if nE and child_ok:
                parent_ok = trusted_parent is None or bool(trusted_parent(f["parent_epoch"], f["parent_cids"]))
        if child_ok and (nS or (parent_ok and nE)):
            w = c.witness
            store = C.c_void_p()
            st = L.ipcfp_store_create(w.cids, w.offsets, w.lengths, w.blob, w.blob_size, w.n_blocks, device, A.STORE_VERIFY_CIDS, C.byref(store))
            try:
                if st != A.OK:
                    return ("err", st, int(L.ipcfp_last_error_index()))
                if nS:
                    st = L.ipcfp_verify_storage_proofs(store, C.byref(c.tipset), c.storage_proofs, nS, sres.ctypes.data)
                    if st != A.OK:
                        return ("err", st, int(L.ipcfp_last_error_index()))
                if nE and parent_ok:
                    st = L.ipcfp_verify_event_proofs(store, C.byref(c.tipset), c.event_proofs, nE, c.data_blob, c.data_blob_size,
                                                     C.addressof(filter_spec) if filter_spec is not None else None, eres.ctypes.data)
                    if st != A.OK:
                        i = int(L.ipcfp_last_error_index())
                        return ("err", st, i + nS if i != NO_INDEX else i)
            finally:
                if store:
                    L.ipcfp_store_destroy(store)
        raw_e, blob = pb.event_proofs_raw
        w = pb.witness
        return ("ok", dict(storage=[bool(x) for x in sres[:nS]], events=[bool(x) for x in eres[:nE]], sp=pb.storage_proofs_raw.tobytes(),
                           ep=raw_e.tobytes(), blob=blob.tobytes(), n_blocks=int(w.n_blocks), witness_bytes=int(np.sum(w.lengths, dtype=np.uint64)),
                           tipset=dict(parent_epoch=f["parent_epoch"], child_epoch=f["child_epoch"], parent_cids=f["parent_cids"],
                                       child_cid=f["child_cid"] or None, parent_state_root=f["parent_state_root"] or None)))
    finally:
        pb.close()


def call(api, text, **kw):
    try:
        v = api.verify_bundle_json(text, **kw)
    except A.IpcfpError as e:
        return ("err", e.status, int(e.index)), None
    return ("ok", dict(storage=v.storage_results, events=v.event_results, sp=v.storage_proofs_raw.tobytes(), ep=v.event_proofs_raw.tobytes(),
                       blob=v.data_blob.tobytes(), n_blocks=v.n_blocks, witness_bytes=v.witness_bytes, tipset=v.tipset)), v


def check(api, text, device_path=None, **kw):
    """The call equals the composition; device_path: the path it must have taken (checked when it succeeds)."""
    got, v = call(api, text, **kw)
    exp = compose(api, text, **kw)
    assert got[0] == exp[0], (got[:3] if got[0] == "err" else "ok", exp[:3] if exp[0] == "err" else "ok")
    if got[0] == "err":
        assert got == exp
    else:
        for k in exp[1]:
            assert got[1][k] == exp[1][k], k
        if device_path is not None:
            assert v.parsed_on_device == device_path
    return got, v


def foreign_spec():
    return A.make_event_spec("SomethingElse(bytes32,uint256)", "not-this-subnet", None)


def event_text(api, ts, flags=A.RESULT_JSON):
    r = api.BlockStore.from_tipset(ts).generate_event_proof(ts, spec_of(ts), flags=flags)
    return r.json, r


@pytest.fixture(scope="module")
def unified3(api, ts3_small, oracle_mod):
    slot = oracle_mod.compute_mapping_slot((b"calib-subnet-1" + bytes(32))[:32], 0)
    b = api.BlockStore.from_tipset(ts3_small, verify_cids=True).generate_proof_bundle(ts3_small, [(1001, slot), (1003, slot)], [spec_of(ts3_small)])
    return J.dumps(J.unified_bundle(ts3_small, b))


@pytest.mark.parametrize("cfg", [1, 2, "shapes", "shapes-nofilter"])
def test_canonical_event_bundles(api, synth_mod, cfg):
    ts = synth_tipset(synth_mod, cfg)
    text, r = event_text(api, ts)
    assert r.proofs
    host_text = J.dumps(J.event_bundle(ts, api.BlockStore.from_tipset(ts).generate_event_proof(ts, spec_of(ts))))
    assert host_text == text   # the same text as ipcfp_event_result_to_json / bundle_json.py
    for spec, verified in ((spec_of(ts), True), (foreign_spec(), False), (None, True)):
        got, v = check(api, text, device_path=True, filter_spec=spec)
        assert got[0] == "ok" and len(got[1]["events"]) == len(r.proofs)
        assert got[1]["events"] == [verified] * len(r.proofs)
        assert v.n_blocks == r.witness.n_blocks and v.ms["total"] > 0


def test_canonical_unified_bundle(api, ts3_small, unified3):
    doc = json.loads(unified3)
    assert doc["storage_proofs"]   # config 3's event specs may match nothing: the event list can be empty
    for spec in (spec_of(ts3_small), foreign_spec(), None):
        got, v = check(api, unified3, device_path=True, filter_spec=spec)
        assert got[0] == "ok" and all(got[1]["storage"])


def test_full_tipset_text(api, synth_mod):
    ts = synth_mod.Tipset(synth_mod.config_params(4))
    text, r = event_text(api, ts, flags=A.RESULT_JSON | A.WITNESS_BY_REFERENCE)
    assert len(text) > 50_000_000
    got, v = check(api, text, device_path=True, filter_spec=spec_of(ts))
    assert got[0] == "ok" and all(got[1]["events"]) and len(got[1]["events"]) == len(r.proofs)


def _tamper(text, fn):
    d = json.loads(text)
    fn(d)
    return J.dumps(d)


def _flip_hex(s, at=2):
    return s[:at] + ("1" if s[at] == "0" else "0") + s[at + 1:]


def _flip_block(d, k):
    b = bytearray(base64.b64decode(d["blocks"][k]["data"]))
    b[len(b) // 2] ^= 0x01
    d["blocks"][k]["data"] = base64.b64encode(bytes(b)).decode()


def test_tampered_bundles(api, ts2, ts3_small, unified3):
    text, r = event_text(api, ts2)
    spec = spec_of(ts2)
    p0 = json.loads(text)["proofs"][0]
    other_cid = J.cid_to_string(bytes(json.loads(text)["blocks"][0]["cid"]))
    edits = [
        lambda d: d["proofs"][0].__setitem__("exec_index", d["proofs"][0]["exec_index"] + 1),
        lambda d: d["proofs"][0].__setitem__("event_index", d["proofs"][0]["event_index"] + 1),
        lambda d: d["proofs"][0]["event_data"].__setitem__("emitter", d["proofs"][0]["event_data"]["emitter"] ^ 1),
        lambda d: d["proofs"][0].__setitem__("message_cid", other_cid),
        lambda d: d["proofs"][0]["event_data"]["topics"].__setitem__(0, _flip_hex(d["proofs"][0]["event_data"]["topics"][0], 10)),
        lambda d: d["proofs"][0]["event_data"].__setitem__("data", _flip_hex(d["proofs"][0]["event_data"]["data"], 2) if len(p0["event_data"]["data"]) > 2 else "0x00"),
        lambda d: [p.__setitem__("child_epoch", p["child_epoch"] + 1) for p in d["proofs"]],
        lambda d: [p.__setitem__("parent_epoch", p["parent_epoch"] - 1) for p in d["proofs"]],
        lambda d: d["proofs"][-1].__setitem__("child_epoch", d["proofs"][-1]["child_epoch"] + 1),   # two tipset pairs: refused
        lambda d: d["blocks"].pop(len(d["blocks"]) // 2),
    ]
    for k, e in enumerate(edits):
        check(api, _tamper(text, e), filter_spec=spec)
    n_blocks = len(json.loads(text)["blocks"])
    for k in (0, n_blocks // 2, n_blocks - 1):
        got, _ = check(api, _tamper(text, lambda d: _flip_block(d, k)), filter_spec=spec)
        assert got == ("err", A.ERR_CID_MISMATCH, k)
    # storage: value, storage root, and an event error indexed after the storage proofs
    uedits = [
        lambda d: d["storage_proofs"][0].__setitem__("value", _flip_hex(d["storage_proofs"][0]["value"], 65)),
        lambda d: d["storage_proofs"][-1].__setitem__("storage_root", d["storage_proofs"][0]["actor_state_cid"]),
        lambda d: d["blocks"].pop(0),
    ]
    for e in uedits:
        check(api, _tamper(unified3, e), filter_spec=spec_of(ts3_small))
    # a unified bundle whose event proofs fail: the index counts the storage proofs first
    doc = json.loads(text)
    uni = J.dumps(dict(storage_proofs=[], event_proofs=doc["proofs"], blocks=doc["blocks"]))
    check(api, uni, device_path=True, filter_spec=spec)
    check(api, _tamper(uni, lambda d: d["event_proofs"][1].__setitem__("exec_index", 10 ** 9)), filter_spec=spec)


def test_non_canonical_texts_take_the_host_parser(api, ts1):
    text, r = event_text(api, ts1)
    spec = spec_of(ts1)
    want, _ = call(api, text, filter_spec=spec)
    doc = json.loads(text)

    def variant(fn):
        d = json.loads(text)
        fn(d)
        return json.dumps(d, separators=(",", ":"))

    cid_str = J.cid_to_string(bytes(doc["blocks"][0]["cid"]))
    texts = [
        json.dumps(doc, indent=2),
        json.dumps(dict(blocks=doc["blocks"], proofs=doc["proofs"]), separators=(",", ":")),                     # reordered keys
        variant(lambda d: d.__setitem__("note", [1, 2.5, None])),                                                # an unknown field
        text.replace('"proofs"', '"\\u0070roofs"', 1),                                                          # an escape
        variant(lambda d: d["blocks"][0].__setitem__("cid", {"/": cid_str})),
        variant(lambda d: d["blocks"][0].__setitem__("cid", cid_str)),
        variant(lambda d: d["proofs"][0]["event_data"]["topics"].__setitem__(0, d["proofs"][0]["event_data"]["topics"][0].upper().replace("0X", "0x"))),
        " " + text,
    ]
    for t in texts:
        got, v = check(api, t, device_path=False, filter_spec=spec)
        assert got[0] == "ok" and got[1]["events"] == want[1]["events"] and got[1]["ep"] == want[1]["ep"]


def test_malformed_texts_return_the_host_parser_status(api, ts1):
    text, _ = event_text(api, ts1)
    rng = np.random.default_rng(5)
    for cut in rng.integers(1, len(text) - 1, 200):
        got, _ = check(api, text[:int(cut)])
        assert got == ("err", A.ERR_INVALID_ARG, NO_INDEX)

    def mutated(fn):
        d = json.loads(text)
        fn(d)
        return json.dumps(d)

    bad = [text + " x", "[]", '{"blocks":[]}',
           mutated(lambda d: d["proofs"][0].__setitem__("exec_index", -1)),
           mutated(lambda d: d["proofs"][0].__setitem__("exec_index", 1.5)),
           mutated(lambda d: d["proofs"][0].__setitem__("exec_index", 2 ** 64)),
           mutated(lambda d: d["proofs"][0]["event_data"].__setitem__("data", "0xabc")),
           mutated(lambda d: d["proofs"][0]["event_data"].__setitem__("data", "abcd")),
           mutated(lambda d: d["proofs"][0].__setitem__("message_cid", "bafy!")),
           mutated(lambda d: d["proofs"][0].__setitem__("message_cid", "baeaaa")),
           mutated(lambda d: d["blocks"][0].__setitem__("data", d["blocks"][0]["data"][:-1])),
           mutated(lambda d: d["blocks"][0].__setitem__("cid", d["blocks"][0]["cid"][:-1])),
           mutated(lambda d: d["proofs"][0]["event_data"].__setitem__("topics", ["0x00"])),
           mutated(lambda d: d["proofs"][0].pop("event_index"))]
    for t in bad:
        got, _ = check(api, t)
        assert got[0] == "err"


def test_seeded_mutations_match_the_composition(api, ts1):
    text, _ = event_text(api, ts1)
    spec = spec_of(ts1)
    rng = np.random.default_rng(2026)
    alpha = b'0123456789abcdefABCDEF",{}[]:- =/+'
    outcomes = {}
    for _ in range(2000):
        b = bytearray(text.encode())
        for _ in range(int(rng.integers(1, 4))):
            at = int(rng.integers(0, len(b)))
            op = int(rng.integers(0, 3))
            if op == 0:
                b[at] = alpha[int(rng.integers(0, len(alpha)))]
            elif op == 1:
                del b[at]
            else:
                b.insert(at, alpha[int(rng.integers(0, len(alpha)))])
        got, v = check(api, bytes(b), filter_spec=spec)
        key = (got[0], got[1] if got[0] == "err" else v.parsed_on_device)
        outcomes[key] = outcomes.get(key, 0) + 1
    assert outcomes.get(("ok", True), 0) > 0 and sum(n for k, n in outcomes.items() if k[0] == "err") > 0, outcomes


def test_trust_callbacks(api, ts2, ts3_small, unified3):
    text, r = event_text(api, ts2)
    calls = []

    def parent(epoch, cids):
        calls.append(("parent", epoch, cids))
        return False

    def child(epoch, cid):
        calls.append(("child", epoch, cid))
        return True

    got, v = check(api, text, device_path=True, trusted_parent=parent, trusted_child=child)
    assert [c[0] for c in calls] == ["child", "parent"] * 2   # once each in the call, once each in the composition
    assert calls[0] == calls[2] and calls[1] == calls[3]
    assert calls[0][1:] == (int(ts2.child_epoch), bytes(ts2.child_cid))
    assert calls[1][1:] == (int(ts2.parent_epoch), bytes(np.asarray(ts2.parent_cids, dtype=np.uint8).reshape(-1)))
    assert got[1]["events"] == [False] * len(r.proofs)
    # untrusted parent on a unified bundle: events false, storage verified
    got, _ = check(api, unified3, device_path=True, trusted_parent=lambda e, c: False)
    assert all(got[1]["storage"]) and not any(got[1]["events"])
    # untrusted child: everything false, and the call succeeds even with a corrupted block (no store is built)
    n_calls = []
    bad = _tamper(unified3, lambda d: _flip_block(d, 0))
    got, _ = check(api, bad, device_path=True, trusted_child=lambda e, c: n_calls.append(1) or False,
                   trusted_parent=lambda e, c: n_calls.append(2) or True)
    assert got[0] == "ok" and not any(got[1]["storage"]) and not any(got[1]["events"])
    assert n_calls == [1, 1]   # once here, once in the composition; the parent is not asked


def test_several_prefixes_and_duplicates(api, synth_mod):
    base = synth_mod.Tipset(synth_mod.config_params(1))
    for family in ("B", "C"):
        ts, _ = adversarial_tipset(base, family, seed=3)
        text, r = event_text(api, ts)
        check(api, text, device_path=None, filter_spec=spec_of(ts))
        prefixes = {bytes(b["cid"][:6]) for b in json.loads(text)["blocks"]}
        assert len(prefixes) > 1
    # duplicate blocks in the text: the first occurrence wins, as in ipcfp_store_create
    text, r = event_text(api, base)
    d = json.loads(text)
    d["blocks"] = d["blocks"] + d["blocks"][:3]
    check(api, J.dumps(d), device_path=True, filter_spec=spec_of(base))


def test_empty_bundles(api):
    for t in ('{"proofs":[],"blocks":[]}', '{"storage_proofs":[],"event_proofs":[],"blocks":[]}'):
        got, v = check(api, t, device_path=True)
        assert got[0] == "ok" and got[1]["storage"] == [] and got[1]["events"] == [] and v.n_blocks == 0


def test_existing_calls_issue_the_same_launches(api, ts2):
    """The host-array front ends of store_create and the verifiers issue the launches they always did (DESIGN.md records the count of this
    flow): the composition's count is the same before and after device-parsed calls, and the device path issues its own kernels."""
    text, _ = event_text(api, ts2)
    spec = spec_of(ts2)

    def launches(fn):
        n0 = api.kernel_launch_count()
        fn()
        return api.kernel_launch_count() - n0

    before = launches(lambda: compose(api, text, filter_spec=spec))
    assert before > 0
    dev = launches(lambda: call(api, text, filter_spec=spec))
    assert dev > before   # the parse kernels on top of the same store and verifier launches
    assert launches(lambda: compose(api, text, filter_spec=spec)) == before
    print(f"launches: composition {before}, device path {dev}")
