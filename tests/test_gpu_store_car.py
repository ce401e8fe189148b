"""ipcfp_store_create_car (include/ipcfp.h) on the GPU: a block store straight from a CARv1 (tests/car_files.py) must be the store of the
composed route — ipcfp_blocks_from_car, then ipcfp_store_create over the CAR's own bytes — on every input: the same blocks, the same
status and index on every refused CAR, and byte-equal results of every resident call, by-reference witnesses included (their offsets
index the CAR). Every valid CAR is parsed on the device, whatever its blocks hold (raw bytes of a CID prefix's form, forged section
headers); only refused CARs reach the host parser, which reports their fault."""
import numpy as np
import pytest

from ipc_filecoin_proofs_b200 import _abi as A
from tests import arena_layouts as L
from tests import car_files as F
from tests.test_gpu_arena_layouts import address_world, event_calls, resolve_calls, storage_calls, storage_world  # noqa: F401
from tests.util import spec_of

pytestmark = pytest.mark.gpu

CHUNK = 64 << 20   # the device path's copy chunk (csrc/car.cu)


def _composed(api, car, verify_cids=False):
    """The composed route: (store, layout over the CAR) or (None, (status, index))."""
    try:
        w = api.blocks_from_car(car)
    except A.IpcfpError as e:
        return None, (e.status, e.index)
    lay = L.Layout(w.cids, w.offsets, w.lengths, np.frombuffer(car, np.uint8) if not isinstance(car, np.ndarray) else car)
    try:
        return api.BlockStore(lay.cids, lay.offsets, lay.lengths, lay.blob, verify_cids=verify_cids), lay
    except A.IpcfpError as e:
        return None, (e.status, e.index)


def _car_store(api, car, verify_cids=False):
    try:
        return api.BlockStore.from_car(car, verify_cids=verify_cids), None
    except A.IpcfpError as e:
        return None, (e.status, e.index)


def _assert_same_blocks(got, ref, lay, sample=None):
    assert got.n_blocks == ref.n_blocks == lay.n_blocks
    idx = range(lay.n_blocks) if sample is None else np.random.default_rng(7).choice(lay.n_blocks, sample, replace=False)
    for i in idx:
        c = lay.cids[i]
        assert got.get(c) == ref.get(c)
    if lay.n_blocks:
        missing = lay.cids[0].copy()
        missing[-1] ^= 0x5A
        assert not got.has(missing)


def _assert_same_events(api, got, ref, ts, lay):
    exp = event_calls(api, ref, ts, lay)
    out = event_calls(api, got, ts, lay)
    for k in exp:
        assert out[k] == exp[k], k
    # by-reference offsets are the parser's offsets into the CAR
    w = got.generate_event_proof(ts, spec_of(ts), A.WITNESS_BY_REFERENCE).witness
    offs = {bytes(lay.cids[i]): int(lay.offsets[i]) for i in reversed(range(lay.n_blocks))}
    assert [int(o) for o in w.offsets] == [offs[bytes(c)] for c in w.cids]


@pytest.mark.parametrize("config", [1, 2, 3])
def test_canonical_cars_are_parsed_on_the_device(api, synth_mod, ts3_small, config):
    ts = ts3_small if config == 3 else synth_mod.Tipset(synth_mod.config_params(config))
    secs = F.of_tipset(ts)
    for k, s in enumerate((secs, F.shuffled(secs, config))):
        car = F.write(s)
        ref, lay = _composed(api, car, verify_cids=True)
        got = api.BlockStore.from_car(car, verify_cids=k == 0)
        # config 3's blocks hold raw bytes of a CID prefix's form (CBOR such as 01 18 cc 82 58 20): the walk steps over them
        assert got.car_info.parsed_on_device and got.car_info.ms_parse > 0 and got.car_info.ms_kernels > 0
        _assert_same_blocks(got, ref, lay, sample=None if lay.n_blocks <= 3000 else 3000)
        _assert_same_events(api, got, ref, ts, lay)
        got.close()
        ref.close()


def _flat_car(flat):
    return F.write([(bytes(flat.cids[i]), bytes(flat.blob[int(flat.offsets[i]):int(flat.offsets[i]) + int(flat.lengths[i])]))
                    for i in range(flat.n_blocks)])


def test_storage_and_resolve(api, storage_world, address_world, monkeypatch):
    w, flat, case = storage_world
    for f, calls in ((flat, lambda st: storage_calls(st, w, case, monkeypatch)), (address_world.flat, lambda st: resolve_calls(st, address_world))):
        car = _flat_car(f)
        ref, lay = _composed(api, car)
        got = api.BlockStore.from_car(car)
        assert got.car_info.parsed_on_device
        assert calls(got) == calls(ref)
        got.close()
        ref.close()


def test_duplicates_first_occurrence_wins(api, ts1):
    secs = F.of_tipset(ts1, 60)
    dup = [(secs[3][0], b"another block under the same CID"), (secs[10][0], secs[10][1])]
    s = secs[:20] + dup + secs[20:] + [(secs[0][0], b"")]
    car = F.write(s)
    got = api.BlockStore.from_car(car)
    ref, lay = _composed(api, car)
    assert got.car_info.parsed_on_device and got.n_blocks == len(s)
    _assert_same_blocks(got, ref, lay)
    assert got.get(secs[3][0]) == secs[3][1] and got.get(secs[0][0]) == secs[0][1]


def test_cid_check_reports_the_section(api, ts1):
    secs = F.of_tipset(ts1)
    k = next(i for i in range(len(secs) * 2 // 3, len(secs)) if secs[i][0][2:6] == b"\xa0\xe4\x02\x20" and secs[i][1])
    bad = list(secs)
    bad[k] = (bad[k][0], bytes([bad[k][1][0] ^ 1]) + bad[k][1][1:])
    car = F.write(bad)
    want = _composed(api, car, verify_cids=True)[1]
    assert want == (A.ERR_CID_MISMATCH, k)
    with pytest.raises(A.IpcfpError) as e:
        api.BlockStore.from_car(car, verify_cids=True)
    assert (e.value.status, e.value.index, e.value.first_bad_block) == (A.ERR_CID_MISMATCH, k, k)
    assert api.BlockStore.from_car(car).n_blocks == len(bad)


def test_forged_prefix_is_stepped_over_on_the_device(api, ts1):
    secs = F.of_tipset(ts1)
    forged = b"abc" + bytes([38]) + F.CBOR_PREFIX + b"\x11" * 40
    s = secs[:30] + [(F.cid_of(F.RAW_PREFIX, 7), forged)] + secs[30:]
    car = F.write(s)
    got = api.BlockStore.from_car(car)
    assert got.car_info.parsed_on_device and got.car_info.ms_kernels > 0
    ref, lay = _composed(api, car)
    _assert_same_blocks(got, ref, lay)
    _assert_same_events(api, got, ref, ts1, lay)
    # a non-minimal length varint is read by the host parser: refused there, with the same outcome
    assert _car_store(api, F.write(secs, nonminimal={5}))[1] == _composed(api, F.write(secs, nonminimal={5}))[1] == (A.ERR_DECODE, 5)


def _rule_table(secs):
    """The CPU suite's hand-made cases (tests/test_car.py), each a CAR."""
    hb = F.header([secs[0][0]])
    base = F.varint(len(hb)) + hb
    body = b"".join(F.section(c, b) for c, b in secs[:3])
    cars = [F.write(secs[:3], header_extra=1), F.write(secs[:3], nonminimal={1}), base + b"\x00" + F.section(*secs[0]),
            F.write(secs[:2]) + b"\x00", base + F.varint(20) + secs[0][0][:20], base + b"\x80" * 9 + b"\x01", b"\x00" + hb, b"",
            F.varint(len(hb) + 1) + hb + b"\x00" + body, F.varint(len(hb) + 500) + hb, F.write([], roots=[]), F.write(secs[:1])]
    cids = [bytes([0x12, 0x20]) + b"\x11" * 32, bytes([0x12, 0x20]) + b"\x11" * 20, bytes([0x01, 0x71, 0x12, 0x20]) + b"\x11" * 32,
            bytes([0x01, 0x55, 0x00, 0x05]) + b"hello", bytes([0x01, 0x81, 0x01, 0xA0, 0xE4, 0x02, 0x20]) + b"\x11" * 32,
            bytes([0x02, 0x71, 0xA0, 0xE4, 0x02, 0x20]) + b"\x11" * 32, bytes([0x01, 0x71, 0xA0, 0xE4, 0x82, 0x00, 0x20]) + b"\x11" * 32]
    cars += [F.write([secs[0], secs[1], (c, b"block"), secs[2]]) for c in cids]
    v1, r0 = ("version", F.cbor_head(0, 1)), ("roots", F.cbor_head(4, 0))
    for entries in ([("version", F.cbor_head(0, 2))], [r0, ("version", F.cbor_head(0, 3))], [v1, r0], [v1], [r0], [r0, v1, v1],
                    [r0, v1, ("extra", F.cbor_head(0, 1))], [("roots", F.cbor_head(4, 1) + F.cbor_head(6, 43) + F.cbor_head(2, 39) + b"\x00" * 39), v1]):
        cars.append(F.write(secs[:3], header_bytes=F.header(entries=entries)))
    car = F.write(secs[:9])
    cars += [car[:cut] for cut in range(0, len(car), 7)]
    rng = np.random.default_rng(5)
    for _ in range(150):
        b = bytearray(car)
        at = int(rng.integers(len(b)))
        b[at] ^= int(rng.integers(1, 256))
        cars.append(bytes(b))
    return cars


def test_rule_table_gives_the_composed_outcome(api, ts1):
    secs = F.of_tipset(ts1, 40)
    for k, car in enumerate(_rule_table(secs)):
        ref, want = _composed(api, car)
        got, status = _car_store(api, car)
        if ref is None:
            assert got is None and status == want, k
        else:
            assert got is not None and got.car_info.parsed_on_device, (k, status)
            _assert_same_blocks(got, ref, want)
            got.close()
            ref.close()


def test_section_headers_straddling_a_copy_chunk(api, ts1):
    """A filler raw block puts section 1 at CHUNK - d for d = 0 … 15: its varint and CID prefix straddle the first chunk's end."""
    secs = F.of_tipset(ts1)
    hb = F.header([secs[0][0]])
    head = len(F.varint(len(hb))) + len(hb)
    for d in range(16):
        size = CHUNK - d - head - 4 - 38   # a 4-byte varint frames the filler section
        filler = (F.cid_of(F.RAW_PREFIX, d), bytes(size))
        car = F.write([filler] + secs)
        assert len(F.section(*filler)) + head == CHUNK - d
        got = api.BlockStore.from_car(car)
        assert got.car_info.parsed_on_device, d
        ref, lay = _composed(api, car)
        _assert_same_blocks(got, ref, lay)
        got.close()
        ref.close()


def test_far_offsets(api, ts2):
    """Config 2 behind more than 4 GiB of filler raw blocks: candidate positions past 2^32 and by-reference offsets >= 2^32."""
    secs = F.of_tipset(ts2)
    n_fill, fill = 5, 900 << 20
    hb = F.header([secs[0][0]])
    tail = b"".join(F.section(c, b) for c, b in secs)
    heads = [F.varint(38 + fill) + F.cid_of(F.RAW_PREFIX, k) for k in range(n_fill)]
    total = len(F.varint(len(hb))) + len(hb) + sum(len(h) + fill for h in heads) + len(tail)
    car = np.zeros(total, np.uint8)
    at = 0
    for piece in [F.varint(len(hb)) + hb]:
        car[at:at + len(piece)] = np.frombuffer(piece, np.uint8)
        at += len(piece)
    for h in heads:
        car[at:at + len(h)] = np.frombuffer(h, np.uint8)
        at += len(h) + fill
    assert at > 1 << 32
    car[at:] = np.frombuffer(tail, np.uint8)
    ref = api.BlockStore.from_tipset(ts2)
    canon = L.Layout(ts2.cids, ts2.offsets, ts2.lengths, ts2.blob)
    exp = event_calls(api, ref, ts2, canon)
    ref.close()
    got = api.BlockStore.from_car(car)   # the fillers' CIDs are not their digests
    assert got.car_info.parsed_on_device and got.n_blocks == n_fill + len(secs)
    w = api.blocks_from_car(car)
    lay = L.Layout(w.cids, w.offsets, w.lengths, car)
    out = event_calls(api, got, ts2, lay)
    for k in exp:
        assert out[k] == exp[k], k
    r = got.generate_event_proof(ts2, spec_of(ts2), A.WITNESS_BY_REFERENCE)
    assert int(r.witness.offsets.min()) >= 1 << 32
    got.close()


def test_full_size_tipset(api, synth_mod):
    """The 1 M-receipt tipset's blocks as one CAR (≈ 1.2 GB), from pinned and from pageable memory: the array store's bundle JSON
    (its blocks hold false candidates, as config 3's do: parsed on the device all the same)."""
    ts = synth_mod.Tipset(synth_mod.config_params(4))
    car = F.write(F.of_tipset(ts))
    spec = spec_of(ts)
    ref = api.BlockStore.from_tipset(ts)
    tip = ref.upload_tipset(ts)
    want = ref.generate_proof_bundle_resident(tip, [], [spec], A.RESULT_JSON).json
    tip.close()
    ref.close()
    pinned = api.PinnedArray(len(car))
    pinned.array[:] = np.frombuffer(car, np.uint8)
    for src in (pinned.array, car):
        got = api.BlockStore.from_car(src, verify_cids=True)
        assert got.car_info.parsed_on_device
        tip = got.upload_tipset(ts)
        assert got.generate_proof_bundle_resident(tip, [], [spec], A.RESULT_JSON).json == want
        tip.close()
        got.close()
    pinned.free()


def test_empty_payload(api):
    got = api.BlockStore.from_car(F.write([], roots=[]), verify_cids=True)
    assert got.n_blocks == 0 and got.car_info.parsed_on_device
