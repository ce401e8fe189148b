"""ipcfp_blocks_from_car (csrc/car_parse.cpp, host C++, no device): the sections of a CARv1 must agree with the rules restated in
tests/car_files.py — the arrays, or the status and the index — on the synthetic tipsets' block sets in any order, on hand-made cases for
every rule, and on seeded byte flips, insertions and deletions."""
import numpy as np
import pytest

import synth
from ipc_filecoin_proofs_b200 import _abi as A
from ipc_filecoin_proofs_b200 import api
from tests import car_files as F

DEC, UNS = A.ERR_DECODE, A.ERR_UNSUPPORTED
NO = F.NO_INDEX


def _got(car):
    try:
        w = api.blocks_from_car(car)
    except A.IpcfpError as e:
        return (e.status, e.index)
    return (w.cids, w.offsets, w.lengths)


def _agree(car):
    """The library and the rules give the same outcome; returns it."""
    want, got = F.expected(car), _got(car)
    if isinstance(want[0], int):
        assert got == want
    else:
        assert not isinstance(got[0], int), got
        for a, b in zip(got, want):
            assert a.dtype == b.dtype and np.array_equal(a, b)
    return want


def _blocks_equal(car, sections):
    w = api.blocks_from_car(car)
    assert w.n_blocks == len(sections) and w.blob.size == len(car)
    for k, (c, b) in enumerate(sections):
        assert bytes(w.cids[k]) == c and w.block(k) == b


@pytest.fixture(scope="module")
def small():
    """The first 40 sections of config 1, one block of them empty."""
    secs = F.of_tipset(synth.Tipset(synth.config_params(1)), 40)
    secs[7] = (secs[7][0], b"")
    return secs


@pytest.mark.parametrize("config", [1, 2, 3])
def test_tipset_block_sets_in_index_order_and_shuffled(config):
    params = synth.config_params(3, hamt_entries=20000) if config == 3 else synth.config_params(config)
    secs = F.of_tipset(synth.Tipset(params))
    for s in (secs, F.shuffled(secs, config)):
        car = F.write(s)
        _blocks_equal(car, s)
        _agree(car)


def test_input_kinds_share_one_result(small):
    import mmap
    car = F.write(small)
    want = _got(car)
    m = mmap.mmap(-1, len(car))
    m.write(car)
    for x in (bytearray(car), np.frombuffer(car, np.uint8).copy(), m):
        got = _got(x)
        assert all(np.array_equal(a, b) for a, b in zip(got, want))


def test_zero_and_one_section(small):
    assert _agree(F.write([], roots=[]))[0].shape == (0, 38)
    assert _agree(F.write([], roots=[small[0][0]]))[0].shape == (0, 38)
    assert len(_agree(F.write(small[:1]))[0]) == 1
    _blocks_equal(F.write(small[:1]), small[:1])


def test_duplicates_empty_and_raw_blocks(small):
    raw = [(F.cid_of(F.RAW_PREFIX, k), bytes([k]) * k) for k in range(5)]
    secs = small[:5] + [small[2], small[0]] + raw + [(small[9][0], b"")] + small[5:10]
    car = F.write(secs)
    _blocks_equal(car, secs)
    _agree(car)


def test_truncation_at_every_byte(small):
    """Every prefix of a CAR cut inside the header, or inside the first, a middle or the last section."""
    secs = small[:9]
    car = F.write(secs)
    hdr_end = len(car) - sum(len(F.section(c, b)) for c, b in secs)
    starts = [hdr_end]
    for c, b in secs:
        starts.append(starts[-1] + len(F.section(c, b)))
    cuts = set(range(0, hdr_end + 1))
    for k in (0, 4, 8):
        cuts |= set(range(starts[k], starts[k + 1] + 1))
    for cut in sorted(cuts):
        out = _agree(car[:cut])
        if cut == 0 or cut < hdr_end:
            assert out == (DEC, NO)
        elif cut in starts:
            assert len(out[0]) == starts.index(cut)
        else:
            assert out == (DEC, max(i for i, s in enumerate(starts) if s <= cut))


def test_length_varints(small):
    hb = F.header([small[0][0]])
    assert _agree(F.write(small[:3], header_extra=1)) == (DEC, NO)   # non-minimal H
    assert _agree(F.write(small[:3], nonminimal={1})) == (DEC, 1)    # non-minimal L
    base = F.varint(len(hb)) + hb
    assert _agree(base + b"\x00" + F.section(*small[0])) == (DEC, 0)     # L = 0
    assert _agree(F.write(small[:2]) + b"\x00") == (DEC, 2)
    assert _agree(base + F.varint(20) + small[0][0][:20]) == (DEC, 0)    # L shorter than the CID
    assert _agree(base + F.varint(37) + small[0][0][:37]) == (DEC, 0)
    assert _agree(base + b"\x80" * 9 + b"\x01") == (DEC, 0)              # a varint of 10 bytes
    assert _agree(b"\x00" + hb) == (DEC, NO)                             # H = 0
    assert _agree(b"") == (DEC, NO)


@pytest.mark.parametrize("name,cid,status", [
    ("cidv0", bytes([0x12, 0x20]) + b"\x11" * 32, UNS),
    ("cidv0-short", bytes([0x12, 0x20]) + b"\x11" * 20, DEC),
    ("sha2-256", bytes([0x01, 0x71, 0x12, 0x20]) + b"\x11" * 32, UNS),
    ("identity", bytes([0x01, 0x55, 0x00, 0x05]) + b"hello", UNS),
    ("two-byte-codec", bytes([0x01, 0x81, 0x01, 0xA0, 0xE4, 0x02, 0x20]) + b"\x11" * 32, UNS),
    ("two-byte-codec-two-byte-code", bytes([0x01, 0x81, 0x01, 0xA0, 0x01, 0x20]) + b"\x11" * 32, UNS),
    ("digest-16", bytes([0x01, 0x71, 0xA0, 0xE4, 0x02, 0x10]) + b"\x11" * 32, UNS),
    ("version-2", bytes([0x02, 0x71, 0xA0, 0xE4, 0x02, 0x20]) + b"\x11" * 32, DEC),
    ("version-0", bytes([0x00, 0x71, 0xA0, 0xE4, 0x02, 0x20]) + b"\x11" * 32, DEC),
    ("digest-past-section", bytes([0x01, 0x71, 0xA0, 0xE4, 0x02, 0x40]) + b"\x11" * 32, DEC),
    ("non-minimal-codec", bytes([0x01, 0xF1, 0x00, 0xA0, 0xE4, 0x02, 0x20]) + b"\x11" * 32, DEC),
    ("non-minimal-code", bytes([0x01, 0x71, 0xA0, 0xE4, 0x82, 0x00, 0x20]) + b"\x11" * 32, DEC),
])
def test_cid_forms(small, name, cid, status):
    car = F.write([small[0], small[1], (cid, b"block"), small[2]])
    assert _agree(car) == (status, 2)


def test_section_that_claims_4_gib_past_the_buffer(small):
    hb = F.header([small[0][0]])
    car = F.varint(len(hb)) + hb + F.section(*small[0]) + F.varint(38 + (1 << 32)) + small[1][0] + b"x" * 8
    assert _agree(car) == (DEC, 1)   # the section does not fit: the bounds rule comes first


@pytest.mark.parametrize("name,entries,status", [
    ("carv2-pragma", [("version", F.cbor_head(0, 2))], UNS),
    ("version-3", None, UNS),
    ("version-0", [("roots", F.cbor_head(4, 0)), ("version", F.cbor_head(0, 0))], UNS),
    ("version-first", [("version", F.cbor_head(0, 1)), ("roots", F.cbor_head(4, 0))], None),
    ("missing-roots", [("version", F.cbor_head(0, 1))], DEC),
    ("missing-version", [("roots", F.cbor_head(4, 0))], DEC),
    ("duplicate-version", [("roots", F.cbor_head(4, 0)), ("version", F.cbor_head(0, 1)), ("version", F.cbor_head(0, 1))], DEC),
    ("duplicate-roots", [("roots", F.cbor_head(4, 0)), ("roots", F.cbor_head(4, 0)), ("version", F.cbor_head(0, 1))], DEC),
    ("unknown-key", [("roots", F.cbor_head(4, 0)), ("version", F.cbor_head(0, 1)), ("extra", F.cbor_head(0, 1))], DEC),
    ("version-not-uint", [("roots", F.cbor_head(4, 0)), ("version", F.cbor_text("1"))], DEC),
    ("roots-not-array", [("roots", F.cbor_head(0, 0)), ("version", F.cbor_head(0, 1))], DEC),
    ("root-not-tag-42", [("roots", F.cbor_head(4, 1) + F.cbor_head(6, 43) + F.cbor_head(2, 39) + b"\x00" + b"\x01" * 38),
                         ("version", F.cbor_head(0, 1))], DEC),
    ("root-untagged", [("roots", F.cbor_head(4, 1) + F.cbor_head(2, 39) + b"\x00" + b"\x01" * 38), ("version", F.cbor_head(0, 1))], DEC),
    ("root-no-zero-byte", [("roots", F.cbor_head(4, 1) + F.cbor_head(6, 42) + F.cbor_head(2, 38) + b"\x01" * 38),
                           ("version", F.cbor_head(0, 1))], DEC),
    ("root-empty-bytes", [("roots", F.cbor_head(4, 1) + F.cbor_head(6, 42) + F.cbor_head(2, 0)), ("version", F.cbor_head(0, 1))], DEC),
    ("non-minimal-version", [("roots", F.cbor_head(4, 0)), ("version", bytes([0x18, 0x01]))], DEC),
    ("indefinite-roots", [("roots", b"\x9f\xff"), ("version", F.cbor_head(0, 1))], DEC),
])
def test_header_rules(small, name, entries, status):
    hb = F.header(version=3) if entries is None else F.header(entries=entries)
    car = F.write(small[:3], header_bytes=hb)
    out = _agree(car)
    if status is None:
        assert len(out[0]) == 3
    else:
        assert out == (status, NO)


def test_header_bytes_left_over_and_not_a_map(small):
    hb = F.header([small[0][0]])
    body = b"".join(F.section(c, b) for c, b in small[:3])
    assert _agree(F.varint(len(hb) + 1) + hb + b"\x00" + body) == (DEC, NO)     # trailing byte inside H
    assert _agree(F.varint(len(hb)) + hb[:-1] + body) == (DEC, NO)               # H one short: the map is cut
    assert _agree(F.varint(1) + b"\x80" + body) == (DEC, NO)                     # an empty array
    assert _agree(F.varint(len(hb) + 500) + hb) == (DEC, NO)                     # H past the buffer


def test_seeded_mutations(small):
    """2 000 byte flips, insertions and deletions of a CAR with roots, duplicates, empty and raw blocks."""
    secs = small[:12] + [small[3], (F.cid_of(F.RAW_PREFIX, 9), b"raw bytes"), (small[20][0], b"")]
    car = F.write(secs, roots=[secs[0][0], secs[5][0]])
    rng = np.random.default_rng(20261018)
    outcomes = set()
    for _ in range(2000):
        b = bytearray(car)
        kind, at = rng.integers(3), int(rng.integers(len(b)))
        if kind == 0:
            b[at] ^= int(rng.integers(1, 256))
        elif kind == 1:
            b[at:at] = bytes(rng.integers(0, 256, int(rng.integers(1, 4)), dtype=np.uint8))
        else:
            del b[at:at + int(rng.integers(1, 4))]
        out = _agree(bytes(b))
        outcomes.add(out[0] if isinstance(out[0], int) else "ok")
    assert {"ok", DEC, UNS} <= outcomes


def test_null_arguments():
    import ctypes as C
    L = api.lib()
    out = C.POINTER(A.ParsedBlocksC)()
    assert L.ipcfp_blocks_from_car(None, 10, C.byref(out)) == A.ERR_INVALID_ARG and not out
    buf = (C.c_uint8 * 4)()
    assert L.ipcfp_blocks_from_car(buf, 4, None) == A.ERR_INVALID_ARG
    h = C.c_void_p()
    assert L.ipcfp_store_create_car(buf, 4, 0, 0, None, None) == A.ERR_INVALID_ARG
    assert L.ipcfp_store_create_car(None, 4, 0, 0, C.byref(h), None) == A.ERR_INVALID_ARG and not h.value
