"""CARv1 archives of a block set, for ipcfp_blocks_from_car / ipcfp_store_create_car (test infrastructure).

* `write(sections, …)` writes a CARv1 (https://ipld.io/specs/transport/car/carv1/): the header {"roots": […], "version": 1} as DAG-CBOR,
  then one section per (cid, block) in the order given, optionally with non-minimal varints; `shuffled` / `of_tipset` give section lists.
* `header(…)` writes header bytes with any keys, order and values, for the header rules.
* `read(car)` states the rules of include/ipcfp.h independently of the library: it returns (cids (n, 38), offsets, lengths) indexing
  the CAR itself, or raises Fault(status, index).
"""
import numpy as np

from ipc_filecoin_proofs_b200 import _abi as A
from tests import rpc_blocks as B

NO_INDEX = (1 << 64) - 1


class Fault(Exception):
    def __init__(self, status, index=NO_INDEX):
        super().__init__(status, index)
        self.status, self.index = status, index


# ------------------------------------------------------------------------------------------ writing
def varint(v, extra=0):
    """Unsigned LEB128 of v; extra > 0 appends that many redundant continuation bytes (a non-minimal encoding of the same value)."""
    out = bytearray()
    while True:
        b = v & 0x7F
        v >>= 7
        out.append(b | 0x80 if v else b)
        if not v:
            break
    if extra:
        out[-1] |= 0x80
    for k in range(extra):
        out.append(0x80 if k + 1 < extra else 0x00)
    return bytes(out)


def cbor_head(major, arg):
    if arg < 24:
        return bytes([major << 5 | arg])
    for ai, nb in ((24, 1), (25, 2), (26, 4), (27, 8)):
        if arg < 1 << (8 * nb):
            return bytes([major << 5 | ai]) + arg.to_bytes(nb, "big")
    raise ValueError(arg)


def cbor_text(s):
    b = s.encode()
    return cbor_head(3, len(b)) + b


def cbor_cid(cid):
    """A CID as DAG-CBOR: tag 42 over a byte string holding 0x00 and the CID's bytes."""
    return cbor_head(6, 42) + cbor_head(2, len(cid) + 1) + b"\x00" + bytes(cid)


def header(roots=(), version=1, entries=None):
    """The header's DAG-CBOR bytes. entries: a list of (key, encoded value) pairs to write instead, in that order."""
    if entries is None:
        entries = [("roots", cbor_head(4, len(roots)) + b"".join(cbor_cid(r) for r in roots)), ("version", cbor_head(0, version))]
    return cbor_head(5, len(entries)) + b"".join(cbor_text(k) + v for k, v in entries)


def section(cid, block, extra=0):
    body = bytes(cid) + bytes(block)
    return varint(len(body), extra) + body


def write(sections, roots=None, header_bytes=None, nonminimal=(), header_extra=0):
    """A CARv1 of (cid, block) pairs in the order given. roots: default the first CID; nonminimal: indices of sections whose length varint
    gets a redundant byte; header_extra: redundant bytes in the header's length varint."""
    if header_bytes is None:
        header_bytes = header([sections[0][0]] if roots is None and sections else (roots or []))
    out = bytearray(varint(len(header_bytes), header_extra) + header_bytes)
    for k, (c, b) in enumerate(sections):
        out += section(c, b, 1 if k in nonminimal else 0)
    return bytes(out)


def of_tipset(ts, n=None):
    """The (cid, block) pairs of a synth.Tipset in store order."""
    cids, blocks = B.blocks_of(ts, n)
    return [(bytes(c), b) for c, b in zip(cids, blocks)]


def shuffled(sections, seed):
    order = np.random.default_rng(seed).permutation(len(sections))
    return [sections[k] for k in order]


def cid_of(prefix, digest_byte=0):
    """A CID of 6 prefix bytes and a 32-byte digest of one repeated byte."""
    return bytes(prefix) + bytes([digest_byte]) * 32


RAW_PREFIX = bytes([0x01, 0x55, 0xA0, 0xE4, 0x02, 0x20])       # CIDv1, raw, blake2b-256
CBOR_PREFIX = bytes([0x01, 0x71, 0xA0, 0xE4, 0x02, 0x20])      # CIDv1, dag-cbor, blake2b-256


# ------------------------------------------------------------------------------------------ the rules, restated
def _varint(buf, at, end):
    """(value, next) of a minimal varint below 2^63 in buf[at:end]; None when truncated, too long or not minimal."""
    v = 0
    for k in range(9):
        if at + k >= end:
            return None
        b = buf[at + k]
        v |= (b & 0x7F) << (7 * k)
        if not b & 0x80:
            if k and b == 0:
                return None
            return v, at + k + 1
    return None


class _Cbor:
    def __init__(self, buf, at, end):
        self.buf, self.at, self.end = buf, at, end

    def head(self):
        if self.at >= self.end:
            raise Fault(A.ERR_DECODE)
        b = self.buf[self.at]
        self.at += 1
        major, ai = b >> 5, b & 31
        if ai < 24:
            return major, ai
        if ai > 27:
            raise Fault(A.ERR_DECODE)
        nb = 1 << (ai - 24)
        if self.end - self.at < nb:
            raise Fault(A.ERR_DECODE)
        arg = int.from_bytes(self.buf[self.at:self.at + nb], "big")
        self.at += nb
        if arg < (24, 1 << 8, 1 << 16, 1 << 32)[ai - 24]:
            raise Fault(A.ERR_DECODE)
        return major, arg

    def expect(self, major):
        m, arg = self.head()
        if m != major:
            raise Fault(A.ERR_DECODE)
        return arg

    def take(self, n):
        if n > self.end - self.at:
            raise Fault(A.ERR_DECODE)
        self.at += n
        return bytes(self.buf[self.at - n:self.at])


def _header(buf):
    r = _varint(buf, 0, len(buf))
    if r is None or r[0] == 0 or r[0] > len(buf) - r[1]:
        raise Fault(A.ERR_DECODE)
    h, at = r
    c = _Cbor(buf, at, at + h)
    seen = set()
    for _ in range(c.expect(5)):
        key = c.take(c.expect(3))
        if key in seen or key not in (b"roots", b"version"):
            raise Fault(A.ERR_DECODE)
        seen.add(key)
        if key == b"version":
            if c.expect(0) != 1:
                raise Fault(A.ERR_UNSUPPORTED)
        else:
            for _ in range(c.expect(4)):
                if c.expect(6) != 42:
                    raise Fault(A.ERR_DECODE)
                root = c.take(c.expect(2))
                if not root or root[0] != 0:
                    raise Fault(A.ERR_DECODE)
    if c.at != c.end or seen != {b"roots", b"version"}:
        raise Fault(A.ERR_DECODE)
    return c.end


def _cid(s, k):
    """The CID rule of section k whose bytes are s."""
    if len(s) >= 2 and s[0] == 0x12 and s[1] == 0x20:
        raise Fault(A.ERR_UNSUPPORTED if len(s) >= 34 else A.ERR_DECODE, k)
    fields, at = [], 0
    for _ in range(4):
        r = _varint(s, at, len(s))
        if r is None:
            raise Fault(A.ERR_DECODE, k)
        fields.append((r[0], r[1] - at))
        at = r[1]
    (version, _), _codec, _code, (size, _) = fields
    if version != 1 or size > len(s) - at:
        raise Fault(A.ERR_DECODE, k)
    if fields[1][1] != 1 or fields[2][1] != 3 or size != 32:
        raise Fault(A.ERR_UNSUPPORTED, k)


def read(car):
    """(cids (n, 38) uint8, offsets uint64, lengths uint32) of a CAR under the rules of include/ipcfp.h, or Fault(status, index)."""
    buf = bytes(car)
    at, k = _header(buf), 0
    cids, offs, lens = [], [], []
    while at < len(buf):
        r = _varint(buf, at, len(buf))
        if r is None or r[0] == 0 or r[0] > len(buf) - r[1]:
            raise Fault(A.ERR_DECODE, k)
        L, s = r
        _cid(buf[s:s + L], k)
        if L - 38 >= 1 << 32:
            raise Fault(A.ERR_UNSUPPORTED, k)
        cids.append(buf[s:s + 38])
        offs.append(s + 38)
        lens.append(L - 38)
        at = s + L
        k += 1
    return (np.frombuffer(b"".join(cids), np.uint8).reshape(-1, 38), np.asarray(offs, np.uint64), np.asarray(lens, np.uint32))


def expected(car):
    """read(car), or (status, index) of its fault."""
    try:
        return read(car)
    except Fault as f:
        return (f.status, f.index)
