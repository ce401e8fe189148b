"""Hand-built message blocks and receipts AMTs for message proofs, and the call restated in Python (cbor2 + hashlib only; a helper module,
not a fixture file).

`world(ts, ...)` turns a synthetic tipset with one parent block into a tipset of two parent blocks whose message AMTs hold real
`Message` and `SignedMessage` blocks (every signature type, every address protocol in `to` / `from`, values of 0 to 32 magnitude
bytes, params at the CBOR length-head edges), one message shared by both parents, and a receipts AMT under a rewritten child header
with exit codes, return data, gas and events roots at their edges. The receipts AMT may be shorter than the execution order and may be
taller than it needs to be.

`prove(blocks, ts, cids, with_body)` restates ipcfp_generate_message_proofs_resident on oracle/pyoracle.py's AMT reader: the
execution order (collect_exec_list), Amtv0<Receipt>::get, the message block decoded by its shape (include/ipcfp.h, "Message proofs"),
and the first fault in request order. `read_set` is the witness the call returns, as a set of CIDs. `cpp_prove` is the second
restatement, tests/oracle_receipts.cpp on oracle/oracle.cpp's decoders."""
import functools
import os
import random
import shutil
import subprocess
import tempfile

import cbor2
import numpy as np

from oracle import pyoracle as P
from tests import event_amts as EA
from tests.event_amts import build_receipts_amt, receipt
from tests.message_amts import base_blocks, build_amt, edit_tipset, exec_order, txmeta
from tests.storage_trees import Blocks, cbytes, cid_of, clink, head

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
U64 = 2 ** 64 - 1
EXECUTED, NOT_EXECUTED, NO_RECEIPT = 0, 1, 2
ERR_MISSING_BLOCK, ERR_DECODE = -2, -3
EDGE_LENGTHS = (0, 23, 24, 255, 256, 65535, 65536)
EXIT_CODES = (0, 1, 16, 33, 2 ** 31, 2 ** 32 - 1)
GAS = (0, 1, 23, 24, 255, 256, 65535, 65536, 2 ** 32 - 1, 2 ** 32, 2 ** 63, U64)


# ------------------------------------------------------------------ blocks
def address(protocol, rng):
    """Address::to_bytes() of each protocol: 0 ID (LEB128), 1 secp256k1 / 2 actor (20 bytes), 3 BLS (48), 4 delegated (namespace, ≤ 54)."""
    if protocol == 0:
        v, out = rng.choice((0, 1, 127, 128, 1000, 2 ** 63, U64)), bytearray()
        while True:
            b = v & 0x7f
            v >>= 7
            out.append(b | (0x80 if v else 0))
            if not v:
                return b"\x00" + bytes(out)
    if protocol in (1, 2):
        return bytes([protocol]) + rng.randbytes(20)
    if protocol == 3:
        return b"\x03" + rng.randbytes(48)
    return b"\x04\x0a" + rng.randbytes(rng.choice((0, 20, 54)))


def token(v):
    """TokenAmount bytes (fvm bigint_ser): empty for 0, else a sign byte and the big-endian magnitude."""
    if v == 0:
        return b""
    m = abs(v)
    return (b"\x01" if v < 0 else b"\x00") + m.to_bytes((m.bit_length() + 7) // 8, "big")


def message(version, to, frm, seq, value, gas_limit, fee_cap, premium, method, params):
    return (head(4, 10) + head(0, version) + cbytes(to) + cbytes(frm) + head(0, seq) + cbytes(token(value)) + head(0, gas_limit)
            + cbytes(token(fee_cap)) + cbytes(token(premium)) + head(0, method) + cbytes(params))


def signed(msg, sig):
    return head(4, 2) + msg + cbytes(sig)


def message_blocks(blocks, rng):
    """Message blocks covering the body's edges → [CID]. Values take 0 to 32 magnitude bytes, params every edge length, signatures
    every type, `to` / `from` every address protocol."""
    out = []
    for k in range(33):
        mag = 0 if k == 0 else (1 << (8 * k - 1)) + rng.getrandbits(8 * k - 1)
        value = -mag if k % 5 == 3 else mag
        params = rng.randbytes(EDGE_LENGTHS[k % len(EDGE_LENGTHS)] if k % 4 == 0 else rng.choice((0, 3, 40)))
        m = message(k % 2, address(k % 5, rng), address((k + 2) % 5, rng), rng.choice((0, 1, 24, 2 ** 40, U64)), value,
                    rng.choice((0, 10_000_000, U64)), rng.getrandbits(8 * (k % 17)), rng.getrandbits(8 * (k % 9)), rng.choice((0, 2, 3844450837, U64)),
                    params)
        kind = k % 4   # 0 unsigned, 1 secp256k1, 2 BLS, 3 delegated
        if kind:
            m = signed(m, bytes([kind]) + rng.randbytes((65, 96, 65)[kind - 1]))
        out.append(blocks.put(m))
    return out


class World:
    """A tipset (EditedTipset) with its blocks, its execution order `exec`, its receipts {position: (exit, ret, gas, events_root)}
    and the receipts AMT."""

    def __init__(self, ts, blocks, exec_, receipts, ramt, never, shared, shared_second):
        self.ts, self.blocks, self.exec, self.receipts, self.ramt, self.never = ts, blocks, exec_, receipts, ramt, never
        self.shared, self.shared_second = shared, shared_second   # the message both parents hold; its position in parent 1's list

    def requests(self):
        """Every executed message, the never-executed CIDs, and duplicates."""
        return list(self.exec) + list(self.never) + [self.exec[0], self.never[0], self.exec[-1]]


def _rewrite_receipts_root(et, blocks, root):
    """The child header of `et` with `[9] ParentMessageReceipts` = root; the tipset's receipts_root and child CID follow."""
    child = cbor2.loads(blocks[bytes(et.child_cid)])
    child[9] = cbor2.CBORTag(42, b"\0" + root)
    new = blocks.put(cbor2.dumps(child))
    cids, offs, lens, blob = blocks.flat()
    et.cids, et.offsets, et.lengths, et.blob, et.n_blocks = cids, offs, lens, blob, len(lens)
    et.child_cid = np.frombuffer(new, dtype=np.uint8).copy()
    et.receipts_root = np.frombuffer(root, dtype=np.uint8).copy()
    return et


def world(ts, seed=1, height=None, short=1, empty_events=False):
    """ts: a synthetic tipset with one parent block. Two parents: parent 0 holds the first half of the messages (BLS: the unsigned ones,
    SECP: the signed ones), parent 1 the rest and, first in its BLS list, parent 0's last SECP message (first position wins). The
    receipts AMT (height: default the minimal one) holds a receipt for every position but the last `short`."""
    rng = random.Random(seed)
    blocks, _, _ = base_blocks(ts)
    blocks = Blocks(blocks)
    msgs = message_blocks(blocks, rng)
    half = len(msgs) // 2
    lists = []
    for part in (msgs[:half], msgs[half:]):
        bls = [c for c in part if blocks[c][0] == 0x8a]
        secp = [c for c in part if blocks[c][0] == 0x82]
        lists.append((bls, secp))
    lists[1] = ([lists[0][1][-1]] + lists[1][0], lists[1][1])
    tms = [txmeta(blocks, build_amt(blocks, dict(enumerate(b))).root, build_amt(blocks, dict(enumerate(s))).root) for b, s in lists]
    et = edit_tipset(ts, blocks, tms)
    ex = exec_order(lists)
    shared_second = sum(len(b) + len(s) for b, s in lists[:1])   # where parent 1's list starts in the concatenated message list
    events = list(blocks)[:4]
    receipts = {}
    for i in range(len(ex) - short):
        ret = rng.randbytes(EDGE_LENGTHS[i % len(EDGE_LENGTHS)] if i % 3 == 0 else rng.choice((0, 1, 32)))
        er = None if empty_events or i % 2 else events[i % len(events)]
        receipts[i] = (EXIT_CODES[i % len(EXIT_CODES)], ret, GAS[i % len(GAS)], er)
    ramt = build_receipts_amt(blocks, {i: receipt(*r) for i, r in receipts.items()}, height=height)
    et = _rewrite_receipts_root(et, blocks, ramt.root)
    never = [cid_of(b"never executed %d" % k) for k in range(3)] + [bytes(P.cid_of(blocks[bytes(et.child_cid)]))]
    return World(et, blocks, ex, receipts, ramt, never, lists[0][1][-1], shared_second)


def forge(w):
    """w's tipset with a forged receipts AMT (every exit code flipped in its lowest bit) under a rewritten child header: every block is
    honestly hashed, the child CID is not w's. → (EditedTipset, blocks)"""
    from tests.util import EditedTipset
    blocks = Blocks(w.blocks)
    ramt = build_receipts_amt(blocks, {i: receipt(r[0] ^ 1, *r[1:]) for i, r in w.receipts.items()}, height=w.ramt.height)
    return _rewrite_receipts_root(EditedTipset(w.ts), blocks, ramt.root), blocks


# ------------------------------------------------------------------ the restatement
class Fault(Exception):
    def __init__(self, status, index):
        super().__init__(status, index)
        self.status, self.index = status, index


def _uint(x):
    if not isinstance(x, int) or isinstance(x, bool) or not 0 <= x <= U64:
        raise ValueError("not a u64")
    return x


def _address(b):
    from tests.address_trees import address_valid
    if not isinstance(b, bytes) or not address_valid(b):
        raise ValueError("not an Address")
    return b


def _token(b):
    if not isinstance(b, bytes):
        raise ValueError("not bytes")
    if not b:
        return 0
    if b[0] > 1 or len(b) - 1 > 32:
        raise ValueError("not a TokenAmount")
    m = int.from_bytes(b[1:], "big")
    return -m if b[0] == 1 else m


def _link(x):
    """A tag-42 link as the engine reads it (csrc/cbor.cuh rd_cid): 39 bytes, the identity multibase 0x00, then a CIDv1 → its 38 bytes."""
    if not isinstance(x, cbor2.CBORTag) or x.tag != 42 or not isinstance(x.value, bytes) or len(x.value) != 39 or x.value[:2] != b"\0\1":
        raise ValueError("not a CID link")
    return bytes(x.value[1:])


def decode_receipt(v):
    if not isinstance(v, list) or len(v) != 4:
        raise ValueError("not a Receipt")
    ec, ret, gas, er = v
    if _uint(ec) > 2 ** 32 - 1 or not isinstance(ret, bytes):
        raise ValueError("receipt field out of range")
    _uint(gas)
    if er is not None:
        er = _link(er)
    return ec, ret, gas, er


def decode_message(raw):
    """The body fields of a message block, decided by its shape."""
    x = EA._strict(raw)
    sig_type = 0
    if isinstance(x, list) and len(x) == 2:
        x, sig = x
        if not isinstance(sig, bytes) or not sig or sig[0] not in (1, 2, 3):
            raise ValueError("not a Signature")
        sig_type = sig[0]
    if not isinstance(x, list) or len(x) != 10:
        raise ValueError("not a Message")
    ver, to, frm, seq, val, gl, fc, gp, meth, params = x
    if not isinstance(params, bytes):
        raise ValueError("params")
    return dict(version=_uint(ver), to=_address(to), from_=_address(frm), sequence=_uint(seq), value=_token(val), gas_limit=_uint(gl),
                gas_fee_cap=_token(fc), gas_premium=_token(gp), method_num=_uint(meth), params=params, sig_type=sig_type)


def _receipts_get(rec, root, i):
    """Amtv0<Receipt>::get(i) → the decoded receipt or None, by the strict AMT restatement of tests/event_amts.py: every node on the
    path is decoded whole, every receipt of the leaf too, before the index is looked at."""
    bw, h, _, node = EA.read_root(rec.get(root), 0)
    in_range = i < 8 ** (h + 1)
    level = h
    while True:
        is_link, items = EA._node_items(node, bw, level)
        for x in node[1]:
            _link(x)
        if not is_link:
            for _, v in items:
                decode_receipt(v)
        hit = dict(items).get((i // 8 ** level) % 8) if in_range else None
        if hit is None:
            return None
        if not is_link:
            return decode_receipt(hit) if level == 0 else None
        raw = rec.get(hit)
        if raw is None:
            raise P.MissingBlock(hit)
        node = EA._strict(raw)
        level -= 1


def prove(blocks, ts, cids, with_body=False):
    """blocks {CID: bytes}, ts a tipset (descriptor attributes) → ([proof dict per request], witness CID set), or raises
    Fault(status, index) for the first fault in request order."""
    txm = [bytes(ts.parent_txmeta_cids[k]) for k in range(int(ts.n_parents))]
    seen = set()

    def get(c):
        seen.add(c)
        return blocks.get(c)

    ex = P.collect_exec_list(get, txm)
    pos = {}
    for i, c in enumerate(ex):
        pos.setdefault(c, i)
    root = bytes(ts.receipts_root)
    wit = set(seen) | {bytes(ts.parent_cids[k]) for k in range(int(ts.n_parents))} | {bytes(ts.child_cid), root}
    out = []
    for j, c in enumerate(cids):
        c = bytes(c)
        p = dict(message_cid=c, status=NOT_EXECUTED, exec_index=None, exit_code=0, return_data=b"", gas_used=0, events_root=None,
                 has_body=False)
        if c in pos:
            e = pos[c]
            p["exec_index"] = e
            rec = P.Recorder(blocks)
            try:
                r = _receipts_get(rec, root, e)
            except P.MissingBlock:
                raise Fault(ERR_MISSING_BLOCK, j)
            except Exception:   # whatever the strict decoders refuse
                raise Fault(ERR_DECODE, j)
            wit |= rec.seen
            if r is None:
                p["status"] = NO_RECEIPT
            else:
                p.update(status=EXECUTED, exit_code=r[0], return_data=r[1], gas_used=r[2], events_root=r[3])
            if with_body:
                raw = blocks.get(c)
                if raw is None:
                    raise Fault(ERR_MISSING_BLOCK, j)
                try:
                    p.update(decode_message(raw))
                except Exception:
                    raise Fault(ERR_DECODE, j)
                p["has_body"] = True
                wit.add(c)
        out.append(p)
    return out, wit


def read_set(blocks, ts, cids, with_body=False):
    """The blocks a complete call reads: the CIDs of its witness."""
    return prove(blocks, ts, cids, with_body)[1]


def proof_dict(mp):
    """A.MessageProof → the restatement's dict (body fields only with the body)."""
    d = dict(message_cid=mp.message_cid, status=mp.status, exec_index=mp.exec_index, exit_code=mp.exit_code, return_data=mp.return_data,
             gas_used=mp.gas_used, events_root=mp.events_root, has_body=mp.has_body)
    if mp.has_body:
        d.update(version=mp.version, to=mp.to, from_=mp.from_, sequence=mp.sequence, value=mp.value, gas_limit=mp.gas_limit,
                 gas_fee_cap=mp.gas_fee_cap, gas_premium=mp.gas_premium, method_num=mp.method_num, params=mp.params, sig_type=mp.sig_type)
    return d


def with_blocks(w, blocks):
    """w's tipset over another block set (dropped or rewritten blocks); CIDs stay as they are."""
    from tests.util import EditedTipset
    cids, offs, lens, blob = Blocks(blocks).flat()
    return EditedTipset(w.ts, cids=cids, offsets=offs, lengths=lens, blob=blob, n_blocks=len(lens))


def receipt_path(w, i):
    """The receipts-AMT nodes (non-root) on the path to position i, top down."""
    out = []
    for level in range(w.ramt.height - 1, -1, -1):
        base = (i // 8 ** (level + 1)) * 8 ** (level + 1)
        if (level, base) in w.ramt.nodes:
            out.append(w.ramt.nodes[(level, base)])
    return out


# ------------------------------------------------------------------ the second restatement: tests/oracle_receipts.cpp
@functools.lru_cache(maxsize=None)
def cpp_lib():
    """tests/oracle_receipts.cpp, compiled with g++ once per process into a temporary directory (the checkout may be read-only)."""
    import ctypes as C
    from ipc_filecoin_proofs_b200 import _abi as A
    gxx = shutil.which("g++")
    if not gxx:
        raise RuntimeError("g++ is needed to build the message-proof oracle")
    out = os.path.join(tempfile.mkdtemp(prefix="oracle_receipts_"), "liboracle_receipts.so")
    subprocess.check_call([gxx, "-std=c++17", "-O2", "-fPIC", "-shared", "-pthread", "-o", out, os.path.join(ROOT, "tests", "oracle_receipts.cpp")])
    L = C.CDLL(out)
    L.oracle_store_create.restype = C.c_void_p
    L.oracle_store_create.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64]
    L.oracle_store_destroy.argtypes = [C.c_void_p]
    L.oracle_message_proofs.restype = C.c_int32
    L.oracle_message_proofs.argtypes = [C.c_void_p, C.POINTER(A.TipsetDesc), C.c_void_p, C.c_uint64, C.c_uint32, C.c_void_p]
    L.oracle_message_blob.restype = C.c_void_p
    L.oracle_message_blob.argtypes = [C.POINTER(C.c_uint64)]
    L.oracle_message_witness.restype = C.c_void_p
    L.oracle_message_witness.argtypes = [C.POINTER(C.c_uint64)]
    L.oracle_last_error_index.restype = C.c_uint64
    return L


def cpp_prove(blocks, ts, cids, with_body=False):
    """prove() by tests/oracle_receipts.cpp over `blocks` → (proofs, witness CID set, data blob), or raises Fault(status, index)."""
    import ctypes as C
    from ipc_filecoin_proofs_b200 import _abi as A
    L = cpp_lib()
    arrays = tuple(np.ascontiguousarray(a, dtype=t) for a, t in zip(Blocks(blocks).flat(), (np.uint8, np.uint64, np.uint32, np.uint8)))
    c, o, n, b = arrays
    h = L.oracle_store_create(c.ctypes.data, o.ctypes.data, n.ctypes.data, b.ctypes.data, len(n))
    try:
        d, keep = A.make_tipset_desc(ts)
        req = np.frombuffer(b"".join(bytes(x) for x in cids), np.uint8) if len(cids) else np.zeros(0, np.uint8)
        recs = (A.MessageProofC * max(len(cids), 1))()
        st = L.oracle_message_proofs(h, C.byref(d), req.ctypes.data if req.size else None, len(cids), A.MESSAGE_WITH_BODY if with_body else 0,
                                     C.addressof(recs))
        if st != 0:
            raise Fault(st, int(L.oracle_last_error_index()))
        k = C.c_uint64()
        p = L.oracle_message_blob(C.byref(k))
        blob = C.string_at(p, k.value) if k.value else b""
        w = L.oracle_message_witness(C.byref(k))
        wit = C.string_at(w, 38 * k.value) if k.value else b""
        witness = {wit[38 * i:38 * i + 38] for i in range(k.value)}
        return [proof_dict(A.message_proof_from_c(recs[i], blob)) for i in range(len(cids))], witness, blob
    finally:
        L.oracle_store_destroy(h)
