"""Filecoin.ChainReadObj JSON-RPC responses of a block set, for ipcfp_blocks_from_rpc_json / ipcfp_store_create_rpc_json (test infrastructure).

* `blocks_of(ts)` gives a synthetic tipset's CIDs and block bytes; request i of a caller's fetch asks for CID i with "id": i.
* `render(blocks, …)` writes the responses as a node would send them: canonical elements (the form the device parser reads), in request
  order or shuffled, split into any number of texts, each a batch or a single object; `element` / `error_element` / `pretty` give the
  other spellings.
* `read(n, texts)` states the rules of include/ipcfp.h independently of the library, on Python's `json` module (the value reader of
  tests/rpc_json.py) and `base64`: it returns the blocks in request order, or raises Fault(status, index).
"""
import base64
import binascii

import numpy as np

from ipc_filecoin_proofs_b200 import _abi as A
from tests import rpc_json as R

NO_INDEX = R.NO_INDEX
Fault = R.Fault


# ------------------------------------------------------------------------------------------ rendering
def blocks_of(ts, n=None):
    """(cids (n, 38), [block bytes]) of a synth.Tipset, in store order; n: only the first n blocks."""
    cids = np.asarray(ts.cids, np.uint8).reshape(-1, 38)
    n = len(cids) if n is None else n
    blob, offs, lens = np.asarray(ts.blob, np.uint8), np.asarray(ts.offsets), np.asarray(ts.lengths)
    mv = memoryview(blob.tobytes())
    return cids[:n].copy(), [bytes(mv[int(offs[i]):int(offs[i]) + int(lens[i])]) for i in range(n)]


def element(i, data):
    """The canonical response to request i: what the device parser reads."""
    return b'{"jsonrpc":"2.0","result":"' + base64.b64encode(data) + b'","id":' + str(i).encode() + b"}"


def error_element(i):
    return b'{"jsonrpc":"2.0","error":{"code":1,"message":"blockstore: block not found"},"id":' + str(i).encode() + b"}"


def pretty(i, data):
    """The same response with another member order and whitespace: read by the host parser only."""
    return b'{ "id": ' + str(i).encode() + b', "jsonrpc": "2.0", "result": "' + base64.b64encode(data) + b'" }'


def render(blocks, n_texts=1, seed=None, single=False, elements=None):
    """The responses as texts: elements (default: canonical, in request order; shuffled with `seed`), split into n_texts batches of
    consecutive elements, or with single=True one object per text."""
    els = list(elements) if elements is not None else [element(i, d) for i, d in enumerate(blocks)]
    if seed is not None:
        order = np.random.default_rng(seed).permutation(len(els))
        els = [els[k] for k in order]
    if single:
        return els
    bounds = np.linspace(0, len(els), n_texts + 1).astype(np.int64)
    return [b"[" + b",".join(els[bounds[k]:bounds[k + 1]]) + b"]" for k in range(n_texts)]


# ------------------------------------------------------------------------------------------ the rules, restated
def _b64(s):
    """Standard base64 with padding and zero unused bits: exactly the strings b64encode writes."""
    try:
        raw = base64.b64decode(s.encode("ascii"), validate=True)
    except (UnicodeEncodeError, binascii.Error, ValueError):
        raise Fault(A.ERR_INVALID_ARG)
    if base64.b64encode(raw).decode() != s:
        raise Fault(A.ERR_INVALID_ARG)
    return raw


def _response(v, n):
    """One response object → (id, block bytes, or None for an error response)."""
    if not isinstance(v, R.Obj):
        raise Fault(A.ERR_INVALID_ARG)
    keys = [k for k, _ in v.pairs]
    if len(set(keys)) != len(keys):
        raise Fault(A.ERR_INVALID_ARG)
    d = dict(v.pairs)
    ver = d.get("jsonrpc")
    if not isinstance(ver, str) or isinstance(ver, R.Num) or ver != "2.0" or "id" not in d or ("result" in d) == ("error" in d):
        raise Fault(A.ERR_INVALID_ARG)
    i = R._u64(d["id"])
    if i >= n:
        raise Fault(A.ERR_INVALID_ARG)
    return i, (_b64(R._string(d["result"])) if "result" in d else None)


def _skip(s, i):
    while i < len(s) and s[i] in R._WS:
        i += 1
    return i


def read(n, texts):
    """The blocks of requests 0 … n-1 the rules give for the texts, or Fault(status, index)."""
    pos, got = 0, []

    def one(s, i):
        nonlocal pos
        try:
            v, i = R._value(s, i, 1)
            got.append(_response(v, n))
        except Fault as f:
            raise Fault(f.status, pos)
        pos += 1
        return i

    for t in texts:
        s = R._as_str(t)
        i = _skip(s, 0)
        if s[i:i + 1] == "[":
            i = _skip(s, i + 1)
            if s[i:i + 1] == "]":
                i += 1
            else:
                while True:
                    i = _skip(s, one(s, i))
                    if s[i:i + 1] == ",":
                        i += 1
                        continue
                    if s[i:i + 1] == "]":
                        i += 1
                        break
                    raise Fault(A.ERR_INVALID_ARG)
        else:
            i = one(s, i)
        if s[i:].strip(R._WS):
            raise Fault(A.ERR_INVALID_ARG)
    count = [0] * n
    by_id = [None] * n
    for i, data in got:
        count[i] += 1
        by_id[i] = data
    for i in range(n):
        if count[i] != 1:
            raise Fault(A.ERR_INVALID_ARG, i)
    for i in range(n):
        if by_id[i] is None:
            raise Fault(A.ERR_MISSING_BLOCK, i)
    return by_id


def expected(n, texts):
    """read(), with a failure as (status, index) instead of an exception."""
    try:
        return read(n, texts)
    except Fault as f:
        return (f.status, f.index)


def arrays(blocks):
    """The block arrays of ipcfp_blocks_from_rpc_json for blocks in request order: 16-aligned offsets, lengths, blob (padding zero)."""
    lens = np.array([len(b) for b in blocks], np.uint32)
    padded = [b + bytes(-len(b) % 16) for b in blocks]
    offs = np.zeros(len(blocks), np.uint64)
    if blocks:
        offs[1:] = np.cumsum([len(p) for p in padded[:-1]], dtype=np.uint64)
    return offs, lens, np.frombuffer(b"".join(padded), np.uint8)


def assert_blocks_equal(w, cids, blocks):
    """An A.WitnessPy from ipcfp_blocks_from_rpc_json holds exactly `blocks` for `cids`, in the documented layout."""
    offs, lens, blob = arrays(blocks)
    assert np.array_equal(w.cids, np.asarray(cids, np.uint8).reshape(-1, 38))
    assert np.array_equal(w.offsets, offs) and np.array_equal(w.lengths, lens)
    assert w.blob.tobytes() == blob.tobytes()


# ------------------------------------------------------------------------------------------ named cases: (name, texts, outcome)
def cases(blocks):
    """Hand-made inputs over `blocks` (at least 4): each with the outcome the rules give (A.OK or the status)."""
    n = len(blocks)
    els = [element(i, d) for i, d in enumerate(blocks)]
    b = lambda es: b"[" + b",".join(es) + b"]"
    swap = lambda k, e: els[:k] + [e] + els[k + 1:]
    d1 = base64.b64encode(blocks[1]).decode()
    return [
        ("canonical", [b(els)], A.OK),
        ("shuffled_three_texts", render(blocks, 3, seed=5), A.OK),
        ("one_object_per_text", render(blocks, single=True, seed=9), A.OK),
        ("empty_batch_text_too", [b"[]", b(els)], A.OK),
        ("pretty_element", [b(swap(1, pretty(1, blocks[1])))], A.OK),
        ("whitespace_around", [b" \n[ " + b" , ".join(els) + b" ]\t"], A.OK),
        ("unknown_member", [b(swap(2, els[2][:-1] + b',"extra":[1,{"x":null}]}'))], A.OK),
        ("escaped_result", [b(swap(1, ('{"jsonrpc":"2.0","result":"%s","id":1}' % d1.replace("A", "\\u0041").replace("/", "\\/")).encode()))], A.OK),
        ("escaped_key", [b(swap(1, ('{"jsonrpc":"2.0","r\\u0065sult":"%s","id":1}' % d1).encode()))], A.OK),
        ("error_response", [b(swap(2, error_element(2)))], A.ERR_MISSING_BLOCK),
        ("duplicate_id", [b(els + [els[1]])], A.ERR_INVALID_ARG),
        ("missing_id", [b(els[:2] + els[3:])], A.ERR_INVALID_ARG),
        ("id_out_of_range", [b(els + [element(n, b"x")])], A.ERR_INVALID_ARG),
        ("id_string", [b(swap(1, els[1].replace(b'"id":1}', b'"id":"1"}')))], A.ERR_INVALID_ARG),
        ("id_negative", [b(swap(1, els[1].replace(b'"id":1}', b'"id":-1}')))], A.ERR_INVALID_ARG),
        ("id_float", [b(swap(1, els[1].replace(b'"id":1}', b'"id":1.0}')))], A.ERR_INVALID_ARG),
        ("id_leading_zero", [b(swap(1, els[1].replace(b'"id":1}', b'"id":01}')))], A.ERR_INVALID_ARG),
        ("repeated_member", [b(swap(1, els[1][:-1] + b',"jsonrpc":"2.0"}'))], A.ERR_INVALID_ARG),
        ("result_and_error", [b(swap(1, els[1][:-1] + b',"error":null}'))], A.ERR_INVALID_ARG),
        ("neither", [b(swap(1, b'{"jsonrpc":"2.0","id":1}'))], A.ERR_INVALID_ARG),
        ("wrong_version", [b(swap(1, els[1].replace(b'"2.0"', b'"1.0"')))], A.ERR_INVALID_ARG),
        ("no_version", [b(swap(1, els[1].replace(b'"jsonrpc":"2.0",', b"")))], A.ERR_INVALID_ARG),
        ("result_not_string", [b(swap(1, b'{"jsonrpc":"2.0","result":null,"id":1}'))], A.ERR_INVALID_ARG),
        ("base64_unpadded", [b(swap(1, element(1, b"ab").replace(b"=", b"")))], A.ERR_INVALID_ARG),
        ("base64_nonzero_trailing_bits", [b(swap(1, element(1, b"ab").replace(b"YWI=", b"YWJ=")))], A.ERR_INVALID_ARG),
        ("base64_nonzero_trailing_bits_2", [b(swap(1, element(1, b"a").replace(b"YQ==", b"YR==")))], A.ERR_INVALID_ARG),
        ("base64_urlsafe", [b(swap(1, element(1, b"\xfb\xff").replace(b"+/8=", b"-_8=")))], A.ERR_INVALID_ARG),
        ("base64_pad_inside", [b(swap(1, element(1, b"abcdef").replace(b"YWJjZGVm", b"YW==ZGVm")))], A.ERR_INVALID_ARG),
        ("element_not_object", [b(swap(1, b"[1]"))], A.ERR_INVALID_ARG),
        ("element_malformed", [b(swap(3, els[3][:-1]))], A.ERR_INVALID_ARG),
        ("trailing_comma", [b(els)[:-1] + b",]"], A.ERR_INVALID_ARG),
        ("missing_bracket", [b(els)[:-1]], A.ERR_INVALID_ARG),
        ("trailing_bytes", [b(els) + b"x"], A.ERR_INVALID_ARG),
        ("empty_text", [b(els), b""], A.ERR_INVALID_ARG),
        ("two_objects_one_text", [els[0] + els[1]] + els[2:], A.ERR_INVALID_ARG),
        ("nested_batch", [b"[" + b(els) + b"]"], A.ERR_INVALID_ARG),
    ]
