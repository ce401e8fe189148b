"""Lotus JSON-RPC texts of a tipset, for ipcfp_tipset_desc_from_json / ipcfp_tipset_upload_json (test infrastructure).

* `texts(ts)` renders, for any synth.Tipset, the three `result` values a caller gets from Lotus: the parent and the child ApiTipset
  (ChainGetTipSetByHeight, with the Lotus block-header fields the reference does not read) and the receipt list (ChainGetParentReceipts)
  in canonical form — compact, struct field order, the form the device parser reads.
* `MUTATORS` rewrites such texts: whitespace, key orders, unknown fields, escapes, missing / null / duplicate fields, wrong types,
  out-of-range and non-integer numbers, bad CID strings, arrays for structs, truncation, trailing bytes. Each names the outcome the rules
  give (OK or the status).
* `read(parent, child, receipts)` states the rules of include/ipcfp.h independently of the library, on Python's `json` module with
  `object_pairs_hook`: it returns the expected descriptor, or raises Fault(status, index).
"""
import base64
import json
import re

import numpy as np

from ipc_filecoin_proofs_b200 import _abi as A

NO_INDEX = 2 ** 64 - 1
_B32 = "abcdefghijklmnopqrstuvwxyz234567"


def cid_str(cid):
    """`Cid::to_string()` of a CIDv1: "b" + RFC 4648 base32, lower case, no padding."""
    return "b" + base64.b32encode(bytes(cid)).decode().lower().rstrip("=")


def cid_map(cid):
    return '{"/":"%s"}' % cid_str(cid)


# ------------------------------------------------------------------------------------------ rendering
class P:
    """A JSON object as ordered (key text, value) pairs: the key text is written verbatim between quotes (escapes allowed)."""

    def __init__(self, pairs):
        self.pairs = list(pairs)


class Raw(str):
    """A JSON text written verbatim (numbers, literals, hand-made fragments)."""


def dump(x, sep=":", comma=",", nl=""):
    if isinstance(x, Raw):
        return str(x)
    if isinstance(x, P):
        return "{" + nl + (comma + nl).join('"%s"%s%s' % (k, sep, dump(v, sep, comma, nl)) for k, v in x.pairs) + nl + "}"
    if isinstance(x, list):
        return "[" + nl + (comma + nl).join(dump(v, sep, comma, nl) for v in x) + nl + "]"
    if isinstance(x, str):
        return json.dumps(x)
    if isinstance(x, bool) or x is None:
        return json.dumps(x)
    return str(int(x))


def _cm(cid):
    return P([("/", cid_str(cid))])


def block_header(miner, parents, state_root, receipts_root, messages, height, k=0):
    """An ApiBlockHeader as Lotus writes a BlockHeader: the six fields the reference reads among the others, in Lotus' order."""
    b64 = base64.b64encode(bytes([k % 251] * 12)).decode()
    return P([("Miner", miner), ("Ticket", P([("VRFProof", b64)])), ("ElectionProof", P([("WinCount", 1), ("VRFProof", b64)])),
              ("BeaconEntries", [P([("Round", 3000000 + k), ("Data", b64)])]), ("WinPoStProof", [P([("PoStProof", 3), ("ProofBytes", b64)])]),
              ("Parents", [_cm(c) for c in parents]), ("ParentWeight", "81960412"), ("Height", height), ("ParentStateRoot", _cm(state_root)),
              ("ParentMessageReceipts", _cm(receipts_root)), ("Messages", _cm(messages)), ("BLSAggregate", P([("Type", 2), ("Data", b64)])),
              ("Timestamp", 1700000000 + k), ("BlockSig", P([("Type", 2), ("Data", b64)])), ("ForkSignaling", 0), ("ParentBaseFee", "100")])


def tipsets(ts):
    """(parent ApiTipset, child ApiTipset) of a synth.Tipset as P structures."""
    pc = [bytes(c) for c in np.asarray(ts.parent_cids).reshape(-1, 38)]
    tx = [bytes(c) for c in np.asarray(ts.parent_txmeta_cids).reshape(-1, 38)]
    other = bytes(ts.receipts_root)
    parent = P([("Cids", [_cm(c) for c in pc]),
                ("Blocks", [block_header("f0%d" % (1000 + i), [other], other, other, tx[i], int(ts.parent_epoch), i) for i in range(len(pc))]),
                ("Height", int(ts.parent_epoch))])
    child = P([("Cids", [_cm(bytes(ts.child_cid))]),
               ("Blocks", [block_header("f01234", pc, bytes(ts.parent_state_root), bytes(ts.receipts_root), bytes(ts.child_cid),
                                        int(ts.child_epoch))]),
               ("Height", int(ts.child_epoch))])
    return parent, child


def _exit_code(i):
    return (0, 0, 0, 7, 33, 4294967295)[i % 6] if i % 3 == 0 else 0


def _return(i):
    return base64.b64encode(bytes(range(i % 7))).decode()


def _gas(i):
    return (i * 2654435761 + 12345) % (2 ** 64) if i % 11 else (2 ** 64 - 1 if i % 22 else 0)


def receipt_pairs(ts, i):
    """ApiReceipt i as P: its canonical fields."""
    root = _cm(bytes(ts.events_roots[i])) if ts.has_events_root[i] else Raw("null")
    return P([("ExitCode", _exit_code(i)), ("Return", _return(i)), ("GasUsed", _gas(i)), ("EventsRoot", root)])


def receipt_records(ts):
    """The canonical text of every receipt, as a list (fast: the 1 M-receipt tipset)."""
    roots = np.asarray(ts.events_roots).reshape(-1, 38)
    has = np.asarray(ts.has_events_root)
    out = []
    for i in range(int(ts.n_receipts)):
        er = '{"/":"b%s"}' % base64.b32encode(roots[i].tobytes()).decode().lower().rstrip("=") if has[i] else "null"
        out.append('{"ExitCode":%d,"Return":"%s","GasUsed":%d,"EventsRoot":%s}' % (_exit_code(i), _return(i), _gas(i), er))
    return out


def texts(ts):
    """(parent, child, receipts) texts of a synth.Tipset: the tipsets compact in Lotus' field order, the receipt list canonical."""
    parent, child = tipsets(ts)
    return dump(parent), dump(child), "[" + ",".join(receipt_records(ts)) + "]"


# ------------------------------------------------------------------------------------------ mutators
def _with_receipt(ts, k, fn):
    """Texts whose receipt k (the list's P structures) is replaced by fn(P) (a P or a Raw)."""
    parent, child = tipsets(ts)
    recs = receipt_records(ts)
    recs[k] = dump(fn(receipt_pairs(ts, k)))
    return dump(parent), dump(child), "[" + ",".join(recs) + "]"


def _with_tipset(ts, which, fn):
    parent, child = tipsets(ts)
    if which == "parent":
        parent = fn(parent)
    else:
        child = fn(child)
    return dump(parent), dump(child), "[" + ",".join(receipt_records(ts)) + "]"


def _pairs(p, fn):
    return P(fn(list(p.pairs)))


def _set(p, key, value):
    return P([(k, value if k == key else v) for k, v in p.pairs])


def _drop(p, key):
    return P([(k, v) for k, v in p.pairs if k != key])


def _first_root(ts, want=True):
    """The index of a receipt deep inside the list with (or without) an events root."""
    has = np.asarray(ts.has_events_root)
    idx = [i for i in range(len(has)) if bool(has[i]) == want]
    return idx[len(idx) * 2 // 3] if idx else None


def _root_string(ts, k, fn):
    return _with_receipt(ts, k, lambda p: _set(p, "EventsRoot", P([("/", fn(cid_str(bytes(ts.events_roots[k]))))])))


def _flip_unused_bit(s):
    return s[:-1] + _B32[_B32.index(s[-1]) ^ 1]


def _bad_char(s):
    return s[:20] + "1" + s[21:]


def _pretty(ts):
    parent, child = tipsets(ts)
    recs = [receipt_pairs(ts, i) for i in range(int(ts.n_receipts))]
    return dump(parent, ": ", ", ", "\n  "), dump(child, ": ", ", "), dump(recs, ": ", ", ", "\n")


def _all_receipts(ts, fn):
    parent, child = tipsets(ts)
    return dump(parent), dump(child), dump([fn(receipt_pairs(ts, i)) for i in range(int(ts.n_receipts))])


def _texts_edit(ts, fn):
    return fn(*texts(ts))


QM = "QmYwAPJzv5CZsnA625s3Xf2nemtYgPpHdWEz79ojWnPbdG"
ZB58 = "zdj7WWeQ43G6JJvLWQWZpyHuAMq6uYWRjkBXFad11vE2LHhQ7"
NESTED = Raw('{"a":[1,2.5e-3,{"b":null,"c":[true,false,"x\\u0041"]}],"d":{}}')

# (name, texts(ts) → (parent, child, receipts), expected outcome: A.OK or the status). k = a receipt deep inside the list.
MUTATORS = [
    ("canonical", lambda ts, k: texts(ts), A.OK),
    ("pretty", lambda ts, k: _pretty(ts), A.OK),
    ("space_around", lambda ts, k: _texts_edit(ts, lambda p, c, r: (" \n" + p + "\t", c, "\r\n " + r)), A.OK),
    ("trailing_space", lambda ts, k: _texts_edit(ts, lambda p, c, r: (p, c, r + " ")), A.OK),
    ("space_in_one", lambda ts, k: _with_receipt(ts, k, lambda p: Raw(dump(p, " : ", " , "))), A.OK),
    ("key_order_one", lambda ts, k: _with_receipt(ts, k, lambda p: _pairs(p, lambda l: l[::-1])), A.OK),
    ("key_order_all", lambda ts, k: _all_receipts(ts, lambda p: _pairs(p, lambda l: l[2:] + l[:2])), A.OK),
    ("unknown_field", lambda ts, k: _with_receipt(ts, k, lambda p: _pairs(p, lambda l: l[:2] + [("Extra", NESTED)] + l[2:])), A.OK),
    ("unknown_field_all", lambda ts, k: _all_receipts(ts, lambda p: P(p.pairs + [("exitCode", 5)])), A.OK),
    ("unknown_in_cidmap", lambda ts, k: _with_receipt(ts, _first_root(ts), lambda p: _set(p, "EventsRoot", P(
        [("x", NESTED)] + [("/", cid_str(bytes(ts.events_roots[_first_root(ts)])))]))), A.OK),
    ("unknown_in_tipset", lambda ts, k: _with_tipset(ts, "child", lambda t: P([("Key", NESTED)] + t.pairs)), A.OK),
    ("escaped_key", lambda ts, k: _with_receipt(ts, k, lambda p: P([("\\u0045xitCode" if a == "ExitCode" else a, v) for a, v in p.pairs])), A.OK),
    ("escaped_slash_key", lambda ts, k: _with_receipt(ts, _first_root(ts), lambda p: _set(p, "EventsRoot", P(
        [("\\/", cid_str(bytes(ts.events_roots[_first_root(ts)])))]))), A.OK),
    ("escaped_cid", lambda ts, k: _root_string(ts, _first_root(ts), lambda s: Raw('"\\u0062' + s[1:] + '"')), A.OK),
    ("events_root_missing", lambda ts, k: _all_receipts(ts, lambda p: _drop(p, "EventsRoot") if dump(p).endswith("null}") else p), A.OK),
    ("return_escaped_record", lambda ts, k: _with_receipt(ts, k, lambda p: _set(p, "Return", Raw('"{\\"ExitCode\\":0,\\"x\\":{}"'))), A.OK),
    ("return_any_string", lambda ts, k: _with_receipt(ts, k, lambda p: _set(p, "Return", "not base64 at all é")), A.OK),
    ("exit_code_u32_max", lambda ts, k: _with_receipt(ts, k, lambda p: _set(p, "ExitCode", 4294967295)), A.OK),
    ("gas_u64_max", lambda ts, k: _with_receipt(ts, k, lambda p: _set(p, "GasUsed", 2 ** 64 - 1)), A.OK),
    ("empty_list", lambda ts, k: _texts_edit(ts, lambda p, c, r: (p, c, "[]")), A.OK),
    ("empty_list_spaced", lambda ts, k: _texts_edit(ts, lambda p, c, r: (p, c, " [ ] ")), A.OK),
    ("height_negative", lambda ts, k: _with_tipset(ts, "parent", lambda t: _set(t, "Height", -5)), A.OK),
    # failures
    ("duplicate_key", lambda ts, k: _with_receipt(ts, k, lambda p: P(p.pairs + [("ExitCode", 0)])), A.ERR_INVALID_ARG),
    ("duplicate_escaped_key", lambda ts, k: _with_receipt(ts, k, lambda p: P(p.pairs + [("Gas\\u0055sed", 0)])), A.ERR_INVALID_ARG),
    ("duplicate_events_root", lambda ts, k: _with_receipt(ts, k, lambda p: P(p.pairs + [("EventsRoot", Raw("null"))])), A.ERR_INVALID_ARG),
    ("duplicate_in_cidmap", lambda ts, k: _with_receipt(ts, _first_root(ts), lambda p: _set(p, "EventsRoot", P(
        [("/", cid_str(bytes(ts.events_roots[_first_root(ts)])))] * 2))), A.ERR_INVALID_ARG),
    ("duplicate_height", lambda ts, k: _with_tipset(ts, "child", lambda t: P(t.pairs + [("Height", 1)])), A.ERR_INVALID_ARG),
    ("return_null", lambda ts, k: _with_receipt(ts, k, lambda p: _set(p, "Return", Raw("null"))), A.ERR_INVALID_ARG),
    ("return_number", lambda ts, k: _with_receipt(ts, k, lambda p: _set(p, "Return", 5)), A.ERR_INVALID_ARG),
    ("exit_code_string", lambda ts, k: _with_receipt(ts, k, lambda p: _set(p, "ExitCode", "0")), A.ERR_INVALID_ARG),
    ("exit_code_2_32", lambda ts, k: _with_receipt(ts, k, lambda p: _set(p, "ExitCode", 2 ** 32)), A.ERR_INVALID_ARG),
    ("exit_code_negative", lambda ts, k: _with_receipt(ts, k, lambda p: _set(p, "ExitCode", Raw("-1"))), A.ERR_INVALID_ARG),
    ("exit_code_minus_zero", lambda ts, k: _with_receipt(ts, k, lambda p: _set(p, "ExitCode", Raw("-0"))), A.ERR_INVALID_ARG),
    ("gas_2_64", lambda ts, k: _with_receipt(ts, k, lambda p: _set(p, "GasUsed", 2 ** 64)), A.ERR_INVALID_ARG),
    ("gas_fraction", lambda ts, k: _with_receipt(ts, k, lambda p: _set(p, "GasUsed", Raw("1.0"))), A.ERR_INVALID_ARG),
    ("gas_exponent", lambda ts, k: _with_receipt(ts, k, lambda p: _set(p, "GasUsed", Raw("1e3"))), A.ERR_INVALID_ARG),
    ("gas_null", lambda ts, k: _with_receipt(ts, k, lambda p: _set(p, "GasUsed", Raw("null"))), A.ERR_INVALID_ARG),
    ("height_minus_zero", lambda ts, k: _with_tipset(ts, "parent", lambda t: _set(t, "Height", Raw("-0"))), A.ERR_INVALID_ARG),
    ("height_2_63", lambda ts, k: _with_tipset(ts, "child", lambda t: _set(t, "Height", 2 ** 63)), A.ERR_INVALID_ARG),
    ("missing_gas", lambda ts, k: _with_receipt(ts, k, lambda p: _drop(p, "GasUsed")), A.ERR_INVALID_ARG),
    ("missing_return", lambda ts, k: _with_receipt(ts, k, lambda p: _drop(p, "Return")), A.ERR_INVALID_ARG),
    ("missing_slash", lambda ts, k: _with_receipt(ts, _first_root(ts), lambda p: _set(p, "EventsRoot", P([("cid", "x")]))), A.ERR_INVALID_ARG),
    ("events_root_string", lambda ts, k: _with_receipt(ts, _first_root(ts), lambda p: _set(
        p, "EventsRoot", cid_str(bytes(ts.events_roots[_first_root(ts)])))), A.ERR_INVALID_ARG),
    ("events_root_slash_number", lambda ts, k: _with_receipt(ts, k, lambda p: _set(p, "EventsRoot", P([("/", 5)]))), A.ERR_INVALID_ARG),
    ("bad_base32_char", lambda ts, k: _root_string(ts, _first_root(ts), _bad_char), A.ERR_INVALID_ARG),
    ("upper_case_base32", lambda ts, k: _root_string(ts, _first_root(ts), lambda s: s[:30] + s[30:].upper()), A.ERR_INVALID_ARG),
    ("unused_bit_set", lambda ts, k: _root_string(ts, _first_root(ts), _flip_unused_bit), A.ERR_INVALID_ARG),
    ("cid_v0_qm", lambda ts, k: _root_string(ts, _first_root(ts), lambda s: QM), A.ERR_UNSUPPORTED),
    ("cid_base58_z", lambda ts, k: _root_string(ts, _first_root(ts), lambda s: ZB58), A.ERR_UNSUPPORTED),
    ("cid_upper_multibase", lambda ts, k: _root_string(ts, _first_root(ts), lambda s: "B" + s[1:].upper()), A.ERR_UNSUPPORTED),
    ("cid_36_bytes", lambda ts, k: _root_string(ts, _first_root(ts), lambda s: cid_str(bytes(ts.events_roots[_first_root(ts)])[:36])),
     A.ERR_UNSUPPORTED),
    ("cid_empty", lambda ts, k: _root_string(ts, _first_root(ts), lambda s: ""), A.ERR_UNSUPPORTED),
    ("receipt_as_array", lambda ts, k: _with_receipt(ts, k, lambda p: [v for _, v in p.pairs]), A.ERR_UNSUPPORTED),
    ("cidmap_as_array", lambda ts, k: _with_receipt(ts, _first_root(ts), lambda p: _set(
        p, "EventsRoot", [cid_str(bytes(ts.events_roots[_first_root(ts)]))])), A.ERR_UNSUPPORTED),
    ("header_as_array", lambda ts, k: _with_tipset(ts, "child", lambda t: _set(t, "Blocks", [[v for _, v in t.pairs[1][1][0].pairs]])),
     A.ERR_UNSUPPORTED),
    ("receipt_number", lambda ts, k: _with_receipt(ts, k, lambda p: Raw("7")), A.ERR_INVALID_ARG),
    ("bad_json_in_unknown", lambda ts, k: _with_receipt(ts, k, lambda p: Raw(dump(p)[:-1] + ',"x":[1,}')), A.ERR_INVALID_ARG),
    ("lone_surrogate", lambda ts, k: _with_receipt(ts, k, lambda p: _set(p, "Return", Raw('"\\ud800"'))), A.ERR_INVALID_ARG),
    ("control_char", lambda ts, k: _with_receipt(ts, k, lambda p: _set(p, "Return", Raw('"a\tb"'))), A.ERR_INVALID_ARG),
    ("truncated", lambda ts, k: _texts_edit(ts, lambda p, c, r: (p, c, r[:len(r) * 3 // 5])), A.ERR_INVALID_ARG),
    ("truncated_end", lambda ts, k: _texts_edit(ts, lambda p, c, r: (p, c, r[:-1])), A.ERR_INVALID_ARG),
    ("trailing_bytes", lambda ts, k: _texts_edit(ts, lambda p, c, r: (p, c, r + "x")), A.ERR_INVALID_ARG),
    ("trailing_comma", lambda ts, k: _texts_edit(ts, lambda p, c, r: (p, c, r[:-1] + ",]")), A.ERR_INVALID_ARG),
    ("missing_comma", lambda ts, k: _texts_edit(ts, lambda p, c, r: (p, c, r.replace("},{", "}{", 1))), A.ERR_INVALID_ARG),
    ("list_is_object", lambda ts, k: _texts_edit(ts, lambda p, c, r: (p, c, "{}")), A.ERR_INVALID_ARG),
    ("list_empty_text", lambda ts, k: _texts_edit(ts, lambda p, c, r: (p, c, "")), A.ERR_INVALID_ARG),
    ("two_lists", lambda ts, k: _texts_edit(ts, lambda p, c, r: (p, c, r + r)), A.ERR_INVALID_ARG),
    ("child_no_cids", lambda ts, k: _with_tipset(ts, "child", lambda t: _set(t, "Cids", [])), A.ERR_INVALID_ARG),
    ("child_no_blocks", lambda ts, k: _with_tipset(ts, "child", lambda t: _set(t, "Blocks", [])), A.ERR_INVALID_ARG),
    ("parent_lengths_differ", lambda ts, k: _with_tipset(ts, "parent", lambda t: _set(t, "Cids", t.pairs[0][1] + [t.pairs[0][1][0]])),
     A.ERR_UNSUPPORTED),
    ("parent_missing_miner", lambda ts, k: _with_tipset(ts, "parent", lambda t: _set(t, "Blocks", [_drop(b, "Miner") for b in t.pairs[1][1]])),
     A.ERR_INVALID_ARG),
    ("parent_bad_messages", lambda ts, k: _with_tipset(ts, "parent", lambda t: _set(t, "Blocks", [_set(b, "Messages", P([("/", QM)]))
                                                                                                 for b in t.pairs[1][1]])), A.ERR_UNSUPPORTED),
    ("child_bad_cid", lambda ts, k: _with_tipset(ts, "child", lambda t: _set(t, "Cids", [P([("/", "bafy!")])])), A.ERR_INVALID_ARG),
    ("child_text_truncated", lambda ts, k: _texts_edit(ts, lambda p, c, r: (p, c[:-1], r)), A.ERR_INVALID_ARG),
    ("parent_text_trailing", lambda ts, k: _texts_edit(ts, lambda p, c, r: (p + "]", c, r)), A.ERR_INVALID_ARG),
]


# ------------------------------------------------------------------------------------------ the rules, restated
class Fault(Exception):
    def __init__(self, status, index=NO_INDEX):
        super().__init__(status, index)
        self.status, self.index = status, index


class Obj:
    def __init__(self, pairs):
        self.pairs = pairs


class Num(str):
    pass


def _no_constant(s):
    raise ValueError(s)


_DEC = json.JSONDecoder(object_pairs_hook=Obj, parse_int=Num, parse_float=Num, parse_constant=_no_constant, strict=True)
_WS = " \t\n\r"


def _deep_ok(v, level, limit=64):
    """The host parser's nesting limit (a value deeper than 64 levels is refused) and its refusal of unpaired surrogate escapes."""
    if level > limit:
        return False
    if isinstance(v, Obj):
        return all(not re.search("[\ud800-\udfff]", k) and _deep_ok(x, level + 1) for k, x in v.pairs)
    if isinstance(v, list):
        return all(_deep_ok(x, level + 1) for x in v)
    if isinstance(v, str) and not isinstance(v, Num):
        return not re.search("[\ud800-\udfff]", v)
    return True


def _value(s, i, level):
    """One JSON value at s[i:] (after whitespace) → (value, end)."""
    while i < len(s) and s[i] in _WS:
        i += 1
    try:
        v, end = _DEC.raw_decode(s, i)
    except ValueError:
        raise Fault(A.ERR_INVALID_ARG)
    if not _deep_ok(v, level):
        raise Fault(A.ERR_INVALID_ARG)
    return v, end


def _struct(v, names, f):
    if isinstance(v, list):
        raise Fault(A.ERR_UNSUPPORTED)
    if not isinstance(v, Obj):
        raise Fault(A.ERR_INVALID_ARG)
    got = {}
    for k, x in v.pairs:
        if k in names:
            if k in got:
                raise Fault(A.ERR_INVALID_ARG)
            got[k] = x
            f(k, x)
    return got


def _require(got, names):
    if any(n not in got for n in names):
        raise Fault(A.ERR_INVALID_ARG)


def _u64(v):
    if not isinstance(v, Num) or not re.fullmatch("[0-9]+", v) or int(v) >= 2 ** 64:
        raise Fault(A.ERR_INVALID_ARG)
    return int(v)


def _i64(v):
    if not isinstance(v, Num) or not re.fullmatch("-?[0-9]+", v) or v == "-0" or not -2 ** 63 <= int(v) < 2 ** 63:
        raise Fault(A.ERR_INVALID_ARG)
    return int(v)


def _string(v):
    if not isinstance(v, str) or isinstance(v, Num):
        raise Fault(A.ERR_INVALID_ARG)
    return v


def _cid_map(v):
    got = _struct(v, ("/",), lambda k, x: _string(x))
    _require(got, ("/",))
    return got["/"]


def _cid(s):
    """parse_cid with the rule of ipcfp_bundle_from_json: "b" + base32 → exactly 38 bytes."""
    if not s or s[0] != "b":
        raise Fault(A.ERR_UNSUPPORTED)
    if any(c not in _B32 for c in s[1:]):
        raise Fault(A.ERR_INVALID_ARG)
    bits = 0
    for c in s[1:]:
        bits = (bits << 5) | _B32.index(c)
    nbits = 5 * (len(s) - 1)
    extra = nbits % 8
    if bits & ((1 << extra) - 1):
        raise Fault(A.ERR_INVALID_ARG)
    if nbits // 8 != 38:
        raise Fault(A.ERR_UNSUPPORTED)
    return (bits >> extra).to_bytes(38, "big")


def _list(v, each):
    if not isinstance(v, list):
        raise Fault(A.ERR_INVALID_ARG)
    for x in v:
        each(x)


HEADER = ("Miner", "Parents", "ParentStateRoot", "ParentMessageReceipts", "Messages", "Height")


def _header(b):
    def field(k, x):
        if k == "Miner":
            _string(x)
        elif k == "Parents":
            _list(x, _cid_map)
        elif k == "Height":
            _i64(x)
        else:
            _cid_map(x)
    _require(_struct(b, HEADER, field), HEADER)


def _tipset(text):
    v, end = _value(text, 0, 0)
    if text[end:].strip(_WS):
        raise Fault(A.ERR_INVALID_ARG)

    def field(k, x):
        if k == "Cids":
            _list(x, _cid_map)
        elif k == "Blocks":
            _list(x, _header)
        else:
            _i64(x)
    got = _struct(v, ("Cids", "Blocks", "Height"), field)
    _require(got, ("Cids", "Blocks", "Height"))
    return got


def _field(obj, name):
    return next(x for k, x in obj.pairs if k == name)


def _receipt(v):
    def field(k, x):
        if k == "ExitCode":
            if _u64(x) >= 2 ** 32:
                raise Fault(A.ERR_INVALID_ARG)
        elif k == "Return":
            _string(x)
        elif k == "GasUsed":
            _u64(x)
        elif x is not None:
            _cid_map(x)
    got = _struct(v, ("ExitCode", "Return", "GasUsed", "EventsRoot"), field)
    _require(got, ("ExitCode", "Return", "GasUsed"))
    if got.get("EventsRoot") is None:
        return None
    return _cid(_cid_map(got["EventsRoot"]))


def _receipts(s):
    roots = []
    i = 0
    while i < len(s) and s[i] in _WS:
        i += 1
    if s[i:i + 1] != "[":
        raise Fault(A.ERR_INVALID_ARG)
    i += 1
    while i < len(s) and s[i] in _WS:
        i += 1
    if s[i:i + 1] == "]":
        i += 1
    else:
        while True:
            idx = len(roots)
            try:
                v, i = _value(s, i, 1)
                roots.append(_receipt(v))
            except Fault as f:
                raise Fault(f.status, idx)
            while i < len(s) and s[i] in _WS:
                i += 1
            if s[i:i + 1] == ",":
                i += 1
                continue
            if s[i:i + 1] == "]":
                i += 1
                break
            raise Fault(A.ERR_INVALID_ARG)
    if s[i:].strip(_WS):
        raise Fault(A.ERR_INVALID_ARG)
    return roots


def _as_str(t):
    return t.decode("latin-1") if isinstance(t, (bytes, bytearray)) else t


def read(parent, child, receipts):
    """The descriptor the rules give for the three texts, as a dict of numpy arrays / ints, or Fault(status, index)."""
    parent, child, receipts = _as_str(parent), _as_str(child), _as_str(receipts)
    p = _tipset(parent)
    pcids = [_cid(_cid_map(c)) for c in p["Cids"]]
    if len(p["Blocks"]) != len(p["Cids"]):
        raise Fault(A.ERR_UNSUPPORTED)
    txmeta = [_cid(_cid_map(_field(b, "Messages"))) for b in p["Blocks"]]
    c = _tipset(child)
    if not c["Cids"] or not c["Blocks"]:
        raise Fault(A.ERR_INVALID_ARG)
    child_cid = _cid(_cid_map(c["Cids"][0]))
    receipts_root = _cid(_cid_map(_field(c["Blocks"][0], "ParentMessageReceipts")))
    state_root = _cid(_cid_map(_field(c["Blocks"][0], "ParentStateRoot")))
    roots = _receipts(receipts)
    n = len(roots)
    u8 = lambda bs: np.frombuffer(b"".join(bs), dtype=np.uint8).reshape(len(bs), 38) if bs else np.zeros((0, 38), np.uint8)
    return dict(parent_epoch=int(p["Height"]), child_epoch=int(c["Height"]), n_parents=len(pcids), parent_cids=u8(pcids), parent_txmeta_cids=u8(txmeta),
                child_cid=np.frombuffer(child_cid, np.uint8), receipts_root=np.frombuffer(receipts_root, np.uint8),
                parent_state_root=np.frombuffer(state_root, np.uint8), n_receipts=n,
                events_roots=u8([r if r is not None else bytes(38) for r in roots]),
                has_events_root=np.array([r is not None for r in roots], dtype=np.uint8))


def expected(parent, child, receipts):
    """read(), with a failure as (status, index) instead of an exception."""
    try:
        return read(parent, child, receipts)
    except Fault as f:
        return (f.status, f.index)


def desc_dict(x):
    """The descriptor fields of a synth.Tipset or an A.TipsetInfoPy, in read()'s form."""
    return dict(parent_epoch=int(x.parent_epoch), child_epoch=int(x.child_epoch), n_parents=int(x.n_parents),
                parent_cids=np.asarray(x.parent_cids, np.uint8).reshape(-1, 38), parent_txmeta_cids=np.asarray(x.parent_txmeta_cids, np.uint8).reshape(-1, 38),
                child_cid=np.asarray(x.child_cid, np.uint8), receipts_root=np.asarray(x.receipts_root, np.uint8),
                parent_state_root=np.asarray(x.parent_state_root, np.uint8), n_receipts=int(x.n_receipts),
                events_roots=np.asarray(x.events_roots, np.uint8).reshape(-1, 38), has_events_root=np.asarray(x.has_events_root, np.uint8))


def assert_desc_equal(got, want):
    g, w = (x if isinstance(x, dict) else desc_dict(x) for x in (got, want))
    assert g.keys() == w.keys()
    for k in w:
        if isinstance(w[k], np.ndarray):
            assert g[k].shape == w[k].shape and np.array_equal(g[k], w[k]), k
        else:
            assert g[k] == w[k], k
