"""ipcfp_blocks_from_rpc_json (csrc/rpc_blocks_parse.cpp, host C++, no device): the block arrays of Filecoin.ChainReadObj responses must be
the synthetic tipset's own blocks on the canonical texts of configs 1-3 however they are split and ordered, and must agree with the rules
restated in tests/rpc_blocks.py on every hand-made case and on seeded byte edits — the arrays, or the status and the index."""
import ctypes as C

import numpy as np
import pytest

import synth
from ipc_filecoin_proofs_b200 import _abi as A
from ipc_filecoin_proofs_b200 import api
from tests import rpc_blocks as B


def _got(cids, texts):
    try:
        return api.blocks_from_rpc_json(cids, texts)
    except A.IpcfpError as e:
        return (e.status, e.index)


def _agree(cids, texts):
    """The library and the rules give the same outcome; returns it."""
    want, got = B.expected(len(cids), texts), _got(cids, texts)
    if isinstance(want, tuple):
        assert got == want
    else:
        assert not isinstance(got, tuple), got
        B.assert_blocks_equal(got, cids, want)
    return want


@pytest.fixture(scope="module")
def small():
    """The first 40 blocks of config 1: a zero-length block among them as well."""
    cids, blocks = B.blocks_of(synth.Tipset(synth.config_params(1)), 40)
    blocks[7] = b""
    return cids, blocks


@pytest.mark.parametrize("config", [1, 2, 3])
def test_canonical_texts_give_the_tipset_blocks(config):
    params = synth.config_params(3, hamt_entries=20000) if config == 3 else synth.config_params(config)
    cids, blocks = B.blocks_of(synth.Tipset(params))
    for n, texts in ((len(blocks), B.render(blocks)), (len(blocks), B.render(blocks, 7, seed=config)),
                     (min(500, len(blocks)), B.render(blocks[:500], single=True, seed=1))):
        B.assert_blocks_equal(api.blocks_from_rpc_json(cids[:n], texts), cids[:n], blocks[:n])
    # the rules agree on a shuffled split of the whole set
    assert B.read(len(blocks), B.render(blocks, 3, seed=2)) == blocks


def test_empty_input():
    w = api.blocks_from_rpc_json(np.zeros((0, 38), np.uint8), [b"[]"])
    assert w.n_blocks == 0 and w.blob.size == 0
    assert api.blocks_from_rpc_json(np.zeros((0, 38), np.uint8), []).n_blocks == 0
    assert _got(np.zeros((0, 38), np.uint8), [B.element(0, b"x")]) == (A.ERR_INVALID_ARG, 0)


def test_zero_length_block(small):
    cids, blocks = small
    assert blocks[7] == b"" and b'"result":"","id":7}' in B.render(blocks)[0]
    w = _agree(cids, B.render(blocks, 2, seed=3))
    assert w[7] == b""


@pytest.mark.parametrize("case", range(36))
def test_named_case_agrees_with_the_rules(small, case):
    cids, blocks = small
    name, texts, outcome = B.cases(blocks)[case]
    want = _agree(cids, texts)
    if outcome == A.OK:
        assert not isinstance(want, tuple), name
    else:
        assert isinstance(want, tuple) and want[0] == outcome, (name, want)


def test_every_case_is_numbered(small):
    assert len(B.cases(small[1])) == 36


def test_check_order(small):
    """Element faults first (by position over all texts), then ids not there exactly once, then error responses, each the smallest."""
    cids, blocks = small
    els = [B.element(i, d) for i, d in enumerate(blocks)]
    bad = els[5][:-1] + b',"id":5}'                                  # repeated member: element fault at position 30 below
    texts = [b"[" + b",".join(els[10:40]) + b"]", b"[" + bad + b"," + b",".join(els[:5]) + b"]"]
    assert _agree(cids, texts) == (A.ERR_INVALID_ARG, 30)
    texts = [b"[" + b",".join([B.error_element(3)] + els[4:20] + els[21:] + els[:3]) + b"]"]
    assert _agree(cids, texts) == (A.ERR_INVALID_ARG, 20)            # missing 20 comes before the error response at 3
    texts = [b"[" + b",".join([B.error_element(9)] + els[:9] + [B.error_element(3)] + els[10:]) + b"]"]
    assert _agree(cids, texts[:1]) == (A.ERR_INVALID_ARG, 3)         # 3 twice
    texts = [b"[" + b",".join([B.error_element(9)] + els[:3] + [B.error_element(3)] + els[4:9] + els[10:]) + b"]"]
    assert _agree(cids, texts) == (A.ERR_MISSING_BLOCK, 3)
    assert _agree(cids, [b"[" + b",".join(els) + b"],"]) == (A.ERR_INVALID_ARG, B.NO_INDEX)


def test_seeded_byte_edits(small):
    """400 seeded edits of a split, shuffled canonical input: status, index and blocks as the rules give them."""
    cids, blocks = small
    base = B.render(blocks, 3, seed=11)
    rng = np.random.default_rng(20261016)
    alphabet = b'{}[]",:0123456789 \nabAZ=+/\\-.enulid'
    n_ok = n_fail = 0
    for _ in range(400):
        texts = [bytearray(t) for t in base]
        for _ in range(int(rng.integers(1, 3))):
            t = texts[int(rng.integers(0, len(texts)))]
            i = int(rng.integers(0, len(t)))
            op = int(rng.integers(0, 4))
            if op == 0:
                t[i] = alphabet[int(rng.integers(0, len(alphabet)))]
            elif op == 1:
                del t[i]
            elif op == 2:
                t.insert(i, alphabet[int(rng.integers(0, len(alphabet)))])
            else:
                j = int(rng.integers(0, len(t)))
                t[i:i] = t[j:j + int(rng.integers(1, 60))]
        want = _agree(cids, [bytes(t) for t in texts])
        n_ok += not isinstance(want, tuple)
        n_fail += isinstance(want, tuple)
    assert n_ok > 0 and n_fail > 0


def test_null_arguments():
    L = api.lib()
    out = C.POINTER(A.ParsedBlocksC)()
    cid = np.zeros(38, np.uint8)
    texts = (C.c_char_p * 1)(b"[]")
    lens = (C.c_uint64 * 1)(2)
    assert L.ipcfp_blocks_from_rpc_json(None, 0, texts, lens, 1, None) == A.ERR_INVALID_ARG
    assert L.ipcfp_blocks_from_rpc_json(None, 1, texts, lens, 1, C.byref(out)) == A.ERR_INVALID_ARG and not out
    assert L.ipcfp_blocks_from_rpc_json(cid.ctypes.data, 1, None, None, 1, C.byref(out)) == A.ERR_INVALID_ARG and not out
    assert L.ipcfp_last_error_index() == B.NO_INDEX


def test_ctypes_layout_matches_c_header(tmp_path):
    import os
    import subprocess
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    structs = (("ipcfp_parsed_blocks", A.ParsedBlocksC), ("ipcfp_store_json_info", A.StoreJsonInfoC))
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "ipcfp.h"', "int main(void) {"]
    for cname, st in structs:
        lines.append(f'printf("{cname} %zu\\n", sizeof({cname}));')
        lines += [f'printf("{cname}.{f} %zu\\n", offsetof({cname}, {f}));' for f, _ in st._fields_]
    lines += ["return 0; }"]
    src, exe = tmp_path / "layout.c", tmp_path / "layout"
    src.write_text("\n".join(lines))
    subprocess.check_call(["gcc", "-I", os.path.join(root, "include"), "-o", str(exe), str(src)])
    got = dict(l.split() for l in subprocess.check_output([str(exe)], text=True).strip().splitlines())
    for cname, st in structs:
        assert int(got[cname]) == C.sizeof(st)
        for f, _ in st._fields_:
            assert int(got[f"{cname}.{f}"]) == getattr(st, f).offset, f
