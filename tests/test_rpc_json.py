"""ipcfp_tipset_desc_from_json (csrc/rpc_parse.cpp, host C++, no device): the tipset descriptor from the Lotus JSON-RPC texts must be the
synthetic tipset's own descriptor on the canonical texts of configs 1 and 2, and must agree with the rules restated in tests/rpc_json.py
(Python's json module) on every mutator — the descriptor, or the status and the receipt index."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import synth
from ipc_filecoin_proofs_b200 import _abi as A
from ipc_filecoin_proofs_b200 import api
from tests import rpc_json as R


@pytest.fixture(scope="module")
def ts_nulls():
    """config 1 with a quarter of the events roots None, so that both spellings of EventsRoot occur."""
    ts = synth.Tipset(synth.config_params(1, null_root_permille=250))
    assert 0 < int(np.asarray(ts.has_events_root).sum()) < ts.n_receipts
    return ts


def _got(parent, child, receipts):
    try:
        return api.tipset_desc_from_json(parent, child, receipts)
    except A.IpcfpError as e:
        return (e.status, e.index)


@pytest.mark.parametrize("config", [1, 2])
def test_canonical_texts_give_the_synthetic_descriptor(config):
    ts = synth.Tipset(synth.config_params(config))
    p, c, r = R.texts(ts)
    got = api.tipset_desc_from_json(p, c, r)
    R.assert_desc_equal(got, ts)
    R.assert_desc_equal(R.read(p, c, r), ts)


@pytest.mark.parametrize("name", [m[0] for m in R.MUTATORS])
def test_mutator_agrees_with_the_rules(ts_nulls, name):
    fn, outcome = next((f, o) for n, f, o in R.MUTATORS if n == name)
    texts = fn(ts_nulls, int(ts_nulls.n_receipts) * 2 // 3)
    want = R.expected(*texts)
    if outcome == A.OK:
        assert isinstance(want, dict), want
    else:
        assert isinstance(want, tuple) and want[0] == outcome, want
    got = _got(*texts)
    if isinstance(want, dict):
        assert not isinstance(got, tuple), got
        R.assert_desc_equal(got, want)
    else:
        assert got == want


def test_receipt_faults_name_their_receipt(ts_nulls):
    """A fault inside element k is reported with index k, wherever k is; a framing fault has no index."""
    n = int(ts_nulls.n_receipts)
    for k in (0, 1, n // 2, n - 1):
        texts = R._with_receipt(ts_nulls, k, lambda p: R._set(p, "Return", R.Raw("null")))
        assert _got(*texts) == (A.ERR_INVALID_ARG, k) == R.expected(*texts)
    p, c, r = R.texts(ts_nulls)
    assert _got(p, c, r + ",") == (A.ERR_INVALID_ARG, R.NO_INDEX) == R.expected(p, c, r + ",")


def test_random_truncations_and_byte_edits(ts_nulls):
    """Seeded edits of the receipt list anywhere in the text: status, index and values as the rules give them."""
    p, c, r = R.texts(ts_nulls)
    rng = np.random.default_rng(20261016)
    alphabet = '{}[]",:0123456789 abx\\-.enul/'
    n_ok = 0
    for _ in range(400):
        b = list(r)
        for _ in range(int(rng.integers(1, 3))):
            i = int(rng.integers(0, len(b)))
            op = int(rng.integers(0, 3))
            if op == 0:
                b[i] = alphabet[int(rng.integers(0, len(alphabet)))]
            elif op == 1:
                del b[i]
            else:
                b.insert(i, alphabet[int(rng.integers(0, len(alphabet)))])
        t = "".join(b)
        want, got = R.expected(p, c, t), _got(p, c, t)
        if isinstance(want, dict):
            n_ok += 1
            assert not isinstance(got, tuple), (got, t)
            R.assert_desc_equal(got, want)
        else:
            assert got == want, t
    assert n_ok > 0


def test_null_arguments():
    L = api.lib()
    out = C.POINTER(A.ParsedTipsetC)()
    assert L.ipcfp_tipset_desc_from_json(b"{}", 2, b"{}", 2, b"[]", 2, None) == A.ERR_INVALID_ARG
    assert L.ipcfp_tipset_desc_from_json(None, 5, b"{}", 2, b"[]", 2, C.byref(out)) == A.ERR_INVALID_ARG and not out


def test_tipset_info_ctypes_layout_matches_c_header(tmp_path):
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "ipcfp.h"', "int main(void) {"]
    for cname, st in (("ipcfp_parsed_tipset", A.ParsedTipsetC), ("ipcfp_tipset_info", A.TipsetInfoC)):
        lines.append(f'printf("{cname} %zu\\n", sizeof({cname}));')
        lines += [f'printf("{cname}.{f} %zu\\n", offsetof({cname}, {f}));' for f, _ in st._fields_]
    lines += ["return 0; }"]
    src, exe = tmp_path / "layout.c", tmp_path / "layout"
    src.write_text("\n".join(lines))
    subprocess.check_call(["gcc", "-I", os.path.join(root, "include"), "-o", str(exe), str(src)])
    got = dict(l.split() for l in subprocess.check_output([str(exe)], text=True).strip().splitlines())
    for cname, st in (("ipcfp_parsed_tipset", A.ParsedTipsetC), ("ipcfp_tipset_info", A.TipsetInfoC)):
        assert int(got[cname]) == C.sizeof(st)
        for f, _ in st._fields_:
            assert int(got[f"{cname}.{f}"]) == getattr(st, f).offset, f
