"""The adversarial CID families of tests/util.py (no GPU): the bijections have the shapes the GPU tests rely on, and the CPU oracle
on a rewritten tipset equals the image of its result on the original one."""
import os
import re

import numpy as np
import pytest

from tests import util as U
from tests.util import spec_of

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FAMILIES = ["A", "B", "C", "D"]


def test_mixed_prefixes_are_valid_and_raw_order_is_not_cid_order():
    from oracle import pyoracle as P
    keys = [P.cid_sort_key(p + bytes(32)) for p in U.MIXED_PREFIXES]
    assert all(k[0] == 1 and k[3] == 32 and len(k[4]) == 32 for k in keys)        # 6-byte prefixes: 1-byte codec, 3-byte code
    assert keys == sorted(keys) and len(set(U.MIXED_PREFIXES)) == 8
    assert sorted(U.MIXED_PREFIXES) != U.MIXED_PREFIXES
    assert [k[2] for k in keys] == [0x7fff, 0xb220, 0x8001, 0x407f, 0x8000, 0xb212, 0xb220, 0xffff]


def test_clustered_digests_shape():
    d = U.clustered_digests(4000, np.random.default_rng(1))
    s = sorted(d)
    firsts = {U.first_difference(a, b) for a, b in zip(s, s[1:]) if a[:4] == b[:4]}
    assert set(range(4, 32)) <= firsts
    assert any(U.first_difference(a, b) == 31 and a[:31] == b[:31] for a, b in zip(s, s[1:]))
    groups = {}
    for x in d:
        groups[x[0:8] + x[16:24]] = groups.get(x[0:8] + x[16:24], 0) + 1
    assert max(groups.values()) == 512 and min(groups.values()) >= 2
    run, longest = 1, 1
    for a, b in zip(s, s[1:]):
        run = run + 1 if a[:4] == b[:4] else 1
        longest = max(longest, run)
    assert longest > 256
    assert len({U.digest_hash(x, 0) for x in d}) == len(groups)   # one hash per group


@pytest.fixture(scope="module")
def originals(synth_mod, oracle_mod):
    cache = {}

    def get(cfg):
        if cfg not in cache:
            ts = synth_mod.Tipset(synth_mod.config_params(cfg))
            cache[cfg] = (ts, oracle_mod.Store.from_tipset(ts).generate_event_proof(ts, spec_of(ts)))
        return cache[cfg]
    return get


@pytest.mark.parametrize("family", FAMILIES)
@pytest.mark.parametrize("cfg", [1, 2])
def test_oracle_on_rewritten_tipset_equals_image(oracle_mod, originals, cfg, family):
    from oracle import pyoracle as P
    ts, exp = originals(cfg)
    rt, cm = U.adversarial_tipset(ts, family)
    got = oracle_mod.Store.from_tipset(rt).generate_event_proof(rt, spec_of(rt))
    U.assert_event_image(got, exp, cm)
    assert exp.proofs and got.n_exec > 0
    if family == "D":
        assert rt.n_blocks > ts.n_blocks + 1000
        return
    u = U.cid_universe(ts)
    assert len(cm.m) == len(u) and all(cm.cid(c) != c for c in u)
    assert cm.proof_keys(exp.proofs) != [p.key() for p in exp.proofs]        # message CIDs are rewritten too
    assert np.array_equal(rt.cids[0], np.frombuffer(cm.cid(ts.cids[0]), dtype=np.uint8))
    cids = [bytes(c) for c in got.witness.cids]
    if family == "A" and cfg == 2:   # the store's own blocks hold a run of equal 4-byte radix keys longer than 256
        keys = sorted(bytes(c[6:10]) for c in rt.cids)
        assert max(keys.count(k) for k in set(keys)) > 256
    if family in ("B", "C"):
        assert bytes(rt.cids[0][:6]) == U.MIXED_PREFIXES[-1]
        assert {c[:6] for c in cids} == set(U.MIXED_PREFIXES) or cfg == 1
        if cfg == 2:
            assert sorted(cids) != cids                                    # raw byte order is not `Cid` order here
            flat = {bytes(c) for c in rt.cids}
            digs = {}
            for c in cm.m.values():
                digs.setdefault(c[6:], []).append(c)
            shared = [v for v in digs.values() if len(v) > 1]
            assert any(all(c in flat for c in v) for v in shared) and any(not any(c in flat for c in v) for v in shared)
    assert cids == sorted(cids, key=P.cid_sort_key)


@pytest.mark.parametrize("family", FAMILIES)
def test_oracle_storage_on_rewritten_tipset_equals_image(oracle_mod, ts3_small, family):
    ts = ts3_small
    rt, cm = U.adversarial_tipset(ts, family)
    n = int(ts.params.hamt_entries)
    keys = [ts.storage_entry(k)[0] for k in (0, 1, 2, 77, n)] + [ts.storage_absent_key(1)]
    slots = [oracle_mod.compute_mapping_slot(k, 0) for k in keys]
    exp = oracle_mod.Store.from_tipset(ts).read_storage_slots(ts.storage_root, np.frombuffer(b"".join(slots), dtype=np.uint8))
    got = oracle_mod.Store.from_tipset(rt).read_storage_slots(rt.storage_root, np.frombuffer(b"".join(slots), dtype=np.uint8))
    assert np.array_equal(got.found, exp.found) and np.array_equal(got.values, exp.values) and got.found.any()
    assert ([bytes(c) for c in got.witness.cids], got.witness.blocks()) == cm.witness(exp.witness)
    specs = [(actor, s) for actor in (1001, 1003, 1006) for s in slots]
    exp = oracle_mod.Store.from_tipset(ts).generate_storage_proofs(ts, specs)
    got = oracle_mod.Store.from_tipset(rt).generate_storage_proofs(rt, specs)
    assert [vars(p) for p in got.proofs] == cm.storage_proofs(exp.proofs)
    assert ([bytes(c) for c in got.witness.cids], got.witness.blocks()) == cm.witness(exp.witness)
    assert got.spec_witness == cm.spec_witness(exp)


def test_python_hash_copy_matches_the_device_source():
    """The store tests aim CIDs at chosen hash-table slots with tests/util.py's copy of the device hash: a change of the hash or of
    the table size must fail here instead of quietly losing those cases."""
    src = open(os.path.join(ROOT, "ipc_filecoin_proofs_b200", "csrc", "common.cuh")).read()
    mix = re.search(r"uint64_t mix64\(uint64_t x\) \{\s*(.*?)\s*return x;", src, re.S).group(1)
    assert mix.replace(" ", "") == "x^=x>>33;x*=0xff51afd7ed558ccdULL;x^=x>>33;x*=0xc4ceb9fe1a85ec53ULL;x^=x>>33;"
    assert "digest_hash(const Digest& d, uint32_t cls) { return mix64(d.w[0] ^ (d.w[2] * 0x9E3779B97F4A7C15ULL) ^ cls); }" in src
    # tests/gpu_prims/shard_check.cu builds message CIDs to chosen owners and claim-table slots with its own copy of this hash (and
    # checks that copy against the device on every input)
    raw = open(os.path.join(ROOT, "ipc_filecoin_proofs_b200", "csrc", "rawcid.cuh")).read()
    assert "uint64_t rawcid_hash(const RawCid& c) { return mix64(c.w[0] ^ (c.w[2] * 0x9E3779B97F4A7C15ULL) ^ c.w[4]); }" in raw
    check = open(os.path.join(ROOT, "tests", "gpu_prims", "shard_check.cu")).read()
    assert "static uint64_t rawcid_hash_h(const RawCid& c) { return mix64_h(c.w[0] ^ (c.w[2] * GOLD) ^ c.w[4]); }" in check
    assert "x ^= x >> 33; x *= M1; x ^= x >> 33; x *= M2; x ^= x >> 33;" in check
    assert "M1 = 0xff51afd7ed558ccdULL, M2 = 0xc4ceb9fe1a85ec53ULL" in check and "GOLD = 0x9E3779B97F4A7C15ULL" in check
    store = open(os.path.join(ROOT, "ipc_filecoin_proofs_b200", "csrc", "store.cu")).read()
    assert re.search(r"uint64_t slots = 64;\s*while \(slots < 2 \* n\) slots <<= 1;", store)
    assert [U.table_slots(n) for n in (0, 1, 31, 32, 33, 63, 64, 65, 1023, 1024, 1025)] == [64, 64, 64, 64, 128, 128, 128, 256, 2048, 2048, 4096]
