#!/usr/bin/env python
"""Extracts the Keccak-256 known answers that the REFERENCE TREE ITSELF holds and writes tests/golden/reference_keccak_vectors.json.

consensus-shipyard/ipc-filecoin-proofs has no tests of its own (SURVEY.md §4), but it vendors forge-std under
topdown-messenger/lib/forge-std/, and that library's sources and test-suite carry constants that are *defined* as Keccak-256 results:

  * src/StdConstants.sol: VM = address(uint160(uint256(keccak256("hevm cheat code")))), DEFAULT_SENDER = …keccak256("foundry default
    caller"), DEFAULT_TEST_CONTRACT = computeCreateAddress(computeCreateAddress(DEFAULT_SENDER, 1), 1)  (asserted in test/StdConstants.t.sol);
  * test/StdUtils.t.sol: hashInitCode(hex"6080") == 0x1a578b7a…, two CREATE2 addresses (keccak256(0xff ‖ deployer ‖ salt ‖ initcodeHash)[12:]),
    one CREATE address (keccak256(rlp([deployer, nonce]))[12:]);
  * src/StdUtils.sol: the selector comment `0x70a08231 = bytes4("balanceOf(address)")`;
  * every mixed-case address literal: solc only accepts it when its EIP-55 checksum — keccak256 of the lower-case hex — is right.

Keccak-256 is on the hot path (topic0 = keccak256(event signature), events/generator.rs:30-35 via common/evm.rs:62-69; mapping slots,
storage/utils.rs:5-12). These are the only vectors in the reference tree that pin anything the path computes; AMT / HAMT / DAG-CBOR stay
unpinned by the reference. Usage: make_reference_keccak_vectors.py <reference checkout>; the JSON is what the tests read. No hashing happens in this script: it only copies
constants and states how each expected value is derived, the tests do the hashing with the implementation under test."""
import json
import os
import re
import sys

if len(sys.argv) != 2:
    raise SystemExit(__doc__.splitlines()[0] + "\nusage: make_reference_keccak_vectors.py <reference checkout>")
REF = sys.argv[1]
FORGE = os.path.join(REF, "topdown-messenger", "lib", "forge-std")
OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "reference_keccak_vectors.json")


def find(path, pattern, group=1):
    """(match group, 'relative path:line') of the first line matching `pattern`."""
    rel = os.path.relpath(path, REF)
    for ln, line in enumerate(open(path, encoding="utf-8"), 1):
        m = re.search(pattern, line)
        if m:
            return m.group(group), f"{rel}:{ln}"
    raise SystemExit(f"pattern {pattern!r} not found in {rel}")


def main():
    consts = os.path.join(FORGE, "src", "StdConstants.sol")
    utils_t = os.path.join(FORGE, "test", "StdUtils.t.sol")
    utils = os.path.join(FORGE, "src", "StdUtils.sol")
    V = []
    vm, src = find(consts, r"constant VM = Vm\((0x[0-9a-fA-F]{40})\)")
    V.append(dict(kind="low20", message_ascii="hevm cheat code", expect=vm, source=src))
    sender, src = find(consts, r"constant DEFAULT_SENDER = (0x[0-9a-fA-F]{40})")
    V.append(dict(kind="low20", message_ascii="foundry default caller", expect=sender, source=src))
    test_contract, src = find(consts, r"constant DEFAULT_TEST_CONTRACT = (0x[0-9a-fA-F]{40})")
    V.append(dict(kind="create_chain", deployer=sender, nonces=[1, 1], expect=test_contract, source=src))
    factory, fsrc = find(consts, r"constant CREATE2_FACTORY = (0x[0-9a-fA-F]{40})")
    multicall, msrc = find(consts, r"MULTICALL3_ADDRESS = IMulticall3\((0x[0-9a-fA-F]{40})\)")
    init_hash, src = find(utils_t, r"assertEq\(initcodeHash, (0x[0-9a-f]{64})\)")
    V.append(dict(kind="digest", message_hex="6080", expect=init_hash, source=src))
    deployer, dsrc = find(utils_t, r"address deployer = (0x[0-9a-fA-F]{40});")
    c2, src = find(utils_t, r"assertEq\(create2Address, (0xB1[0-9a-fA-F]{38})\)")
    salt_int, _ = find(utils_t, r"bytes32 salt = bytes32\(uint256\((\d+)\)\);")
    V.append(dict(kind="create2", deployer=deployer, salt_hex="%064x" % int(salt_int), initcode_preimage_hex="%064x" % 0x6080, expect=c2, source=src,
                  note="initcodeHash = keccak256(abi.encode(0x6080)): the 32-byte big-endian word"))
    salt2, _ = find(utils_t, r"bytes32 salt = (0x[0-9a-f]{64});")
    c2b, src = find(utils_t, r"assertEq\(create2Address, (0xc0ff[0-9a-fA-F]{36})\)")
    V.append(dict(kind="create2", deployer=factory, salt_hex=salt2[2:], initcode_preimage_hex="6080", expect=c2b, source=src,
                  note="default CREATE2 deployer (StdConstants.CREATE2_FACTORY); initcodeHash = hashInitCode(hex\"6080\")"))
    nonce, _ = find(utils_t, r"uint256 nonce = (\d+);")
    c1, src = find(utils_t, r"assertEq\(createAddress, (0x[0-9a-fA-F]{40})\)")
    V.append(dict(kind="create_chain", deployer=deployer, nonces=[int(nonce)], expect=c1, source=src))
    sel, src = find(utils, r"// (0x[0-9a-f]{8}) = bytes4\(\"balanceOf\(address\)\"\)")
    V.append(dict(kind="prefix4", message_ascii="balanceOf(address)", expect=sel, source=src))
    for addr, s in ((vm, "VM"), (factory, fsrc), (sender, "DEFAULT_SENDER"), (test_contract, "DEFAULT_TEST_CONTRACT"), (multicall, msrc), (deployer, dsrc),
                    (c2, "create2Address"), (c2b, "create2Address (default deployer)"), (c1, "createAddress")):
        V.append(dict(kind="eip55", address=addr, source=s if ":" in s else f"{s} literal, see above"))
    doc = dict(what="Keccak-256 known answers held by the reference tree (vendored forge-std); made by tests/golden/make_reference_keccak_vectors.py",
               reference_subtree="topdown-messenger/lib/forge-std", vectors=V)
    with open(OUT, "w") as f:
        json.dump(doc, f, indent=1)
        f.write("\n")
    print(f"{len(V)} vectors -> {OUT}")


if __name__ == "__main__":
    main()
