"""CPU tests of the recursion-key helpers against the reference's own vk map (tests/golden/recursion_vks.json, written by
tools/gen_recursion_vks_pins.py from the reference's vk_map.bin, verifier_vks.bin and VK_ROOT_BYTES): bytes32 of the pinned root is
VK_ROOT_BYTES; every sampled opening verifies against the pinned root as verify_merkle_proof does, and fails after a one-word change;
the library's vk hash and public-values digest equal the oracle's sponge; the public-value offsets follow the struct's field list."""
import json
import os

import numpy as np
import pytest

from tests import oracle_lib as O
from tests import recursion_ref as RR

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def golden():
    with open(os.path.join(ROOT, "tests", "golden", "recursion_vks.json")) as f:
        return json.load(f)


def test_pinned_root_packs_to_vk_root_bytes(golden):
    from sp1_b200 import lib as B
    root = O.to_monty(np.array(golden["root"]))
    assert B.digest_bytes32(root) == bytes.fromhex(golden["vk_root_bytes"])
    assert RR.bytes32(root) == bytes.fromhex(golden["vk_root_bytes"])
    assert golden["num_keys"] == 185862 and golden["log_height"] == 18 and golden["vk_verification"] is True


def test_digest_bytes32_is_the_31_bit_concatenation():
    from sp1_b200 import lib as B
    rng = np.random.default_rng(3)
    for d in [np.zeros(8, np.int64), np.full(8, O.P - 1)] + [rng.integers(0, O.P, 8) for _ in range(20)]:
        v = 0
        for w in d:
            v = (v << 31) | int(w)
        got = B.digest_bytes32(O.to_monty(d))
        assert got == v.to_bytes(32, "big") and got[0] == 0
    with pytest.raises(B.Sp1B200Error, match="not canonical"):
        B.digest_bytes32(np.full(8, O.P, np.uint32))


def test_sampled_openings_verify_against_the_reference_root(golden):
    root = O.to_monty(np.array(golden["root"]))
    ops = golden["openings"]
    n, h = golden["num_keys"], 1 << golden["log_height"]
    assert {0, n - 1, n, h - 1} <= {o["index"] for o in ops} and len(ops) >= 64
    for o in ops:
        leaf, path, i = O.to_monty(np.array(o["leaf"])), O.to_monty(np.array(o["path"])), o["index"]
        assert path.shape == (golden["log_height"], 8)
        if i >= n:
            assert not leaf.any(), "a padding leaf is the zero digest"
        assert RR.merkle_proof_holds(leaf, i, path, root), i
        # reverse_bits_len ignores the index bits above the path length
        assert RR.merkle_proof_holds(leaf, i | (5 << golden["log_height"]), path, root), i
    for o in ops[:8]:
        leaf, path, i = O.to_monty(np.array(o["leaf"])), O.to_monty(np.array(o["path"])), o["index"]
        bad = path.copy(); bad[3, 2] = (int(bad[3, 2]) + 1) % O.P
        assert not RR.merkle_proof_holds(leaf, i, bad, root)
        assert not RR.merkle_proof_holds(leaf, i ^ 1, path, root)   # wrong low index bit: the root compression's orientation
        # the leaf's own compression with the sibling on the other side
        assert not RR.merkle_proof_holds(leaf, i ^ (1 << (golden["log_height"] - 1)), path, root)


def test_pinned_keys_are_in_canonical_order(golden):
    n = golden["num_keys"]
    keys = sorted((o["index"], tuple(o["leaf"])) for o in golden["openings"] if o["index"] < n)
    assert [k for _, k in keys] == sorted(k for _, k in keys)


def test_vk_hash_matches_the_oracle_sponge():
    from sp1_b200 import lib as B
    rng = np.random.default_rng(11)
    for _ in range(8):
        key = O.rand_field(rng, 32)
        got = B.vk_hash(key[:8], key[8:])
        assert (got == RR.vk_hash(key)).all()
        assert (got == O.hash_(key[:26])).all()
        pad = key.copy(); pad[26:] = O.rand_field(rng, 6)    # the padding words are not hashed
        assert (B.vk_hash(pad[:8], pad[8:]) == got).all()
    with pytest.raises(B.Sp1B200Error, match="n_vk_tail"):
        B.vk_hash(key[:8], key[8:31])


def test_recursion_pv_digest_matches_the_oracle_sponge():
    from sp1_b200 import lib as B
    rng = np.random.default_rng(12)
    for _ in range(8):
        pv = O.rand_field(rng, 187)
        got = B.recursion_pv_digest(pv)
        assert (got == RR.pv_digest(pv)).all() and (got == O.hash_(pv[:175])).all()
        tail = pv.copy(); tail[175:] = O.rand_field(rng, 12)    # digest and proof_nonce are not hashed
        assert (B.recursion_pv_digest(tail) == got).all()


def test_public_value_offsets_follow_the_field_list():
    from sp1_b200 import lib as B
    assert RR.RPV_NUM_ELTS == 187 == B.PV_MAX_NUM
    assert RR.NUM_PV_ELMS_TO_HASH == 175 == B.RPV_NUM_TO_HASH
    for name, (at, w) in B.RPV.items():
        assert RR.RPV[name] == (at, w), name
    assert RR.RPV["proof_nonce"] == (183, 4)


def test_compressed_verdict_names():
    from sp1_b200 import lib as B
    assert B.verdict_name(76) == "Unknown"
    names = {77: "InvalidPublicValues(recursion public values are invalid)", 78: "InvalidPublicValues(vk_root mismatch)",
             79: "InvalidVerificationKey", 80: "InvalidPublicValues(is_complete is not 1)",
             81: "InvalidPublicValues(sp1 vk hash mismatch)", 82: "UninitializedVerificationKey"}
    for v, n in names.items():
        assert B.verdict_name(v) == n
    assert B.verdict_name(83) == "Unknown"
    assert B.verdict_name(46) == "InvalidPublicValues(invalid public values length)"
