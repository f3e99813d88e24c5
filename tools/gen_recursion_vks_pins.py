"""Pins the recursion vk map to the reference's own data: writes tests/golden/recursion_vks.json.

    python tools/gen_recursion_vks_pins.py --reference PATH_TO_SP1 [--samples 60]

Reads the reference's crates/prover/src/vk_map.bin (bincode BTreeMap<[SP1Field; 8], usize>: the digests of every allowed recursion
verifying key), crates/verifier/vk-artifacts/verifier_vks.bin (bincode VerifierRecursionVks: root, vk_verification, num_keys) and
VK_ROOT_BYTES in crates/verifier/src/lib.rs.  Builds MerkleTree::commit (crates/recursion/circuit/src/basefold/merkle_tree.rs:24-64)
over the map's keys in canonical lexicographic order with the oracle's Poseidon2 compression (oracle/liboracle.so), and asserts, before
writing anything, that the keys' indices are 0..n-1 in that order, that the root is verifier_vks.bin's root and that its
koalabears_to_bn254 packing is VK_ROOT_BYTES.  The fixture records the source files' SHA-256s, the counts, the root, VK_ROOT_BYTES and
sampled openings (index, leaf, path; canonical words): key 0, the last key, the first and the last padding leaf, and seeded picks.
The 7.4 MB map itself is not committed."""
import argparse
import hashlib
import json
import os
import re
import struct
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

P = 0x7F000001


def read_vk_map(data):
    (n,) = struct.unpack_from("<Q", data, 0)
    assert len(data) == 8 + n * 40, "vk_map.bin is not a bincode BTreeMap<[u32; 8], u64>"
    rec = np.frombuffer(data, dtype=np.uint8, offset=8).reshape(n, 40)
    keys = rec[:, :32].copy().view("<u4").reshape(n, 8).astype(np.uint32)
    idx = rec[:, 32:].copy().view("<u8").reshape(n)
    return keys, idx


def bytes32(canonical8):
    v = 0
    for w in canonical8:
        v = (v << 31) | int(w)
    return v.to_bytes(32, "big")


def reverse_bits_len(x, bits):
    r = 0
    for _ in range(bits):
        r = (r << 1) | (x & 1)
        x >>= 1
    return r


def commit(keys_monty):
    """MerkleTree::commit -> (log_h, layers: list of [2^(log_h-k), 8] Montgomery arrays, k = 0 .. log_h)"""
    from tests import oracle_lib as O
    n = keys_monty.shape[0]
    log_h = max(1, (n - 1).bit_length())
    h = 1 << log_h
    leaves = np.zeros((h, 8), np.uint32)
    rev = np.array([reverse_bits_len(i, log_h) for i in range(n)])
    leaves[rev] = keys_monty
    layers = [leaves]
    while layers[-1].shape[0] > 1:
        c = layers[-1]
        layers.append(np.stack([O.compress(c[2 * j], c[2 * j + 1]) for j in range(c.shape[0] // 2)]))
    return log_h, layers


def open_path(log_h, layers, index):
    pos = reverse_bits_len(index, log_h)
    leaf = layers[0][pos]
    path = []
    for k in range(log_h):
        path.append(layers[k][pos ^ 1])
        pos >>= 1
    return leaf, np.stack(path)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reference", required=True, help="the reference SP1 checkout")
    ap.add_argument("--samples", type=int, default=60, help="seeded openings besides the four fixed ones")
    ap.add_argument("--out", default=os.path.join(ROOT, "tests", "golden", "recursion_vks.json"))
    args = ap.parse_args()
    from tests import oracle_lib as O
    map_path = os.path.join(args.reference, "crates", "prover", "src", "vk_map.bin")
    vvk_path = os.path.join(args.reference, "crates", "verifier", "vk-artifacts", "verifier_vks.bin")
    lib_path = os.path.join(args.reference, "crates", "verifier", "src", "lib.rs")
    map_bytes, vvk_bytes = open(map_path, "rb").read(), open(vvk_path, "rb").read()
    keys, idx = read_vk_map(map_bytes)
    n = keys.shape[0]
    assert (keys < P).all(), "a key word is not canonical"
    assert [tuple(k) for k in keys.tolist()] == sorted(tuple(k) for k in keys.tolist()), "keys are not in canonical lexicographic order"
    assert (idx == np.arange(n)).all(), "the map's indices are not 0..n-1 in key order"
    assert len(vvk_bytes) == 41, "verifier_vks.bin is not bincode(VerifierRecursionVks)"
    want_root = np.frombuffer(vvk_bytes[:32], "<u4").astype(np.uint32)
    vk_verification = bool(vvk_bytes[32])
    (num_keys,) = struct.unpack_from("<Q", vvk_bytes, 33)
    assert num_keys == n, (num_keys, n)
    m = re.search(r"VK_ROOT_BYTES: \[u8; 32\] = \[(.*?)\]", open(lib_path).read(), re.S)
    vk_root_bytes = bytes(int(x, 16) for x in re.findall(r"0x([0-9a-fA-F]{2})", m.group(1)))
    assert len(vk_root_bytes) == 32

    log_h, layers = commit(O.to_monty(keys))
    root = O.from_monty(layers[-1][0])
    assert (root == want_root).all(), f"oracle root {root.tolist()} != verifier_vks.bin root {want_root.tolist()}"
    assert bytes32(root) == vk_root_bytes, "koalabears_to_bn254(root) != VK_ROOT_BYTES"

    h = 1 << log_h
    rng = np.random.default_rng(2024)
    picks = [0, n - 1, n, h - 1] + sorted(int(x) for x in rng.choice(np.arange(1, h - 1), size=args.samples, replace=False))
    openings = []
    for i in picks:
        leaf, path = open_path(log_h, layers, i)
        openings.append(dict(index=i, leaf=O.from_monty(leaf).tolist(), path=O.from_monty(path).tolist()))
    out = dict(
        source=dict(vk_map_sha256=hashlib.sha256(map_bytes).hexdigest(), verifier_vks_sha256=hashlib.sha256(vvk_bytes).hexdigest()),
        num_keys=n, vk_verification=vk_verification, log_height=log_h, root=root.tolist(), vk_root_bytes=vk_root_bytes.hex(),
        words="canonical", openings=openings)
    with open(args.out, "w") as f:
        json.dump(out, f, separators=(",", ":"))
        f.write("\n")
    print(f"{args.out}: {n} keys, root {vk_root_bytes.hex()}, {len(openings)} openings")


if __name__ == "__main__":
    main()
