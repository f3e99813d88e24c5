"""An independent restatement, on the oracle's Poseidon2 (tests/oracle_lib.py), of what SP1Prover::verify_compressed / verify_shrink add
around one verify_shard: the verifying-key hash, its bytes32 packing, the digest of RecursionPublicValues, the recursion vk map
(RecursionVks::from_map, MerkleTree::commit / open), verify_merkle_proof, and the checks themselves on top of the oracle's
orc_verify_shard.  Test infrastructure only; words are u32 Montgomery words unless a name says canonical."""
import numpy as np

from tests import oracle_lib as O
from tests.machines import widths

# RecursionPublicValues<F> (crates/recursion/executor/src/public_values.rs:39-143), field by field: (name, width)
RPV_FIELDS = [("prev_committed_value_digest", 32), ("committed_value_digest", 32), ("prev_deferred_proofs_digest", 8),
              ("deferred_proofs_digest", 8), ("prev_deferred_proof", 1), ("deferred_proof", 1), ("pc_start", 3), ("next_pc", 3),
              ("initial_timestamp", 4), ("last_timestamp", 4), ("previous_init_addr", 3), ("last_init_addr", 3),
              ("previous_finalize_addr", 3), ("last_finalize_addr", 3), ("previous_init_page_idx", 3), ("last_init_page_idx", 3),
              ("previous_finalize_page_idx", 3), ("last_finalize_page_idx", 3), ("start_reconstruct_deferred_digest", 8),
              ("end_reconstruct_deferred_digest", 8), ("sp1_vk_digest", 8), ("vk_root", 8), ("global_cumulative_sum", 14),
              ("contains_first_shard", 1), ("num_included_shard", 1), ("is_complete", 1), ("prev_exit_code", 1), ("exit_code", 1),
              ("prev_commit_syscall", 1), ("commit_syscall", 1), ("prev_commit_deferred_syscall", 1), ("commit_deferred_syscall", 1),
              ("digest", 8), ("proof_nonce", 4)]
RPV = {}
_at = 0
for _name, _w in RPV_FIELDS:
    RPV[_name] = (_at, _w)
    _at += _w
RPV_NUM_ELTS = _at
NUM_PV_ELMS_TO_HASH = RPV["digest"][0]
ONE = int(O.to_monty(1))

# verdict codes (include/sp1b200.h)
ACCEPT, INVALID_SHARD_PROOF, PV_LENGTH = 0, 45, 46
PV_DIGEST, VK_ROOT, INVALID_VK, IS_COMPLETE, SP1_VK_DIGEST, UNINITIALIZED_VK = 77, 78, 79, 80, 81, 82


def sponge(words):
    """PaddingFreeSponge<16, 8, 8> (overwrite mode) on the oracle's permutation"""
    s = np.zeros(16, np.uint32)
    w = [int(x) for x in words]
    for i in range(0, len(w), 8):
        chunk = w[i:i + 8]
        s[:len(chunk)] = chunk
        s = O.permute(s)
    return s[:8].copy()


def vk_hash(key32):
    """hash_koalabear without mprotect (crates/hypercube/src/verifier/hashable_key.rs:94-118): the commitment and tail words 0..17"""
    return sponge(np.asarray(key32, np.uint32)[:26])


def pv_digest(pv):
    """recursion_public_values_digest (crates/prover/src/utils.rs:22-28)"""
    return sponge(np.asarray(pv, np.uint32)[:NUM_PV_ELMS_TO_HASH])


def bytes32(digest):
    """koalabears_to_bn254 (hashable_key.rs:23-33) as 32 big-endian bytes"""
    v = 0
    for w in O.from_monty(np.asarray(digest, np.uint32)).tolist():
        v = (v << 31) | int(w)
    return v.to_bytes(32, "big")


def reverse_bits_len(x, bits):
    r = 0
    for _ in range(bits):
        r = (r << 1) | (x & 1)
        x >>= 1
    return r


class VkMap:
    """RecursionVks::from_map (crates/prover/src/recursion.rs:59-87) and MerkleTree::commit / open
    (crates/recursion/circuit/src/basefold/merkle_tree.rs:24-88)"""

    def __init__(self, digests, pad_to=0):
        keys = {tuple(int(x) for x in O.from_monty(np.asarray(d, np.uint32))) for d in np.asarray(digests, np.uint32).reshape(-1, 8)}
        for i in range(len(keys), pad_to):
            keys.add((i,) * 8)
        self.keys = sorted(keys)   # canonical lexicographic order
        self.index = {k: i for i, k in enumerate(self.keys)}
        n = len(self.keys)
        assert n >= 2, "MerkleTree::commit needs two leaves"
        self.log_h = (n - 1).bit_length()
        h = 1 << self.log_h
        leaves = np.zeros((h, 8), np.uint32)
        for i, k in enumerate(self.keys):
            leaves[reverse_bits_len(i, self.log_h)] = O.to_monty(np.array(k))
        self.layers = [leaves]
        while self.layers[-1].shape[0] > 1:
            c = self.layers[-1]
            self.layers.append(np.stack([O.compress(c[2 * j], c[2 * j + 1]) for j in range(c.shape[0] // 2)]))
        self.root = self.layers[-1][0].copy()

    def open_index(self, index):
        pos = reverse_bits_len(index, self.log_h)
        leaf = self.layers[0][pos].copy()
        path = []
        for k in range(self.log_h):
            path.append(self.layers[k][pos ^ 1])
            pos >>= 1
        return leaf, np.stack(path)

    def open(self, digest):
        i = self.index[tuple(int(x) for x in O.from_monty(np.asarray(digest, np.uint32)))]
        return i, self.open_index(i)[1]


def merkle_proof_holds(leaf, index, path, root):
    """verify_merkle_proof (crates/hypercube/src/verifier/proof.rs:121-143)"""
    path = np.asarray(path, np.uint32).reshape(-1, 8)
    v = np.asarray(leaf, np.uint32)
    idx = reverse_bits_len(int(index), path.shape[0])
    for sib in path:
        v = O.compress(sib, v) if idx & 1 else O.compress(v, sib)
        idx >>= 1
    return bool((v == np.asarray(root, np.uint32)).all())


def verify_compressed(blob, heights, names, log_stack, max_log_rows, prm, key32, words, n_pv, vk_root, vk_verification, merkle_proof,
                      sp1_vk_digest, shrink=False, shrink_vk=None):
    """SP1Prover::verify_compressed / verify_shrink (crates/prover/src/verify.rs:527-642) -> (verdict, orc_verify_shard result or None).
    n_pv: the proof's public-value count; the public values are the last n_pv proof words."""
    key32 = np.asarray(key32, np.uint32)
    if shrink:
        if shrink_vk is None:
            return UNINITIALIZED_VK, None
        if not (np.asarray(shrink_vk, np.uint32) == key32).all():
            return INVALID_VK, None
    if n_pv != RPV_NUM_ELTS:
        return PV_LENGTH, None
    ch = O.Challenger()
    ch.observe(key32)
    pc = key32[:8] if any(pw for _, pw in widths(blob)) else None
    r = O.verify_shard(blob, heights, names, log_stack, max_log_rows, ch, pc, words, **prm)
    if r != 0:
        return INVALID_SHARD_PROOF, r
    pv = np.asarray(words, np.uint32)[-n_pv:]
    at = lambda f: pv[RPV[f][0]:RPV[f][0] + RPV[f][1]]
    if not (pv_digest(pv) == at("digest")).all():
        return PV_DIGEST, 0
    if not (at("vk_root") == np.asarray(vk_root, np.uint32)).all():
        return VK_ROOT, 0
    if vk_verification and not merkle_proof_holds(vk_hash(key32), merkle_proof[0], merkle_proof[1], vk_root):
        return INVALID_VK, 0
    if int(at("is_complete")[0]) != ONE:
        return IS_COMPLETE, 0
    if not (at("sp1_vk_digest") == np.asarray(sp1_vk_digest, np.uint32)).all():
        return SP1_VK_DIGEST, 0
    return ACCEPT, 0
