"""ctypes binding of oracle/liboracle.so — the CPU checker.  Test infrastructure only."""
import ctypes as C
import os
import subprocess

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_SO = os.path.join(ROOT, "oracle", "liboracle.so")
P = 0x7F000001

u32p = C.POINTER(C.c_uint32)


def _build():
    if not os.path.exists(_SO):
        subprocess.check_call(["make", "-C", os.path.join(ROOT, "oracle")])


_lib = None


def lib():
    global _lib
    if _lib is None:
        _build()
        L = C.CDLL(_SO)
        L.orc_num_threads.restype = C.c_int
        for n in ("orc_to_monty", "orc_from_monty", "orc_inv", "orc_two_adic_generator"):
            getattr(L, n).restype = C.c_uint32
            getattr(L, n).argtypes = [C.c_uint32]
        for n in ("orc_mul", "orc_add", "orc_sub"):
            getattr(L, n).restype = C.c_uint32
            getattr(L, n).argtypes = [C.c_uint32, C.c_uint32]
        L.orc_challenger_sample_bits.restype = C.c_uint32
        L.orc_challenger_grind.restype = C.c_uint32
        L.orc_challenger_check_witness.restype = C.c_int
        L.orc_stacked_prove_verify.restype = C.c_int64
        _lib = L
    return _lib


def ptr(a):
    assert a.dtype == np.uint32 and a.flags["C_CONTIGUOUS"]
    return a.ctypes.data_as(u32p)


def to_monty(x):
    """canonical -> Montgomery, vectorised in numpy"""
    x = np.asarray(x, dtype=np.uint64)
    return ((x << np.uint64(32)) % np.uint64(P)).astype(np.uint32)


def from_monty(x):
    x = np.asarray(x, dtype=np.uint64)
    # x * 2^-32 mod p ; 2^-32 mod p computed with python ints
    rinv = pow(1 << 32, P - 2, P)
    return ((x * np.uint64(rinv)) % np.uint64(P)).astype(np.uint32)


def rand_field(rng, shape):
    """uniform canonical field elements, returned as Montgomery words"""
    return to_monty(rng.integers(0, P, size=shape, dtype=np.uint64))


ONE = (1 << 32) % P                    # the Montgomery word of 1
WORD_KINDS = ("max", "zero", "one", "minus_one", "mixed")
# the words of the `mixed` kind besides uniform ones: the ends of [0, p), 1 and -1 in Montgomery form, and 2^30 (p - 1 is also
# 2^31 - 2^24, so it appears once)
SPECIAL_WORDS = np.array([0, 1, 2, P - 2, P - 1, ONE, P - ONE, 1 << 30], np.uint32)


def words(rng, shape, kind=None):
    """Montgomery WORDS of a given kind (the canonical values follow through from_monty).  The lazily reducing kernels see words, and
    only words near p - 1 bring their 64-bit accumulators close to the reduction's bound:
      None       uniform canonical values (rand_field; the same draws, so a seed gives the same words as rand_field)
      "max"      every word p - 1 (the canonical value 0x3FFF0001)
      "zero"     every word 0
      "one"      every word ONE (the value 1)
      "minus_one" every word p - ONE (the value p - 1)
      "mixed"    blocks of 16 words: uniform words, one special word (SPECIAL_WORDS) repeated, or specials and uniform words alternating
                 at random"""
    if kind is None:
        return rand_field(rng, shape)
    fill = {"max": P - 1, "zero": 0, "one": ONE, "minus_one": P - ONE}
    if kind in fill:
        return np.full(shape, fill[kind], np.uint32)
    assert kind == "mixed", f"unknown word kind {kind!r}"
    n = int(np.prod(shape, dtype=np.int64))
    nb = (n + 15) // 16
    u = rand_field(rng, nb * 16).reshape(nb, 16)
    spec = SPECIAL_WORDS[rng.integers(0, SPECIAL_WORDS.size, (nb, 16))]
    mode = rng.integers(0, 4, nb)                                # 0, 1: uniform, 2: a run of one special word, 3: singletons
    pick = rng.integers(0, 2, (nb, 16)).astype(bool) & (mode == 3)[:, None]
    out = np.where(pick, spec, u)
    out = np.where((mode == 2)[:, None], spec[:, :1], out)
    return np.ascontiguousarray(out.reshape(-1)[:n].reshape(shape))


def permute(state):
    s = np.ascontiguousarray(state, dtype=np.uint32).copy()
    lib().orc_poseidon2_permute(ptr(s))
    return s


def hash_(vals):
    v = np.ascontiguousarray(vals, dtype=np.uint32)
    out = np.zeros(8, dtype=np.uint32)
    lib().orc_hash(ptr(v), C.c_uint64(v.size), ptr(out))
    return out


def compress(l, r):
    l = np.ascontiguousarray(l, dtype=np.uint32)
    r = np.ascontiguousarray(r, dtype=np.uint32)
    out = np.zeros(8, dtype=np.uint32)
    lib().orc_compress(ptr(l), ptr(r), ptr(out))
    return out


def rs_encode(msg, log_blowup):
    """msg: [ncols, 2^log_h] uint32 (each column contiguous) -> [ncols, 2^(log_h+log_blowup)]"""
    msg = np.ascontiguousarray(msg, dtype=np.uint32)
    ncols, h = msg.shape
    log_h = h.bit_length() - 1
    assert 1 << log_h == h
    out = np.zeros((ncols, h << log_blowup), dtype=np.uint32)
    lib().orc_rs_encode(ptr(msg), C.c_uint64(ncols), C.c_uint32(log_h), C.c_uint32(log_blowup), ptr(out))
    return out


def dft_naive(msg, log_n):
    msg = np.ascontiguousarray(msg, dtype=np.uint32)
    out = np.zeros(1 << log_n, dtype=np.uint32)
    lib().orc_dft_naive(ptr(msg), C.c_uint64(msg.size), C.c_uint32(log_n), ptr(out))
    return out


def merkle_commit(mat, want_layers=False):
    """mat: [width, 2^log_h] (each column contiguous).  -> (root, commitment[, layers flat [2^(log_h+1)-1, 8]])"""
    mat = np.ascontiguousarray(mat, dtype=np.uint32)
    width, h = mat.shape
    log_h = h.bit_length() - 1
    root = np.zeros(8, dtype=np.uint32)
    commit = np.zeros(8, dtype=np.uint32)
    layers = np.zeros((2 * h - 1, 8), dtype=np.uint32) if want_layers else None
    lib().orc_merkle_commit(ptr(mat), C.c_uint64(width), C.c_uint32(log_h),
                            ptr(layers) if want_layers else None, ptr(root), ptr(commit))
    return (root, commit, layers) if want_layers else (root, commit)


class Challenger:
    def __init__(self, state=None):
        self.st = np.zeros(34, dtype=np.uint32)
        if state is None:
            lib().orc_challenger_init(ptr(self.st))
        else:
            self.st[:] = state

    def clone(self):
        return Challenger(self.st.copy())

    def observe(self, vals):
        v = np.ascontiguousarray(np.atleast_1d(vals), dtype=np.uint32)
        lib().orc_challenger_observe(ptr(self.st), ptr(v), C.c_uint64(v.size))

    def sample(self, n=1):
        out = np.zeros(n, dtype=np.uint32)
        lib().orc_challenger_sample(ptr(self.st), ptr(out), C.c_uint64(n))
        return out

    def sample_bits(self, bits):
        return int(lib().orc_challenger_sample_bits(ptr(self.st), C.c_uint32(bits)))

    def grind(self, bits):
        return int(lib().orc_challenger_grind(ptr(self.st), C.c_uint32(bits)))

    def check_witness(self, bits, w):
        return bool(lib().orc_challenger_check_witness(ptr(self.st), C.c_uint32(bits), C.c_uint32(w)))


def stacked_prove_verify(dense_rounds, log_h, point, challenger, log_blowup=2, num_queries=124, pow_bits=16,
                         batch_pow_bits=5, replay=None):
    """dense_rounds: list of [ncols, 2^log_h] arrays.  point: [k,4] uint32 with k >= log_h.
    Returns (commits [n_rounds,8], proof words) — raises if the restated verifier rejects."""
    rounds = [np.ascontiguousarray(d, dtype=np.uint32) for d in dense_rounds]
    n = len(rounds)
    arr = (u32p * n)(*[ptr(r) for r in rounds])
    ncols = (C.c_uint64 * n)(*[r.shape[0] for r in rounds])
    point = np.ascontiguousarray(point, dtype=np.uint32)
    commits = np.zeros((n, 8), dtype=np.uint32)
    cap = 1 << 24
    proof = np.zeros(cap, dtype=np.uint32)
    rw = None
    if replay is not None:
        rw = np.ascontiguousarray(replay, dtype=np.uint32)
    nwords = lib().orc_stacked_prove_verify(arr, ncols, C.c_uint32(n), C.c_uint32(log_h), ptr(point),
                                            C.c_uint32(point.shape[0]), C.c_uint32(log_blowup), C.c_uint32(num_queries),
                                            C.c_uint32(pow_bits), C.c_uint32(batch_pow_bits),
                                            ptr(rw) if rw is not None else None, ptr(challenger.st), ptr(commits),
                                            ptr(proof), C.c_uint64(cap))
    if nwords < 0:
        raise RuntimeError(f"oracle stacked_prove_verify failed ({nwords})")
    return commits, proof[:nwords].copy()


def jagged_prove_verify(rounds_tables, log_stack, max_log_rows, z_row, challenger, log_blowup=2, num_queries=124,
                        pow_bits=16, batch_pow_bits=5, replay=None):
    """rounds_tables: list (rounds) of lists of tables; a table is an array [cols, rows] (each column contiguous,
    rows <= 2^max_log_rows; rows may be 0: pass np.zeros((cols, 0))).  z_row: [max_log_rows, 4].
    Returns (commits [n_rounds, 8], claims [total_cols, 4], proof words); raises if the restated verifier rejects."""
    n = len(rounds_tables)
    dense, n_tables, rows, cols = [], [], [], []
    for tabs in rounds_tables:
        n_tables.append(len(tabs))
        parts = []
        for t in tabs:
            t = np.ascontiguousarray(t, dtype=np.uint32)
            cols.append(t.shape[0]); rows.append(t.shape[1])
            if t.shape[1]:
                parts.append(t.reshape(-1))
        dense.append(np.ascontiguousarray(np.concatenate(parts)) if parts else np.zeros(1, np.uint32))
    arr = (u32p * n)(*[ptr(d) for d in dense])
    nt = (C.c_uint32 * n)(*n_tables)
    R = (C.c_uint64 * len(rows))(*rows)
    Cc = (C.c_uint64 * len(cols))(*cols)
    z = np.ascontiguousarray(z_row, dtype=np.uint32)
    commits = np.zeros((n, 8), np.uint32)
    claims = np.zeros((sum(cols), 4), np.uint32)
    cap = 1 << 24
    proof = np.zeros(cap, np.uint32)
    rw = None if replay is None else np.ascontiguousarray(replay, dtype=np.uint32)
    f = lib().orc_jagged_prove_verify
    f.restype = C.c_int64
    nwords = f(arr, C.c_uint32(n), nt, R, Cc, C.c_uint32(log_stack), C.c_uint32(max_log_rows), ptr(z),
               C.c_uint32(log_blowup), C.c_uint32(num_queries), C.c_uint32(pow_bits), C.c_uint32(batch_pow_bits),
               ptr(rw) if rw is not None else None, ptr(challenger.st), ptr(commits), ptr(claims), ptr(proof),
               C.c_uint64(cap))
    if nwords < 0:
        raise RuntimeError(f"oracle jagged_prove_verify failed ({nwords})")
    return commits, claims, proof[:nwords].copy()


def random_tables(rng, shapes, kind=None):
    """shapes: list of (rows, cols) -> list of [cols, rows] Montgomery arrays of the given word kind (words; None: uniform)"""
    return [words(rng, (c, r), kind) if r else np.zeros((c, 0), np.uint32) for r, c in shapes]


def zerocheck_prove_verify(blob, heights, mains, preps, pv, max_log_rows, gkr_point, challenger):
    """mains/preps: per chip [w, height] arrays (preps[k] None when the chip has no preprocessed columns).
    Returns (gkr openings per chip flat [sum(main_w+prep_w), 4], proof+opened words)."""
    n = len(heights)
    keep = []

    def arr_ptr(a):
        a = np.ascontiguousarray(a if a is not None and a.size else np.zeros(1, np.uint32), dtype=np.uint32)
        keep.append(a)
        return ptr(a)
    M = (u32p * n)(*[arr_ptr(m) for m in mains])
    Pp = (u32p * n)(*[arr_ptr(p) for p in preps])
    H = (C.c_uint64 * n)(*heights)
    blob = np.ascontiguousarray(blob, dtype=np.uint32)
    pv = np.ascontiguousarray(pv, dtype=np.uint32)
    gp = np.ascontiguousarray(gkr_point, dtype=np.uint32)
    ncols = sum(m.shape[0] for m in mains) + sum(p.shape[0] for p in preps if p is not None)
    openings = np.zeros((ncols, 4), np.uint32)
    cap = 1 << 22
    out = np.zeros(cap, np.uint32)
    f = lib().orc_zerocheck_prove_verify
    f.restype = C.c_int64
    nw = f(ptr(blob), H, M, Pp, ptr(pv), C.c_uint32(pv.size), C.c_uint32(max_log_rows), ptr(gp), ptr(challenger.st),
           ptr(openings), ptr(out), C.c_uint64(cap))
    if nw < 0:
        raise RuntimeError(f"oracle zerocheck failed ({nw})")
    return openings, out[:nw].copy()


def gkr_prove_verify(blob, heights, mains, preps, max_log_rows, challenger, gkr_pow_bits=12, replay=None):
    n = len(heights)
    keep = []

    def arr_ptr(a):
        a = np.ascontiguousarray(a if a is not None and a.size else np.zeros(1, np.uint32), dtype=np.uint32)
        keep.append(a)
        return ptr(a)
    M = (u32p * n)(*[arr_ptr(m) for m in mains])
    Pp = (u32p * n)(*[arr_ptr(p) for p in preps])
    H = (C.c_uint64 * n)(*heights)
    blob = np.ascontiguousarray(blob, dtype=np.uint32)
    cap = 1 << 22
    out = np.zeros(cap, np.uint32)
    rw = None if replay is None else np.ascontiguousarray([replay], dtype=np.uint32)
    f = lib().orc_gkr_prove_verify
    f.restype = C.c_int64
    nw = f(ptr(blob), H, M, Pp, C.c_uint32(max_log_rows), C.c_uint32(gkr_pow_bits), ptr(rw) if rw is not None else None,
           ptr(challenger.st), ptr(out), C.c_uint64(cap))
    if nw < 0:
        raise RuntimeError(f"oracle gkr failed ({nw})")
    return out[:nw].copy()


def prove_shard_verify(blob, heights, mains, preps, names, pv, log_stack, max_log_rows, challenger, log_blowup=2, num_queries=124,
                       pow_bits=16, batch_pow_bits=5, gkr_pow_bits=12):
    """Whole-shard oracle: returns (prep_commit[8], proof words).  Raises if the restated ShardVerifier rejects."""
    pd = [np.ascontiguousarray(p, dtype=np.uint32).reshape(-1) for p in preps if p is not None and p.size]
    md = [np.ascontiguousarray(m, dtype=np.uint32).reshape(-1) for m in mains if m.size]
    prep_dense = np.concatenate(pd) if pd else np.zeros(1, np.uint32)
    main_dense = np.concatenate(md) if md else np.zeros(1, np.uint32)
    H = (C.c_uint64 * len(heights))(*heights)
    nm = b"".join(n.encode() + b"\0" for n in names)
    blob = np.ascontiguousarray(blob, dtype=np.uint32)
    pv = np.ascontiguousarray(pv, dtype=np.uint32)
    pc = np.zeros(8, np.uint32)
    cap = 1 << 24
    out = np.zeros(cap, np.uint32)
    f = lib().orc_prove_shard_verify
    f.restype = C.c_int64
    nw = f(ptr(blob), H, ptr(prep_dense), ptr(main_dense), C.c_char_p(nm), ptr(pv), C.c_uint32(pv.size), C.c_uint32(log_stack),
           C.c_uint32(max_log_rows), C.c_uint32(log_blowup), C.c_uint32(num_queries), C.c_uint32(pow_bits), C.c_uint32(batch_pow_bits),
           C.c_uint32(gkr_pow_bits), ptr(challenger.st), ptr(pc), ptr(out), C.c_uint64(cap))
    if nw < 0:
        raise RuntimeError(f"oracle prove_shard failed ({nw})")
    return pc, out[:nw].copy()


def verify_shard(blob, heights, names, log_stack, max_log_rows, challenger, prep_commit, words, log_blowup=2, num_queries=124, pow_bits=16,
                 batch_pow_bits=5, gkr_pow_bits=12):
    """Verify-only: the restated ShardVerifier::verify_shard on proof words produced elsewhere (e.g. by the CUDA library).
    `challenger`: the state the prover started from; updated to the verifier's final state.  Returns 0 (accepted), -1 (rejected),
    -2 (the words do not parse)."""
    H = (C.c_uint64 * len(heights))(*heights)
    nm = b"".join(n.encode() + b"\0" for n in names)
    blob = np.ascontiguousarray(blob, dtype=np.uint32)
    words = np.ascontiguousarray(words, dtype=np.uint32)
    pc = np.ascontiguousarray(prep_commit if prep_commit is not None else np.zeros(8), dtype=np.uint32)
    f = lib().orc_verify_shard
    f.restype = C.c_int64
    return int(f(ptr(blob), H, C.c_char_p(nm), C.c_uint32(log_stack), C.c_uint32(max_log_rows), C.c_uint32(log_blowup), C.c_uint32(num_queries),
                 C.c_uint32(pow_bits), C.c_uint32(batch_pow_bits), C.c_uint32(gkr_pow_bits), ptr(challenger.st), ptr(pc), ptr(words),
                 C.c_uint64(words.size)))


def partial_lagrange(point):
    """eq table of an ext point [n, 4] -> [2^n, 4]; the first coordinate is the most significant bit of the index"""
    point = np.ascontiguousarray(point, dtype=np.uint32)
    out = np.zeros((1 << point.shape[0], 4), np.uint32)
    lib().orc_partial_lagrange(ptr(point), C.c_uint64(point.shape[0]), ptr(out))
    return out


def jagged_last_inputs():
    """z_col [n, 4] and the Hadamard sumcheck claim [4] of this thread's last oracle jagged proof"""
    claim = np.zeros(4, np.uint32)
    f = lib().orc_jagged_last_inputs
    f.restype = C.c_uint32
    n = f(None, C.c_uint32(0), ptr(claim))
    z_col = np.zeros((n, 4), np.uint32)
    f(ptr(z_col), C.c_uint32(n), ptr(claim))
    return z_col, claim


def gkr_last_inputs():
    """the inputs of this thread's last oracle LogUp-GKR prove that the proof does not carry:
    -> (alpha [4], beta_seed [n, 4], per GKR layer in proof order (lambda [4], claim [4], evaluation point [m, 4]))"""
    f = lib().orc_gkr_last_inputs
    f.restype = C.c_uint64
    n = f(None, C.c_uint64(0))
    w = np.zeros(n, np.uint32)
    f(ptr(w), C.c_uint64(n))
    alpha = w[0:4]; nb = int(w[4]); o = 5
    beta = w[o:o + 4 * nb].reshape(nb, 4); o += 4 * nb
    layers = []
    nl = int(w[o]); o += 1
    for _ in range(nl):
        lam, claim = w[o:o + 4], w[o + 4:o + 8]; m = int(w[o + 8]); o += 9
        layers.append((lam, claim, w[o:o + 4 * m].reshape(m, 4))); o += 4 * m
    assert o == n
    return alpha, beta, layers


def zerocheck_last_inputs():
    """the inputs of this thread's last oracle zerocheck prove: -> (alpha [4], gamma [4], lambda [4], claimed sum [4], the round
    challenges in round order [n, 4])"""
    f = lib().orc_zerocheck_last_inputs
    f.restype = C.c_uint64
    n = f(None, C.c_uint64(0))
    w = np.zeros(n, np.uint32)
    f(ptr(w), C.c_uint64(n))
    m = int(w[16])
    assert n == 17 + 4 * m
    return w[0:4], w[4:8], w[8:12], w[12:16], w[17:].reshape(m, 4)
