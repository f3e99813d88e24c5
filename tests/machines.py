"""Machines with numpy traces for the parity tests: the benchmark's workloads at reduced size, hand-written chip specs with the
calibrated features of those workloads (constraint counts, filler columns, several preprocessed columns, long LogUp messages), the
hand-made interaction machines of the shard checks, the shared case tables, and the one reader of the machine-blob layout.

Every builder returns (blob, heights, mains, preps, pv, names); mains[k] / preps[k] are [w, height] Montgomery arrays (preps[k] is
None for a chip without preprocessed columns).  Traces are drawn from the generator in chip order, one synth_trace per chip and
nothing else in between, so a seed always gives the same words."""
import collections

import numpy as np

from tests import oracle_lib as O

PV0 = 12345
PV = O.to_monty(np.array([PV0, 5, 6, 7]))

# the small protocol parameters of most whole-shard tests
SMALL = dict(num_queries=8, pow_bits=4, batch_pow_bits=2, gkr_pow_bits=3)

# one hand-written chip.  vps (values per send) selects the interactions: None = the light template (synth_air.synth_interactions),
# () = none at all (a chip with constraints but no LogUp interactions), a list = synth_air.synth_interactions_calibrated with one
# send + one receive per entry, each message that many values long.  deep: the same constraints in an order with long-lived
# intermediates (synth_air.synth_chip)
Chip = collections.namedtuple("Chip", "h g wp n_constraints extra extra_prep vps deep", defaults=(False, None, 0, 0, None, False))


def traces(specs, seed, pv0=PV0):
    """numpy traces of chips with fields h, g, wp, extra, extra_prep (Chip, or the specs of sp1_b200.workload.synthetic_machine)
    drawn from `seed` (an int or a numpy Generator, which is drawn from in place) -> (mains, preps).  A multi-shard test calls this
    with the same seed for every shard, so that the preprocessed tables agree, and each shard's own public value 0."""
    from sp1_b200 import synth_air as SA
    rng = np.random.default_rng(seed)
    mains, preps = [], []
    for c in specs:
        m, p = SA.synth_trace(rng, c.h, c.g, c.wp, pv0, extra_cols=c.extra, extra_prep=c.extra_prep)
        mains.append(m); preps.append(p)
    return mains, preps


def workload_machine(workload, seed, max_log_rows=22, scale=1.0, machine_seed=42):
    """the benchmark machine of `workload` (sp1_b200.workload.synthetic_machine: heights from `machine_seed`, scaled by `scale`) with
    numpy traces drawn from `seed`"""
    from sp1_b200 import workload as W
    mach = W.synthetic_machine(workload, seed=machine_seed, max_log_rows=max_log_rows, scale=scale)
    mains, preps = traces(mach["specs"], seed)
    return mach["blob"], [sp.h for sp in mach["specs"]], mains, preps, PV.copy(), list(mach["names"])


def spec_machine(rng, chips, interactions=True, names="Chip{:03d}"):
    """chips: list of Chip (or plain tuples in Chip's field order).  interactions=False builds the blob without an interaction
    section (synth_air.machine_blob).  names: the chip-name format; the names are observed into the transcript."""
    from sp1_b200 import synth_air as SA
    chips = [Chip(*c) for c in chips]
    words, iwords = [], []
    for c in chips:
        words.append(SA.synth_chip(c.g, c.wp, deep=c.deep, n_constraints=c.n_constraints, extra_cols=c.extra, extra_prep=c.extra_prep)[0])
        if c.vps is None:
            iwords.append(SA.synth_interactions(c.g, c.wp))
        elif len(c.vps) == 0:
            iwords.append([0])
        else:
            iwords.append(SA.synth_interactions_calibrated(c.g, c.wp, list(c.vps)))
    mains, preps = traces(chips, rng)
    blob = SA.machine_blob_with_interactions(words, iwords) if interactions else SA.machine_blob(words)
    return blob, [c.h for c in chips], mains, preps, PV.copy(), [names.format(i) for i in range(len(chips))]


def shard_inputs(spec, seed):
    """the seeded whole-shard inputs of the golden fixtures and the shard tests: spec_machine with names Chip00, Chip01, ..., then a
    challenger that has observed 9 random words from the same generator -> (blob, heights, mains, preps, pv, names, challenger)"""
    rng = np.random.default_rng(seed)
    inp = spec_machine(rng, spec, names="Chip{:02d}")
    ch = O.Challenger(); ch.observe(O.rand_field(rng, 9))
    return inp + (ch,)


def silent(spec, silent_chips):
    """spec's (height, groups, with_prep) chips, those listed in silent_chips without LogUp interactions"""
    return [Chip(*c, vps=() if k in silent_chips else None) for k, c in enumerate(spec)]


# ---- the machine-blob layout (include/sp1b200.h, sp1b200_machine_create) ----------------------------------------------------------
def chip_segments(blob):
    """-> per chip (main_w, prep_w, program words, interaction words); the interaction words are None for a blob without an
    interaction section.  Program: 9 header words main_w prep_w _ _ n_instrs n_leaves n_consts n_publics n_assert, then the records.
    Interactions: a count, then per interaction is_send kind n_values and n_values + 1 virtual columns (multiplicity first), each
    n_terms constant {source col weight}*."""
    b = [int(x) for x in blob]
    progs, p = [], 1
    for _ in range(b[0]):
        ni, nl, nc, npub, na = b[p + 4:p + 9]
        ln = 9 + 2 * ni + 2 * nl + nc + npub + 2 * na
        progs.append(b[p:p + ln]); p += ln
    inters = [None] * b[0]
    if p < len(b):
        for k in range(b[0]):
            q = p + 1
            for _ in range(b[p]):
                nv = b[q + 2]; q += 3
                for _ in range(nv + 1):
                    q += 2 + 3 * b[q]
            inters[k] = b[p:q]; p = q
    assert p == len(b), "malformed machine blob"
    return [(w[0], w[1], w, iw) for w, iw in zip(progs, inters)]


def widths(blob):
    """(main_w, prep_w) per chip"""
    return [(mw, pw) for mw, pw, _, _ in chip_segments(blob)]


def n_interactions(blob):
    """total LogUp interactions of a machine blob"""
    return sum(iw[0] for _, _, _, iw in chip_segments(blob))


# ---- shared case tables ---------------------------------------------------------------------------------------------------------------
SHARD_SPECS = [
    # spec (height, groups, with_prep), log_stack, max_log_rows
    ([(8, 1, False)], 3, 3),
    ([(5, 1, False), (0, 2, False), (6, 1, True)], 3, 3),
    ([(32, 2, True), (96, 1, False), (128, 1, False), (0, 1, True)], 5, 7),
]

GKR_EDGE_CASES = [
    # spec, chips without interactions, max_log_rows
    ([(64, 1, False), (32, 2, False), (16, 1, True)], (1,), 7),       # a chip with constraints but no interactions
    ([(2, 1, False), (1, 1, False)], (0,), 3),                          # 4 interactions in all, heights 2 and 1
    ([(8, 3, False), (0, 1, False), (8, 1, True)], (2,), 4),            # absent chip + silent chip with preprocessed columns
]

# the core-proof tests' machines, with and without preprocessed columns
WITH_PREP = [Chip(256, 2, True), Chip(64 + 8, 3, False), Chip(0, 1, False), Chip(128, 1, True)]
NO_PREP = [Chip(128, 2, False), Chip(32, 1, False)]

# verify_shard's checks of the jagged table shapes against the chips (shard.rs:506-523, :662-742): the oracle's restated verifier does
# not make them, so where the library stops at one of them the oracle can only be required to reject as well
ORACLE_LACKS = ("InvalidShape(preprocessed widths)", "InvalidShape(chip tables)")


def full_table_spec(n_chips, seed, absent=True):
    """n_chips tiny chips with varied heights (1 included, and 0 when `absent`), some with preprocessed columns or filler columns,
    light and calibrated interactions.  With absent=False every chip takes a slot of the GKR batch table."""
    rng = np.random.default_rng(seed)
    heights = ([0] if absent else []) + [1, 2, 3, 32]
    heights += [int(x) for x in rng.integers(0 if absent else 1, 33, n_chips - len(heights))]
    spec = []
    for k, h in enumerate(heights):
        vps = None if k % 3 == 0 else [int(x) for x in rng.integers(1, 13, 1 + k % 4)]
        spec.append(Chip(h, 1 + k % 2, k % 4 == 1, None, int(k % 5 == 2), 1 if k % 8 == 5 else 0, vps))
    return spec


# ---- hand-made interaction machines of the shard checks (oracle/debug.hpp) ---------------------------------------------------------
def _inter_words(inters):
    """inters: [(is_send, kind, mult vcol words, [value vcol words])] -> the chip's interaction words"""
    w = [len(inters)]
    for is_send, kind, mult, vals in inters:
        w += [is_send, kind, len(vals)] + mult
        for v in vals:
            w += v
    return w


def cross_chip_machine(rng, h=64, mult_col_kind4=False):
    """two one-group chips whose sends (chip 0) and receives (chip 1) sit in different chips: chip 1's trace is chip 0's with the rows
    reversed.  Interactions (sends in chip 0, receives in chip 1, same order): kind 4 (a, 9) with multiplicity 1 (or column d when
    mult_col_kind4), kind 6 (b) with multiplicity d."""
    from sp1_b200 import synth_air as SA
    w, _, _ = SA.synth_chip(1, False)
    m0, _ = SA.synth_trace(rng, h, 1, False, PV0)
    m1 = np.ascontiguousarray(m0[:, ::-1])
    a, b, d = (SA.LEAF_MAIN, 0, 1), (SA.LEAF_MAIN, 1, 1), (SA.LEAF_MAIN, 3, 1)
    mult4 = SA._vcol([d]) if mult_col_kind4 else SA._vcol([], constant=1)
    inter = lambda s: [(s, 4, mult4, [SA._vcol([a]), SA._vcol([], constant=9)]), (s, 6, SA._vcol([d]), [SA._vcol([b])])]
    blob = SA.machine_blob_with_interactions([w, w], [_inter_words(inter(1)), _inter_words(inter(0))])
    return blob, [h, h], [m0, m1], [None, None]


def fingerprint(kind, values):
    """the interaction check's key fingerprint (the library's host code, libsp1b200_hostcheck.so)"""
    import ctypes as C
    from tests import hostcheck_lib
    f = hostcheck_lib.load().sp1b200_hostcheck_fingerprint
    f.restype = C.c_uint64
    v = np.ascontiguousarray(values, dtype=np.uint32)
    return int(f(C.c_uint32(kind), C.c_uint32(v.size), v.ctypes.data_as(C.POINTER(C.c_uint32)) if v.size else None))


def colliding_keys(rng, kind=5):
    """two different 3-value keys (canonical values) with equal fingerprints, from the two linear forms read off basis vectors"""
    P = O.P

    def forms(vals):
        x = fingerprint(kind, O.to_monty(np.array(vals)))
        return x >> 31, x & 0x7fffffff
    base = forms([0, 0, 0])
    c = []
    for t in range(3):
        e = [0, 0, 0]; e[t] = 1
        f = forms(e)
        c.append(((f[0] - base[0]) % P, (f[1] - base[1]) % P))
    # d = c0 x c1 (componentwise forms over the three values) is in the kernel of both forms
    u, v = [x[0] for x in c], [x[1] for x in c]
    d = [(u[1] * v[2] - u[2] * v[1]) % P, (u[2] * v[0] - u[0] * v[2]) % P, (u[0] * v[1] - u[1] * v[0]) % P]
    A = [int(x) for x in rng.integers(0, P, 3)]
    B = [(x + y) % P for x, y in zip(A, d)]
    assert A != B
    return A, B


def constant_key_machine(rng, chip_inters, heights):
    """one-group chips whose interactions have constant values: chip_inters[k] = [(is_send, kind, canonical values)], multiplicity 1"""
    from sp1_b200 import synth_air as SA
    words, iws, mains = [], [], []
    for inters, h in zip(chip_inters, heights):
        w, _, _ = SA.synth_chip(1, False)
        words.append(w)
        iws.append(_inter_words([(s, k, SA._vcol([], constant=1), [SA._vcol([], constant=x) for x in vals]) for s, k, vals in inters]))
        mains.append(SA.synth_trace(rng, h, 1, False, PV0)[0])
    return SA.machine_blob_with_interactions(words, iws), list(heights), mains, [None] * len(heights)


# ---- oracle and product calls on these machines ----------------------------------------------------------------------------------
def oracle_zerocheck(rng, blob, heights, mains, preps, pv, mlr):
    """the oracle's zerocheck proof of a machine at a random GKR point from a random transcript state, both drawn from rng.
    -> (GKR point, challenger state before the proof, the column openings at the GKR point, proof words, challenger state after it)"""
    gp = O.rand_field(rng, (mlr, 4))
    ch = O.Challenger(); ch.observe(O.rand_field(rng, 4))
    st0 = ch.st.copy()
    openings, owords = O.zerocheck_prove_verify(blob, heights, mains, preps, pv, mlr, gp, ch)
    return gp, st0, openings, owords, ch.st.copy()


def _ext_mul(a, b):
    out = np.zeros(4, np.uint32)
    O.lib().orc_ext_mul(O.ptr(np.ascontiguousarray(a, dtype=np.uint32)), O.ptr(np.ascontiguousarray(b, dtype=np.uint32)), O.ptr(out))
    return out


def _ext_add(a, b):
    return ((a.astype(np.uint64) + b) % O.P).astype(np.uint32)


def product_zerocheck(lib, mach, heights, mains, preps, pv, gp, st0, openings, device=None):
    """the product's zerocheck (Lib.zerocheck) on the inputs of oracle_zerocheck: alpha and gamma sampled from st0 as the oracle samples
    them, the per-chip claims sum_j gamma^(j+1) * opening_j (main then prep).  device: (per chip main, per chip preprocessed) device
    tensors holding mains / preps, or None to upload them here.  -> (proof words, challenger state after the proof)"""
    import torch
    from sp1_b200.lib import HostChallenger
    hc = HostChallenger(st0.copy())
    alpha = hc.sample(4); gamma = hc.sample(4)
    claims, k = [], 0
    for m, p in zip(mains, preps):
        w = m.shape[0] + (p.shape[0] if p is not None else 0)
        acc, g = np.zeros(4, np.uint32), gamma.copy()
        for j in range(w):
            acc = _ext_add(acc, _ext_mul(openings[k + j], g))
            g = _ext_mul(g, gamma)
        claims.append(acc); k += w
    if device is None:
        d_mains = [torch.from_numpy(np.ascontiguousarray(m).view(np.int32)).cuda() for m in mains]
        d_preps = [torch.from_numpy(np.ascontiguousarray(p).view(np.int32)).cuda() if p is not None else None for p in preps]
        torch.cuda.synchronize()
    else:
        d_mains, d_preps = device
    words = lib.zerocheck(mach, heights, d_mains, d_preps, pv, gp, alpha, gamma, np.stack(claims), hc.st)
    return words, hc.st


def dense_main(mains):
    """the main traces back to back (the prove_shard input)"""
    parts = [np.ascontiguousarray(m).reshape(-1) for m in mains if m.size]
    return np.ascontiguousarray(np.concatenate(parts)) if parts else np.zeros(1, np.uint32)


def first_diff(words, owords, what="words"):
    """"first differing words ..." message for a proof that differs from the oracle's"""
    if words.size != owords.size:
        return f"{what}: {words.size} words, the oracle has {owords.size}"
    bad = np.nonzero(words != owords)[0]
    return f"{what}: first differing words {bad[:8].tolist()} of {words.size}"


SECTIONS = ["main commitment", "LogUp-GKR", "zerocheck", "evaluation proof", "public values"]


def shard_diff(words, owords):
    """as first_diff, naming the first differing section of a whole-shard proof (section lengths in words[1:1 + words[0]])"""
    msg = first_diff(words, owords, "shard proof")
    n_sec = int(owords[0])
    lens = [int(x) for x in owords[1:1 + n_sec]]
    n = min(words.size, owords.size)
    bad = np.nonzero(words[:n] != owords[:n])[0]
    at = int(bad[0]) if bad.size else n
    off = 1 + n_sec
    if at < off:
        return f"{msg}; first difference in the section header"
    for s, ln in enumerate(lens):
        if at < off + ln:
            name = SECTIONS[s] if s < len(SECTIONS) else f"section {s}"
            return f"{msg}; first difference in the {name} section (words {off}..{off + ln}) at offset {at - off}"
        off += ln
    return f"{msg}; first difference past the last section"
