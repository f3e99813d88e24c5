"""Machines with numpy traces for the parity tests: the benchmark's workloads at reduced size, and hand-written chip specs with the
calibrated features of those workloads (constraint counts, filler columns, several preprocessed columns, long LogUp messages).

Every builder returns (blob, heights, mains, preps, pv, names); mains[k] / preps[k] are [w, height] Montgomery arrays (preps[k] is
None for a chip without preprocessed columns), the same layout as tests.test_oracle._synth_machine_gkr."""
import collections

import numpy as np

from tests import oracle_lib as O

PV0 = 12345

# one hand-written chip.  vps (values per send) selects the interactions: None = the light template (synth_air.synth_interactions),
# () = none at all (a chip with constraints but no LogUp interactions), a list = synth_air.synth_interactions_calibrated with one
# send + one receive per entry, each message that many values long
Chip = collections.namedtuple("Chip", "h g wp n_constraints extra extra_prep vps", defaults=(False, None, 0, 0, None))


def workload_machine(workload, seed, max_log_rows=22, scale=1.0, machine_seed=42):
    """the benchmark machine of `workload` (sp1_b200.workload.synthetic_machine: heights from `machine_seed`, scaled by `scale`) with
    numpy traces drawn from `seed`"""
    from sp1_b200 import synth_air as SA
    from sp1_b200 import workload as W
    mach = W.synthetic_machine(workload, seed=machine_seed, max_log_rows=max_log_rows, scale=scale)
    rng = np.random.default_rng(seed)
    mains, preps = [], []
    for sp in mach["specs"]:
        m, p = SA.synth_trace(rng, sp.h, sp.g, sp.wp, PV0, extra_cols=sp.extra, extra_prep=sp.extra_prep)
        mains.append(m); preps.append(p)
    pv = O.to_monty(np.array([PV0, 5, 6, 7]))
    return mach["blob"], [sp.h for sp in mach["specs"]], mains, preps, pv, list(mach["names"])


def spec_machine(rng, chips):
    """chips: list of Chip (or plain tuples in Chip's field order)"""
    from sp1_b200 import synth_air as SA
    words, iwords, mains, preps, heights = [], [], [], [], []
    for c in chips:
        c = Chip(*c)
        w, _, _ = SA.synth_chip(c.g, c.wp, n_constraints=c.n_constraints, extra_cols=c.extra, extra_prep=c.extra_prep)
        if c.vps is None:
            iw = SA.synth_interactions(c.g, c.wp)
        elif len(c.vps) == 0:
            iw = [0]
        else:
            iw = SA.synth_interactions_calibrated(c.g, c.wp, list(c.vps))
        words.append(w); iwords.append(iw)
        m, p = SA.synth_trace(rng, c.h, c.g, c.wp, PV0, extra_cols=c.extra, extra_prep=c.extra_prep)
        mains.append(m); preps.append(p); heights.append(c.h)
    pv = O.to_monty(np.array([PV0, 5, 6, 7]))
    names = [f"Chip{i:03d}" for i in range(len(chips))]
    return SA.machine_blob_with_interactions(words, iwords), heights, mains, preps, pv, names


def n_interactions(blob):
    """total LogUp interactions of a machine blob (the interaction section follows the chips' constraint programs)"""
    b = [int(x) for x in blob]
    n, p = b[0], 1
    for _ in range(n):
        ni, nl, nc, npub, na = b[p + 4:p + 9]
        p += 9 + 2 * ni + 2 * nl + nc + npub + 2 * na
    total = 0
    for _ in range(n):
        k = b[p]; p += 1
        total += k
        for _ in range(k):
            nv = b[p + 2]; p += 3
            for _ in range(nv + 1):
                p += 2 + 3 * b[p]
    assert p == len(b), "malformed machine blob"
    return total


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


def product_zerocheck(lib, mach, heights, mains, preps, pv, gp, st0, openings):
    """the product's zerocheck (Lib.zerocheck) on the inputs of oracle_zerocheck: alpha and gamma sampled from st0 as the oracle samples
    them, the per-chip claims sum_j gamma^(j+1) * opening_j (main then prep).  -> (proof words, challenger state after the proof)"""
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
    d_mains = [torch.from_numpy(np.ascontiguousarray(m).view(np.int32)).cuda() for m in mains]
    d_preps = [torch.from_numpy(np.ascontiguousarray(p).view(np.int32)).cuda() if p is not None else None for p in preps]
    torch.cuda.synchronize()
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
