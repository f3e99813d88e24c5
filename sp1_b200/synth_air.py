"""Synthetic AIRs in the reference GPU prover's bytecode format, with traces that satisfy them.

The reference lowers each chip's Rust `Air::eval` to `ChunkBytecode` (sp1-gpu/crates/air/src/ir/bytecode.rs, consumed by
sp1-gpu/crates/sys/lib/zerocheck/sequential.cu:52-110).  That lowering needs cargo, which this image lacks, so tests and
bench use synthetic chips expressed directly in the same instruction set (DagInstr / LeafRef / BcOp, layout of
sp1-gpu/crates/sys/include/zerocheck/sequential.cuh:13-49): the prover input contract is unchanged.

Column template (repeated `groups` times in the main trace), constraints of degree <= 3:
    a, b free;  d in {0,1};  c = a*b;  e = a*b*d;  f = a + K*pv[0]      (+ with preprocessed column g:  h = g*a)
so all-zero padding rows violate the `f` constraint by a constant — exercising the padded-row correction.
Test/bench input generation only.
"""
import numpy as np

P = 0x7F000001
LOAD_LEAF, LOAD_CONST, LOAD_PUBLIC, ADD, SUB, MUL, NEG = range(7)
LEAF_PREP, LEAF_MAIN = 2, 4


def to_monty(x):
    x = np.asarray(x, dtype=np.uint64)
    return ((x << np.uint64(32)) % np.uint64(P)).astype(np.uint32)


class Asm:
    def __init__(self):
        self.instrs, self.leaves, self.consts, self.publics, self.asserts = [], [], [], [], []
        self.nreg = 0

    def _r(self):
        self.nreg += 1
        return self.nreg - 1

    def leaf(self, source, col):
        self.leaves.append((source, col))
        r = self._r()
        self.instrs.append((LOAD_LEAF, r, len(self.leaves) - 1, 0))
        return r

    def const(self, canonical):
        self.consts.append(int(to_monty(np.array([canonical]))[0]))
        r = self._r()
        self.instrs.append((LOAD_CONST, r, len(self.consts) - 1, 0))
        return r

    def public(self, idx):
        self.publics.append(idx)
        r = self._r()
        self.instrs.append((LOAD_PUBLIC, r, len(self.publics) - 1, 0))
        return r

    def op(self, opc, a, b=0):
        r = self._r()
        self.instrs.append((opc, r, a, b))
        return r

    def assert_zero(self, reg):
        self.asserts.append(reg)

    def words(self, main_w, prep_w, alphas=None):
        """the chip's words of the machine blob; alphas[k] = the reversed-powers index of assert k (default: k)"""
        n = len(self.asserts)
        w = [main_w, prep_w, n, self.nreg, len(self.instrs), len(self.leaves), len(self.consts), len(self.publics), n]
        for opc, out, a, b in self.instrs:
            w += [opc | (out << 16), a | (b << 16)]
        for src, col in self.leaves:
            w += [src, col]
        w += self.consts + self.publics + self.asserts + (list(range(n)) if alphas is None else list(alphas))
        return w


def synth_chip(groups, with_prep, kconst=7, deep=False, n_constraints=None, extra_cols=0, extra_prep=0):
    """-> (machine words for this chip, main_w, prep_w).
    n_constraints (calibrated chips): further constraints of degree 2-3 are added round-robin over the groups until the chip has
    that many (at most 9 per group); each is implied by the template's relations, so the same traces satisfy them and they vanish on
    the all-zero padding row.  extra_cols: unconstrained filler columns after the template (exact reference widths, e.g. 682).
    extra_prep (needs with_prep): further preprocessed columns; they are committed, opened and batched like any column but appear in
    no constraint (recursion chips keep most of their columns preprocessed).
    deep=True emits the SAME constraints in an order with long-lived intermediates (all products a_g b_g first, consumed in
    reverse order afterwards): the register pressure of the program grows with `groups`, which exercises the larger
    register-file tiers of the zerocheck kernels (the flat order needs a handful of registers whatever the chip size)."""
    a = Asm()
    main_w = 6 * groups + (1 if with_prep else 0) + extra_cols
    prep_w = (1 + extra_prep) if with_prep else 0
    pv0 = a.public(0)
    kc = a.const(kconst)
    one = a.const(1)
    kpv = a.op(MUL, kc, pv0)

    def tail(g, ab, A=None):
        Cc, D, E, Fc = (a.leaf(LEAF_MAIN, 6 * g + i) for i in range(2, 6))
        if A is None:
            A = a.leaf(LEAF_MAIN, 6 * g)
        a.assert_zero(a.op(SUB, Cc, ab))                       # c - a b
        a.assert_zero(a.op(MUL, D, a.op(SUB, D, one)))         # d (d - 1)
        a.assert_zero(a.op(SUB, E, a.op(MUL, ab, D)))          # e - a b d   (degree 3)
        a.assert_zero(a.op(SUB, Fc, a.op(ADD, A, kpv)))        # f - (a + K pv0)

    if deep:
        abs_ = []
        for g in range(groups):
            A, B = a.leaf(LEAF_MAIN, 6 * g), a.leaf(LEAF_MAIN, 6 * g + 1)
            abs_.append(a.op(MUL, A, B))
        for g in reversed(range(groups)):
            tail(g, abs_[g])
    else:
        for g in range(groups):
            A, B = a.leaf(LEAF_MAIN, 6 * g), a.leaf(LEAF_MAIN, 6 * g + 1)
            tail(g, a.op(MUL, A, B), A)
    if with_prep:
        G = a.leaf(LEAF_PREP, 0)
        H = a.leaf(LEAF_MAIN, 6 * groups)
        A0 = a.leaf(LEAF_MAIN, 0)
        a.assert_zero(a.op(ADD, a.op(NEG, a.op(MUL, G, A0)), H))  # -(g a) + h
    if n_constraints is not None:
        have = len(a.asserts)
        kind, g = 0, 0
        while have < n_constraints and kind < 5:
            A, B, Cc, D, E, Fc = (a.leaf(LEAF_MAIN, 6 * g + i) for i in range(6))
            if kind == 0:
                a.assert_zero(a.op(MUL, D, a.op(SUB, Cc, a.op(MUL, A, B))))     # d (c - a b)          degree 3
            elif kind == 1:
                a.assert_zero(a.op(SUB, E, a.op(MUL, Cc, D)))                   # e - c d
            elif kind == 2:
                a.assert_zero(a.op(MUL, D, a.op(SUB, E, Cc)))                   # d (e - c)            (d boolean, e = c d)
            elif kind == 3:
                a.assert_zero(a.op(MUL, B, a.op(SUB, Fc, a.op(ADD, A, kpv))))   # b (f - a - K pv0)
            else:
                a.assert_zero(a.op(MUL, E, a.op(SUB, D, one)))                  # e (d - 1)
            have += 1
            g += 1
            if g == groups:
                g, kind = 0, kind + 1
    return a.words(main_w, prep_w), main_w, prep_w


def synth_trace(rng, height, groups, with_prep, pv0_canonical, kconst=7, extra_cols=0, extra_prep=0):
    """canonical-domain generation, returned as Montgomery words, column-major [w, height]"""
    cols = []
    prep = None
    a0 = None
    for g in range(groups):
        a = rng.integers(0, P, height, dtype=np.uint64)
        b = rng.integers(0, P, height, dtype=np.uint64)
        d = rng.integers(0, 2, height, dtype=np.uint64)
        c = a * b % P
        e = c * d % P
        f = (a + kconst * pv0_canonical) % P
        cols += [a, b, c, d, e, f]
        if g == 0:
            a0 = a
    if with_prep:
        gcol = rng.integers(0, P, height, dtype=np.uint64)
        cols.append(gcol * a0 % P)
        prep = to_monty(np.stack([gcol] + [rng.integers(0, P, height, dtype=np.uint64) for _ in range(extra_prep)]))
    for _ in range(extra_cols):
        cols.append(rng.integers(0, P, height, dtype=np.uint64))
    main = to_monty(np.stack(cols)) if height else np.zeros((len(cols), 0), np.uint32)
    if with_prep and not height:
        prep = np.zeros((1 + extra_prep, 0), np.uint32)
    return main, prep


def machine_blob(chip_words):
    w = [len(chip_words)]
    for cw in chip_words:
        w += cw
    return np.array(w, dtype=np.uint32)


# ---- LogUp interactions (crates/hypercube/src/lookup/interaction.rs:11-22; VirtualPairCol = Σ weight·column + constant) ----
def _vcol(terms, constant=0):
    """terms: [(source, col, weight_canonical)] -> words: n_terms constant {source col weight}*"""
    w = [len(terms), int(to_monty(np.array([constant]))[0])]
    for src, col, wt in terms:
        w += [src, col, int(to_monty(np.array([wt]))[0])]
    return w


def synth_interactions(groups, with_prep, inter_groups=None):
    """Balanced sends/receives for a synth_chip: every tuple that is sent is received with the same multiplicity, so the
    cumulative LogUp sum is zero.  Words for one chip: n_interactions then per interaction
    is_send arg_index n_values, multiplicity vcol, value vcols."""
    inter = []
    ig = groups if inter_groups is None else max(1, min(groups, inter_groups))
    for g in range(ig):
        base = 6 * g
        a, b, c, d, e, f = (base + i for i in range(6))
        vals3 = [_vcol([(LEAF_MAIN, a, 1)]), _vcol([(LEAF_MAIN, b, 1), (LEAF_MAIN, a, 2)]), _vcol([(LEAF_MAIN, c, 1)], constant=5)]
        mult_d = _vcol([(LEAF_MAIN, d, 1)])
        inter.append((1, 5, mult_d, vals3))                     # send, kind Byte(5), multiplicity d
        vals1 = [_vcol([(LEAF_MAIN, e, 3)])]
        inter.append((1, 7, _vcol([], constant=1), vals1))      # send, kind State(7), multiplicity 1
    for g in range(ig):
        base = 6 * g
        a, b, c, d, e, f = (base + i for i in range(6))
        vals3 = [_vcol([(LEAF_MAIN, a, 1)]), _vcol([(LEAF_MAIN, a, 2), (LEAF_MAIN, b, 1)]), _vcol([(LEAF_MAIN, c, 1)], constant=5)]
        inter.append((0, 5, _vcol([(LEAF_MAIN, d, 1)]), vals3))  # receive the same tuples
        inter.append((0, 7, _vcol([], constant=1), [_vcol([(LEAF_MAIN, e, 3)])]))
    if with_prep:
        gv = [_vcol([(LEAF_PREP, 0, 1)]), _vcol([(LEAF_MAIN, 6 * groups, 1)])]
        inter.insert(2 * ig, (1, 2, _vcol([(LEAF_MAIN, 3, 1)]), gv))   # send (g, h) with multiplicity d0
        inter.append((0, 2, _vcol([(LEAF_MAIN, 3, 1)]), gv))
    w = [len(inter)]
    for is_send, kind, mult, vals in inter:
        w += [is_send, kind, len(vals)] + mult
        for v in vals:
            w += v
    return w


def synth_interactions_calibrated(groups, with_prep, values_per_send):
    """Interactions with the message statistics of a real chip (sp1_b200/chip_stats.json): one send + one receive of the same
    tuple and multiplicity per entry of `values_per_send` (value counts, e.g. 4 = byte lookup, 5 = CPU state, 9 = memory access),
    so the cumulative LogUp sum is zero.  Values are linear combinations of the group columns."""
    kinds = [5, 7, 3, 2, 6, 9]   # InteractionKind indices: Byte, State, Memory, Program, Syscall, Global (any stable labels)
    sends, recvs = [], []
    for i, nv in enumerate(values_per_send):
        g = i % groups
        a, b, c, d, e, f = (6 * g + j for j in range(6))
        menu = [
            [(LEAF_MAIN, a, 1)], [(LEAF_MAIN, b, 1), (LEAF_MAIN, a, 2)], ([(LEAF_MAIN, c, 1)], 5), [(LEAF_MAIN, e, 3)], [(LEAF_MAIN, f, 1)],
            [(LEAF_MAIN, a, 1), (LEAF_MAIN, b, 1), (LEAF_MAIN, c, 1)], ([(LEAF_MAIN, d, 1)], 1), [(LEAF_MAIN, f, 2), (LEAF_MAIN, e, 1)],
            [(LEAF_MAIN, b, 7)], [(LEAF_MAIN, c, 1), (LEAF_MAIN, d, 4)], [(LEAF_MAIN, a, 3), (LEAF_MAIN, f, 1)], [(LEAF_MAIN, e, 1), (LEAF_MAIN, b, 2)],
        ]
        vals = []
        for k in range(nv):
            m = menu[(k + i) % len(menu)]
            vals.append(_vcol(*m) if isinstance(m, tuple) else _vcol(m))
        mult = _vcol([(LEAF_MAIN, d, 1)]) if i % 3 else _vcol([], constant=1)   # boolean column or the constant 1
        kind = kinds[i % len(kinds)]
        sends.append((1, kind, mult, vals))
        recvs.append((0, kind, mult, vals))
    inter = sends + recvs
    if with_prep:
        gv = [_vcol([(LEAF_PREP, 0, 1)]), _vcol([(LEAF_MAIN, 6 * groups, 1)])]
        inter.insert(len(sends), (1, 2, _vcol([(LEAF_MAIN, 3, 1)]), gv))
        inter.append((0, 2, _vcol([(LEAF_MAIN, 3, 1)]), gv))
    w = [len(inter)]
    for is_send, kind, mult, vals in inter:
        w += [is_send, kind, len(vals)] + mult
        for v in vals:
            w += v
    return w


def machine_blob_with_interactions(chip_words, inter_words):
    w = [len(chip_words)]
    for cw in chip_words:
        w += cw
    for iw in inter_words:
        w += iw
    return np.array(w, dtype=np.uint32)


def synth_trace_cuda(height, groups, with_prep, pv0_canonical, seed, device, kconst=7, extra_cols=0, extra_prep=0):
    """same trace family generated on the GPU with torch (bench input only): -> (main [w*height] int32 Montgomery words
    column-major, prep [height] or None)"""
    import torch
    g = torch.Generator(device=device)
    g.manual_seed(seed)
    w = 6 * groups + (1 if with_prep else 0) + extra_cols
    if height == 0:
        return torch.zeros(0, dtype=torch.int32, device=device), (torch.zeros(0, dtype=torch.int32, device=device) if with_prep else None)
    out = torch.empty((w, height), dtype=torch.int32, device=device)

    def mont(x):  # canonical int64 -> Montgomery word
        return ((x << 32) % P).to(torch.int32)
    a0 = None
    for gi in range(groups):
        a = torch.randint(0, P, (height,), dtype=torch.int64, device=device, generator=g)
        b = torch.randint(0, P, (height,), dtype=torch.int64, device=device, generator=g)
        d = torch.randint(0, 2, (height,), dtype=torch.int64, device=device, generator=g)
        c = a * b % P
        e = c * d % P
        f = (a + kconst * pv0_canonical) % P
        for i, col in enumerate((a, b, c, d, e, f)):
            out[6 * gi + i] = mont(col)
        if gi == 0:
            a0 = a
    prep = None
    if with_prep:
        gc = torch.randint(0, P, (height,), dtype=torch.int64, device=device, generator=g)
        out[6 * groups] = mont(gc * a0 % P)
        prep = mont(gc)
        if extra_prep:
            prep = torch.cat([prep] + [mont(torch.randint(0, P, (height,), dtype=torch.int64, device=device, generator=g)) for _ in range(extra_prep)])
    for j in range(extra_cols):
        out[6 * groups + (1 if with_prep else 0) + j] = mont(torch.randint(0, P, (height,), dtype=torch.int64, device=device, generator=g))
    return out.reshape(-1), prep
