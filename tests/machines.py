"""Machines with numpy traces for the parity tests: the benchmark's workloads at reduced size, hand-written chip specs with the
calibrated features of those workloads (constraint counts, filler columns, several preprocessed columns, long LogUp messages), chips
whose constraints are random programs with satisfying traces (random_program), the hand-made interaction machines of the shard checks, the shared case tables, and the one reader of the machine-blob layout.

Every builder returns (blob, heights, mains, preps, pv, names); mains[k] / preps[k] are [w, height] Montgomery arrays (preps[k] is
None for a chip without preprocessed columns).  Traces are drawn from the generator in chip order, one synth_trace (or one
RandomProgram.trace for a random-program chip) per chip and nothing else in between, so a seed always gives the same words."""
import collections
import functools

import numpy as np

from sp1_b200 import synth_air as SA
from tests import oracle_lib as O

PV0 = 12345
PV = O.to_monty(np.array([PV0, 5, 6, 7]))

# the small protocol parameters of most whole-shard tests
SMALL = dict(num_queries=8, pow_bits=4, batch_pow_bits=2, gkr_pow_bits=3)

# one hand-written chip.  vps (values per send) selects the interactions: None = the light template (synth_air.synth_interactions),
# () = none at all (a chip with constraints but no LogUp interactions), a list = synth_air.synth_interactions_calibrated with one
# send + one receive per entry, each message that many values long.  deep: the same constraints in an order with long-lived
# intermediates (synth_air.synth_chip).  program: a Prog, for a chip whose constraints are a random program (random_program) instead
# of the template; such a chip has no interactions and ignores g, wp, n_constraints, extra, extra_prep, vps and deep.
Chip = collections.namedtuple("Chip", "h g wp n_constraints extra extra_prep vps deep program",
                              defaults=(False, None, 0, 0, None, False, None))

# ---- random constraint programs ---------------------------------------------------------------------------------------------------
# The knobs of one random program (random_program), the seed first:
#   n_asserts  constraints (0: an empty program, a chip without constraints); one of them sums the constant and public loads, one
#              the live products, and direct / dup take 3 / 1 more;
#   live       products computed before the body and summed in reverse order after it: the live set of the re-scheduled program,
#              that is its register-file tier (<= 8, <= 16, <= 32 registers in shared memory, <= 128 local, <= 1024 global);
#   cols       free (random) main columns, at least 1;  prep: preprocessed columns;  n_ops: instructions of the random body;
#   wide       unread filler columns between two blocks of `cols` free columns: wide >= 2^16 puts loaded columns above 2^16;
#   direct     one assert each on a leaf (a main column that is zero on every row), on the constant 0 and on a public value that is 0;
#   dup        one register asserted under two alpha indices;
#   max_deg    the highest degree of any value (1, 2 or 3);
#   max_word   the constant table also holds the canonical value 0x3FFF0001, whose Montgomery word is p - 1 (the largest word)
#   sat        False: a program no trace needs to satisfy (the host lowering checks): asserts name any register at any point of the
#              body, which later instructions may still read or overwrite, direct asserts land on loads that ops also read, there is
#              no sum over the constants and public values, the register file can be as small as one register, and n_asserts is
#              what the body asserts besides the live sum, the direct asserts and the duplicate.
Prog = collections.namedtuple("Prog", "seed n_asserts live cols prep n_ops wide direct dup max_deg sat max_word",
                              defaults=(8, 0, 6, 1, 40, 0, True, False, 3, True, False))
MAX_WORD_VALUE = 0x3FFF0001     # the canonical value whose Montgomery word is p - 1

# the public values of a machine with random-program chips: every program loads each of them; index 4 is 0 (the public assert)
PROG_PV_CANONICAL = [PV0, 5, 6, 7, 0, O.P - 1, 1, 987654321]
PROG_PV = O.to_monty(np.array(PROG_PV_CANONICAL))
OPCODE_NAMES = ["LOAD_LEAF", "LOAD_CONST", "LOAD_PUBLIC", "ADD", "SUB", "MUL", "NEG"]   # synth_air's opcodes 0 .. 6


def prog_chip(h, seed, **knobs):
    """a Chip of height h whose constraints are random_program(Prog(seed, **knobs))"""
    return Chip(h, 0, False, program=Prog(seed, **knobs))


class RandomProgram(collections.namedtuple("RandomProgram", "words main_w prep_w instrs leaves consts publics asserts witness zero_col features")):
    """A random non-SSA constraint program in the machine-blob layout (words, from synth_air.Asm) and what its trace generator needs:
    instrs (opcode, out, a, b), leaves (source, column), consts (canonical), publics (indices into the public values), asserts
    [(register, alpha index)], witness[k] = the main column that assert k subtracts (None for a direct assert), zero_col = the main
    column that is zero on every row (the direct leaf assert reads it), and the set of features the program exercises (opcode names,
    "assert_leaf", "assert_const", "assert_public", "alpha_permuted", "dup_assert", "cube", "alias", "overwrite", "dead_code",
    "high_column", and "degree_d" for the highest degree d of its constraints)."""

    def trace(self, rng, h, pv, kind=None):
        """a main and preprocessed trace of height h (Montgomery, [w, h]) that satisfies every constraint under the canonical public
        values pv: free and preprocessed columns of Montgomery words of the given kind (O.words; None: uniform values), the zero
        column, and each witness column filled with its asserted expression evaluated row by row mod p"""
        if kind is None:
            main = rng.integers(0, O.P, (self.main_w, h), dtype=np.uint64)
            prep = rng.integers(0, O.P, (self.prep_w, h), dtype=np.uint64)
        else:
            main = O.from_monty(O.words(rng, (self.main_w, h), kind)).astype(np.uint64)
            prep = O.from_monty(O.words(rng, (self.prep_w, h), kind)).astype(np.uint64)
        if self.asserts:                                      # the zero column and the witness columns close the main trace
            main[self.zero_col:] = 0
        regs = self._eval(main, prep, pv, h)
        for (r, _), w in zip(self.asserts, self.witness):
            if w is not None:
                main[w] = regs[r]
        regs = self._eval(main, prep, pv, h)
        assert all((regs[r] == 0).all() for r, _ in self.asserts), "random_program: the trace does not satisfy the program"
        return O.to_monty(main), (O.to_monty(prep) if self.prep_w else None)

    def _eval(self, main, prep, pv, h):
        """the program over all rows at once, exact integers mod p: -> the registers at the end"""
        P = np.uint64(O.P)
        regs = {}
        for opc, out, a, b in self.instrs:
            if opc == SA.LOAD_LEAF:
                src, col = self.leaves[a]
                v = (main if src == SA.LEAF_MAIN else prep)[col].copy()
            elif opc == SA.LOAD_CONST:
                v = np.full(h, self.consts[a], np.uint64)
            elif opc == SA.LOAD_PUBLIC:
                v = np.full(h, pv[self.publics[a]] % O.P, np.uint64)
            elif opc == SA.ADD:
                v = (regs[a] + regs[b]) % P
            elif opc == SA.SUB:
                v = (regs[a] + P - regs[b]) % P
            elif opc == SA.MUL:
                v = regs[a] * regs[b] % P
            else:
                v = (P - regs[a]) % P
            regs[out] = v
        return regs


@functools.lru_cache(maxsize=None)
def random_program(prog):
    """A random constraint program (RandomProgram) from the knobs `prog` (a Prog); with prog.sat, one that traces can satisfy.
    Registers are overwritten at will (also an operand by the result: x = x * y), operands alias (x * x), results go unused (dead
    code); loads cover main and preprocessed columns, every entry of a constant table holding 0, 1, p - 1 and random values, and every
    public value index; no value exceeds degree prog.max_deg.  With prog.sat each constraint is `e - w` for an expression e that reads
    no witness column and a witness column w of its own (the trace fills w with e), or a direct assert on a zero leaf, the constant 0 or
    a zero public value.  The constraints take a random permutation of the alpha indices."""
    LOAD_LEAF, LOAD_CONST, LOAD_PUBLIC, ADD, SUB, MUL, NEG = SA.LOAD_LEAF, SA.LOAD_CONST, SA.LOAD_PUBLIC, SA.ADD, SA.SUB, SA.MUL, SA.NEG
    rng = np.random.default_rng(prog.seed)
    n_a, n_pv, sat = prog.n_asserts, len(PROG_PV_CANONICAL), prog.sat
    free = list(range(prog.cols)) + (list(range(prog.cols + prog.wide, 2 * prog.cols + prog.wide)) if prog.wide else [])
    zero_col = free[-1] + 1 if free else 0
    consts = [0, 1, O.P - 1] + ([MAX_WORD_VALUE] if prog.max_word else []) + [int(x) for x in rng.integers(2, O.P - 1, 3)]
    publics = [int(x) for x in rng.permutation(n_pv)] + [int(x) for x in rng.integers(0, n_pv, 2)]
    zero_pub = [j for j, i in enumerate(publics) if PROG_PV_CANONICAL[i] == 0]
    instrs, leaves, asserts, witness = [], [], [], []
    feats = set()
    # register states: "val" (readable), "taint" (depends on a witness column: never read, may be overwritten), "frozen" (asserted:
    # never written again), "held" (a long-lived product: readable, not written until it is consumed).  Without `sat` nothing is
    # tainted and asserted registers stay readable and writable.
    state = {}
    deg = {}
    assert_deg = [0]

    def new_reg():
        r = len(state)
        state[r] = "free"
        return r

    def out_reg(exclude=()):
        cand = [r for r, s in state.items() if s in ("free", "val", "taint") and r not in exclude]
        if len(cand) < (3 if sat else 1):
            return new_reg()
        return int(rng.choice(cand))

    def readable():
        return [r for r, s in state.items() if s in ("val", "held")]

    def emit(opc, out, a=0, b=0, d=0, s="val"):
        if state.get(out, "free") != "free":
            feats.add("overwrite")
        if opc >= ADD and (out in ((a,) if opc == NEG else (a, b)) or (opc != NEG and a == b)):
            feats.add("alias")
        instrs.append((opc, out, a, b))
        state[out], deg[out] = s, d
        feats.add(OPCODE_NAMES[opc])
        return out

    def leaf(out, src, col, s="val"):
        leaves.append((src, col))
        if col >= 1 << 16:
            feats.add("high_column")
        return emit(LOAD_LEAF, out, len(leaves) - 1, 0, 1, s)

    def rand_leaf(out):
        if prog.prep and rng.integers(0, 4) == 0:
            return leaf(out, SA.LEAF_PREP, int(rng.integers(0, prog.prep)))
        return leaf(out, SA.LEAF_MAIN, int(rng.choice(free)))

    def add_assert(r, w=None):
        asserts.append(r); witness.append(w)
        assert_deg[0] = max(assert_deg[0], deg[r])

    def random_step():
        k = int(rng.integers(0, 10))
        rd = readable()
        out = out_reg()
        if k == 0 or not rd:
            rand_leaf(out)
        elif k == 1:
            emit(LOAD_CONST, out, int(rng.integers(0, len(consts))))
        elif k == 2:
            emit(LOAD_PUBLIC, out, int(rng.integers(0, len(publics))))
        elif k == 3:
            x = int(rng.choice(rd))
            emit(NEG, out, x, 0, deg[x])
        elif k == 4:                                                        # x^3 as (x * x) * x, the second product in place
            x = int(rng.choice([r for r in rd if deg[r] <= 1] or rd))
            if deg[x] <= 1 and 3 * deg[x] <= prog.max_deg:
                out = out_reg(exclude=(x,))
                emit(MUL, out, x, x, 2 * deg[x])
                emit(MUL, out, out, x, 3 * deg[x])
                feats.add("cube")
            else:
                emit(ADD, out, x, x, deg[x])
        else:
            x, y = int(rng.choice(rd)), int(rng.choice(rd))
            opc = [ADD, SUB, MUL][int(rng.integers(0, 3))]
            if opc == MUL and deg[x] + deg[y] > prog.max_deg:
                opc = SUB
            emit(opc, out, x, y, deg[x] + deg[y] if opc == MUL else max(deg[x], deg[y]))

    def assert_expr(e):
        """assert e - w for a fresh witness column w; the result lands in e's own register, in w's or in another one"""
        if not sat:                                                         # e itself, which stays readable and writable
            return add_assert(e)
        w = zero_col + 1 + sum(x is not None for x in witness)
        t = out_reg(exclude=(e,))
        leaf(t, SA.LEAF_MAIN, w, s="taint")
        choice = int(rng.integers(0, 3))
        out = e if choice == 0 and state[e] == "val" else t if choice == 1 else out_reg(exclude=(e, t))
        emit(SUB, out, e, t, max(deg[e], 1), s="frozen")
        add_assert(out, w)

    def direct_assert(kind):
        """an assert on a leaf of the zero column, on the constant 0 or on a zero public value: a register of its own with `sat`,
        otherwise a register that the rest of the body may read or overwrite"""
        r = new_reg() if sat else out_reg()
        s = "frozen" if sat else "val"
        if kind == "leaf":
            leaf(r, SA.LEAF_MAIN, zero_col, s=s)
        elif kind == "const":
            emit(LOAD_CONST, r, 0, s=s)
        else:
            emit(LOAD_PUBLIC, r, zero_pub[int(rng.integers(0, len(zero_pub)))], s=s)
        feats.add("assert_" + kind)
        add_assert(r)

    if n_a:
        held = []
        for _ in range(prog.live):                                          # long-lived products
            r = new_reg()
            rand_leaf(r)
            x = int(rng.choice(readable()))
            if deg[x] + 1 > prog.max_deg:
                x = r if prog.max_deg >= 2 else emit(LOAD_CONST, new_reg(), int(rng.integers(0, len(consts))))
            emit(MUL, r, r, x, deg[r] + deg[x], s="held")
            held.append(r)
        n_direct = 3 if prog.direct else 0
        if sat:
            # a sum over every constant and public value entry: sum_j c_j * leaf_j + sum_j pv_j * leaf_j (degree 1)
            acc = new_reg()
            emit(LOAD_CONST, acc, int(rng.integers(0, len(consts))))
            for opc, n in ((LOAD_CONST, len(consts)), (LOAD_PUBLIC, len(publics))):
                for j in rng.permutation(n):
                    t = out_reg(exclude=(acc,))
                    emit(opc, t, int(j))
                    u = out_reg(exclude=(acc, t))
                    rand_leaf(u)
                    emit(MUL, t, t, u, 1)
                    emit([ADD, SUB][int(rng.integers(0, 2))], acc, acc, t, 1)
            n_body = n_a - n_direct - 1 - (1 if held else 0) - (1 if prog.dup else 0)
            assert n_body >= 0, "too few asserts for the program's parts"
            assert_expr(acc)
        else:
            n_body = n_a
        at = sorted(int(x) for x in rng.integers(0, prog.n_ops + 1, n_body))
        direct_at = [] if sat else sorted(int(x) for x in rng.integers(0, prog.n_ops + 1, n_direct))
        for step in range(prog.n_ops + 1):
            while direct_at and direct_at[0] == step:
                direct_at.pop(0)
                direct_assert(["leaf", "const", "public"][len(direct_at) % 3])
            while at and at[0] == step:
                at.pop(0)
                rd = [r for r in readable() if state[r] == "val"]
                if not rd:
                    rand_leaf(out_reg())
                    rd = [r for r in readable() if state[r] == "val"]
                assert_expr(int(rng.choice(rd)))
            if step < prog.n_ops:
                random_step()
        if held:                                                            # consume the products in reverse order
            s = held[-1]
            state[s] = "val"
            for r in reversed(held[:-1]):
                emit([ADD, SUB][int(rng.integers(0, 2))], s, s, r, max(deg[s], deg[r]))
                state[r] = "val"
            assert_expr(s)
        if prog.direct and sat:
            for kind in ("leaf", "const", "public"):
                direct_assert(kind)
        if prog.dup:
            k = int(rng.choice([i for i, w in enumerate(witness) if w is not None or not sat]))  # an `e - w`: a nudged w fails both
            asserts.append(asserts[k]); witness.append(witness[k])
            feats.add("dup_assert")
        feats.add(f"degree_{max(assert_deg[0], 1)}")
    # dead code: results overwritten or never read before the end, and not asserted
    live_regs, dead = set(asserts), 0
    for opc, out, a, b in reversed(instrs):
        if out not in live_regs:
            dead += 1
            continue
        live_regs.discard(out)
        if opc >= ADD:
            live_regs.add(a)
            if opc != NEG:
                live_regs.add(b)
    if dead:
        feats.add("dead_code")
    alphas = [int(x) for x in rng.permutation(len(asserts))]
    if alphas != sorted(alphas):
        feats.add("alpha_permuted")
    if not n_a:
        consts, publics = [], []
    n_witness = len({w for w in witness if w is not None})
    main_w = (zero_col + 1 + n_witness) if n_a else max(len(free), 1)
    a = SA.Asm()
    a.instrs, a.leaves, a.asserts, a.publics = instrs, leaves, asserts, publics
    a.consts = [int(x) for x in O.to_monty(np.array(consts, dtype=np.uint64))]
    a.nreg = max(len(state), 1)
    return RandomProgram(a.words(main_w, prog.prep, alphas), main_w, prog.prep, instrs, leaves, consts, publics,
                         list(zip(asserts, alphas)), witness, zero_col, frozenset(feats))


TIER_NAMES = ["shared <= 8", "shared <= 16", "shared <= 32", "local", "global"]


def zc_tier(regs):
    """the zerocheck kernels' register-file tier of a program with `regs` live registers (TIER_NAMES; sp1_b200/csrc/zerocheck.cu)"""
    return next((t for t, n in enumerate((8, 16, 32, 128)) if regs <= n), 4)


def lowered_shape(words):
    """a chip's program as zc_lower re-schedules it (the library's host code, libsp1b200_hostcheck.so) -> (register pressure of the
    whole stream, lowered instructions, whether sp1b200_machine_create also splits it into pieces: >= 8 asserts and >= 128 lowered
    instructions)"""
    import ctypes as C
    from tests import hostcheck_lib
    cw = np.ascontiguousarray(words, dtype=np.uint32)
    main_w, prep_w, n_c = (int(x) for x in cw[:3])
    rows = [np.zeros(max(n, 1), np.uint32) for n in (main_w, prep_w, 64, 4 * max(n_c, 1), 12)]
    nl = C.c_uint32(0)
    regs = hostcheck_lib.load().sp1b200_hostcheck_zc_lower(*(O.ptr(a) for a in [cw] + rows[:4]), C.c_uint32(24), O.ptr(rows[4]),
                                                           C.byref(nl))
    assert regs > 0, "zc_lower rejected the program"
    return regs, nl.value, int(cw[8]) >= 8 and nl.value >= 128


def traces(specs, seed, pv0=PV0, kind=None):
    """numpy traces of chips with fields h, g, wp, extra, extra_prep (Chip, or the specs of sp1_b200.workload.synthetic_machine)
    drawn from `seed` (an int or a numpy Generator, which is drawn from in place) -> (mains, preps).  A multi-shard test calls this
    with the same seed for every shard, so that the preprocessed tables agree, and each shard's own public value 0.  A random-program
    chip's trace satisfies its program under PROG_PV with public value 0 replaced by pv0.  kind: the word kind of the free columns
    (O.words); None keeps the uniform draws, so that a seed gives the same traces as before the argument existed."""
    rng = np.random.default_rng(seed)
    mains, preps = [], []
    for c in specs:
        if getattr(c, "program", None) is not None:
            m, p = random_program(c.program).trace(rng, c.h, [pv0] + PROG_PV_CANONICAL[1:], kind=kind)
        else:
            m, p = SA.synth_trace(rng, c.h, c.g, c.wp, pv0, extra_cols=c.extra, extra_prep=c.extra_prep)
            if kind is not None:
                m, p = refill_template_trace(rng, m, p, c.g, c.wp, pv0, kind)
        mains.append(m); preps.append(p)
    return mains, preps


def refill_template_trace(rng, main, prep, groups, with_prep, pv0, kind, kconst=7):
    """a synth_air.synth_trace trace (main [6 groups + with_prep + extra, h], prep [1 + extra_prep, h] or None) with its free columns
    redrawn as words of the given kind (O.words): per group a and b, the filler columns, and the preprocessed columns; then the
    constrained columns recomputed mod p from them: c = a b, e = c d, f = a + kconst pv0, and the product g a_0 of the first
    preprocessed column with group 0's a.  The boolean column d is kept."""
    h = main.shape[1]
    if not h:
        return main, prep
    cols = O.from_monty(main).astype(np.uint64)
    P = np.uint64(O.P)
    free = [6 * g + k for g in range(groups) for k in (0, 1)] + list(range(6 * groups + (1 if with_prep else 0), main.shape[0]))
    cols[free] = O.from_monty(O.words(rng, (len(free), h), kind))
    for g in range(groups):
        a, b, d = cols[6 * g], cols[6 * g + 1], cols[6 * g + 3]
        cols[6 * g + 2] = a * b % P
        cols[6 * g + 4] = cols[6 * g + 2] * d % P
        cols[6 * g + 5] = (a + np.uint64(kconst * pv0 % O.P)) % P
    if with_prep:
        prep = O.words(rng, prep.shape, kind)
        cols[6 * groups] = O.from_monty(prep[0]).astype(np.uint64) * cols[0] % P
    return O.to_monty(cols), prep


def workload_machine(workload, seed, max_log_rows=22, scale=1.0, machine_seed=42):
    """the benchmark machine of `workload` (sp1_b200.workload.synthetic_machine: heights from `machine_seed`, scaled by `scale`) with
    numpy traces drawn from `seed`"""
    from sp1_b200 import workload as W
    mach = W.synthetic_machine(workload, seed=machine_seed, max_log_rows=max_log_rows, scale=scale)
    mains, preps = traces(mach["specs"], seed)
    return mach["blob"], [sp.h for sp in mach["specs"]], mains, preps, PV.copy(), list(mach["names"])


def spec_machine(rng, chips, interactions=True, names="Chip{:03d}", kind=None):
    """chips: list of Chip (or plain tuples in Chip's field order).  interactions=False builds the blob without an interaction
    section (synth_air.machine_blob).  names: the chip-name format; the names are observed into the transcript.  The public values are
    PV, or PROG_PV when a chip has a random program.  kind: the word kind of the traces' free columns (traces)."""
    chips = [Chip(*c) for c in chips]
    words, iwords = [], []
    for c in chips:
        if c.program is not None:
            words.append(random_program(c.program).words)
            iwords.append([0])
            continue
        words.append(SA.synth_chip(c.g, c.wp, deep=c.deep, n_constraints=c.n_constraints, extra_cols=c.extra, extra_prep=c.extra_prep)[0])
        if c.vps is None:
            iwords.append(SA.synth_interactions(c.g, c.wp))
        elif len(c.vps) == 0:
            iwords.append([0])
        else:
            iwords.append(SA.synth_interactions_calibrated(c.g, c.wp, list(c.vps)))
    mains, preps = traces(chips, rng, kind=kind)
    blob = SA.machine_blob_with_interactions(words, iwords) if interactions else SA.machine_blob(words)
    pv = PROG_PV if any(c.program is not None for c in chips) else PV
    return blob, [c.h for c in chips], mains, preps, pv.copy(), [names.format(i) for i in range(len(chips))]


def shard_inputs(spec, seed, kind=None):
    """the seeded whole-shard inputs of the golden fixtures and the shard tests: spec_machine with names Chip00, Chip01, ... (traces of
    the word kind `kind`), then a challenger that has observed 9 random words from the same generator -> (blob, heights, mains, preps,
    pv, names, challenger)"""
    rng = np.random.default_rng(seed)
    inp = spec_machine(rng, spec, names="Chip{:02d}", kind=kind)
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

# zerocheck machines of random-program chips (spec, max_log_row_count): every register-file tier (live 0 / 10 / 24 / 80 / 300), the
# pieces path (16 asserts, >= 128 lowered instructions), chips without constraints between constrained ones, chips of degree 1 and 2,
# heights 0, 1, 2, 3, odd, 2^k, 2^k + 1 and 2^max_log_row_count, max_log_row_count 1 to 13, and a chip of more than 2^16 main columns
PROGRAM_ZC_CASES = [
    ([prog_chip(64, 11), prog_chip(0, 12), prog_chip(48, 13, live=10), prog_chip(16, 14, n_asserts=0), prog_chip(33, 15, live=24, dup=True),
      prog_chip(100, 16, live=80, n_asserts=12), prog_chip(17, 17, live=300, n_asserts=12), prog_chip(128, 18, n_asserts=16, n_ops=150),
      Chip(32, 1, True)], 7),
    ([prog_chip(1, 21), prog_chip(2, 22, dup=True), prog_chip(3, 23), prog_chip(4, 24, n_asserts=0), prog_chip(4, 25, n_asserts=16, n_ops=150),
      prog_chip(3, 26, max_deg=1), prog_chip(4, 27, max_deg=2)], 2),
    ([prog_chip(1, 31), prog_chip(0, 32), prog_chip(2, 33, dup=True)], 1),
    ([prog_chip(8192, 41, live=24, prep=3), prog_chip(4097, 42, n_asserts=16, n_ops=150), prog_chip(1500, 43, live=300, n_asserts=10),
      Chip(4096, 2, True)], 13),
    ([prog_chip(4, 51, wide=65600, n_asserts=6, n_ops=20), prog_chip(5, 52)], 3),
]

# a whole shard of random-program chips (one without constraints, one absent) next to template chips with and without interactions
RANDOM_SHARD_SPEC = ([prog_chip(64, 61, prep=2), Chip(32, 1, True), prog_chip(0, 62), prog_chip(17, 63, live=10, dup=True),
                      prog_chip(8, 64, n_asserts=0), Chip(16, 2, False, vps=()), prog_chip(40, 65, n_asserts=16, n_ops=150)], 5, 7)

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
