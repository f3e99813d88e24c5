"""NumPy restatement of the main (multiplicity) trace generators of the core machine's Byte, Range and Program chips and of the Byte and
Range chips' public-value dependencies, from the Rust (crates/core/machine/src), as canonical integers: the reference the device tables
of sp1b200_lookup_traces are checked against.  It shares no code with the CUDA.  Each table is returned row-major [rows, cols] as the Rust
fills it; main_words() gives the library's layout (each table column-major, Montgomery words)."""
import numpy as np

P = 0x7F000001
BYTE_NUM_ROWS = 1 << 16    # bytes/trace.rs:15
RANGE_NUM_ROWS = 1 << 17   # range/trace.rs:15
NUM_BYTE_OPS = 6           # executor/src/events/byte.rs:11, the width of ByteMultCols
AND, OR, XOR, U8RANGE, LTU, MSB, RANGE = range(7)   # ByteOpcode (executor/src/opcode.rs:163-178)

# PublicValues<[F; 4], [F; 3], [F; 4], F> word offsets (crates/hypercube/src/air/public_values.rs, without mprotect)
PREV_COMMITTED_VALUE_DIGEST, COMMITTED_VALUE_DIGEST = 0, 32
PC_START, NEXT_PC = 80, 83
PREVIOUS_INIT_ADDR, LAST_INIT_ADDR, PREVIOUS_FINALIZE_ADDR, LAST_FINALIZE_ADDR = 89, 92, 95, 98
INITIAL_TIMESTAMP, LAST_TIMESTAMP = 113, 117
PV_DIGEST_NUM_WORDS = 8


def _histogram(keys, counts, size):
    """exact integer sum of counts per key (np.bincount sums in float64: split each count into 16-bit halves so no sum passes 2^53)"""
    keys = np.asarray(keys, np.int64)
    counts = np.asarray(counts, np.uint64)
    lo = np.bincount(keys, weights=(counts & np.uint64(0xFFFF)).astype(np.float64), minlength=size)
    hi = np.bincount(keys, weights=(counts >> np.uint64(16)).astype(np.float64), minlength=size)
    return hi.astype(np.uint64) * np.uint64(1 << 16) + lo.astype(np.uint64)


def byte_trace(lookups):
    """ByteChip::generate_trace_into (bytes/trace.rs:68-92) over (lookup, mult) records: row (b << 8) + c, column opcode; Range skipped"""
    op = lookups["opcode"].astype(np.int64)
    assert (op <= RANGE).all(), "invalid ByteOpcode"
    keep = op != RANGE                                        # if lookup.opcode == ByteOpcode::Range { continue; }
    row = (lookups["b"].astype(np.int64) << 8) + lookups["c"].astype(np.int64)
    index = op                                                # lookup.opcode as usize
    flat = _histogram((row * NUM_BYTE_OPS + index)[keep], lookups["count"][keep], BYTE_NUM_ROWS * NUM_BYTE_OPS)
    return flat.reshape(BYTE_NUM_ROWS, NUM_BYTE_OPS)          # values[row * NUM_BYTE_MULT_COLS + index]


def range_trace(lookups):
    """RangeChip::generate_trace_into (range/trace.rs:98-121): row a + (1 << b) for Range records"""
    keep = lookups["opcode"] == RANGE                         # if lookup.opcode != ByteOpcode::Range { continue; }
    b = lookups["b"].astype(np.int64)[keep]
    assert (b <= 16).all(), "Range records check at most 16 bits"
    row = lookups["a"].astype(np.int64)[keep] + (np.int64(1) << b)
    return _histogram(row, lookups["count"][keep], RANGE_NUM_ROWS).reshape(RANGE_NUM_ROWS, 1)


def next_multiple_of_32(n):
    """hypercube/src/util.rs:50-59 with no fixed height"""
    return max(-(-n // 32) * 32, 16)


def program_trace(pc_base, n_instrs, pcs):
    """ProgramChip::generate_trace_into (program/trusted.rs:134-292): instruction_counts[pc] summed over the events; row idx < nb_instructions
    reads instruction_counts.get(pc_base + 4 idx), padding rows are zero"""
    padded_nb_rows = next_multiple_of_32(n_instrs)
    pc = pcs["pc"].astype(np.uint64)
    off = pc - np.uint64(pc_base)                             # wraps for pc < pc_base: such a pc is no row's
    idx = off >> np.uint64(2)
    keep = (pc >= np.uint64(pc_base)) & ((off & np.uint64(3)) == 0) & (idx < np.uint64(n_instrs))
    values = _histogram(idx[keep].astype(np.int64), pcs["count"][keep], padded_nb_rows)
    return values.reshape(padded_nb_rows, 1)


def _timestamp_from_limbs(limbs):
    """public_values.rs:383-389"""
    return (limbs[0] << 32) + (limbs[1] << 24) + (limbs[2] << 16) + limbs[3]


def _addr(limbs):
    """previous_init_addr() and friends: the limbs folded from the top, 16 bits each"""
    acc = 0
    for x in reversed(limbs):
        acc = acc * (1 << 16) + x
    return acc


def _u8_range_checks(bytes_):
    """ByteRecord::add_u8_range_checks (events/byte.rs): pairs, an odd last byte paired with 0"""
    out = []
    i = 0
    while i + 1 < len(bytes_):
        out.append((U8RANGE, 0, bytes_[i], bytes_[i + 1]))
        i += 2
    if i < len(bytes_):
        out.append((U8RANGE, 0, bytes_[i], 0))
    return out


def byte_dependencies(pv):
    """ByteChip::generate_dependencies (bytes/trace.rs:50-66) -> [(opcode, a, b, c)]; pv: the canonical field words of the public values"""
    pv = [int(x) for x in pv]
    initial = _timestamp_from_limbs(pv[INITIAL_TIMESTAMP:INITIAL_TIMESTAMP + 4])
    last = _timestamp_from_limbs(pv[LAST_TIMESTAMP:LAST_TIMESTAMP + 4])
    out = [(U8RANGE, 0, (initial >> 24) & 0xFF, (initial >> 16) & 0xFF), (U8RANGE, 0, (last >> 24) & 0xFF, (last >> 16) & 0xFF)]
    for i in range(PV_DIGEST_NUM_WORDS):
        # the u32 word of the u64-form record is the little-endian join of the four byte words of the field form
        for base in (PREV_COMMITTED_VALUE_DIGEST, COMMITTED_VALUE_DIGEST):
            word = sum(pv[base + 4 * i + k] << (8 * k) for k in range(4))
            out += _u8_range_checks(list(word.to_bytes(4, "little")))
    return out


def range_dependencies(pv):
    """RangeChip::generate_dependencies (range/trace.rs:54-96, without mprotect) -> [(opcode, a, b, c)]"""
    pv = [int(x) for x in pv]
    out = []
    for at in (INITIAL_TIMESTAMP, LAST_TIMESTAMP):
        ts = _timestamp_from_limbs(pv[at:at + 4])
        ts_0 = (ts >> 32) & 0xFFFF
        ts_3 = ts & 0xFFFF
        out.append((RANGE, ts_0, 16, 0))
        out.append((RANGE, ((ts_3 - 1) & 0xFFFF) // 8, 13, 0))   # u16 subtraction, wrapping as in the release build
    for at in (PC_START, NEXT_PC, PREVIOUS_INIT_ADDR, LAST_INIT_ADDR, PREVIOUS_FINALIZE_ADDR, LAST_FINALIZE_ADDR):
        addr = _addr(pv[at:at + 3])
        for s in (0, 16, 32):
            out.append((RANGE, (addr >> s) & 0xFFFF, 16, 0))
    return out


def dependency_records(pv):
    """both chips' dependencies as count-1 records of sp1_b200.lib.BYTE_LOOKUP_DTYPE"""
    from sp1_b200.lib import pack_byte_lookups
    ev = np.array(byte_dependencies(pv) + range_dependencies(pv), np.int64)
    return pack_byte_lookups(ev[:, 0], ev[:, 1], ev[:, 2], ev[:, 3], 1)


def to_monty(x):
    x = np.asarray(x, dtype=np.uint64)
    assert (x < np.uint64(P)).all(), "multiplicity >= p (F::from_canonical_usize)"
    return ((x << np.uint64(32)) % np.uint64(P)).astype(np.uint32)


def tables(pc_base, n_instrs, lookups, pcs, pv=None):
    """-> {name: row-major canonical table} for Byte, Program, Range; pv (canonical) adds the dependencies"""
    if pv is not None:
        lookups = np.concatenate([lookups, dependency_records(pv)])
    return dict(Byte=byte_trace(lookups), Program=program_trace(pc_base, n_instrs, pcs), Range=range_trace(lookups))


def main_words(pc_base, n_instrs, lookups, pcs, pv=None):
    """-> (byte [6, 2^16], program [1, h], range [1, 2^17]): each column-major as [cols, rows] Montgomery words"""
    t = tables(pc_base, n_instrs, lookups, pcs, pv)
    return tuple(to_monty(t[name].T) for name in ("Byte", "Program", "Range"))
