"""NumPy restatement of the core machine's three preprocessed trace generators, line by line from the Rust (crates/core/machine/src),
as canonical integers: the reference the device tables of sp1b200_program_preprocessed_traces are checked against.  It shares no code with
the CUDA.  Each table is returned row-major [rows, cols] as the Rust fills it; dense() lays the three out as the library does (chip-name
order Byte, Program, Range; each column-major; Montgomery words)."""
import numpy as np

P = 0x7F000001

BYTE_NUM_ROWS = 1 << 16    # bytes/trace.rs:15
RANGE_NUM_ROWS = 1 << 17   # range/trace.rs:15
NUM_BYTE_PREPROCESSED_COLS = 7      # bytes/columns.rs BytePreprocessedCols {b, c, and, or, xor, ltu, msb}
NUM_RANGE_PREPROCESSED_COLS = 2     # range/columns.rs RangePreprocessedCols {a, bits}
NUM_PROGRAM_PREPROCESSED_COLS = 16  # program/trusted.rs ProgramPreprocessedCols {pc[3], InstructionCols (program/instruction.rs)}
X0 = 0                     # Register::X0


def byte_trace():
    """ByteChip::trace (bytes/mod.rs:31-80)"""
    values = np.zeros((BYTE_NUM_ROWS, NUM_BYTE_PREPROCESSED_COLS), np.int64)
    # bytes/mod.rs:41: for (row_index, (b, c)) in (0..=u8::MAX).cartesian_product(0..=u8::MAX).enumerate()
    b, c = np.divmod(np.arange(BYTE_NUM_ROWS, dtype=np.int64), 256)
    values[:, 0] = b                      # col.b
    values[:, 1] = c                      # col.c
    # opcodes of ByteOpcode::byte_table() (executor/src/events/byte.rs:166-176): AND, OR, XOR, U8Range, LTU, MSB
    values[:, 2] = b & c                  # ByteOpcode::AND -> col.and
    values[:, 3] = b | c                  # ByteOpcode::OR -> col.or
    values[:, 4] = b ^ c                  # ByteOpcode::XOR -> col.xor
    # ByteOpcode::U8Range => {}
    values[:, 5] = b < c                  # ByteOpcode::LTU -> col.ltu = F::from_bool(b < c)
    values[:, 6] = (b & 0b1000_0000) != 0   # ByteOpcode::MSB -> col.msb
    return values


def range_trace():
    """RangeChip::trace (range/mod.rs:18-39)"""
    values = np.zeros((RANGE_NUM_ROWS, NUM_RANGE_PREPROCESSED_COLS), np.int64)
    values[0] = (0, 0)                    # range/mod.rs:24-27: the first row is (0, 0)
    for bits in range(0, 17):             # range/mod.rs:30: for bits in 0..=16
        a = np.arange(1 << bits, dtype=np.int64)
        row_index = (1 << bits) + a       # range/mod.rs:32
        values[row_index, 0] = a          # col.a
        values[row_index, 1] = bits       # col.bits
    return values


def next_multiple_of_32(n, fixed_height=None):
    """hypercube/src/util.rs:50-59"""
    if fixed_height is not None:
        assert n <= fixed_height, "fixed height is too small"
        return fixed_height
    return max(-(-n // 32) * 32, 16)


def _word_from_u64(v):
    """Word::from(u64) (hypercube/src/word.rs:167-176): four 16-bit limbs, low first"""
    v = np.asarray(v, np.uint64)
    return [((v >> np.uint64(s)) & np.uint64(0xFFFF)).astype(np.int64) for s in (0, 16, 32, 48)]


def program_trace(pc_base, instrs):
    """ProgramChip::generate_preprocessed_trace_into (program/trusted.rs:80-127) with preprocessed_shape None.  instrs: a structured array
    with fields opcode, op_a, op_b, op_c, imm_b, imm_c (sp1_b200.lib.INSTRUCTION_DTYPE)"""
    nb_rows = len(instrs)                                    # trusted.rs:90
    assert nb_rows > 0, "empty program"                      # trusted.rs:85-88
    padded_nb_rows = next_multiple_of_32(nb_rows, None)      # trusted.rs:91-92
    assert padded_nb_rows * 4 < P                            # trusted.rs:93-96
    values = np.zeros((padded_nb_rows, NUM_PROGRAM_PREPROCESSED_COLS), np.int64)
    idx = np.arange(padded_nb_rows, dtype=np.int64)          # trusted.rs:112: i * chunk_size + j
    idx[idx >= nb_rows] = 0                                  # trusted.rs:113-115: padding rows repeat instruction 0
    pc = np.uint64(pc_base) + idx.astype(np.uint64) * np.uint64(4)   # trusted.rs:117
    assert (pc < np.uint64(1 << 48)).all()                   # trusted.rs:118
    values[:, 0] = (pc & np.uint64(0xFFFF)).astype(np.int64)                     # trusted.rs:119-123
    values[:, 1] = ((pc >> np.uint64(16)) & np.uint64(0xFFFF)).astype(np.int64)
    values[:, 2] = ((pc >> np.uint64(32)) & np.uint64(0xFFFF)).astype(np.int64)
    ins = instrs[idx]                                        # trusted.rs:124
    # InstructionCols::populate (program/instruction.rs:36-45)
    values[:, 3] = ins["opcode"]                             # opcode.as_field(): the #[repr(u8)] discriminant
    values[:, 4] = ins["op_a"]
    values[:, 5:9] = np.stack(_word_from_u64(ins["op_b"]), axis=1)
    values[:, 9:13] = np.stack(_word_from_u64(ins["op_c"]), axis=1)
    values[:, 13] = ins["op_a"] == X0                        # op_a_0
    values[:, 14] = ins["imm_b"].astype(bool)                # F::from_bool(imm_b)
    values[:, 15] = ins["imm_c"].astype(bool)
    return values


def to_monty(x):
    x = np.asarray(x, dtype=np.uint64) % np.uint64(P)
    return ((x << np.uint64(32)) % np.uint64(P)).astype(np.uint32)


def tables(pc_base, instrs):
    """-> [(name, row-major canonical table)] in chip-name order"""
    return [("Byte", byte_trace()), ("Program", program_trace(pc_base, instrs)), ("Range", range_trace())]


def dense(pc_base, instrs):
    """-> (dense Montgomery words: the tables back to back, each column-major, shapes [(rows, cols)])"""
    ts = [t for _, t in tables(pc_base, instrs)]
    return np.concatenate([to_monty(t.T.reshape(-1)) for t in ts]), [t.shape for t in ts]
