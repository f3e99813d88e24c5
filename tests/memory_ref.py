"""NumPy restatement of the core machine's memory chips MemoryGlobalInit / MemoryGlobalFinalize (crates/core/machine/src/memory/global.rs)
and MemoryLocal (memory/local.rs): their generate_trace_into and generate_dependencies, read line by line from the Rust, as canonical
integers.  It is the reference the device output of sp1b200_memory_traces is checked against and shares no code with the CUDA.

Traces come back row-major [rows, cols] as the Rust fills them; main_words() gives the library's layout (column-major Montgomery
words).  Byte lookups come back as the Rust emits them, (opcode, a, b, c) per event; global events as (message [n, 8], is_receive [n],
kind [n])."""
import numpy as np

P = 0x7F000001
U8RANGE, RANGE = 3, 6                  # ByteOpcode (executor/src/opcode.rs:163-178)
KIND_MEMORY = 1                        # InteractionKind::Memory (hypercube/src/lookup/interaction.rs)

# MemoryInitCols (global.rs:254-304) with LtOperationUnsigned (operations/slt.rs:29-38), U16CompareOperation (u16_compare.rs:27-30) and
# IsZeroOperation (is_zero.rs:31-37) inlined in field order
INIT_COLS = (["clk_high", "clk_low", "index"] + [f"prev_addr[{k}]" for k in range(3)] + [f"addr[{k}]" for k in range(3)]
             + ["lt.bit"] + [f"lt.u16_flags[{k}]" for k in range(4)] + ["lt.not_eq_inv", "lt.comparison_limbs[0]", "lt.comparison_limbs[1]"]
             + [f"value[{k}]" for k in range(4)] + ["value_lower", "value_upper", "is_real", "is_comp", "prev_valid",
                                                      "is_prev_addr_zero.inverse", "is_prev_addr_zero.result",
                                                      "is_index_zero.inverse", "is_index_zero.result"])
# SingleMemoryLocal (local.rs:27-65), NUM_LOCAL_MEMORY_ENTRIES_PER_ROW = 1
LOCAL_COLS = ([f"addr[{k}]" for k in range(3)] + ["initial_clk_high", "final_clk_high", "initial_clk_low", "final_clk_low"]
              + [f"initial_value[{k}]" for k in range(4)] + [f"final_value[{k}]" for k in range(4)]
              + ["initial_value_lower", "initial_value_upper", "final_value_lower", "final_value_upper", "is_real"])
NUM_MEMORY_INIT_COLS = len(INIT_COLS)          # 30
NUM_MEMORY_LOCAL_INIT_COLS = len(LOCAL_COLS)   # 20
IC = {name: k for k, name in enumerate(INIT_COLS)}
LC = {name: k for k, name in enumerate(LOCAL_COLS)}


def next_multiple_of_32(n):
    """hypercube/src/util.rs:50-59 with no fixed height"""
    return max(-(-n // 32) * 32, 16)


def num_rows(n):
    """the chip's height in a shard: not included without events (global.rs:238-247, local.rs:240-246), else next_multiple_of_32"""
    return next_multiple_of_32(n) if n else 0


def inverse(x):
    """F::inverse of non-zero canonical elements, x^(p-2) mod p"""
    x = np.asarray(x, np.uint64) % np.uint64(P)
    r = np.ones_like(x)
    e = P - 2
    while e:
        if e & 1:
            r = r * x % np.uint64(P)
        x = x * x % np.uint64(P)
        e >>= 1
    return r


def is_zero_populate(a):
    """IsZeroOperation::populate_from_field_element (is_zero.rs:44-55) -> (inverse, result)"""
    a = np.asarray(a, np.uint64) % np.uint64(P)
    z = a == 0
    inv = np.where(z, np.uint64(0), inverse(np.where(z, np.uint64(1), a)))
    return inv, z.astype(np.uint64)


def u64_to_u16_limbs(x):
    """sp1_primitives::consts::u64_to_u16_limbs: [4, n] low limb first"""
    x = np.asarray(x, np.uint64)
    return np.stack([(x >> np.uint64(16 * k)) & np.uint64(0xFFFF) for k in range(4)])


def _sorted(events):
    """memory_events.sort_by_key(|event| event.addr) (a stable sort)"""
    return events[np.argsort(events["addr"], kind="stable")]


def _prev_addrs(ev, previous_addr):
    """prev_addr = if i == 0 { previous_addr } else { memory_events[i - 1].addr }"""
    return np.concatenate([np.array([previous_addr], np.uint64), ev["addr"][:-1]]).astype(np.uint64)


def populate_unsigned(b, c):
    """LtOperationUnsigned::populate_unsigned(_, 1, b, c) (slt.rs:155-194) over arrays -> (bit, u16_flags [4, n], not_eq_inv,
    comparison_limbs [2, n], the Range lookup's a = b_limb.wrapping_sub(c_limb))"""
    n = len(b)
    b_limbs, c_limbs = u64_to_u16_limbs(b), u64_to_u16_limbs(c)
    flags = np.zeros((4, n), np.uint64)
    comp = np.zeros((2, n), np.uint64)
    not_eq_inv = np.zeros(n, np.uint64)
    done = np.zeros(n, bool)
    for k in (3, 2, 1, 0):                       # izip!(b_limbs.iter().rev(), c_limbs.iter().rev(), self.u16_flags.iter_mut().rev())
        hit = ~done & (b_limbs[k] != c_limbs[k])
        flags[k] = np.where(hit, 1, flags[k])
        comp[0] = np.where(hit, b_limbs[k], comp[0])
        comp[1] = np.where(hit, c_limbs[k], comp[1])
        diff = (b_limbs[k] + np.uint64(P) - c_limbs[k]) % np.uint64(P)      # b_limb - c_limb in F
        not_eq_inv = np.where(hit, inverse(np.where(hit, diff, np.uint64(1))), not_eq_inv)
        done |= hit
    bit = np.ones(n, np.uint64)                  # U16CompareOperation::populate: bit = a_u16 = 1
    range_a = (comp[0] - comp[1]) & np.uint64(0xFFFF)   # comparison_limbs[0].wrapping_sub(comparison_limbs[1])
    return bit, flags, not_eq_inv, comp, range_a


def global_trace(events, previous_addr):
    """MemoryGlobalChip::generate_trace_into (global.rs:155-236) -> [num_rows(n), 30] canonical"""
    ev = _sorted(events)
    n = len(ev)
    t = np.zeros((num_rows(n), NUM_MEMORY_INIT_COLS), np.uint32)   # canonical elements < p < 2^32
    if n == 0:
        return t
    addr, value, ts = ev["addr"], ev["value"], ev["timestamp"]
    a = u64_to_u16_limbs(addr)
    for k in range(3):
        t[:n, IC[f"addr[{k}]"]] = a[k]
    t[:n, IC["clk_high"]] = ts >> np.uint64(24)
    t[:n, IC["clk_low"]] = ts & np.uint64(0xFFFFFF)
    v = u64_to_u16_limbs(value)                  # Word::from(value)
    for k in range(4):
        t[:n, IC[f"value[{k}]"]] = v[k]
    t[:n, IC["is_real"]] = 1
    t[:n, IC["value_lower"]] = (value >> np.uint64(32)) & np.uint64(0xFF)
    t[:n, IC["value_upper"]] = (value >> np.uint64(40)) & np.uint64(0xFF)
    i = np.arange(n, dtype=np.uint64)
    prev = _prev_addrs(ev, previous_addr)
    t[:n, IC["prev_valid"]] = np.where((prev == 0) & (i != 0), 0, 1)
    t[:n, IC["index"]] = i
    p = u64_to_u16_limbs(prev)
    for k in range(3):
        t[:n, IC[f"prev_addr[{k}]"]] = p[k]
    inv, res = is_zero_populate(p[0] + p[1] + p[2])
    t[:n, IC["is_prev_addr_zero.inverse"]], t[:n, IC["is_prev_addr_zero.result"]] = inv, res
    inv, res = is_zero_populate(i)
    t[:n, IC["is_index_zero.inverse"]], t[:n, IC["is_index_zero.result"]] = inv, res
    comp = (prev != 0) | (i != 0)
    bit, flags, not_eq_inv, limbs, _ = populate_unsigned(prev, addr)
    t[:n, IC["is_comp"]] = comp
    t[:n, IC["lt.bit"]] = np.where(comp, bit, 0)            # else: LtOperationUnsigned::default()
    for k in range(4):
        t[:n, IC[f"lt.u16_flags[{k}]"]] = np.where(comp, flags[k], 0)
    t[:n, IC["lt.not_eq_inv"]] = np.where(comp, not_eq_inv, 0)
    for k in range(2):
        t[:n, IC[f"lt.comparison_limbs[{k}]"]] = np.where(comp, limbs[k], 0)
    return t


def global_dependencies(events, previous_addr, is_receive):
    """MemoryGlobalChip::generate_dependencies (global.rs:63-142) -> (byte lookups [(opcode, a, b, c)] in emission order, message [n, 8],
    is_receive [n], kind [n]); is_receive: False for Initialize, True for Finalize"""
    ev = _sorted(events)
    n = len(ev)
    lookups = []
    if n:
        addr, value = ev["addr"], ev["value"]
        prev = _prev_addrs(ev, previous_addr)
        v, p, a = u64_to_u16_limbs(value), u64_to_u16_limbs(prev), u64_to_u16_limbs(addr)
        lower = (value >> np.uint64(32)) & np.uint64(0xFF)
        upper = (value >> np.uint64(40)) & np.uint64(0xFF)
        i = np.arange(n, dtype=np.uint64)
        _, _, _, _, range_a = populate_unsigned(prev, addr)
        comp = (i != 0) | (prev != 0)
        cols = ([(RANGE, v[k], 16, 0) for k in range(4)] + [(RANGE, p[k], 16, 0) for k in range(3)]
                + [(RANGE, a[k], 16, 0) for k in range(3)] + [(U8RANGE, 0, lower, upper), (RANGE, range_a, 16, 0)])
        rows = np.zeros((n, len(cols), 4), np.int32)
        for j, fields in enumerate(cols):
            for f, x in enumerate(fields):
                rows[:, j, f] = np.asarray(x, np.int64)
        keep = np.ones((n, len(cols)), bool)
        keep[:, -1] = comp                       # populate_unsigned only when i != 0 || prev_addr != 0
        lookups = rows[keep]
    lookups = np.asarray(lookups, np.int32).reshape(-1, 4)
    return (lookups,) + global_interaction_events(ev, is_receive)


def global_interaction_events(events, is_receive):
    """the GlobalInteractionEvents of MemoryGlobalChip::generate_dependencies (global.rs:117-141), in address order -> (message [n, 8],
    is_receive [n], kind [n])"""
    ev = _sorted(events)
    n = len(ev)
    msg = np.zeros((n, 8), np.uint64)
    if n:
        ts, value, addr = ev["timestamp"], ev["value"], ev["addr"]
        if is_receive:
            msg[:, 0] = ts >> np.uint64(24)
            msg[:, 1] = ts & np.uint64(0xFFFFFF)
        for k in range(3):
            msg[:, 2 + k] = (addr >> np.uint64(16 * k)) & np.uint64(0xFFFF)
        msg[:, 5] = (value & np.uint64(0xFFFF)) + np.uint64(1 << 16) * ((value >> np.uint64(32)) & np.uint64(0xFF))
        msg[:, 6] = ((value >> np.uint64(16)) & np.uint64(0xFFFF)) + np.uint64(1 << 16) * ((value >> np.uint64(40)) & np.uint64(0xFF))
        msg[:, 7] = (value >> np.uint64(48)) & np.uint64(0xFFFF)
    return msg, np.full(n, int(is_receive), np.uint8), np.full(n, KIND_MEMORY, np.uint8)


def local_trace(events):
    """MemoryLocalChip::generate_trace_into (local.rs:166-238) -> [num_rows(n), 20] canonical"""
    n = len(events)
    t = np.zeros((num_rows(n), NUM_MEMORY_LOCAL_INIT_COLS), np.uint32)
    if n == 0:
        return t
    a = u64_to_u16_limbs(events["addr"])
    for k in range(3):
        t[:n, LC[f"addr[{k}]"]] = a[k]
    it, ft = events["initial_timestamp"], events["final_timestamp"]
    t[:n, LC["initial_clk_high"]] = it >> np.uint64(24)
    t[:n, LC["final_clk_high"]] = ft >> np.uint64(24)
    t[:n, LC["initial_clk_low"]] = it & np.uint64(0xFFFFFF)
    t[:n, LC["final_clk_low"]] = ft & np.uint64(0xFFFFFF)
    iv, fv = events["initial_value"], events["final_value"]
    for k, (x, y) in enumerate(zip(u64_to_u16_limbs(iv), u64_to_u16_limbs(fv))):
        t[:n, LC[f"initial_value[{k}]"]] = x
        t[:n, LC[f"final_value[{k}]"]] = y
    t[:n, LC["is_real"]] = 1
    t[:n, LC["initial_value_lower"]] = (iv >> np.uint64(32)) & np.uint64(0xFF)
    t[:n, LC["initial_value_upper"]] = (iv >> np.uint64(40)) & np.uint64(0xFF)
    t[:n, LC["final_value_lower"]] = (fv >> np.uint64(32)) & np.uint64(0xFF)
    t[:n, LC["final_value_upper"]] = (fv >> np.uint64(40)) & np.uint64(0xFF)
    return t


def local_dependencies(events):
    """MemoryLocalChip::generate_dependencies (local.rs:105-157) -> (byte lookups [(opcode, a, b, c)], message [2n, 8], is_receive [2n],
    kind [2n]): per event the initial access (a receive), then the final access (a send)"""
    n = len(events)
    lookups = np.zeros((n, 10, 4), np.int32)
    msg = np.zeros((n, 2, 8), np.uint64)
    for j, (ts, value) in enumerate(((events["initial_timestamp"], events["initial_value"]),
                                     (events["final_timestamp"], events["final_value"]))):
        b0 = (value >> np.uint64(32)) & np.uint64(0xFF)
        b1 = (value >> np.uint64(40)) & np.uint64(0xFF)
        lookups[:, 5 * j] = np.stack([np.full(n, U8RANGE), np.zeros(n), b0, b1], axis=1)   # add_u8_range_check
        for k, limb in enumerate(u64_to_u16_limbs(value)):                  # add_u16_range_checks_field(Word::from(value))
            lookups[:, 5 * j + 1 + k] = np.stack([np.full(n, RANGE), limb, np.full(n, 16), np.zeros(n)], axis=1)
        m = msg[:, j]
        m[:, 0] = ts >> np.uint64(24)
        m[:, 1] = ts & np.uint64(0xFFFFFF)
        for k in range(3):
            m[:, 2 + k] = (events["addr"] >> np.uint64(16 * k)) & np.uint64(0xFFFF)
        m[:, 5] = (value & np.uint64(0xFFFF)) + np.uint64(1 << 16) * b0
        m[:, 6] = ((value >> np.uint64(16)) & np.uint64(0xFFFF)) + np.uint64(1 << 16) * b1
        m[:, 7] = (value >> np.uint64(48)) & np.uint64(0xFFFF)
    is_receive = np.tile(np.array([1, 0], np.uint8), n)
    return lookups.reshape(-1, 4), msg.reshape(-1, 8), is_receive, np.full(2 * n, KIND_MEMORY, np.uint8)


def to_monty(x):
    return ((np.asarray(x, np.uint64) % np.uint64(P)) << np.uint64(32)) % np.uint64(P)


def main_words(trace):
    """a row-major canonical trace -> the library's layout: column-major [cols, rows] Montgomery words"""
    return np.stack([to_monty(trace[:, k]).astype(np.uint32) for k in range(trace.shape[1])]) if trace.size else \
        np.zeros(trace.shape[::-1], np.uint32)


def shard(init, finalize, previous_init_addr, previous_finalize_addr, local):
    """the three chips of one shard -> dict(traces=(init, finalize, local) row-major canonical, lookups [(opcode, a, b, c)] of the three
    chips in the order init, finalize, local, and global events (message, is_receive, kind) in the same order)"""
    di = global_dependencies(init, previous_init_addr, False)
    df = global_dependencies(finalize, previous_finalize_addr, True)
    dl = local_dependencies(local)
    return dict(traces=(global_trace(init, previous_init_addr), global_trace(finalize, previous_finalize_addr), local_trace(local)),
                lookups=np.concatenate([di[0], df[0], dl[0]]),
                globals=tuple(np.concatenate([d[k] for d in (di, df, dl)]) for k in (1, 2, 3)))
