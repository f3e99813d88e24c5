"""ctypes binding of oracle/_ref/libsp1ref.so — the REFERENCE's own CUDA kernels (sp1-gpu/crates/sys, compiled unmodified by
oracle/Makefile) behind oracle/ref_launcher.cu.  Test infrastructure only: imported by tests/ and by bench.py's
`vs_ref_kernels` leg, never by the product."""
import ctypes as C
import os

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SO = os.path.join(ROOT, "oracle", "_ref", "libsp1ref.so")
u32p = C.POINTER(C.c_uint32)
_lib = None


def available():
    return os.path.exists(SO)


class RefError(RuntimeError):
    pass


def _chk(e):
    if e:
        raise RefError(e.decode())


def lib():
    global _lib
    if _lib is None:
        if not available():
            raise RefError("oracle/_ref/libsp1ref.so missing: run `make -C oracle ref` where /root/reference exists")
        L = C.CDLL(SO)
        for n in ("ref_init", "ref_malloc", "ref_free", "ref_h2d", "ref_d2h", "ref_field_op", "ref_ext_op", "ref_permute", "ref_hash",
                  "ref_compress", "ref_merkle_tree", "ref_batch_coset_dft", "ref_batch", "ref_fold_mle_ext", "ref_fix_last_variable_ext",
                  "ref_partial_lagrange_ext", "ref_grind", "ref_challenger_script", "ref_gkr_populate", "ref_zerocheck_node_sums",
                  "ref_jagged_sumcheck", "ref_logup_gkr", "ref_zerocheck", "ref_bp_transitions", "ref_jagged_eval"):
            getattr(L, n).restype = C.c_char_p
        _chk(L.ref_init())
        _lib = L
    return _lib


def _p(a):
    assert a.dtype == np.uint32 and a.flags["C_CONTIGUOUS"]
    return a.ctypes.data_as(u32p)


class DevBuf:
    """plain cudaMalloc buffer owned by the reference library's process (independent of torch and of libsp1b200)"""

    def __init__(self, words):
        self.words = int(words)
        p = C.c_void_p()
        _chk(lib().ref_malloc(C.c_size_t(max(4, self.words * 4)), C.byref(p)))
        self.ptr = p

    @classmethod
    def from_host(cls, a):
        a = np.ascontiguousarray(a, dtype=np.uint32)
        b = cls(a.size)
        _chk(lib().ref_h2d(b.ptr, _p(a.reshape(-1)), C.c_size_t(a.size * 4)))
        return b

    def to_host(self, shape=None):
        out = np.zeros(self.words, np.uint32)
        _chk(lib().ref_d2h(_p(out), self.ptr, C.c_size_t(self.words * 4)))
        return out if shape is None else out.reshape(shape)

    def free(self):
        if self.ptr:
            lib().ref_free(self.ptr)
            self.ptr = None

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


FIELD_OPS = {"add": 0, "sub": 1, "mul": 2, "inv": 3, "cube": 4, "neg": 5}
EXT_OPS = {"add": 0, "sub": 1, "mul": 2, "inv": 3, "mul_base": 4, "interpolate_linear": 5}


def field_op(op, a, b=None):
    a = np.ascontiguousarray(a, np.uint32)
    b = a if b is None else np.ascontiguousarray(b, np.uint32)
    out = np.zeros_like(a)
    _chk(lib().ref_field_op(FIELD_OPS[op], _p(a), _p(b), _p(out), C.c_size_t(a.size)))
    return out


def ext_op(op, a, b=None, c=None):
    a = np.ascontiguousarray(a, np.uint32)
    b = a if b is None else np.ascontiguousarray(b, np.uint32)
    c = a if c is None else np.ascontiguousarray(c, np.uint32)
    out = np.zeros_like(a)
    _chk(lib().ref_ext_op(EXT_OPS[op], _p(a), _p(b), _p(c), _p(out), C.c_size_t(a.size // 4)))
    return out


def permute(states):
    s = np.ascontiguousarray(states, np.uint32).copy()
    _chk(lib().ref_permute(_p(s), C.c_size_t(s.size // 16)))
    return s


def hash_(items):
    """items: [n_items, n_in] -> [n_items, 8]"""
    v = np.ascontiguousarray(items, np.uint32)
    out = np.zeros((v.shape[0], 8), np.uint32)
    _chk(lib().ref_hash(_p(v), C.c_size_t(v.shape[1]), _p(out), C.c_size_t(v.shape[0])))
    return out


def compress(l, r):
    l = np.ascontiguousarray(l, np.uint32)
    r = np.ascontiguousarray(r, np.uint32)
    out = np.zeros_like(l)
    _chk(lib().ref_compress(_p(l), _p(r), _p(out), C.c_size_t(l.size // 8)))
    return out


def merkle_tree(mat, d_mat=None, d_digests=None):
    """mat: [width, 2^h] column-major.  -> (digests [2^(h+1)-1, 8] in HEAP order (root first), (leaf_ms, compress_ms))"""
    width, rows = mat.shape if d_mat is None else mat
    h = rows.bit_length() - 1
    own = d_mat is None
    if own:
        d_mat = DevBuf.from_host(mat)
    dg = d_digests or DevBuf(((2 << h) - 1) * 8)
    ms = (C.c_float * 2)()
    _chk(lib().ref_merkle_tree(d_mat.ptr, dg.ptr, C.c_size_t(width), C.c_size_t(h), ms))
    if d_digests is not None:
        return None, (ms[0], ms[1])
    out = dg.to_host(((2 << h) - 1, 8))
    dg.free()
    if own:
        d_mat.free()
    return out, (ms[0], ms[1])


def heap_to_layers(heap, h):
    """heap order (root at 0, leaves at 2^h - 1) -> the bottom-up layer order of sp1b200_merkle_commit / orc_merkle_commit"""
    return np.concatenate([heap[(1 << k) - 1:(2 << k) - 1] for k in range(h, -1, -1)])


INV3_MONTY = None


def batch_coset_dft(msg, log_blowup, shift_monty=None, bit_rev=True, d_in=None, d_out=None, shape=None):
    """the reference's RS-encode call (encode_batch -> coset_dft_into -> batch_coset_dft): shift word = 1 / generator"""
    global INV3_MONTY
    if shift_monty is None:
        if INV3_MONTY is None:
            INV3_MONTY = int(field_op("inv", np.array([((3 << 32) % 0x7F000001)], np.uint32))[0])
        shift_monty = INV3_MONTY
    ncols, n = msg.shape if shape is None else shape
    lg = n.bit_length() - 1
    own = d_in is None
    if own:
        d_in = DevBuf.from_host(msg)
        d_out = DevBuf(ncols * (n << log_blowup))
    ms = C.c_float()
    _chk(lib().ref_batch_coset_dft(d_out.ptr, d_in.ptr, C.c_uint32(lg), C.c_uint32(log_blowup), C.c_uint32(shift_monty), C.c_uint32(ncols),
                                   C.c_int(1 if bit_rev else 0), C.byref(ms)))
    if not own:
        return None, ms.value
    out = d_out.to_host((ncols, n << log_blowup))
    d_in.free(); d_out.free()
    return out, ms.value


def batch(mat, beta_powers):
    """batchKernel: out[row] = sum_c beta_powers[c] * mat[c][row]  (ext)"""
    width, height = mat.shape
    d_in, d_b = DevBuf.from_host(mat), DevBuf.from_host(beta_powers)
    d_out = DevBuf(height * 4)
    ms = C.c_float()
    _chk(lib().ref_batch(d_in.ptr, d_out.ptr, d_b.ptr, C.c_size_t(height), C.c_size_t(width), C.byref(ms)))
    out = d_out.to_host((height, 4))
    for b in (d_in, d_b, d_out):
        b.free()
    return out, ms.value


def fold_mle_ext(vals, beta):
    """foldMle<ext, ext>: out[i] = beta * in[2i+1] + in[2i]; vals: [2m, 4]"""
    vals = np.ascontiguousarray(vals, np.uint32)
    m = vals.shape[0] // 2
    d_in, d_out = DevBuf.from_host(vals), DevBuf(m * 4)
    beta = np.ascontiguousarray(beta, np.uint32)
    ms = C.c_float()
    _chk(lib().ref_fold_mle_ext(d_in.ptr, d_out.ptr, _p(beta), C.c_size_t(m), C.c_size_t(1), C.byref(ms)))
    out = d_out.to_host((m, 4))
    d_in.free(); d_out.free()
    return out


def fix_last_variable_ext(vals, alpha):
    """fixLastVariableInPlace<ext>: out[i] = in[2i] * (1 - alpha) + in[2i+1] * alpha"""
    vals = np.ascontiguousarray(vals, np.uint32)
    m = vals.shape[0] // 2
    d = DevBuf.from_host(vals)
    alpha = np.ascontiguousarray(alpha, np.uint32)
    _chk(lib().ref_fix_last_variable_ext(d.ptr, _p(alpha), C.c_size_t(m), C.c_size_t(1)))
    out = d.to_host((2 * m, 4))[:m]
    d.free()
    return out


def partial_lagrange_ext(point):
    """eq table of an ext point: [2^n, 4]; the first coordinate is the most significant bit of the index"""
    point = np.ascontiguousarray(point, np.uint32)
    n = point.shape[0]
    d_p, d_o = DevBuf.from_host(point), DevBuf((1 << n) * 4)
    _chk(lib().ref_partial_lagrange_ext(d_o.ptr, d_p.ptr, C.c_size_t(n)))
    out = d_o.to_host((1 << n, 4))
    d_p.free(); d_o.free()
    return out


def grind(st34, bits):
    st = np.ascontiguousarray(st34, np.uint32)
    w = C.c_uint32()
    ms = C.c_float()
    _chk(lib().ref_grind(_p(st), C.c_uint32(bits), C.byref(w), C.byref(ms)))
    return w.value, ms.value


def challenger_script(st34, ops, vals):
    st = np.ascontiguousarray(st34, np.uint32).copy()
    ops = np.ascontiguousarray(ops, np.uint32)
    vals = np.ascontiguousarray(vals, np.uint32)
    out = np.zeros(ops.size, np.uint32)
    _chk(lib().ref_challenger_script(_p(st), _p(ops), _p(vals), _p(out), C.c_size_t(ops.size)))
    return st, out


# ---- machine-blob parsing (the product's blob format, include/sp1b200.h) for the reference's own data layouts ---------------------------
def parse_chip_words(blob):
    """-> list of dicts per chip {main_w, prep_w, n_constraints, n_regs, instrs, leaves, consts, publics, assert_regs, assert_alphas}, and
    the offset where the interaction section starts"""
    b = np.asarray(blob, np.uint32)
    n = int(b[0]); o = 1
    chips = []
    for _ in range(n):
        main_w, prep_w, n_c, n_regs, ni, nl, nc, npub, na = [int(x) for x in b[o:o + 9]]; o += 9
        c = dict(main_w=main_w, prep_w=prep_w, n_constraints=n_c, n_regs=n_regs)
        c["instrs"] = b[o:o + 2 * ni].copy(); o += 2 * ni
        c["leaves"] = b[o:o + 2 * nl].copy(); o += 2 * nl
        c["consts"] = b[o:o + nc].copy(); o += nc
        c["publics"] = b[o:o + npub].copy(); o += npub
        c["assert_regs"] = b[o:o + na].copy(); o += na
        c["assert_alphas"] = b[o:o + na].copy(); o += na
        chips.append(c)
    return chips, o


def parse_interactions(blob, offset, n_chips):
    """-> per chip: list of (is_send, arg_index, mult vcol, [value vcols]); vcol = (constant, [(source, col, weight)])"""
    b = np.asarray(blob, np.uint32); o = offset
    out = []

    def vcol():
        nonlocal o
        nt, const = int(b[o]), int(b[o + 1]); o += 2
        terms = [(int(b[o + 3 * t]), int(b[o + 3 * t + 1]), int(b[o + 3 * t + 2])) for t in range(nt)]
        o += 3 * nt
        return const, terms
    for _ in range(n_chips):
        n = int(b[o]); o += 1
        chip = []
        for _ in range(n):
            is_send, arg, nv = int(b[o]), int(b[o + 1]), int(b[o + 2]); o += 3
            mult = vcol()
            vals = [vcol() for _ in range(nv)]
            chip.append((is_send, arg, mult, vals))
        out.append(chip)
    return out


LEAF_PREP = 2


def _interaction_csr(inter):
    """one chip of parse_interactions in the flattened CSR form of the reference's `Interactions<F>` (sys/include/logup_gkr/tracegen.cuh),
    indices local to the chip: dict of the arrays ref_gkr_populate / ref_logup_gkr take"""
    values_ptr, mult_ptr, vcw_ptr = [0], [0], [0]
    vcw, mcw, vconst, mconst, args, send = [], [], [], [], [], []
    for is_send, arg, (mc, mterms), vals in inter:
        for const, terms in vals:
            vconst.append(const)
            vcw += [(col, src == LEAF_PREP, wt) for src, col, wt in terms]
            vcw_ptr.append(len(vcw))
        values_ptr.append(len(vconst))
        mconst.append(mc)
        mcw += [(col, src == LEAF_PREP, wt) for src, col, wt in mterms]
        mult_ptr.append(len(mcw))
        args.append(int(((arg << 32) % 0x7F000001)))
        send.append(1 if is_send else 0)
    return dict(values_ptr=(values_ptr, np.uint64), mult_ptr=(mult_ptr, np.uint64), vcw_ptr=(vcw_ptr, np.uint64),
                vcw_col=([c for c, _, _ in vcw], np.uint64), vcw_is_prep=([p for _, p, _ in vcw], np.uint8), vcw_weight=([w for _, _, w in vcw], np.uint32),
                values_constants=(vconst, np.uint32), mcw_col=([c for c, _, _ in mcw], np.uint64), mcw_is_prep=([p for _, p, _ in mcw], np.uint8),
                mcw_weight=([w for _, _, w in mcw], np.uint32), mult_constants=(mconst, np.uint32), arg_indices=(args, np.uint32),
                is_send=(send, np.uint8))


def _arr(x, dt):
    """a contiguous array of dtype dt, one zero entry when empty (never a null pointer)"""
    return np.ascontiguousarray(np.array(x if len(x) else [0], dtype=dt))


_CTYPES = {np.uint64: C.c_uint64, np.uint32: C.c_uint32, np.uint8: C.c_uint8}


def _ptr(a):
    return a.ctypes.data_as(C.POINTER(_CTYPES[a.dtype.type]))


def gkr_populate(inter, main, prep, alpha, betas):
    """the reference's populateLastCircuitLayer for one chip.  inter: one chip of parse_interactions; main / prep: [w, h] column-major.
    -> (num [n_inter, h] uint32, den [n_inter, h, 4])"""
    h = main.shape[1]
    n = len(inter)
    a = {k: _arr(x, dt) for k, (x, dt) in _interaction_csr(inter).items()}
    n_values, n_vcw, n_mcw = int(a["values_ptr"][-1]), int(a["vcw_ptr"][-1]), int(a["mult_ptr"][-1])
    half = (h + 1) // 2 if h else 1
    q = (half + 1) // 2
    outH = 2 * q * n
    num = np.zeros(4 * outH, np.uint32)
    den = np.zeros((4 * outH, 4), np.uint32)
    oh = C.c_uint64()
    mainf = np.ascontiguousarray(main, np.uint32).reshape(-1)
    prepf = np.ascontiguousarray(prep, np.uint32).reshape(-1) if prep is not None and prep.size else np.zeros(1, np.uint32)
    alpha = np.ascontiguousarray(alpha, np.uint32); betas = np.ascontiguousarray(betas, np.uint32)
    _chk(lib().ref_gkr_populate(_p(prepf), C.c_uint64(prepf.size if prep is not None and prep.size else 0), _p(mainf), C.c_uint64(mainf.size), C.c_uint64(h),
                                C.c_uint32(n), _ptr(a["values_ptr"]), _ptr(a["mult_ptr"]), _ptr(a["vcw_ptr"]), C.c_uint64(n_values), _ptr(a["vcw_col"]),
                                _ptr(a["vcw_is_prep"]), _ptr(a["vcw_weight"]), C.c_uint64(n_vcw), _ptr(a["values_constants"]), _ptr(a["mcw_col"]),
                                _ptr(a["mcw_is_prep"]), _ptr(a["mcw_weight"]), C.c_uint64(n_mcw), _ptr(a["mult_constants"]), _ptr(a["arg_indices"]),
                                _ptr(a["is_send"]), _p(alpha), _p(betas.reshape(-1)), C.c_uint32(betas.shape[0]), _p(num), _p(den.reshape(-1)), C.byref(oh)))
    assert oh.value == outH
    out_num = np.zeros((n, h), np.uint32); out_den = np.zeros((n, h, 4), np.uint32)
    for j in range(n):
        base = 2 * q * j
        out_num[j, 0::2] = num[base:base + half][: (h + 1) // 2]
        out_num[j, 1::2] = num[base + 2 * outH:base + 2 * outH + half][: h // 2]
        out_den[j, 0::2] = den[base:base + half][: (h + 1) // 2]
        out_den[j, 1::2] = den[base + 2 * outH:base + 2 * outH + half][: h // 2]
    return out_num, out_den


def gkr_layer_words(v, p):
    """the words ref_logup_gkr returns for GKR layer p (in proof order: p + 1 row variables, n = v + p + 1 rounds): the 10-value grid and
    3 sums per round from round 2 on for a lookahead layer (more than 2 row variables), 3 sums per round otherwise, then n0, n1, d0, d1"""
    n = v + p + 1
    return 4 * ((10 + 3 * (n - 2) if p + 1 > 2 else 3 * n) + 4)


def gkr_raw_words(v, mlr):
    """the number of words ref_logup_gkr returns for 2^v padded interactions and max_log_row_count mlr: the output numerators and
    denominators (2^(v+1) ext each), then every layer"""
    return 8 * (2 << v) + sum(gkr_layer_words(v, p) for p in range(mlr - 1))


def logup_gkr(chip_inters, heights, mains, preps, alpha, betas, mlr, lambdas, points, challenges):
    """the reference's LogUp-GKR kernels (ref_logup_gkr): first layer, forward circuit and every layer's sumcheck rounds with the challenges
    supplied.  chip_inters: parse_interactions of the machine; mains / preps: [w, h] column-major (preps[k] None without preprocessed
    columns); lambdas [L, 4], points / challenges: per GKR layer in proof order, [v + p + 1, 4] each.  -> the raw words (see ref_launcher.cu)"""
    csr = [_interaction_csr(i) for i in chip_inters]
    a = {k: _arr([x for c in csr for x in c[k][0]], csr[0][k][1]) for k in csr[0]}
    main_parts = [np.ascontiguousarray(m, np.uint32).reshape(-1) for m in mains]
    prep_parts = [np.ascontiguousarray(p, np.uint32).reshape(-1) if p is not None else np.zeros(0, np.uint32) for p in preps]
    main_off = np.ascontiguousarray(np.cumsum([0] + [m.size for m in main_parts])[:-1], np.uint64)
    prep_off = np.ascontiguousarray(np.cumsum([0] + [p.size for p in prep_parts])[:-1], np.uint64)
    mainf = _arr(np.concatenate(main_parts), np.uint32)
    prepf = _arr(np.concatenate(prep_parts), np.uint32)
    hs = np.ascontiguousarray(heights, np.uint64)
    ni = np.ascontiguousarray([len(i) for i in chip_inters], np.uint32)
    total = int(ni.sum())
    v = max(total - 1, 0).bit_length()
    out = np.zeros(gkr_raw_words(v, mlr), np.uint32)
    pts = np.ascontiguousarray(np.concatenate([np.asarray(p, np.uint32).reshape(-1) for p in points]), np.uint32)
    chs = np.ascontiguousarray(np.concatenate([np.asarray(c, np.uint32).reshape(-1) for c in challenges]), np.uint32)
    assert pts.size == chs.size
    lam = np.ascontiguousarray(lambdas, np.uint32).reshape(-1)
    alpha = np.ascontiguousarray(alpha, np.uint32); betas = np.ascontiguousarray(betas, np.uint32).reshape(-1)
    _chk(lib().ref_logup_gkr(C.c_uint32(len(heights)), _ptr(hs), _ptr(ni), _p(mainf), _ptr(main_off), C.c_uint64(mainf.size), _p(prepf), _ptr(prep_off),
                             C.c_uint64(prepf.size), *[_ptr(a[k]) for k in ("values_ptr", "mult_ptr", "vcw_ptr", "vcw_col", "vcw_is_prep", "vcw_weight",
                                                                            "values_constants", "mcw_col", "mcw_is_prep", "mcw_weight", "mult_constants",
                                                                            "arg_indices", "is_send")],
                             _p(alpha), _p(betas), C.c_uint32(betas.size // 4), C.c_uint32(mlr), _p(lam), _p(pts), _p(chs), C.c_uint64(pts.size),
                             _p(out), C.c_uint64(out.size)))
    return out


def zerocheck_raw_words(n_chips, n_cols, mlr):
    """the number of words ref_zerocheck returns: the padded-row adjustment of every chip, the 16 totals of the fused first two rounds,
    3 totals per later round and one value per column of the jagged trace (ext each)"""
    return 4 * (n_chips + 16 + 3 * (mlr - 2) + n_cols)


def zerocheck(blob, heights, mains, preps, prep_pad_rows, pv, alpha_pows, gkr_pows, lambda_pows, mlr, zeta, challenges):
    """the reference's zerocheck kernels (ref_zerocheck) with the host tables and challenges supplied: mains / preps [w, h] column-major
    (preps[k] None without preprocessed columns); alpha_pows, gkr_pows, lambda_pows, zeta, challenges [*, 4].  -> the raw words (see
    ref_launcher.cu)"""
    main_parts = [np.ascontiguousarray(m, np.uint32).reshape(-1) for m in mains]
    prep_parts = [np.ascontiguousarray(p, np.uint32).reshape(-1) if p is not None else np.zeros(0, np.uint32) for p in preps]
    main_off = np.ascontiguousarray(np.cumsum([0] + [m.size for m in main_parts])[:-1], np.uint64)
    prep_off = np.ascontiguousarray(np.cumsum([0] + [p.size for p in prep_parts])[:-1], np.uint64)
    mainf = _arr(np.concatenate(main_parts), np.uint32)
    prepf = _arr(np.concatenate(prep_parts), np.uint32)
    n_cols = sum(m.shape[0] for m in mains) + sum(p.shape[0] for p in preps if p is not None) + 1
    out = np.zeros(zerocheck_raw_words(len(heights), n_cols, mlr), np.uint32)
    t = {k: np.ascontiguousarray(np.asarray(v, np.uint32).reshape(-1, 4)) for k, v in
         dict(a=alpha_pows, g=gkr_pows, l=lambda_pows, z=zeta, c=challenges).items()}
    pv = _arr(pv, np.uint32)
    _chk(lib().ref_zerocheck(_p(np.ascontiguousarray(blob, np.uint32)), _ptr(np.ascontiguousarray(heights, np.uint64)), _p(mainf), _ptr(main_off),
                             C.c_uint64(sum(m.size for m in main_parts)), _p(prepf), _ptr(prep_off), C.c_uint64(sum(p.size for p in prep_parts)),
                             C.c_uint32(prep_pad_rows), _p(pv), C.c_uint32(len(pv)), _p(_arr(t["a"].reshape(-1), np.uint32)), C.c_uint32(t["a"].shape[0]),
                             _p(_arr(t["g"].reshape(-1), np.uint32)), C.c_uint32(t["g"].shape[0]), _p(t["l"].reshape(-1)), C.c_uint32(mlr),
                             _p(t["z"].reshape(-1)), _p(t["c"].reshape(-1)), _p(out), C.c_uint64(out.size)))
    return out


def zerocheck_node_sums(chip, main, prep, pv, alpha_pows, E):
    """the reference's zerocheck_fused_sequential<felt, 1024> over one chip (chip = one entry of parse_chip_words).  E: eq table over the
    row PAIRS [2^k, 4].  -> [3, 4] sums at the nodes {0, 2, 4}"""
    h = main.shape[1]
    out = np.zeros(12, np.uint32)
    mainf = np.ascontiguousarray(main, np.uint32).reshape(-1)
    prepf = np.ascontiguousarray(prep, np.uint32).reshape(-1) if prep is not None and prep.size else np.zeros(1, np.uint32)
    pw = 0 if prep is None else prep.shape[0]
    pv = np.ascontiguousarray(pv, np.uint32); ap = np.ascontiguousarray(alpha_pows, np.uint32); E = np.ascontiguousarray(E, np.uint32)
    k = E.shape[0].bit_length() - 1
    z = lambda a: a if a.size else np.zeros(1, np.uint32)
    _chk(lib().ref_zerocheck_node_sums(_p(z(chip["instrs"])), C.c_uint32(chip["instrs"].size // 2), _p(z(chip["leaves"])), C.c_uint32(chip["leaves"].size // 2),
                                       _p(z(chip["consts"])), C.c_uint32(chip["consts"].size), _p(z(chip["publics"])), C.c_uint32(chip["publics"].size),
                                       _p(z(chip["assert_regs"])), _p(z(chip["assert_alphas"])), C.c_uint32(chip["assert_regs"].size), _p(mainf),
                                       C.c_uint32(main.shape[0]), _p(prepf), C.c_uint32(pw), C.c_uint32(h), _p(pv), C.c_uint32(pv.size), _p(ap.reshape(-1)),
                                       C.c_uint32(ap.shape[0]), _p(E.reshape(-1)), C.c_uint32(k), _p(out)))
    return out.reshape(3, 4)


def jagged_sumcheck(dense, col_heights, eq_row, eq_col, challenges, log_stacking_height):
    """the reference's jagged Hadamard sumcheck kernels (ref_jagged_sumcheck) on the base-field dense words, the element heights of its
    columns, the eq tables of z_row and z_col and the round challenges in sampling order.  -> the raw sums, flat words: grid8 (8 ext) |
    round 2 (2 ext) | rounds 3 .. log_m - 1 (2 ext each) | p_eval, q_eval | stacked evals (len(dense) >> log_stacking_height ext)"""
    dense = np.ascontiguousarray(dense, np.uint32).reshape(-1)
    eq_row = np.ascontiguousarray(eq_row, np.uint32).reshape(-1, 4)
    eq_col = np.ascontiguousarray(eq_col, np.uint32).reshape(-1, 4)
    ch = np.ascontiguousarray(challenges, np.uint32).reshape(-1, 4)
    log_m = ch.shape[0]
    h = np.ascontiguousarray(col_heights, np.uint64)
    grid8, r2 = np.zeros(32, np.uint32), np.zeros(8, np.uint32)
    rounds = np.zeros(max(1, 8 * (log_m - 3)), np.uint32)
    pq = np.zeros(8, np.uint32)
    stacked = np.zeros(4 * (dense.size >> log_stacking_height), np.uint32)
    _chk(lib().ref_jagged_sumcheck(_p(dense), C.c_uint64(dense.size), h.ctypes.data_as(C.POINTER(C.c_uint64)), C.c_uint32(h.size),
                                   _p(eq_row.reshape(-1)), C.c_uint64(eq_row.shape[0]), _p(eq_col.reshape(-1)), C.c_uint64(eq_col.shape[0]),
                                   _p(ch.reshape(-1)), C.c_uint32(log_m), C.c_uint32(log_stacking_height), _p(grid8), _p(r2), _p(rounds), _p(pq),
                                   _p(stacked)))
    return np.concatenate([grid8, r2, rounds[:8 * (log_m - 3)], pq, stacked])


def bp_transitions():
    """the reference's TRANSITIONS table as its transition_kernel writes it (ref_bp_transitions): [16 bit states, 5 input memory states]
    -> output memory state, FAIL = 4; bit state = row * 8 + index * 4 + current prefix-sum bit * 2 + next prefix-sum bit, memory state =
    comparison_so_far * 2 + carry"""
    out = np.zeros(80, np.uint64)
    _chk(lib().ref_bp_transitions(out.ctypes.data_as(C.POINTER(C.c_uint64))))
    return out.reshape(16, 5)


def jagged_eval(merged, zc, z_row, z_index, claim, st34):
    """the reference's jagged evaluation sumcheck kernels (ref_jagged_eval) on the condensed merged prefix sums [nk, 2 (log_m + 1)] (field
    words), the condensed z_col eq values [nk, 4], z_row, z_index (the Hadamard sumcheck point) and the claimed sum, from the challenger
    state before the claim is observed.  -> (the round_num = -1 program values [2, nk, 4], sum values [2 (log_m + 1), 3, 4] = (y_0, y_1/2,
    y_1) per round, the sampled point [2 (log_m + 1), 4] most recent first, the final challenger state [34])"""
    merged = np.ascontiguousarray(merged, np.uint32)
    nk, dim = merged.shape
    zc = np.ascontiguousarray(zc, np.uint32).reshape(-1)
    z_row = np.ascontiguousarray(z_row, np.uint32).reshape(-1, 4)
    z_index = np.ascontiguousarray(z_index, np.uint32).reshape(-1, 4)
    claim = np.ascontiguousarray(claim, np.uint32).reshape(4)
    st = np.ascontiguousarray(st34, np.uint32).copy()
    bp = np.zeros((2, nk, 4), np.uint32)
    sums = np.zeros((dim, 3, 4), np.uint32)
    point = np.zeros((dim, 4), np.uint32)
    z = lambda a: a if a.size else np.zeros(4, np.uint32)
    _chk(lib().ref_jagged_eval(_p(merged.reshape(-1)), C.c_uint32(nk), C.c_uint32(dim // 2 - 1), _p(zc), _p(z(z_row).reshape(-1)),
                               C.c_uint32(z_row.shape[0]), _p(z(z_index).reshape(-1)), C.c_uint32(z_index.shape[0]), _p(claim), _p(st),
                               _p(bp.reshape(-1)), _p(sums.reshape(-1)), _p(point.reshape(-1))))
    return bp, sums, point, st
