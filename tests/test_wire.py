"""ShardProof wire format (SURVEY 8f.4): the product's flat proof words <-> bincode(ShardProof) through the C ABI (host-only entry points),
checked against an independent schema-driven reader of the Rust struct definitions (tests/bincode_ref.py), the reference-held bincode
files that pin the leaf encodings (tests/golden/bincode_pins.json), and the restated verifier on the round-tripped words."""
import json
import os
import struct

import numpy as np
import pytest

from sp1_b200 import lib as PL
from tests import bincode_ref as BR
from tests import machines as M
from tests import oracle_lib as O

HERE = os.path.dirname(os.path.abspath(__file__))


PARAMS = dict(log_blowup=2, num_queries=6, pow_bits=3, batch_pow_bits=2, gkr_pow_bits=3)


def _proof(spec, log_stack, mlr, seed=71):
    rng = np.random.default_rng(seed)
    blob, heights, mains, preps, pv, names = M.spec_machine(rng, spec, names="Chip{:02d}")
    ch = O.Challenger(); ch.observe(O.rand_field(rng, 5))
    start = ch.clone()
    pc, words = O.prove_shard_verify(blob, heights, mains, preps, names, pv, log_stack, mlr, ch, **PARAMS)
    w = M.widths(blob)
    return dict(blob=blob, heights=heights, names=names, words=words, main_w=[a for a, _ in w], prep_w=[b for _, b in w], start=start,
                final=ch, prep_commit=pc, params=dict(PARAMS, log_stacking_height=log_stack, max_log_row_count=mlr))


def test_leaf_encoding_pins():
    """what the reference-held bincode files say about the leaves: canonical u32 field words, arrays without length, usize = u64"""
    pins = json.load(open(os.path.join(HERE, "golden", "bincode_pins.json")))
    head = bytes.fromhex(pins["dummy"]["head_hex"])
    r = BR.Reader(head)
    assert r.u64() == pins["dummy"]["entries"]
    for i in range(3):
        assert BR.DIGEST(r) == [i] * 8 and BR.USIZE(r) == i        # [F::from_canonical_u32(i); 8] -> i  (recursion.rs:72-75)
    assert (1 << 32) % BR.P == 33554430 != 1                        # the Montgomery word of 1 is not what the file holds
    r = BR.Reader(bytes.fromhex(pins["vk_map"]["head_hex"]))
    assert r.u64() == pins["vk_map"]["entries"]
    k0, _, k1, _ = BR.DIGEST(r), BR.USIZE(r), BR.DIGEST(r), BR.USIZE(r)
    assert k0 < k1 and pins["vk_map"]["max_word"] < BR.P


@pytest.mark.parametrize("spec,log_stack,mlr", M.SHARD_SPECS)
def test_bincode_matches_the_struct_definitions(spec, log_stack, mlr):
    p = _proof(spec, log_stack, mlr)
    data = PL.shard_proof_to_bincode(p["words"], p["names"], p["heights"], p["main_w"], p["prep_w"], **p["params"])
    tree = BR.decode_shard_proof(data)                 # every byte consumed by the restated struct definitions
    words, names, heights = BR.flatten(tree)
    assert names == p["names"] and heights == list(p["heights"])
    assert len(words) == p["words"].size and (np.array(words, dtype=np.uint64) == p["words"]).all()
    # spot checks in the reference's own terms
    assert len(tree["opened_values"]["chips"][0][1]["degree"]["values"]) == mlr + 1
    assert tree["evaluation_proof"]["max_log_row_count"] == mlr
    bf = tree["evaluation_proof"]["pcs_proof"]["basefold_proof"]
    assert len(bf["univariate_messages"]) == len(bf["fri_commitments"]) == len(bf["query_phase_openings_and_proofs"]) == log_stack
    assert bf["component_polynomials_query_openings_and_proofs"][0]["values"]["dimensions"][0] == PARAMS["num_queries"]
    assert tree["public_values"] == [int(x) for x in O.from_monty(p["words"][-len(tree["public_values"]):])]


@pytest.mark.parametrize("spec,log_stack,mlr", M.SHARD_SPECS)
def test_bincode_round_trip_and_verifier(spec, log_stack, mlr):
    p = _proof(spec, log_stack, mlr)
    data = PL.shard_proof_to_bincode(p["words"], p["names"], p["heights"], p["main_w"], p["prep_w"], **p["params"])
    words, heights = PL.shard_proof_from_bincode(data, p["names"], p["main_w"], p["prep_w"], **p["params"])
    assert heights == list(p["heights"]) and words.size == p["words"].size and (words == p["words"]).all()
    ch = p["start"].clone()
    prm = {k: v for k, v in p["params"].items() if k not in ("log_stacking_height", "max_log_row_count")}
    assert O.verify_shard(p["blob"], heights, p["names"], log_stack, mlr, ch, p["prep_commit"], words, **prm) == 0
    assert (ch.st == p["final"].st).all()


def test_bincode_rejects_malformed_input():
    spec, log_stack, mlr = M.SHARD_SPECS[1]
    p = _proof(spec, log_stack, mlr)
    args = (p["names"], p["main_w"], p["prep_w"])
    data = bytearray(PL.shard_proof_to_bincode(p["words"], p["names"], p["heights"], p["main_w"], p["prep_w"], **p["params"]))
    with pytest.raises(PL.Sp1B200Error, match="truncated|exceeds"):
        PL.shard_proof_from_bincode(bytes(data[:-3]), *args, **p["params"])
    with pytest.raises(PL.Sp1B200Error, match="trailing"):
        PL.shard_proof_from_bincode(bytes(data) + b"\0", *args, **p["params"])
    bad = bytearray(data); bad[8:12] = struct.pack("<I", BR.P)            # first public value := p (not canonical)
    with pytest.raises(PL.Sp1B200Error, match="canonical"):
        PL.shard_proof_from_bincode(bytes(bad), *args, **p["params"])
    bad = bytearray(data); bad[0:8] = struct.pack("<Q", 1 << 40)          # absurd length prefix
    with pytest.raises(PL.Sp1B200Error, match="exceeds"):
        PL.shard_proof_from_bincode(bytes(bad), *args, **p["params"])
    with pytest.raises(PL.Sp1B200Error, match="name"):
        PL.shard_proof_from_bincode(bytes(data), ["Chip00", "Chip01", "Chip0X"], p["main_w"], p["prep_w"], **p["params"])
    with pytest.raises(PL.Sp1B200Error, match="ascending"):
        PL.shard_proof_to_bincode(p["words"], p["names"][::-1], p["heights"], p["main_w"], p["prep_w"], **p["params"])
    with pytest.raises(PL.Sp1B200Error, match="width"):
        PL.shard_proof_from_bincode(bytes(data), p["names"], [w + 1 for w in p["main_w"]], p["prep_w"], **p["params"])
    short = p["words"][:-1].copy()
    with pytest.raises(PL.Sp1B200Error, match="add up"):
        PL.shard_proof_to_bincode(short, p["names"], p["heights"], p["main_w"], p["prep_w"], **p["params"])
    # a flipped proof byte still parses but the restated verifier rejects the round-tripped words
    bad = bytearray(data); bad[len(bad) // 2] ^= 1
    try:
        words, heights = PL.shard_proof_from_bincode(bytes(bad), *args, **p["params"])
    except PL.Sp1B200Error:
        return
    prm = {k: v for k, v in p["params"].items() if k not in ("log_stacking_height", "max_log_row_count")}
    assert O.verify_shard(p["blob"], heights, p["names"], log_stack, mlr, p["start"].clone(), p["prep_commit"], words, **prm) != 0


def test_bincode_reader_survives_random_corruption():
    """memory safety of the byte reader: random byte flips, length-prefix overwrites and truncations must end in an error message or a
    parsed proof - never in a crash or an over-read (every length prefix is checked against the bytes that remain)"""
    spec, log_stack, mlr = M.SHARD_SPECS[2]
    p = _proof(spec, log_stack, mlr)
    args = (p["names"], p["main_w"], p["prep_w"])
    data = PL.shard_proof_to_bincode(p["words"], p["names"], p["heights"], p["main_w"], p["prep_w"], **p["params"])
    rng = np.random.default_rng(2024)
    outcomes = {"error": 0, "parsed": 0}
    for trial in range(400):
        b = bytearray(data)
        kind = trial % 4
        if kind == 0:                                   # a few random byte flips
            for pos in rng.integers(0, len(b), size=int(rng.integers(1, 6))):
                b[pos] ^= 1 << int(rng.integers(0, 8))
        elif kind == 1:                                 # overwrite 8 bytes somewhere with a huge / random u64 (hits length prefixes often)
            pos = int(rng.integers(0, len(b) - 8))
            b[pos:pos + 8] = struct.pack("<Q", int(rng.integers(0, 1 << 62)) if trial % 8 == 1 else (1 << 63) + 5)
        elif kind == 2:                                 # truncate
            b = b[:int(rng.integers(0, len(b)))]
        else:                                           # splice a random window out
            a = int(rng.integers(0, len(b) - 16)); b = b[:a] + b[a + int(rng.integers(1, 16)):]
        try:
            words, heights = PL.shard_proof_from_bincode(bytes(b), *args, **p["params"])
            assert words[0] == 5 and len(heights) == len(p["names"])
            outcomes["parsed"] += 1
        except PL.Sp1B200Error as e:
            assert str(e).startswith("shard_proof_from_bincode:")
            outcomes["error"] += 1
    assert outcomes["error"] > 200 and outcomes["parsed"] + outcomes["error"] == 400, outcomes


def test_bincode_reader_under_sanitizers(tmp_path):
    """the wire code (host-only) compiled as plain C++ with -fsanitize=address,undefined and driven by tools/fuzz_wire.cpp over mutated
    proofs in exact-size heap buffers: any over-read, overflow or UB aborts the run"""
    import shutil
    import subprocess
    root = os.path.dirname(HERE)
    if shutil.which("g++") is None:
        pytest.skip("no g++")
    exe = str(tmp_path / "fuzz_wire")
    cc = subprocess.run(["g++", "-std=c++17", "-O1", "-g", "-fsanitize=address,undefined", "-fno-sanitize-recover=all", "-x", "c++",
                         f"-I{root}/include", f"-I{root}/sp1_b200/csrc", "-I/usr/local/cuda/include", f"{root}/tools/fuzz_wire.cpp",
                         f"{root}/sp1_b200/csrc/wire.cu", "-o", exe], capture_output=True, text=True)
    if cc.returncode != 0:
        pytest.skip("sanitizer build unavailable here: " + cc.stderr[-300:])
    spec, log_stack, mlr = M.SHARD_SPECS[2]
    p = _proof(spec, log_stack, mlr)
    data = PL.shard_proof_to_bincode(p["words"], p["names"], p["heights"], p["main_w"], p["prep_w"], **p["params"])
    f = tmp_path / "proof.bin"
    f.write_bytes(data)
    widths = [str(x) for pair in zip(p["main_w"], p["prep_w"]) for x in pair]
    run = subprocess.run([exe, str(f), str(log_stack), str(mlr), str(len(p["names"]))] + widths, capture_output=True, text=True,
                         env=dict(os.environ, FUZZ_TRIALS="6000"), timeout=300)
    assert run.returncode == 0, run.stderr[-2000:]
    assert run.stdout.startswith("parsed ")


def test_bincode_golden_fixtures():
    """committed SHA-256 of the wire bytes of the golden proofs (tests/golden/shard_proofs_bincode.json, tools/gen_golden_proofs.py --bincode):
    pins the byte layout against accidental change; the proof words behind them are the ones tests/golden/shard_proofs.json pins"""
    import hashlib
    from tools import gen_golden_proofs as GG
    gold = {c["name"]: c for c in json.load(open(os.path.join(HERE, "golden", "shard_proofs_bincode.json")))["cases"]}
    words_gold = {c["name"]: c for c in json.load(open(os.path.join(HERE, "golden", "shard_proofs.json")))["cases"]}
    for case in GG.CASES:
        got = GG.bincode_case(*case)
        g = gold[case[0]]
        assert got["words_sha256"] == words_gold[case[0]]["sha256"] == g["words_sha256"]
        assert got["bincode_bytes"] == g["bincode_bytes"] and got["bincode_sha256"] == g["bincode_sha256"], case[0]
