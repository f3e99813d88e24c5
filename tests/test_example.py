"""The compiled host above the C ABI (examples/prove_shard.cpp over include/sp1b200_air_prover.hpp, the C++ mirror of the
reference's AirProver trait): it must build with a plain C++ compiler against the header (CPU), and on a GPU reproduce a golden
shard proof without Python in the loop."""
import os
import struct
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXE = os.path.join(ROOT, "examples", "prove_shard")


def _build():
    # the library itself is built by __graft_entry__.build() (nvcc); here only the plain-C++ host is (re)linked against it
    assert os.path.exists(os.path.join(ROOT, "sp1_b200", "libsp1b200.so")), "run python __graft_entry__.py first"
    subprocess.check_call(["make", "-C", os.path.join(ROOT, "examples")], stdout=subprocess.DEVNULL)


def test_example_host_builds_and_reports_usage():
    _build()
    r = subprocess.run([EXE], capture_output=True, text=True)
    assert r.returncode == 2 and "usage" in r.stderr


def test_wire_example_host_on_the_cpu(tmp_path):
    """examples/proof_wire.cpp (plain C++ over include/sp1b200.h, no GPU): golden proof words -> bincode(ShardProof) -> words, and the
    bytes it writes are the committed golden wire bytes"""
    import hashlib
    import json
    from tests import machines as M
    from tools import gen_golden_proofs as GG
    _build()
    name, spec, log_stack, mlr, seed, nq, pw, bpw, gpw = GG.CASES[2]
    rng_case = GG.bincode_case(*GG.CASES[2])
    # the same seeded proof as the golden generator
    blob, heights, _, _, names, _, words, _ = GG.prove_case(spec, log_stack, mlr, seed, nq, pw, bpw, gpw)
    job = _u32(log_stack, mlr, 2, nq, len(names))
    for nm, h, (a, b) in zip(names, heights, M.widths(blob)):
        raw = nm.encode()
        job += _u32(len(raw)) + raw + b"\0" * (-len(raw) % 4) + _u32(h & 0xffffffff, h >> 32, a, b)
    job += _u32(words.size) + words.astype("<u4").tobytes()
    jf, out = tmp_path / "job.bin", tmp_path / "proof.bincode"
    jf.write_bytes(job)
    r = subprocess.run([os.path.join(ROOT, "examples", "proof_wire"), str(jf), str(out)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    assert "round trip identical" in r.stdout
    assert hashlib.sha256(out.read_bytes()).hexdigest() == rng_case["bincode_sha256"]
    gold = {c["name"]: c for c in json.load(open(os.path.join(ROOT, "tests", "golden", "shard_proofs_bincode.json")))["cases"]}
    assert gold[name]["bincode_sha256"] == rng_case["bincode_sha256"]


def _u32(*xs):
    return struct.pack("<%dI" % len(xs), *[int(x) for x in xs])


def _vec(a):
    a = np.ascontiguousarray(a, dtype=np.uint32).reshape(-1)
    return _u32(a.size) + a.astype("<u4").tobytes()


@pytest.mark.gpu
def test_example_host_reproduces_golden_proof(tmp_path):
    from tests import golden_util as G
    _build()
    case = [c for c in G.cases() if c["name"] == "four_chips"][0]
    blob, heights, mains, preps, pv, names, ch = G.inputs_of(case)
    params = [case["log_stacking_height"], case["max_log_row_count"], 2, case["num_queries"], case["pow_bits"], case["batch_pow_bits"],
              case["gkr_pow_bits"], 0]
    buf = _u32(0x42315053, 1) + _u32(*params) + _u32(len(heights))
    for name, h, m, p in zip(names, heights, mains, preps):
        nb = name.encode()
        buf += _u32(len(nb)) + nb + b"\0" * (-len(nb) % 4) + _u32(m.shape[0], 0 if p is None else p.shape[0], h)
    prep_dense = np.concatenate([np.ascontiguousarray(p).reshape(-1) for p in preps if p is not None and p.size] or [np.zeros(0, np.uint32)])
    main_dense = np.concatenate([np.ascontiguousarray(m).reshape(-1) for m in mains if m.size])
    buf += _vec(blob) + _vec(pv) + np.ascontiguousarray(ch.st, dtype="<u4").tobytes() + _vec(prep_dense) + _vec(main_dense)
    fin, fout = tmp_path / "in.bin", tmp_path / "out.bin"
    fin.write_bytes(buf)
    r = subprocess.run([EXE, str(fin), str(fout)], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr
    out = np.frombuffer(fout.read_bytes(), dtype="<u4")
    pc, n = out[:8], int(out[8])
    words, st = out[9:9 + n], out[9 + n:9 + n + 34]
    G.check_words(case, pc, words, st)
