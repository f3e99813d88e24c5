"""Stored outputs of the reference's own CUDA kernels (oracle/_ref/libsp1ref.so) on seeded inputs, kept under tests/golden/ so that the
comparison with the reference runs from this repository alone.  Each test module that pins kernels to the reference owns one `Store` (one
JSON file): tests/test_gpu_ref_kernels.py writes tests/golden/ref_kernels.json, tests/test_ref_sumcheck.py tests/golden/ref_sumcheck.json,
tests/test_ref_gkr.py tests/golden/ref_gkr.json, tests/test_ref_zerocheck.py tests/golden/ref_zerocheck.json, tests/test_ref_jagged_eval.py
tests/golden/ref_jagged_eval.json.

Every entry holds the SHA-256 of an output's little-endian u32 words, and the words themselves for the outputs a test reads (keep=True).
With SP1B200_RECORD_REF=1 (and oracle/_ref built) the tests run the reference kernels instead, compare against them directly, and
rewrite their module's file at the end of the module: `SP1B200_RECORD_REF=1 python -m pytest tests/test_gpu_ref_kernels.py`."""
import hashlib
import json
import os

import numpy as np

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
RECORD = os.environ.get("SP1B200_RECORD_REF") == "1"


class Store:
    """the reference outputs of one test module: tests/golden/<name>.json"""

    def __init__(self, name, generator):
        self.path = os.path.join(GOLDEN, name + ".json")
        self.generator = generator
        self._entries = None

    def entries(self):
        if self._entries is None:
            self._entries = {} if RECORD else json.load(open(self.path))["outputs"]
        return self._entries

    def save(self):
        """write the recorded entries (recording runs only)"""
        if RECORD:
            write(self.path, self.entries(), self.generator)


KERNELS = Store("ref_kernels", "tests/test_gpu_ref_kernels.py")
PATH = KERNELS.path


def _digest(a):
    return hashlib.sha256(np.ascontiguousarray(a, np.uint32).astype("<u4").tobytes()).hexdigest()


def _entry(a, keep=False):
    a = np.ascontiguousarray(a, np.uint32)
    e = {"size": int(a.size), "sha256": _digest(a)}
    if keep:
        e["words"] = [int(x) for x in a.reshape(-1)]
    return e


class Ref:
    """one reference output: the live array while recording, the stored entry otherwise"""

    def __init__(self, key, compute, keep=False, store=KERNELS):
        self.key = key
        self.store = store
        if RECORD:
            self.value = np.ascontiguousarray(compute(), np.uint32)
            store.entries()[key] = _entry(self.value, keep)
        elif key not in store.entries():
            raise KeyError(f"{key} is not in {store.path}: record it with SP1B200_RECORD_REF=1 on a machine with oracle/_ref built")

    @property
    def words(self):
        """the output's words (flat); stored for outputs recorded with keep=True"""
        if RECORD:
            return self.value.reshape(-1)
        return np.array(self.store.entries()[self.key]["words"], np.uint32)

    def eq(self, got, part=None, sel=None):
        """got (or got[sel]) equals the reference output (or its part `sel`, stored under `part`) word for word"""
        got = np.asarray(got)
        if sel is not None:
            got = got[sel]
        key = self.key if part is None else f"{self.key}/{part}"
        if RECORD:
            ref = self.value if sel is None else self.value[sel]
            if part is not None:
                self.store.entries()[key] = _entry(ref)
            return ref.size == got.size and bool((ref.reshape(-1) == np.asarray(got, np.uint32).reshape(-1)).all())
        e = self.store.entries()[key]
        return e["size"] == got.size and e["sha256"] == _digest(got)


def save():
    """write the recorded entries of tests/golden/ref_kernels.json (recording runs only)"""
    KERNELS.save()


def write(path, entries, generator="tests/test_gpu_ref_kernels.py"):
    """one output per line"""
    with open(path, "w") as f:
        f.write(f'{{"generator": "{generator} with SP1B200_RECORD_REF=1 (oracle/_ref/libsp1ref.so: the reference\'s '
                'sp1-gpu/crates/sys kernels compiled unmodified by oracle/Makefile)",\n"outputs": {\n')
        f.write(",\n".join(f"{json.dumps(k)}: {json.dumps(v)}" for k, v in sorted(entries.items())))
        f.write("\n}}\n")
