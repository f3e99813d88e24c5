"""Contexts that prove the inputs of the whole-proof verifiers: Core proves the shards of a core proof under one verifying key, Rec
proves recursion proofs under distinct keys with a recursion vk map over them.  Machines are (blob, heights, names, chip specs); every
shard draws its traces with machines.traces."""
import numpy as np

from tests import core_chain as CC
from tests import gpu_prove as GP
from tests import machines as M
from tests import oracle_lib as O
from tests import recursion_ref as RR


def specs_machine(chips):
    """-> (blob, heights, names, chips) of hand-written chips"""
    blob, heights, _, _, _, names = M.spec_machine(np.random.default_rng(1), chips)
    return blob, heights, names, chips


def workload_specs_machine(workload, mlr, scale):
    """-> (blob, heights, names, specs) of a benchmark machine (machine seed 42)"""
    from sp1_b200 import workload as W
    mach = W.synthetic_machine(workload, seed=42, max_log_rows=mlr, scale=scale)
    return mach["blob"], [s.h for s in mach["specs"]], list(mach["names"]), mach["specs"]


class Core:
    """a context + machine proving shards of one program under one verifying key"""

    def __init__(self, machine, log_stack, mlr, prm=M.SMALL, seed=5, **ctx):
        from sp1_b200 import Lib
        self.blob, self.heights, self.names, self.specs = machine
        self.log_stack, self.mlr, self.prm, self.seed = log_stack, mlr, prm, seed
        self.lib = Lib(0, log_stacking_height=log_stack, max_log_row_count=mlr, **prm, **ctx)
        self.mach = self.lib.machine_create(self.blob)
        self.pc, self.prep_round = GP.commit_prep(self.lib, M.traces(self.specs, seed, 0)[1])

    def start(self, tail):
        from sp1_b200.lib import HostChallenger
        hc = HostChallenger(); hc.observe(self.pc); hc.observe(tail)
        return hc.st.copy()

    def prove(self, pvs, tail, before_each=None):
        """-> (words per shard, final prover state per shard); tail, pvs: canonical.  before_each(): called before every shard's proof"""
        tail = O.to_monty(np.array(tail))
        words, finals = [], []
        for pv in pvs:
            mains, _ = M.traces(self.specs, self.seed, CC.pv0_of(pv))
            st = self.start(tail)
            if before_each is not None:
                before_each()
            words.append(GP.prove(self.lib, self.mach, self.prep_round, mains, self.heights, self.names, O.to_monty(np.array(pv)), st))
            finals.append(st)
        return words, finals, tail

    def verify(self, words, tail, heights=None, threads=0):
        hs = [self.heights] * len(words) if heights is None else heights
        return self.lib.verify_core_proof(self.mach, self.pc, tail, hs, self.names, words, host_threads=threads)

    def close(self):
        if self.prep_round is not None:
            self.lib.jagged_round_free(self.prep_round)
        self.lib.machine_free(self.mach)
        self.lib.close()


class Rec:
    """a context + recursion machine proving shards under distinct verifying keys, with a vk map over those keys"""

    def __init__(self, machine, log_stack, mlr, n_keys=6, prm=M.SMALL, seed=5, extra_keys=20):
        from sp1_b200 import Lib
        from sp1_b200 import lib as B
        self.blob, self.heights, self.names, self.specs = machine
        self.log_stack, self.mlr, self.prm, self.seed = log_stack, mlr, prm, seed
        self.lib = Lib(0, log_stacking_height=log_stack, max_log_row_count=mlr, **prm)
        self.mach = self.lib.machine_create(self.blob)
        self.pc, self.prep_round = GP.commit_prep(self.lib, M.traces(self.specs, seed, 0)[1])
        rng = np.random.default_rng(300 + seed)
        self.keys = [np.concatenate([self.pc, O.rand_field(rng, 18), np.zeros(6, np.uint32)]) for _ in range(n_keys + 1)]
        self.outsider = self.keys.pop()   # a key the map does not hold
        self.digests = np.concatenate([np.stack([B.vk_hash(k[:8], k[8:]) for k in self.keys]), O.rand_field(rng, (extra_keys, 8))])
        self.vks = self.lib.recursion_vks(self.digests)
        self.vks_off = self.lib.recursion_vks(self.digests, vk_verification=False)
        self.root = self.vks.root()
        self.sp1 = O.rand_field(rng, 8)
        self.rng = rng

    def pv(self, **faults):
        """valid recursion public values, then the faults: vk_root, is_complete, digest (a word of the digest changed after hashing)"""
        from sp1_b200 import lib as B
        pv = O.rand_field(self.rng, 187)
        pv[0] = O.to_monty(int(self.rng.integers(1, 1 << 20)))
        pv[136:144] = self.sp1
        pv[144:152] = self.root
        pv[168] = RR.ONE
        if faults.get("vk_root"):
            pv[147] = (int(pv[147]) + 1) % O.P
        if faults.get("is_complete"):
            pv[168] = 0
        pv[175:183] = B.recursion_pv_digest(pv)
        if faults.get("digest"):
            pv[176] = (int(pv[176]) + 1) % O.P
        return pv

    def prove(self, key, pv):
        from sp1_b200.lib import HostChallenger
        mains, _ = M.traces(self.specs, self.seed, int(O.from_monty(pv[:1])[0]))
        hc = HostChallenger(); hc.observe(key)
        st = hc.st.copy()
        return GP.prove(self.lib, self.mach, self.prep_round, mains, self.heights, self.names, pv, st), st

    def merkle(self, key):
        from sp1_b200 import lib as B
        return self.vks.open(B.vk_hash(key[:8], key[8:]))

    def verify(self, cases, vks=None, **kw):
        """cases: list of (key, words, merkle proof, expected sp1 digest)"""
        return self.lib.verify_compressed(self.mach, vks or self.vks, [c[0] for c in cases], [self.heights] * len(cases), self.names,
                                          [c[1] for c in cases], [c[2] for c in cases], [c[3] for c in cases], **kw)

    def oracle(self, key, words, n_pv, merkle, sp1, vk_verification=True, **kw):
        return RR.verify_compressed(self.blob, self.heights, self.names, self.log_stack, self.mlr, self.prm, key, words, n_pv, self.root,
                                    vk_verification, merkle, sp1, **kw)[0]

    def close(self):
        self.vks.close(); self.vks_off.close()
        if self.prep_round is not None:
            self.lib.jagged_round_free(self.prep_round)
        self.lib.machine_free(self.mach)
        self.lib.close()
