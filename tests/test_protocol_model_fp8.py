"""CPU: the kDenseFp8 part of the barrier-protocol model (scripts/protocol_model.py, DenseFp8Sim) -- K filled by TMA,
V^T by the three converter warps, each ring with its own depth and arrival counts.  It must accept the shipped
protocol at every depth combination it draws and reject the two converter mistakes that break it."""
import os
import random
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "scripts"))
import protocol_model as pm  # noqa: E402

SRC = open(os.path.join(ROOT, "scripts", "protocol_model.py")).read()
WAIT_EMPTY = "                yield lambda s=vs, p=((tile // V) & 1) ^ 1: self.vt_empty[s].done(p)\n"
STORE = "                yield from self._store_vt(w, vs, rs, tag)\n"
ARRIVE = "                self.vt_full[vs].arrive()                     # after the last store (and its proxy fence)\n"


def _mutated(old, new):
    assert SRC.count(old) == 1
    ns = {"__name__": "mutated_model"}
    exec(compile(SRC.replace(old, new), "mutated_model", "exec"), ns)
    return ns


def _caught(ns, trials=80):
    caught = 0
    for trial in range(trials):
        rng = random.Random(4242 + trial)
        items, depths = ns["random_dense_fp8"](rng)
        try:
            ns["DenseFp8Sim"](items, *depths, rng).run()
        except AssertionError:
            caught += 1
    return caught


def test_dense_fp8_protocol_has_no_violation():
    for trial in range(400):
        rng = random.Random(7654321 + trial)
        items, depths = pm.random_dense_fp8(rng)
        pm.DenseFp8Sim(items, *depths, rng).run()


def test_model_catches_converter_arriving_before_its_last_store():
    """Mutation: each converter warp arrives on vt_full before its V^T stores -> PV reads a slot still being written
    (or not yet holding the tile)."""
    assert _caught(_mutated(STORE + ARRIVE, ARRIVE + STORE)) > 10


def test_model_catches_converter_writing_before_the_empty_wait():
    """Mutation: each converter warp stores into its V^T slot before waiting on that slot's vt_empty -> it overwrites a
    tile a PV wgmma still reads, or that the warpgroups have not read yet."""
    assert _caught(_mutated(WAIT_EMPTY + STORE, STORE + WAIT_EMPTY)) > 10


def test_existing_modes_unchanged_by_the_dense_fp8_model():
    """The 16-bit and FP8-cache modes still run on the Sim class and generators they had; main() draws the kDenseFp8
    trials from a generator of their own, so the other modes' random trials are those they were."""
    for trial in range(100):
        rng = random.Random(1000003 + trial)
        pm.Sim(pm.random_items(rng), rng.choice([4, 8]), rng).run()
        items, empty = pm.random_varlen_items(rng)
        pm.Sim(items, rng.choice([4, 8]), rng, empty).run()
        items, empty, vtail = pm.random_cache_items(rng)
        pm.Sim(items, rng.choice([4, 8]), rng, empty, vtail).run()
        for varlen in (False, True):
            items, empty, vtail, nraw = pm.random_fp8_cache_items(rng, varlen)
            pm.Sim(items, rng.choice([4, 8]), rng, empty, vtail, fp8=True, nraw=nraw).run()
