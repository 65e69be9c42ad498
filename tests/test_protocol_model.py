"""CPU: the randomized model of the forward kernel's barrier protocol (scripts/protocol_model.py) -- the roles of
csrc/fa_fwd_sm90.cuh as coroutines under a random scheduler, with shadow state for every shared-memory
buffer.  It must accept the shipped protocol and reject broken ones (mutation check), so that a protocol change is
vetted here before it costs GPU time."""
import os
import random
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "scripts"))
import protocol_model as pm  # noqa: E402


def test_shipped_protocol_has_no_violation():
    for trial in range(400):
        rng = random.Random(1234567 + trial)
        items = pm.random_items(rng)
        pm.Sim(items, rng.choice([4, 8]), rng).run()


def test_model_catches_an_early_release():
    """Mutation: each warpgroup releases the Q buffer after every KV tile instead of after its last S -> the producer
    loads the next item's Q while an S wgmma of the current item still reads it."""
    src = open(os.path.join(ROOT, "scripts", "protocol_model.py")).read()
    needle = "last_q_user = (j == n - 1)"
    assert needle in src
    ns = {"__name__": "mutated_model"}
    exec(compile(src.replace(needle, "last_q_user = True"), "mutated_model", "exec"), ns)
    caught = 0
    for trial in range(60):
        rng = random.Random(99 + trial)
        items = ns["random_items"](rng)
        try:
            ns["Sim"](items, 4, rng).run()
        except AssertionError:
            caught += 1
    assert caught > 10
