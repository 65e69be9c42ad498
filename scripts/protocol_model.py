#!/usr/bin/env python
"""CPU-only randomized model of the forward kernel's barrier protocol (csrc/fa_fwd_sm90.cuh).

The three roles -- the TMA producer and the two softmax / wgmma warpgroups -- are Python generators that mirror the
kernel's control flow statement by statement (same barriers, arrival counts, ring-entry and parity bookkeeping, same
release points) and yield at every mbarrier wait.  A random scheduler interleaves them; TMA loads complete after random
delays, and each warpgroup's wgmma groups complete in order after random delays (wgmma.wait_group N returns once at most
N groups are still in flight).  One CTA walks a list of work items, as the persistent schedule does; a list of one item
is the one-CTA-per-item schedule.  An item with no KV tiles is skipped by the producer; the softmax warpgroups skip it
too, except for a live one (`empty`: every dense and cache item, and a variable-length item inside its sequence), for
which they write O = 0 and LSE = +inf (-inf for a split-KV partial) without waiting on any barrier.  For a KV-cache
item (`vtail`) both warpgroups also WRITE into the ring: they zero the V rows past the sequence's keys in the slot of
its last tile before PV reads it.  The stores take time (they span a scheduling point), and are legal only between
that slot's kv_full and the warpgroup's release.  Shadow state catches what a deadlock-only test would miss:

  * a Q buffer or ring slot overwritten by TMA while an issued, unfinished wgmma still reads it, or while a warpgroup
    still stores into it,
  * a warpgroup storing into a slot that no longer holds the tile it waited for,
  * a wgmma that reads a buffer holding the wrong (item, tile) -- a release that came too early or a parity slip,
  * every warpgroup consumes every item's K/V tiles exactly once and in order, and finishes every item.

With `fp8` (the FP8-cache modes) a fourth role joins: the converter (producer warps 1-3).  The TMA lane then loads
each K/V tile into a ring of raw e4m3 tiles (raw_full / raw_empty); the converter waits on the entry's raw_full and
on its K/V slot's kv_empty, widens the raw tile into the slot (stores spanning a scheduling point), arrives on
kv_full and releases the raw tile.  The softmax warpgroups are unchanged, but do not zero V tails (the converter
writes those rows as zeros).  Shadow state adds: a raw tile overwritten by TMA while the converter reads it, and the
converter storing into a slot a wgmma still reads.

DenseFp8Sim models kDenseFp8 (Q, K and V in e4m3) with three rings of their own depths and barriers: K (nk slots,
filled by TMA: k_full one arrival, k_empty one per warpgroup), raw V (nraw slots, filled by TMA: raw_full one arrival;
raw_empty one per converter warp) and V^T (nvt slots, written by the converter: vt_full one arrival per converter warp,
vt_empty one per warpgroup).  Tile j of the running tile count takes slot j % depth of each ring.  The three converter
warps are roles of their own: each waits on the tile's raw_full and its V^T slot's vt_empty, stores its part (spanning
a scheduling point), then arrives on vt_full and raw_empty.  Shadow state adds: a V^T slot read by a wgmma before every
converter warp's part of that tile is stored, or while one still stores into it, and a converter warp storing into a
slot a wgmma still reads.  With `empty` (kVarlenFp8) an item without tiles is written only when listed there; the
others lie past their sequence's end and every role skips them, as in Sim.

Run:  python scripts/protocol_model.py [trials]      (exit code 0 = no violation found)
"""
import random
import sys


class Bar:
    def __init__(self, name, count):
        self.name, self.count, self.pending, self.phase = name, count, count, 0

    def arrive(self):
        self.pending -= 1
        assert self.pending >= 0, f"{self.name}: too many arrivals"
        if self.pending == 0:
            self.pending = self.count
            self.phase ^= 1

    def done(self, parity):          # try_wait.parity
        return self.phase != parity


class Sim:
    def __init__(self, items, nstage, rng, empty=None, vtail=(), fp8=False, nraw=2):
        self.items, self.N, self.rng = items, nstage, rng     # items: KV tiles per work item (0 = none)
        # items with 0 tiles whose rows are still written; None: all of them (the dense and cache rule), a list: those
        # of a packed batch that lie inside their sequence (the others are skipped by every role)
        self.empty = {i for i, n in enumerate(items) if n == 0} if empty is None else set(empty)
        self.fp8, self.R = fp8, nraw                          # FP8 cache: raw ring of nraw tiles + the converter
        # items whose last V tile the consumers zero in place (FP8: the converter zeroes it, not the consumers)
        self.vtail = set() if fp8 else set(vtail)
        self.raw_full = [Bar(f"raw_full{i}", 1) for i in range(nraw)]
        self.raw_empty = [Bar(f"raw_empty{i}", 1) for i in range(nraw)]   # one arrival per converter warp
        self.raw_buf = [None] * nraw
        self.raw_readers = [0] * nraw
        self.q_full = Bar("q_full", 1)
        self.q_empty = Bar("q_empty", 2)                      # one arrival per warpgroup (per warp in the kernel)
        self.kv_full = [Bar(f"kv_full{i}", 1) for i in range(nstage)]
        self.kv_empty = [Bar(f"kv_empty{i}", 2) for i in range(nstage)]
        # shadow state
        self.q_buf = None                                     # item resident in the Q buffer; "busy" while TMA writes
        self.kv_buf = [None] * nstage                         # (item, j, 'K'|'V')
        self.q_readers = 0
        self.kv_readers = [0] * nstage
        self.kv_writers = [0] * nstage                        # warpgroups storing into the slot
        self.tma_q = []                                       # in-flight loads: [remaining, fn]
        self.mma_q = [[], []]                                 # per warpgroup, in order: [remaining, fn_done]
        self.seen = [[], []]                                  # (item, j) consumed, per warpgroup
        self.finished = [[], []]

    # ---- async engines ----
    def tma(self, fn):
        self.tma_q.append([self.rng.randint(1, 12), fn])

    def tick(self):
        for e in self.tma_q:
            e[0] -= 1
        for e in [e for e in self.tma_q if e[0] <= 0]:
            self.tma_q.remove(e)
            e[1]()
        for q in self.mma_q:
            if q:
                q[0][0] -= 1
                if q[0][0] <= 0:
                    q.pop(0)[1]()

    def in_flight(self, t):
        return len(self.mma_q[t])

    # ---- roles ----
    def producer(self):
        N, ent, qcnt = self.N, 0, 0
        for item, n in enumerate(self.items):
            if n == 0:
                continue
            if qcnt > 0:
                yield lambda p=(qcnt - 1) & 1: self.q_empty.done(p)
            qcnt += 1
            assert self.q_readers == 0, f"Q buffer overwritten while a wgmma reads it (item {item})"
            self.q_buf = "busy"

            def q_landed(item=item):
                assert self.q_readers == 0, "Q buffer written under a reader"
                self.q_buf = item
                self.q_full.arrive()
            self.tma(q_landed)
            for j in range(n):
                for kv in "KV":
                    if self.fp8:                              # the raw tile; the converter fills the slot
                        rs = ent % self.R
                        yield lambda s=rs, p=((ent // self.R) & 1) ^ 1: self.raw_empty[s].done(p)
                        assert self.raw_readers[rs] == 0, f"raw tile {rs} overwritten while the converter reads it"
                        self.raw_buf[rs] = "busy"

                        def raw_landed(rs=rs, tag=(item, j, kv)):
                            assert self.raw_readers[rs] == 0, "raw tile written under the converter"
                            self.raw_buf[rs] = tag
                            self.raw_full[rs].arrive()
                        self.tma(raw_landed)
                        ent += 1
                        continue
                    slot = ent % N
                    yield lambda s=slot, p=((ent // N) & 1) ^ 1: self.kv_empty[s].done(p)
                    assert self.kv_readers[slot] == 0, f"slot {slot} overwritten while a wgmma reads it"
                    assert self.kv_writers[slot] == 0, f"slot {slot} overwritten while a warpgroup stores into it"
                    self.kv_buf[slot] = "busy"

                    def kv_landed(slot=slot, tag=(item, j, kv)):
                        assert self.kv_readers[slot] == 0, "slot written under a reader"
                        assert self.kv_writers[slot] == 0, "slot written under a warpgroup's stores"
                        self.kv_buf[slot] = tag
                        self.kv_full[slot].arrive()
                    self.tma(kv_landed)
                    ent += 1

    def converter(self):
        """Producer warps 1-3 of the FP8-cache modes: raw ring entry -> K/V ring slot, over the TMA lane's entries."""
        N, R, ent = self.N, self.R, 0
        for item, n in enumerate(self.items):
            if n == 0:
                continue
            for j in range(n):
                for kv in "KV":
                    slot, rs, tag = ent % N, ent % R, (item, j, kv)
                    yield lambda s=rs, p=(ent // R) & 1: self.raw_full[s].done(p)
                    yield lambda s=slot, p=((ent // N) & 1) ^ 1: self.kv_empty[s].done(p)
                    # widen: read the raw tile, store into the slot; the stores span a scheduling point
                    assert self.raw_buf[rs] == tag, f"converter: raw tile {rs} holds {self.raw_buf[rs]}, not {tag}"
                    assert self.kv_readers[slot] == 0, f"converter stores into slot {slot} while a wgmma reads it"
                    self.raw_readers[rs] += 1
                    self.kv_writers[slot] += 1
                    self.kv_buf[slot] = "converting"
                    yield lambda: True
                    assert self.kv_readers[slot] == 0, f"slot {slot} read by a wgmma under the converter's stores"
                    self.kv_buf[slot] = tag
                    self.kv_writers[slot] -= 1
                    self.raw_readers[rs] -= 1
                    self.kv_full[slot].arrive()               # after the last store (and its proxy fence)
                    self.raw_empty[rs].arrive()
                    ent += 1

    def consumer(self, t):
        N, ent, qcnt = self.N, 0, 0

        def issue(reads):
            """One wgmma group reading the Q buffer and/or ring slots; the reads last until the group completes."""
            for what, slot, tag in reads:
                if what == "Q":
                    assert self.q_buf == tag, f"wg{t}: Q buffer holds {self.q_buf}, expected item {tag}"
                    self.q_readers += 1
                else:
                    assert self.kv_buf[slot] == tag, f"wg{t}: slot {slot} holds {self.kv_buf[slot]}, expected {tag}"
                    self.kv_readers[slot] += 1

            def done():
                for what, slot, _ in reads:
                    if what == "Q":
                        self.q_readers -= 1
                    else:
                        self.kv_readers[slot] -= 1
            self.mma_q[t].append([self.rng.randint(1, 6), done])

        def wait_group(k):
            yield lambda: self.in_flight(t) <= k

        def wait_full(e):
            yield lambda s=e % N, p=(e // N) & 1: self.kv_full[s].done(p)

        def store_into(slot, tag):
            """The warpgroup's zeroing stores into a ring slot: they start and end at different scheduling points."""
            assert self.kv_buf[slot] == tag, f"wg{t}: stores into slot {slot} holding {self.kv_buf[slot]}, not {tag}"
            self.kv_writers[slot] += 1
            yield lambda: True
            assert self.kv_buf[slot] == tag, f"wg{t}: slot {slot} refilled under its stores ({self.kv_buf[slot]})"
            self.kv_writers[slot] -= 1

        for item, n in enumerate(self.items):
            if n == 0:
                if item in self.empty:                        # epilogue only: no barrier is touched
                    yield lambda: True
                    self.finished[t].append(item)
                continue
            yield lambda p=qcnt & 1: self.q_full.done(p)
            qcnt += 1
            # KV tile 0: S_0
            last_q_user = (0 == n - 1)
            yield from wait_full(ent)
            issue([("Q", None, item), ("KV", ent % N, (item, 0, "K"))])
            self.seen[t].append((item, 0))
            yield from wait_group(0)
            self.kv_empty[ent % N].arrive()
            if last_q_user:
                self.q_empty.arrive()
            # KV tiles 1 .. n-1: S_j and PV_{j-1} in flight together
            for j in range(1, n):
                ek, ev = ent + 2 * j, ent + 2 * j - 1
                yield from wait_full(ek)
                issue([("Q", None, item), ("KV", ek % N, (item, j, "K"))])
                self.seen[t].append((item, j))
                yield from wait_full(ev)
                issue([("KV", ev % N, (item, j - 1, "V"))])
                yield from wait_group(1)
                self.kv_empty[ek % N].arrive()
                last_q_user = (j == n - 1)
                if last_q_user:
                    self.q_empty.arrive()
                yield from wait_group(0)
                self.kv_empty[ev % N].arrive()
            ev = ent + 2 * n - 1
            yield from wait_full(ev)
            if item in self.vtail:                            # zero the V rows past the keys, then PV reads the slot
                yield from store_into(ev % N, (item, n - 1, "V"))
            issue([("KV", ev % N, (item, n - 1, "V"))])
            yield from wait_group(0)
            self.kv_empty[ev % N].arrive()
            ent += 2 * n
            self.finished[t].append(item)

    def run(self, max_steps=200000):
        roles = [self.producer(), self.consumer(0), self.consumer(1)] + ([self.converter()] if self.fp8 else [])
        nr = len(roles)
        waits = [None] * nr
        alive = [True] * nr
        for _ in range(max_steps):
            ready = [i for i in range(nr) if alive[i] and (waits[i] is None or waits[i]())]
            busy = bool(self.tma_q) or any(self.mma_q)
            if not ready and not busy:
                if not any(alive):
                    break
                raise AssertionError("deadlock: " + ", ".join(f"role{i}" for i in range(nr) if alive[i]))
            if ready and (not busy or self.rng.random() < 0.6):
                i = self.rng.choice(ready)
                try:
                    waits[i] = next(roles[i])
                except StopIteration:
                    alive[i] = False
                    waits[i] = None
            else:
                self.tick()
        else:
            raise AssertionError("did not finish")
        want = [(it, j) for it, n in enumerate(self.items) for j in range(n)]
        done = [it for it, n in enumerate(self.items) if n > 0 or it in self.empty]
        for t in range(2):
            assert self.seen[t] == want, f"wg{t} consumed {self.seen[t]}, expected {want}"
            assert self.finished[t] == done


class DenseFp8Sim:
    """kDenseFp8 / kVarlenFp8: the TMA lane (Q, K, raw V), three converter warps (raw V -> V^T) and the two softmax
    warpgroups.  `empty` as Sim's: the tile-less items whose rows are written (default: every one)."""
    WARPS = 3                                                 # converter warps (producer warps 1-3)

    def __init__(self, items, nk, nraw, nvt, rng, empty=None):
        self.items, self.NK, self.R, self.V, self.rng = items, nk, nraw, nvt, rng
        self.empty = {i for i, n in enumerate(items) if n == 0} if empty is None else set(empty)
        self.q_full, self.q_empty = Bar("q_full", 1), Bar("q_empty", 2)
        self.k_full = [Bar(f"k_full{i}", 1) for i in range(nk)]
        self.k_empty = [Bar(f"k_empty{i}", 2) for i in range(nk)]
        self.raw_full = [Bar(f"raw_full{i}", 1) for i in range(nraw)]
        self.raw_empty = [Bar(f"raw_empty{i}", self.WARPS) for i in range(nraw)]
        self.vt_full = [Bar(f"vt_full{i}", self.WARPS) for i in range(nvt)]
        self.vt_empty = [Bar(f"vt_empty{i}", 2) for i in range(nvt)]
        # shadow state
        self.q_buf, self.q_readers = None, 0
        self.k_buf, self.k_readers = [None] * nk, [0] * nk
        self.raw_buf, self.raw_readers = [None] * nraw, [0] * nraw
        self.vt_part = [[None] * self.WARPS for _ in range(nvt)]   # the tile each warp's part of the slot holds
        self.vt_readers, self.vt_writers = [0] * nvt, [0] * nvt
        self.tma_q, self.mma_q = [], [[], []]
        self.seen, self.finished = [[], []], [[], []]

    tma = Sim.tma
    tick = Sim.tick
    in_flight = Sim.in_flight

    def producer(self):
        NK, R, tile, qcnt = self.NK, self.R, 0, 0
        for item, n in enumerate(self.items):
            if n == 0:
                continue
            if qcnt > 0:
                yield lambda p=(qcnt - 1) & 1: self.q_empty.done(p)
            qcnt += 1
            assert self.q_readers == 0, f"Q buffer overwritten while a wgmma reads it (item {item})"
            self.q_buf = "busy"

            def q_landed(item=item):
                assert self.q_readers == 0, "Q buffer written under a reader"
                self.q_buf = item
                self.q_full.arrive()
            self.tma(q_landed)
            for j in range(n):
                ks, rs, tag = tile % NK, tile % R, (item, j)
                yield lambda s=ks, p=((tile // NK) & 1) ^ 1: self.k_empty[s].done(p)
                assert self.k_readers[ks] == 0, f"K slot {ks} overwritten while a wgmma reads it"
                self.k_buf[ks] = "busy"

                def k_landed(ks=ks, tag=tag):
                    assert self.k_readers[ks] == 0, "K slot written under a reader"
                    self.k_buf[ks] = tag
                    self.k_full[ks].arrive()
                self.tma(k_landed)
                yield lambda s=rs, p=((tile // R) & 1) ^ 1: self.raw_empty[s].done(p)
                assert self.raw_readers[rs] == 0, f"raw tile {rs} overwritten while the converter reads it"
                self.raw_buf[rs] = "busy"

                def raw_landed(rs=rs, tag=tag):
                    assert self.raw_readers[rs] == 0, "raw tile written under the converter"
                    self.raw_buf[rs] = tag
                    self.raw_full[rs].arrive()
                self.tma(raw_landed)
                tile += 1

    def _store_vt(self, w, vs, rs, tag):
        """Converter warp w's part of the transpose of raw tile rs into V^T slot vs: the stores span a scheduling
        point."""
        assert self.raw_buf[rs] == tag, f"converter {w}: raw tile {rs} holds {self.raw_buf[rs]}, not {tag}"
        assert self.vt_readers[vs] == 0, f"converter {w} stores into V^T slot {vs} while a wgmma reads it"
        self.raw_readers[rs] += 1
        self.vt_writers[vs] += 1
        self.vt_part[vs][w] = "converting"
        yield lambda: True
        assert self.vt_readers[vs] == 0, f"V^T slot {vs} read by a wgmma under converter {w}'s stores"
        self.vt_part[vs][w] = tag
        self.vt_writers[vs] -= 1
        self.raw_readers[rs] -= 1

    def converter(self, w):
        R, V, tile = self.R, self.V, 0
        for item, n in enumerate(self.items):
            for j in range(n):
                rs, vs, tag = tile % R, tile % V, (item, j)
                yield lambda s=rs, p=(tile // R) & 1: self.raw_full[s].done(p)
                yield lambda s=vs, p=((tile // V) & 1) ^ 1: self.vt_empty[s].done(p)
                yield from self._store_vt(w, vs, rs, tag)
                self.vt_full[vs].arrive()                     # after the last store (and its proxy fence)
                self.raw_empty[rs].arrive()
                tile += 1

    def consumer(self, t):
        NK, V, ent, qcnt = self.NK, self.V, 0, 0

        def issue(reads):
            for what, slot, tag in reads:
                if what == "Q":
                    assert self.q_buf == tag, f"wg{t}: Q buffer holds {self.q_buf}, expected item {tag}"
                    self.q_readers += 1
                elif what == "K":
                    assert self.k_buf[slot] == tag, f"wg{t}: K slot {slot} holds {self.k_buf[slot]}, expected {tag}"
                    self.k_readers[slot] += 1
                else:
                    assert self.vt_writers[slot] == 0 and self.vt_part[slot] == [tag] * self.WARPS, \
                        f"wg{t}: V^T slot {slot} holds {self.vt_part[slot]}, expected {tag}"
                    self.vt_readers[slot] += 1

            def done():
                for what, slot, _ in reads:
                    if what == "Q":
                        self.q_readers -= 1
                    elif what == "K":
                        self.k_readers[slot] -= 1
                    else:
                        self.vt_readers[slot] -= 1
            self.mma_q[t].append([self.rng.randint(1, 6), done])

        def wait_group(k):
            yield lambda: self.in_flight(t) <= k

        def wait_k(e):
            yield lambda s=e % NK, p=(e // NK) & 1: self.k_full[s].done(p)

        def wait_vt(e):
            yield lambda s=e % V, p=(e // V) & 1: self.vt_full[s].done(p)

        for item, n in enumerate(self.items):
            if n == 0:
                if item in self.empty:                        # live without tiles: epilogue only, no barrier
                    yield lambda: True
                    self.finished[t].append(item)
                continue                                      # else past its sequence's end: skipped
            yield lambda p=qcnt & 1: self.q_full.done(p)
            qcnt += 1
            yield from wait_k(ent)
            issue([("Q", None, item), ("K", ent % NK, (item, 0))])
            self.seen[t].append((item, 0))
            yield from wait_group(0)
            self.k_empty[ent % NK].arrive()
            if n == 1:
                self.q_empty.arrive()
            for j in range(1, n):
                ek, ev = ent + j, ent + j - 1
                yield from wait_k(ek)
                issue([("Q", None, item), ("K", ek % NK, (item, j))])
                self.seen[t].append((item, j))
                yield from wait_vt(ev)
                issue([("VT", ev % V, (item, j - 1))])
                yield from wait_group(1)
                self.k_empty[ek % NK].arrive()
                if j == n - 1:
                    self.q_empty.arrive()
                yield from wait_group(0)
                self.vt_empty[ev % V].arrive()
            ev = ent + n - 1
            yield from wait_vt(ev)
            issue([("VT", ev % V, (item, n - 1))])
            yield from wait_group(0)
            self.vt_empty[ev % V].arrive()
            ent += n
            self.finished[t].append(item)

    def run(self, max_steps=200000):
        roles = [self.producer(), self.consumer(0), self.consumer(1)] + [self.converter(w) for w in range(self.WARPS)]
        nr = len(roles)
        waits, alive = [None] * nr, [True] * nr
        for _ in range(max_steps):
            ready = [i for i in range(nr) if alive[i] and (waits[i] is None or waits[i]())]
            busy = bool(self.tma_q) or any(self.mma_q)
            if not ready and not busy:
                if not any(alive):
                    break
                raise AssertionError("deadlock: " + ", ".join(f"role{i}" for i in range(nr) if alive[i]))
            if ready and (not busy or self.rng.random() < 0.6):
                i = self.rng.choice(ready)
                try:
                    waits[i] = next(roles[i])
                except StopIteration:
                    alive[i] = False
                    waits[i] = None
            else:
                self.tick()
        else:
            raise AssertionError("did not finish")
        want = [(it, j) for it, n in enumerate(self.items) for j in range(n)]
        done = [it for it, n in enumerate(self.items) if n > 0 or it in self.empty]
        for t in range(2):
            assert self.seen[t] == want, f"wg{t} consumed {self.seen[t]}, expected {want}"
            assert self.finished[t] == done


def random_dense_fp8(rng):
    """kDenseFp8: the dense items of random_items and ring depths (K, raw V, V^T), the shipped 4 / 3 / 4 and 8 / 4 / 8
    among them."""
    depths = rng.choice([(4, 3, 4), (8, 4, 8), (1, 1, 1), (2, 3, 1), (3, 1, 2)])
    return random_items(rng), depths


def random_varlen_fp8(rng):
    """kVarlenFp8: the items of a packed batch as random_varlen_items draws them -- past a sequence's end (skipped by
    every role), inside it without a key (causal Sq_b > Sk_b, or Sk_b = 0: written without a barrier), with tiles --
    and ring depths as random_dense_fp8.  Returns (items, empty, depths)."""
    depths = rng.choice([(4, 3, 4), (8, 4, 8), (1, 1, 1), (2, 3, 1), (3, 1, 2)])
    items, empty = random_varlen_items(rng)
    return items, empty, depths


def random_items(rng):
    """Tiles per item of a dense problem.  Items without tiles (causal rows above the first key when Sq > Sk, or a split
    past a Q tile's causal diagonal) are live: Sim's default writes their rows."""
    kind = rng.choice(["one", "causal", "noncausal", "split"])
    if kind == "one":
        return [rng.randint(1, 8)]
    items = []
    for _ in range(rng.randint(1, 9)):
        if kind == "causal":
            items.append(rng.randint(0, 6))
        elif kind == "noncausal":
            items.append(4)
        else:
            items.append(rng.choice([0, 1, 2, 3]))
    return items


def random_varlen_items(rng):
    """Items of a variable-length batch: tiles per item, and the items that lie inside their sequence but see no key
    (causal Sq_b > Sk_b, or Sk_b = 0).  Items past a sequence's end are skipped by every role, like a 0 here."""
    items, empty = [], []
    for i in range(rng.randint(1, 12)):
        kind = rng.random()
        if kind < 0.3:
            items.append(0)
            empty.append(i)
        elif kind < 0.45:
            items.append(0)
        else:
            items.append(rng.randint(1, 6))
    return items, empty


def random_cache_items(rng):
    """Items of a KV-cache problem: tiles per item (0 = a split past the sequence's keys, or a row block that sees
    none: its rows are still written), and the items whose last tile holds the sequence's last key with slots past
    it, whose V rows the consumers zero."""
    items, empty, vtail = [], [], []
    for i in range(rng.randint(1, 12)):
        n = rng.choice([0, 0, 1, 2, 3, 5])
        items.append(n)
        if n == 0:
            empty.append(i)
        elif rng.random() < 0.7:
            vtail.append(i)
    return items, empty, vtail


def random_varlen_cache_items(rng):
    """Items of a variable-length batch against a KV cache (kVarlenCache): items past a sequence's end, skipped by
    every role (0, not empty); items inside it whose rows see no key (cached length 0 without appended keys, or causal
    rows above the first key), written without a barrier (0, empty); items with tiles, most of which end on a page
    with slots past the sequence's keys, whose V rows the consumers zero (vtail)."""
    items, empty, vtail = [], [], []
    for i in range(rng.randint(1, 12)):
        kind = rng.random()
        if kind < 0.25:
            items.append(0)
        elif kind < 0.45:
            items.append(0)
            empty.append(i)
        else:
            items.append(rng.randint(1, 6))
            if rng.random() < 0.7:
                vtail.append(i)
    return items, empty, vtail


def random_fp8_cache_items(rng, varlen):
    """Items of an FP8-cache problem (kCacheFp8, or kVarlenCacheFp8 when `varlen`): those of its 16-bit mode -- items
    skipped by every role, items without tiles whose rows are still written, items whose last tile has rows past the
    sequence's keys (which the converter writes as zeros) -- and a raw-ring depth."""
    items, empty, vtail = random_varlen_cache_items(rng) if varlen else random_cache_items(rng)
    return items, empty, vtail, rng.choice([2, 4])


def main():
    trials = int(sys.argv[1]) if len(sys.argv) > 1 else 3000
    for trial in range(trials):
        rng = random.Random(1000003 + trial)
        Sim(random_items(rng), rng.choice([4, 8]), rng).run()
        items, empty = random_varlen_items(rng)
        Sim(items, rng.choice([4, 8]), rng, empty).run()
        items, empty, vtail = random_cache_items(rng)
        Sim(items, rng.choice([4, 8]), rng, empty, vtail).run()
        items, empty, vtail = random_varlen_cache_items(rng)
        Sim(items, rng.choice([4, 8]), rng, empty, vtail).run()
        for varlen in (False, True):
            items, empty, vtail, nraw = random_fp8_cache_items(rng, varlen)
            Sim(items, rng.choice([4, 8]), rng, empty, vtail, fp8=True, nraw=nraw).run()
        rng8 = random.Random(2000003 + trial)             # kDenseFp8, on a generator of its own
        items, depths = random_dense_fp8(rng8)
        DenseFp8Sim(items, *depths, rng8).run()
        rngv = random.Random(3000003 + trial)             # kVarlenFp8, on a generator of its own
        items, empty, depths = random_varlen_fp8(rngv)
        DenseFp8Sim(items, *depths, rngv, empty).run()
    print(f"{trials} trials: no violation")


if __name__ == "__main__":
    main()
