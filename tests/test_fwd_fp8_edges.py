"""The e4m3-wgmma forwards (kDenseFp8, kVarlenFp8, kCacheQkv8, kVarlenCacheQkv8) and the widened FP8-cache forwards
(kCacheFp8, kVarlenCacheFp8) against float64 at tile, k-step, page and split edges, on inputs that make the FP8 checker
decisive.

Why needles.  The FP8 budget (test_fwd_fp8.fp8_reference / compare) allows O about 2^-4 A for the e4m3 rounding of P and
LSE the logit error eta = s 2^-8 sum_d |q k|, about 0.007 at D = 128 on N(0, 0.5^2) inputs.  One key more or less in a
row of N keys moves LSE by about 1/N and O by about |v| / N, so on random inputs the FP8 checker stops seeing a mask or
length off-by-one at N ~ 150 (LSE) or N ~ 20 (O): a decode row against 1,000 keys passes "one key short"
(test_random_decode_row_hides_one_key_short records that).  The needle inputs put each row's softmax mass on one chosen
visible key, so a kernel that drops, shifts or misplaces that key is off by O(1).

Needle inputs.  Key j of every sequence (every kv head) is the e4m3 code CODE = 16 in two dimensions and 0 elsewhere:
a(j) = j % 32, its place in a 32-key PV k-step, and b(j) = 32 + (j // 32) % (D - 32), its k-step; no two keys of a
sequence share both (K <= 32 (D - 32): 1024 keys at D = 64, 3072 at D = 128).  A row whose needle is key n holds CODE
in a(n) and b(n): its logit against n is T = 16 nats (the softmax scale is chosen so), against a key that shares one
of the two dimensions T / 2, against any other key 0.  With at most K / 32 + 32 keys sharing a dimension, the needle
holds at least 0.9 of l at every shape here, and eta = T / 256 keeps the budget near 0.2 A.  All values are exact in
e4m3, so the float64 reference sees what the kernel sees.  V is random: every key its own row.  Rows take their needle
round-robin over: the row's last visible key (K_b - 1, or the causal diagonal i + K_b - Sq); the first key past it
(causal rows only: the mass a diagonal moved by +1 would take); keys 0, 2, 31, 32, 61, 127 and 128 (32-key block and
tile boundaries; 2 and 61 are moved by the PV key order pi, 0 / 31 / 32 / 127 / 128 are not); and a split boundary
where the shape has one.  A fixed position past the row's last visible key falls back to that key.

CPU: the builder puts at least 0.9 of l on every visible needle at every shape below; on those inputs the FP8 budget
rejects the exact result of each wrong problem (causal diagonal +-1, one key short, kv head h % Hkv, a dropped split
partial, V permuted by pi within each 32-key block) and accepts the right one rounded to each output dtype.
GPU: edge sweeps of every e4m3 mode on random and needle inputs and of the widened FP8-cache modes on random inputs
(their 16-bit budget is 16 times tighter), and four kCacheQkv8
/ kVarlenCacheQkv8 workloads at scale (guard buffers, appended pools, three schedules bitwise equal, checker rejection
on the needle run).  Every element within budget, no pass fraction, key-less rows exactly 0 / +inf."""
import math
import os
import subprocess
import sys
import tempfile

import numpy as np
import pytest
import torch

import test_fwd_float64_reference as fr
from test_fwd_float64_reference import W, _decode_lens, assert_guarded, guarded, reference
from test_fwd_fp8 import compare as f8_compare, deq, fp8_reference
from test_kvcache_qkv8 import (FP8, KS, QS, VS, bits, cache_lens_dense, cache_lens_varlen, e4m3, gather,
                               make_pools)
from test_varlen import offsets

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CODE = 16.0                      # e4m3 value of a key's two planted dimensions (exact)
T_NEEDLE = 16.0                  # the needle's logit in nats, against 0 for a key that shares neither dimension
NEEDLE_SCALE = T_NEEDLE / (2 * CODE * CODE * QS * KS)     # softmax_scale: s' (q8 . k8) = T_NEEDLE on the needle
FIXED = (0, 2, 31, 32, 61, 127, 128)
EDGES8 = [1, 31, 32, 33, 63, 64, 65, 96, 127, 128, 129, 160, 255, 256, 257]
PAIRS8 = [(sq, sk) for sq in EDGES8 for sk in EDGES8]
OUT_KINDS = ("bf16", "fp16", "f32")


# ------------------------------------------------------------------ needle inputs -----------------------------------------

def key_dims(j, D):
    """The two planted dimensions of key j: its place in a 32-key k-step and its k-step."""
    return j % 32, 32 + (j // 32) % (D - 32)


def needle_keys(first, n, Hkv, D):
    """Keys [first, first + n) of a sequence, (Hkv, n, D) float: CODE in their two dimensions, 0 elsewhere."""
    assert first + n <= 32 * (D - 32), "keys would share both dimensions"
    j = torch.arange(first, first + n)
    a, b = key_dims(j, D)
    k = torch.zeros((n, D))
    k[torch.arange(n), a] = CODE
    k[torch.arange(n), b] = CODE
    return k[None].expand(Hkv, n, D).contiguous()


def needle_rows(Sq, K, causal, Hq, extra=(), turn=0):
    """(Hq, Sq) needle key of every row of a sequence of K keys, -1 for a row without a visible key.  The (row, head)
    pairs take the positions in turn, starting `turn` places in (so that decode batches cover them across
    sequences)."""
    pos = ["last"] + list(extra) + (["past"] if causal else []) + list(FIXED)
    i = torch.arange(Sq)
    h = torch.arange(Hq)[:, None]
    last = (torch.clamp(i + K - Sq, max=K - 1) if causal else torch.full((Sq,), K - 1)).expand(Hq, Sq)
    cls = (i * Hq + h + turn) % len(pos)
    n = last.clone()
    for c, p in enumerate(pos):
        if p == "last":
            want = last
        elif p == "past":
            want = torch.where(last + 1 < K, last + 1, last)
        else:
            want = torch.clamp(last, max=p)
        n = torch.where(cls == c, want, n)
    return torch.where(last < 0, torch.full_like(n, -1), n)


def needle_q(rows, D):
    """(Hq, Sq, D) float: CODE in the two dimensions of the row's needle key (zeros for a key-less row)."""
    Hq, Sq = rows.shape
    q = torch.zeros((Hq, Sq, D))
    hh, ii = torch.nonzero(rows >= 0, as_tuple=True)
    a, b = key_dims(rows[hh, ii], D)
    q[hh, ii, a] = CODE
    q[hh, ii, b] = CODE
    return q


def needle_seq(Hq, Hkv, Sq, K, D, causal, seed, extra=(), turn=0):
    """One sequence's e4m3 q (Hq, Sq, D), k, v (Hkv, K, D) on the CPU; every key its own random V row."""
    g = torch.Generator().manual_seed(seed)
    q = needle_q(needle_rows(Sq, K, causal, Hq, extra, turn), D).to(FP8)
    return q, needle_keys(0, K, Hkv, D).to(FP8), e4m3(g, VS, Hkv, K, D)


def random_seq(Hq, Hkv, Sq, K, D, seed):
    g = torch.Generator().manual_seed(seed)
    return e4m3(g, QS, Hq, Sq, D), e4m3(g, KS, Hkv, K, D), e4m3(g, VS, Hkv, K, D)


def make_seq(inp, Hq, Hkv, Sq, K, D, causal, seed, extra=(), turn=0):
    """(q8, k8, v8, softmax_scale) of one sequence: inp "needle" or "random" (N(0, 0.5^2) quantized as a caller would)."""
    if inp == "needle":
        return (*needle_seq(Hq, Hkv, Sq, K, D, causal, seed, extra, turn), NEEDLE_SCALE)
    return (*random_seq(Hq, Hkv, Sq, K, D, seed), D ** -0.5)


def needle_mass(q8, k8, causal, scale, rows):
    """(Hq, Sq) share of l on each row's needle key (nan for rows without one), from the exact e4m3 values."""
    Hq, Sq, _ = q8.shape
    Hkv, K, _ = k8.shape
    kk = k8.double()[torch.arange(Hq) // (Hq // Hkv)]
    s = (q8.double() @ kk.transpose(-1, -2)) * (scale * QS * KS)
    vis = (torch.arange(K)[None] <= torch.arange(Sq)[:, None] + K - Sq) if causal else torch.ones(Sq, K).bool()
    p = torch.softmax(s.masked_fill(~vis, -math.inf), -1)
    got = torch.gather(p, -1, rows.clamp(min=0)[..., None])[..., 0]
    shown = (rows >= 0) & vis[torch.arange(Sq)[None].expand(Hq, Sq), rows.clamp(min=0)]
    return torch.where(shown, got, torch.full_like(got, math.nan))


# ------------------------------------------------------------------ CPU: the needle checker -----------------------------

# per-sequence shapes of the GPU sweeps and workloads: name, Hq, Hkv, Sq, K, D, causal, output kind, split_keys
NEEDLE_SHAPES = [
    ("dense edge 257 x 257 causal", 4, 2, 257, 257, 64, True, "bf16", None),
    ("dense edge 1 x 257", 4, 2, 1, 257, 128, False, "fp16", None),
    ("dense edge 129 x 33 causal", 4, 2, 129, 33, 128, True, "bf16", None),
    ("dense edge 33 x 160", 4, 2, 33, 160, 64, False, "f32", None),
    ("split-KV 129 x 1153, 5 splits", 4, 2, 129, 1153, 128, True, "bf16", 256),
    ("split-KV 1 x 1023, 3 splits", 4, 2, 1, 1023, 64, False, "fp16", 384),
    ("cache decode, capacity 1000", 4, 2, 1, 1000, 128, True, "fp16", None),
    ("cache 129 rows on 512 keys, 2 splits", 4, 2, 129, 512, 64, True, "bf16", 256),
    ("varlen-cache 257 rows appended to 257", 4, 2, 257, 514, 128, True, "fp16", None),
    ("qkv8 decode at scale", 8, 2, 1, 1500, 128, True, "bf16", None),
    ("qkv8 split decode at scale", 8, 2, 1, 1500, 128, True, "fp16", 768),
    ("qkv8 Sq 200 causal at scale", 8, 2, 200, 900, 64, True, "fp16", None),
    ("qkv8 varlen-cache prefill at scale", 8, 2, 512, 1500, 128, True, "bf16", None),
]
SHAPE_IDS = [s[0] for s in NEEDLE_SHAPES]


def _budget_kind(kind):
    return "bf16" if kind == "f32" else kind


def _out_dt(kind):
    return torch.float32 if kind == "f32" else (torch.bfloat16 if kind == "bf16" else torch.float16)


@pytest.fixture(scope="module")
def pi(built):
    import tfa_ctypes
    L = tfa_ctypes.lib()
    return torch.tensor([L.tfa_internal_fp8_p_key(c) for c in range(32)])


def pi_permuted(v, pi):
    """V with key 32 b + c read from key 32 b + pi(c): P in fp8_p_key order against a V^T in key order."""
    K = v.shape[2]
    j = torch.arange(K)
    src = 32 * (j // 32) + pi[j % 32]
    return v[:, :, torch.where(src < K, src, j)]


def wrong_references(q, k8, v8, causal, scale, Hq, Hkv, Sq, split_keys, pi):
    """(name, exact result of a wrong problem) for every mutation that changes something at this shape."""
    out = []
    for what, mut in fr.mutations(Hq, Hkv, Sq, causal, split_keys):
        if mut == "drop_last":
            out.append((what, reference(q, k8[:, :, :-1], v8[:, :, :-1], causal, scale, KS, VS)))
        else:
            out.append((what, reference(q, k8, v8, causal, scale, KS, VS, **mut)))
    out.append(("V permuted by pi", reference(q, k8, pi_permuted(v8, pi), causal, scale, KS, VS)))
    return out


@pytest.mark.parametrize("name,Hq,Hkv,Sq,K,D,causal,kind,split_keys", NEEDLE_SHAPES, ids=SHAPE_IDS)
def test_needle_builder_puts_the_mass_on_the_needle(name, Hq, Hkv, Sq, K, D, causal, kind, split_keys):
    extra = (split_keys,) if split_keys else ()
    rows = needle_rows(Sq, K, causal, Hq, extra)
    q8, k8, _ = needle_seq(Hq, Hkv, Sq, K, D, causal, seed=1, extra=extra)
    assert torch.equal(q8.float(), needle_q(rows, D)) and torch.equal(k8.float(), needle_keys(0, K, Hkv, D))
    mass = needle_mass(q8, k8, causal, NEEDLE_SCALE, rows)
    shown = ~torch.isnan(mass)
    assert int(shown.sum()) >= int((rows >= 0).sum()) // 2
    assert float(mass[shown].min()) >= 0.9, float(mass[shown].min())
    # the last key and the split boundary are needles at every shape; with enough (row, head) pairs every position is
    used = set(rows[shown].tolist())
    assert {K - 1, *extra} <= used, sorted({K - 1, *extra} - used)
    if Hq * Sq >= 2 * (len(FIXED) + 3):
        want = {p for p in FIXED if p < K}
        assert want <= used, sorted(want - used)
    if causal and Sq > 1:
        last = torch.clamp(torch.arange(Sq) + K - Sq, max=K - 1)
        assert len(set(rows[(rows == last) & (last >= 0)].tolist())) >= min(8, K, Sq)    # many diagonal positions
        assert bool(((rows == last + 1) & (last >= 0)).any())                            # needles just past it


@pytest.mark.parametrize("name,Hq,Hkv,Sq,K,D,causal,kind,split_keys", NEEDLE_SHAPES, ids=SHAPE_IDS)
def test_fp8_checker_rejects_wrong_results_on_needles(pi, name, Hq, Hkv, Sq, K, D, causal, kind, split_keys):
    """The exact result of each wrong problem, rounded to the output dtype, fails the FP8 budget; the right one passes
    in every output dtype."""
    extra = (split_keys,) if split_keys else ()
    q8, k8, v8 = (t[None] for t in needle_seq(Hq, Hkv, Sq, K, D, causal, seed=K + Sq, extra=extra))
    q = deq(q8, QS)
    ref = fp8_reference(q, k8, v8, causal, NEEDLE_SCALE, KS, VS)
    for k in OUT_KINDS:
        ok, r, _, msg = f8_compare(ref[0].to(_out_dt(k)), ref[1].float(), ref, _budget_kind(k))
        assert ok, (k, msg)
    wrongs = wrong_references(q, k8, v8, causal, NEEDLE_SCALE, Hq, Hkv, Sq, split_keys, pi)
    names = {w for w, _ in wrongs}
    assert "one key short" in names and "V permuted by pi" in names
    if causal:
        assert "causal offset -1" in names and (Sq == 1 or "causal offset +1" in names)
    dt = _out_dt(kind)
    for what, wrong in wrongs:
        ok, r, le, _ = f8_compare(wrong[0].to(dt), wrong[1].float(), ref, _budget_kind(kind))
        assert not ok, f"{name}: {what} passes (ratio {r:.3f}, LSE excess {le:.2e})"


def test_random_decode_row_hides_one_key_short():
    """The gap the needles close: on N(0, 0.5^2) inputs a decode row against 1,000 keys one key short is within the
    FP8 budget (LSE moves by ~1/1000, O by ~|v|/1000), so random inputs cannot judge a K_b off-by-one there.  The
    needle inputs of the same shape reject it (test_fp8_checker_rejects_wrong_results_on_needles)."""
    Hq, Hkv, K, D = 8, 2, 1000, 128
    q8, k8, v8 = (t[None] for t in random_seq(Hq, Hkv, 1, K, D, seed=3))
    q = deq(q8, QS)
    ref = fp8_reference(q, k8, v8, True, D ** -0.5, KS, VS)
    short = reference(q, k8[:, :, :-1], v8[:, :, :-1], True, D ** -0.5, KS, VS)
    ok, r, le, _ = f8_compare(short[0].to(torch.bfloat16), short[1].float(), ref, "bf16")
    assert ok and r < 1.0 and le < 0, (r, le)


# ------------------------------------------------------------------ GPU: helpers --------------------------------------------

@pytest.fixture(scope="module")
def tfa(built):
    import tfa_ctypes
    tfa_ctypes.lib()
    return tfa_ctypes


class Worst:
    """The largest err / budget and |dLSE| over a sweep, and its failures."""

    def __init__(self):
        self.ratio, self.dlse, self.fails, self.rows = 0.0, 0.0, [], 0

    def check(self, label, out, lse, q8, k8, v8, causal, scale, kind, mutate=None):
        """out (1, Hq, Sq, D), lse (1, Hq, Sq) of one sequence; q8 (1, Hq, Sq, D), k8 / v8 (1, Hkv, K, D) e4m3.
        Returns whether it passed."""
        self.rows += out.shape[1] * out.shape[2]
        if k8.shape[2] == 0:
            ok = bool((out == 0).all()) and bool(torch.isposinf(lse).all())
            if not ok:
                self.fails.append(f"{label}: a row without keys is not 0 / +inf")
            return ok
        ref = fp8_reference(deq(q8, QS), k8, v8, causal, scale, KS, VS, **(mutate or {}))
        ok, r, _, msg = f8_compare(out, lse, ref, _budget_kind(kind))
        keyed = ~torch.isinf(ref[1])
        dl = float((lse.double() - ref[1]).abs()[keyed].max()) if bool(keyed.any()) else 0.0
        if mutate is None:
            self.ratio, self.dlse = max(self.ratio, r), max(self.dlse, dl)
            if not ok:
                self.fails.append(f"{label}: {msg}")
        return ok

    def report(self, what):
        print(f"\n[fp8 edges] {what}: {self.rows} rows, max err/budget {self.ratio:.3f}, max |dLSE| {self.dlse:.2e}")
        assert not self.fails, f"{len(self.fails)} failing: " + "; ".join(self.fails[:8])


def _out_kw(kind):
    return dict(out_fp32=kind == "f32", out_dtype=torch.float16 if kind == "fp16" else torch.bfloat16)


# ------------------------------------------------------------------ GPU: kDenseFp8 and its split-KV ---------------------

@pytest.mark.gpu
@pytest.mark.parametrize("causal", [False, True])
@pytest.mark.parametrize("D", [64, 128])
def test_dense_fp8_tile_edges(tfa, D, causal):
    """Every (Sq, Sk) pair of EDGES8, GQA group 2, random and needle inputs, the output dtype cycling."""
    w = Worst()
    for idx, (Sq, Sk) in enumerate(PAIRS8):
        for inp in ("random", "needle"):
            kind = OUT_KINDS[(idx + (inp == "needle")) % 3]
            q8, k8, v8, scale = (t.cuda() if torch.is_tensor(t) else t
                                 for t in make_seq(inp, 4, 2, Sq, Sk, D, causal, seed=idx))
            q8, k8, v8 = q8[None], k8[None], v8[None]
            out, lse = tfa.attn_fwd(q8, k8, v8, causal, scale, num_splits=1, q_scale=QS, k_scale=KS, v_scale=VS,
                                    **_out_kw(kind))
            w.check(f"{inp} Sq {Sq} Sk {Sk} {kind}", out, lse, q8, k8, v8, causal, scale, kind)
    w.report(f"kDenseFp8 edges D {D} causal {causal}")


@pytest.mark.gpu
@pytest.mark.parametrize("causal", [False, True])
def test_dense_fp8_split_kv_edges(tfa, causal):
    """Sk = 128 t +- 1 with 2, 3 and 5 splits asked, Sq 1 and 129, D 64 and 128 in turn (128 past 1024 keys, where
    needle keys would repeat at D 64), random and needle inputs (a needle at the last split's first key); among them
    every split count whose last split holds one KV tile."""
    w, one_tile = Worst(), set()
    for t in range(2, 10):
        for Sk in (128 * t - 1, 128 * t + 1):
            D = 64 if (t + causal) % 2 == 0 and Sk <= 1024 else 128
            for ns in (2, 3, 5):
                for Sq in (1, 129):
                    nkv = -(-Sk // 128)
                    n_want = min(ns, nkv)
                    tiles = -(-nkv // n_want)
                    last_split = 128 * tiles * (-(-nkv // tiles) - 1)
                    for inp in ("random", "needle"):
                        kind = OUT_KINDS[(t + ns + Sq + (inp == "needle")) % 3]
                        q8, k8, v8, scale = make_seq(inp, 4, 2, Sq, Sk, D, causal, seed=Sk * 7 + ns + Sq,
                                                     extra=(last_split,))
                        q8, k8, v8 = q8[None].cuda(), k8[None].cuda(), v8[None].cuda()
                        out, lse, n = tfa.attn_fwd(q8, k8, v8, causal, scale, num_splits=ns, return_splits=True,
                                                   q_scale=QS, k_scale=KS, v_scale=VS, **_out_kw(kind))
                        assert 1 < n <= ns
                        if nkv - (n - 1) * -(-nkv // n) == 1:
                            one_tile.add(n)
                        w.check(f"{inp} Sq {Sq} Sk {Sk} splits {n} {kind}", out, lse, q8, k8, v8, causal, scale, kind)
    assert {2, 3, 5} <= one_tile, one_tile
    w.report(f"kDenseFp8 split-KV edges causal {causal}")


# ------------------------------------------------------------------ GPU: kVarlenFp8 --------------------------------------

def packed(inp, lq, lk, Hq, Hkv, D, causal, seed):
    """Every sequence built on its own, packed: q (total_q, Hq, D), k / v (total_k, Hkv, D) e4m3 on the GPU, cu_q, cu_k,
    the softmax scale."""
    seqs = [make_seq(inp, Hq, Hkv, a, b, D, causal, seed + i, turn=i) for i, (a, b) in enumerate(zip(lq, lk))]
    cat = lambda i: torch.cat([s[i].permute(1, 0, 2) for s in seqs]).cuda()
    cu = lambda ls: torch.tensor([0] + np.cumsum(ls).tolist(), dtype=torch.int32, device="cuda")
    return cat(0), cat(1), cat(2), cu(lq), cu(lk), seqs[0][3]


def _rows(t, a, b):
    return t[a:b].permute(1, 0, 2)[None]


@pytest.mark.gpu
@pytest.mark.parametrize("causal", [False, True])
@pytest.mark.parametrize("D", [64, 128])
def test_varlen_fp8_tile_edges(tfa, D, causal):
    """The 225 EDGES8 pairs as the sequences of one packed call."""
    lq, lk = [p[0] for p in PAIRS8], [p[1] for p in PAIRS8]
    w = Worst()
    for j, inp in enumerate(("random", "needle")):
        kind = OUT_KINDS[(j + D // 64 + causal) % 3]
        q, k, v, cu_q, cu_k, scale = packed(inp, lq, lk, 4, 2, D, causal, seed=31)
        out, lse = tfa.attn_varlen_fwd(q, k, v, cu_q, cu_k, max(lq), causal, scale, q_scale=QS, k_scale=KS,
                                       v_scale=VS, **_out_kw(kind))
        for (q0, q1), (k0, k1) in zip(offsets(lq), offsets(lk)):
            w.check(f"{inp} Sq {q1 - q0} Sk {k1 - k0} {kind}", _rows(out, q0, q1), lse[:, q0:q1][None],
                    _rows(q, q0, q1), _rows(k, k0, k1), _rows(v, k0, k1), causal, scale, kind)
    w.report(f"kVarlenFp8 edges D {D} causal {causal}")


# ------------------------------------------------------------------ GPU: kCacheQkv8 --------------------------------------

def put_keys(pool, table, b, first, codes):
    """Write codes (n, Hkv, D) as keys [first, first + n) of sequence b through the block table (None: contiguous)."""
    n = codes.shape[0]
    if n == 0:
        return
    page = pool.shape[1]
    j = torch.arange(first, first + n, device=pool.device)
    flat = pool.view(torch.uint8)
    if table is None:
        flat[b, j] = codes.view(torch.uint8).to(pool.device)
    else:
        flat[table[b].long()[j // page], j % page] = codes.view(torch.uint8).to(pool.device)


def qkv8_pools(inp, lens, Hkv, D, pool, seed):
    """e4m3 pools holding keys [0, lens[b]) of every sequence (random, or needle keys), NaN codes elsewhere; returns
    (k, v, table, capacity)."""
    name, page, mbps = pool
    kp, vp, table, cap = make_pools(lens, Hkv, D, page or 1, mbps, seed=seed, contiguous=page is None)
    if inp == "needle":
        for b, L in enumerate(lens):
            n = min(max(L, 0), cap)
            put_keys(kp, table, b, 0, needle_keys(0, n, Hkv, D).permute(1, 0, 2).to(FP8))
    return kp, vp, table, cap


def new_rows(inp, starts, n, Hkv, D, dt, g):
    """k_new / v_new rows in the output dtype: the needle keys [starts[b], starts[b] + n) scaled so the append
    quantizes them to CODE, or N(0, 0.5^2); V always random.  (len(starts), n, Hkv, D)."""
    vn = torch.empty((len(starts), n, Hkv, D)).normal_(0, 0.5, generator=g).to(dt)
    if inp == "needle":
        kn = torch.stack([needle_keys(s, n, Hkv, D).permute(1, 0, 2) for s in starts]) * KS
    else:
        kn = torch.empty((len(starts), n, Hkv, D)).normal_(0, 0.5, generator=g)
    return kn.to(dt).cuda(), vn.cuda()


def cache_q(inp, Ks, Sq, Hq, D, causal, seed, extra=()):
    """(B, Sq, Hq, D) e4m3 q of a dense-query cache call whose sequences hold Ks[b] keys after the append."""
    g = torch.Generator().manual_seed(seed)
    if inp == "needle":
        qs = [needle_q(needle_rows(Sq, K, causal, Hq, extra, turn=b), D).permute(1, 0, 2) for b, K in enumerate(Ks)]
        return torch.stack(qs).to(FP8).cuda()
    return e4m3(g, QS, len(Ks), Sq, Hq, D).cuda()


def run_cache_qkv8(tfa, inp, lens, Sq, Hq, Hkv, D, pool, causal, snew, ns, kind, seed, extra=(), out=None, lse=None):
    """One kCacheQkv8 call.  Returns dict(out, lse, splits, Ks, q, pools after, table, cap, pools before, k_new,
    v_new)."""
    kp, vp, table, cap = qkv8_pools(inp, lens, Hkv, D, pool, seed)
    Ls = [min(max(L, 0), cap - snew) for L in lens]
    Ks = [cache_lens_dense(L, cap, snew) for L in lens]
    q = cache_q(inp, Ks, Sq, Hq, D, causal, seed + 1, extra)
    g = torch.Generator().manual_seed(seed + 2)
    kn, vn = new_rows(inp, Ls, snew, Hkv, D, _out_dt("bf16" if kind == "f32" else kind), g) if snew else (None, None)
    sl = torch.tensor(lens, dtype=torch.int32, device="cuda")
    k1, v1 = kp.clone(), vp.clone()
    o, l, n = tfa.attn_kvcache_fwd(q, k1, v1, sl, table, kn, vn, is_causal=causal, scale=scale_of(inp, D),
                                   num_splits=ns, return_splits=True, out=out, lse=lse, q_scale=QS, k_scale=KS,
                                   v_scale=VS, **_out_kw(kind))
    return dict(out=o, lse=l, splits=n, Ks=Ks, q=q, k1=k1, v1=v1, kp=kp, vp=vp, table=table, cap=cap, kn=kn, vn=vn,
                sl=sl, scale=scale_of(inp, D), variant=tfa.lib().tfa_internal_last_variant())


def scale_of(inp, D):
    return NEEDLE_SCALE if inp == "needle" else D ** -0.5


def check_cache_qkv8(w, label, r, causal, kind, mutate=None):
    """Every sequence of a kCacheQkv8 run against the float64 reference of its Ks[b] keys read back from the pools."""
    ok = True
    for b, K in enumerate(r["Ks"]):
        kw = mutate(b, K) if mutate else None
        if kw is False:
            continue
        k8, v8 = gather(r["k1"], r["table"], b, K), gather(r["v1"], r["table"], b, K)
        if kw and kw.get("drop_last"):
            k8, v8, kw = k8[:, :, :-1], v8[:, :, :-1], {}
        qb = r["q"][b].permute(1, 0, 2)[None]
        ok &= w.check(f"{label} seq {b} K {K}", r["out"][b].permute(1, 0, 2)[None], r["lse"][b][None], qb, k8, v8,
                      causal, r["scale"], kind, kw if mutate else None)
    return ok


POOLS = [("page128", 128, 4), ("page256", 256, 2), ("contiguous1000", None, 1000)]
SQ8 = [1, 4, 63, 64, 65, 128, 129]


@pytest.mark.gpu
@pytest.mark.parametrize("causal", [False, True])
@pytest.mark.parametrize("pool", POOLS, ids=[p[0] for p in POOLS])
def test_cache_qkv8_edges(tfa, pool, causal):
    """Cached lengths at EDGES8, capacity - 1 and capacity (unused slots NaN codes), Snew 0, 1 and Sq (a cached length
    past capacity - Snew is cut there, so that the new keys fit), 1 or 3 splits with a workspace, random and needle
    inputs."""
    w = Worst()
    cap = 1000 if pool[1] is None else pool[1] * pool[2]
    lens = EDGES8 + [cap - 1, cap]
    splits = set()
    for i, Sq in enumerate(SQ8):
        for j, snew in enumerate(sorted({0, 1, Sq})):
            ns = (1, 3)[(i + j) % 2]
            D = (64, 128)[(i + j + causal) % 2]
            for inp in ("random", "needle"):
                kind = OUT_KINDS[(i + j + (inp == "needle")) % 3]
                r = run_cache_qkv8(tfa, inp, lens, Sq, 4, 2, D, pool, causal, snew, ns, kind, seed=100 * i + 10 * j)
                splits.add(r["splits"])
                check_cache_qkv8(w, f"{inp} Sq {Sq} Snew {snew} D {D} splits {r['splits']} {kind}", r, causal, kind)
    assert 1 in splits and max(splits) > 1, splits
    w.report(f"kCacheQkv8 edges {pool[0]} causal {causal}")


# ------------------------------------------------------------------ GPU: kVarlenCacheQkv8 --------------------------------

def run_varlen_cache_qkv8(tfa, inp, sq, lens, Hq, Hkv, D, page, mbps, causal, append, kind, seed, out=None, lse=None):
    """One kVarlenCacheQkv8 call on a permuted table.  Returns what check_varlen_cache_qkv8 reads."""
    kp, vp, table, cap = qkv8_pools(inp, lens, Hkv, D, ("paged", page, mbps), seed)
    Ks = [cache_lens_varlen(L, cap, n, append) for L, n in zip(lens, sq)]
    Ls = [K - (min(n, cap) if append else 0) for K, n in zip(Ks, sq)]
    g = torch.Generator().manual_seed(seed + 1)
    qs, kns, vns = [], [], []
    for b, (n, K) in enumerate(zip(sq, Ks)):
        if inp == "needle":
            qs.append(needle_q(needle_rows(n, K, causal, Hq, turn=b), D).permute(1, 0, 2).to(FP8))
        else:
            qs.append(e4m3(g, QS, n, Hq, D))
        if append:
            kn, vn = new_rows(inp, [Ls[b]], n, Hkv, D, _out_dt("bf16" if kind == "f32" else kind), g)
            kns.append(kn[0])
            vns.append(vn[0])
    q = torch.cat(qs).cuda()
    kn = torch.cat(kns) if append else None
    vn = torch.cat(vns) if append else None
    cu = torch.tensor([0] + np.cumsum(sq).tolist(), dtype=torch.int32, device="cuda")
    sl = torch.tensor(lens, dtype=torch.int32, device="cuda")
    k1, v1 = kp.clone(), vp.clone()
    o, l = tfa.attn_varlen_kvcache_fwd(q, k1, v1, cu, max(sq), sl, table, kn, vn, is_causal=causal,
                                       scale=scale_of(inp, D), out=out, lse=lse, q_scale=QS, k_scale=KS, v_scale=VS,
                                       **_out_kw(kind))
    return dict(out=o, lse=l, Ks=Ks, q=q, k1=k1, v1=v1, kp=kp, vp=vp, table=table, cap=cap, kn=kn, vn=vn, cu=cu,
                sl=sl, sq=sq, scale=scale_of(inp, D), variant=tfa.lib().tfa_internal_last_variant())


def check_varlen_cache_qkv8(w, label, r, causal, kind, mutate=None):
    ok = True
    for b, ((r0, r1), K) in enumerate(zip(offsets(r["sq"]), r["Ks"])):
        if r1 == r0:
            continue
        kw = mutate(b, K) if mutate else None
        if kw is False:
            continue
        k8, v8 = gather(r["k1"], r["table"], b, K), gather(r["v1"], r["table"], b, K)
        if kw and kw.get("drop_last"):
            k8, v8, kw = k8[:, :, :-1], v8[:, :, :-1], {}
        ok &= w.check(f"{label} seq {b} Sq {r1 - r0} K {K}", _rows(r["out"], r0, r1), r["lse"][:, r0:r1][None],
                      _rows(r["q"], r0, r1), k8, v8, causal, r["scale"], kind, kw if mutate else None)
    return ok


@pytest.mark.gpu
@pytest.mark.parametrize("causal,append", [(True, True), (True, False), (False, True), (False, False)])
def test_varlen_cache_qkv8_edges(tfa, causal, append):
    """The EDGES8 pairs as (query rows, cached length) of one call, page 128 on a permuted table, with and without the
    append (each sequence then holds its cached length + its query rows)."""
    sq, lens = [p[0] for p in PAIRS8], [p[1] for p in PAIRS8]
    w = Worst()
    D = 128 if causal else 64
    for j, inp in enumerate(("random", "needle")):
        kind = OUT_KINDS[(j + append + 2 * causal) % 3]
        r = run_varlen_cache_qkv8(tfa, inp, sq, lens, 4, 2, D, 128, 5, causal, append, kind, seed=41 + j)
        check_varlen_cache_qkv8(w, f"{inp} {kind}", r, causal, kind)
    w.report(f"kVarlenCacheQkv8 edges causal {causal} append {append}")


# ------------------------------------------------------------------ GPU: the widened FP8-cache modes --------------------

FP8_CACHE_SCALES = (0.0123, 0.00731)


@pytest.mark.gpu
@pytest.mark.parametrize("page", [128, 256])
@pytest.mark.parametrize("causal", [False, True])
def test_widened_fp8_cache_edges(tfa, page, causal):
    """kCacheFp8 through test_fwd_float64_reference's runner: Sq of SQ8, cached lengths at EDGES8 and at the pool's
    last page edge, Snew 0, 1 and Sq, 1 or 3 splits, 16-bit budget with k_scale / v_scale."""
    worst = [0.0, 0.0]
    fails = []
    for i, Sq in enumerate(SQ8):
        for j, snew in enumerate(sorted({0, 1, Sq})):
            top = -(-257 // page) * page
            kind, D = (("bf16", 128), ("fp16", 64))[(i + j + causal) % 2]
            kw = dict(lens=EDGES8 + [top - 1, top], Sq=Sq, Hq=4, Hkv=2, D=D, kind=kind, page=page, causal=causal,
                      snew=snew, ns=(1, 3)[(i + j) % 2], fp8=FP8_CACHE_SCALES)
            r = fr.run_workload(tfa, W("edges", "cache", 500 + 10 * i + j, kw))
            v = fr.check_workload(r)
            worst[0], worst[1] = max(worst[0], v.ratio), max(worst[1], v.lse_err)
            if not v.ok:
                fails.append(f"Sq {Sq} Snew {snew}: {v.msg}")
    print(f"\n[fp8 edges] kCacheFp8 edges page {page} causal {causal}: max err/budget {worst[0]:.3f}, "
          f"max |dLSE| {worst[1]:.2e}")
    assert not fails, "; ".join(fails[:8])


@pytest.mark.gpu
@pytest.mark.parametrize("causal,append", [(True, True), (False, False), (True, False), (False, True)])
def test_widened_fp8_varlen_cache_edges(tfa, causal, append):
    """kVarlenCacheFp8 through test_fwd_float64_reference's runner on the EDGES8 pairs, page 128."""
    sq, lens = [p[0] for p in PAIRS8], [p[1] for p in PAIRS8]
    kw = dict(sq=sq, lens=lens, Hq=4, Hkv=2, D=128 if causal else 64, kind="fp16" if causal else "bf16", page=128,
              causal=causal, append=append, fp8=FP8_CACHE_SCALES)
    r = fr.run_workload(tfa, W("edges", "varlen_cache", 43, kw))
    v = fr.check_workload(r)
    print(f"\n[fp8 edges] kVarlenCacheFp8 edges causal {causal} append {append}: max err/budget {v.ratio:.3f}, "
          f"max |dLSE| {v.lse_err:.2e}")
    assert v.ok, v.msg


# ------------------------------------------------------------------ GPU: e4m3-query cache workloads at scale -----------

VC_SQ = [512] * 4 + [1] * 60
SCALE_WORKLOADS = [
    W("qkv8_decode", "cache", 121, dict(lens=_decode_lens(121, 64, 256, 1500), Sq=1, Hq=32, Hkv=8, D=128, kind="bf16",
                                        page=256, causal=True, snew=1, ns=1)),
    W("qkv8_decode_splits", "cache", 122, dict(lens=_decode_lens(122, 64, 256, 1500), Sq=1, Hq=32, Hkv=8, D=128,
                                               kind="fp16", page=256, causal=True, snew=1, ns=3)),
    W("qkv8_sq200_causal", "cache", 123, dict(lens=[0, 1, 199, 200, 201, 900, 555, 128], Sq=200, Hq=32, Hkv=8, D=64,
                                              kind="fp16", page=128, causal=True, snew=0, ns=1)),
    W("qkv8_varlen_cache_mixed", "varlen_cache", 124, dict(sq=VC_SQ, lens=_decode_lens(124, 64, 256, 1500), Hq=32,
                                                           Hkv=8, D=128, kind="bf16", page=256, causal=True,
                                                           append=True)),
]
SCALE_BY_NAME = {w.name: w for w in SCALE_WORKLOADS}


def _mbps(kw):
    extra = kw.get("snew", 0) if "snew" in kw else max(kw["sq"])
    return -(-(max(kw["lens"]) + extra) // kw["page"]) + 1


def run_scale(tfa, w, inp):
    """Workload w on `inp` inputs, out / lse in NaN guard buffers; checks the guards and that the appended pools equal
    those of tfa_attn_kvcache_fp8_fwd / tfa_attn_varlen_kvcache_fp8_fwd (16-bit q, same k_new / v_new and scales)."""
    kw = w.kw
    dt = _out_dt(kw["kind"])
    mbps = _mbps(kw)
    if w.mode == "cache":
        B, Sq = len(kw["lens"]), kw["Sq"]
        ob, out = guarded((B, Sq, kw["Hq"], kw["D"]), dt)
        lb, lse = guarded((B, kw["Hq"], Sq), torch.float32)
        r = run_cache_qkv8(tfa, inp, kw["lens"], Sq, kw["Hq"], kw["Hkv"], kw["D"], ("paged", kw["page"], mbps),
                           True, kw["snew"], kw["ns"], kw["kind"], w.seed, out=out, lse=lse)
        r["items"] = -(-Sq // 128) * B * kw["Hq"] * r["splits"]
        if kw["snew"]:
            k2, v2 = r["kp"].clone(), r["vp"].clone()
            tfa.attn_kvcache_fwd(torch.zeros(tuple(r["q"].shape), dtype=dt, device="cuda"), k2, v2, r["sl"],
                                 r["table"], r["kn"], r["vn"], is_causal=True, k_scale=KS, v_scale=VS)
    else:
        total = sum(kw["sq"])
        ob, out = guarded((total, kw["Hq"], kw["D"]), dt)
        lb, lse = guarded((kw["Hq"], total), torch.float32)
        r = run_varlen_cache_qkv8(tfa, inp, kw["sq"], kw["lens"], kw["Hq"], kw["Hkv"], kw["D"], kw["page"], mbps,
                                  True, kw["append"], kw["kind"], w.seed, out=out, lse=lse)
        r["items"] = -(-max(kw["sq"]) // 128) * len(kw["sq"]) * kw["Hq"]
        if kw["append"]:
            k2, v2 = r["kp"].clone(), r["vp"].clone()
            tfa.attn_varlen_kvcache_fwd(torch.zeros(tuple(r["q"].shape), dtype=dt, device="cuda"), k2, v2, r["cu"],
                                        max(kw["sq"]), r["sl"], r["table"], r["kn"], r["vn"], is_causal=True,
                                        k_scale=KS, v_scale=VS)
    torch.cuda.synchronize()
    assert_guarded(ob, out)
    assert_guarded(lb, lse)
    if kw.get("snew") or kw.get("append"):
        assert torch.equal(bits(r["k1"]), bits(k2)) and torch.equal(bits(r["v1"]), bits(v2)), f"{w.name}: appends"
        assert not torch.equal(bits(r["k1"]), bits(r["kp"]))
    return r


def scale_check(w, r, inp, mutate=None):
    worst = Worst()
    chk = check_cache_qkv8 if w.mode == "cache" else check_varlen_cache_qkv8
    ok = chk(worst, f"{w.name} {inp}", r, True, w.kw["kind"], mutate)
    return ok, worst


def scale_portable(r):
    return {"out": r["out"].cpu(), "lse": r["lse"].cpu(), "variant": r["variant"]}


@pytest.fixture(scope="module")
def scale_runs(tfa):
    return {(w.name, inp): run_scale(tfa, w, inp) for w in SCALE_WORKLOADS for inp in ("random", "needle")}


@pytest.mark.gpu
@pytest.mark.parametrize("name", [w.name for w in SCALE_WORKLOADS])
def test_qkv8_workload_within_budget(scale_runs, name):
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    w = SCALE_BY_NAME[name]
    for inp in ("random", "needle"):
        r = scale_runs[(name, inp)]
        assert r["items"] >= 3 * sms, f"{r['items']} work items for {sms} SMs"
        ok, worst = scale_check(w, r, inp)
        print(f"\n[fp8 edges] {name} {inp}: {r['items']} items, schedule {r['variant']}, max err/budget "
              f"{worst.ratio:.3f}, max |dLSE| {worst.dlse:.2e}")
        assert ok, worst.fails[:4]


SCALE_SCHEDULE_RUN = r'''
import os, sys, torch
sys.path.insert(0, os.path.join(os.environ["TFA_ROOT"], "tiny-flash-attention_b200"))
sys.path.insert(0, os.path.join(os.environ["TFA_ROOT"], "tests"))
import tfa_ctypes as tfa
from test_fwd_fp8_edges import SCALE_WORKLOADS, run_scale, scale_portable
res = {}
for w in SCALE_WORKLOADS:
    for inp in ("random", "needle"):
        res[(w.name, inp)] = scale_portable(run_scale(tfa, w, inp))
        torch.cuda.empty_cache()
torch.save(res, os.environ["TFA_OUT"])
'''


@pytest.mark.gpu
def test_qkv8_workloads_bitwise_equal_under_both_schedules(scale_runs):
    outs = {}
    with tempfile.TemporaryDirectory() as tmp:
        for variant in ("classic", "persist"):
            path = os.path.join(tmp, variant + ".pt")
            env = dict(os.environ, TFA_ROOT=ROOT, TFA_OUT=path, TFA_KERNEL=variant)
            p = subprocess.run([sys.executable, "-c", SCALE_SCHEDULE_RUN], env=env, capture_output=True, text=True,
                               timeout=1200)
            assert p.returncode == 0, p.stderr[-3000:]
            outs[variant] = torch.load(path)
    for key, r in scale_runs.items():
        want = scale_portable(r)
        for variant, code in (("classic", 0), ("persist", 4)):
            got = outs[variant][key]
            assert got["variant"] == code, (key, variant)
            assert torch.equal(bits(got["out"]), bits(want["out"])) and torch.equal(bits(got["lse"]),
                                                                                    bits(want["lse"])), (key, variant)


@pytest.mark.gpu
@pytest.mark.parametrize("name", [w.name for w in SCALE_WORKLOADS])
def test_checker_rejects_qkv8_workload_against_wrong_reference(scale_runs, name):
    """The kernel's own result on the needle inputs, against a reference wrong by the diagonal (+1, or -1 for decode
    rows), the head mapping or one key of the first sequence with keys: rejected."""
    w = SCALE_BY_NAME[name]
    r = scale_runs[(name, "needle")]
    Sq = w.kw.get("Sq") or max(w.kw["sq"])
    first = next(b for b, K in enumerate(r["Ks"]) if K >= 2 and (w.mode == "cache" or w.kw["sq"][b] > 0))
    for what, mut in (("causal diagonal", dict(shift=1 if Sq > 1 else -1)), ("kv head h % Hkv", dict(heads="mod")),
                      ("one key short", dict(drop_last=True))):
        pick = (lambda b, K, m=mut: m) if what != "one key short" else (lambda b, K: mut if b == first else False)
        ok, _ = scale_check(w, r, "needle", pick)
        assert not ok, f"{name}: {what} passes"
