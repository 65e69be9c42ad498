"""Every sm_90a forward mode (dense, split-KV, varlen, cache, varlen-cache, FP8, rotary) at 128K-256K keys against
the float64 reference, and the accumulations whose error grows with the key count.

The float64 suites stop at about 2K keys.  Here each mode runs one long workload on two input patterns:
  * noise_mean: q and k from N(0, 0.5^2), V = 1 + N(0, 0.5^2), so that O is far from zero and a relative error in l
    or a drift of the PV accumulator shows in O (with V of mean 0, O ~ 0 at long context and hides both);
  * sink_repeat: key 0 of every sequence sits above the rest, and every other key row is one and the same vector, so
    each row's tail of P is constant.  q's dimension 0 is drawn from U(0.5, 8) against a sink that differs from the
    repeated key only in that dimension, so the gap delta between the sink and the tail spreads over about 0.3 to 8
    nats across rows.  This is the input (repeated tokens, padding without rotary, FP8 keys sharing a code) on which a
    running fp32 row sum drifts past the LSE bound (test_fwd_softmax_range.test_row_sum_order_keeps_lse_bound_on_a_
    constant_tail); the FP8 workloads build the same patterns in float and quantize them as a caller would.
Each workload is checked against test_fwd_float64_reference.reference (test_fwd_fp8.fp8_reference for kDenseFp8) and
its budget, which carries the row-sum term L_SUM and the 16-bit PV term E_PV16.  Decode batches are checked on every
row; long prefills on their first 256 rows (where a causal offset shows), their last 256 and 64 random blocks of 8
rows per head, each block against only the keys its rows can see, in chunks that keep a float64 score block near
256 MB.  out and lse are written into NaN guard buffers; the cache workloads' appended rows must be exact.  Every
workload runs under the automatic schedule and, one subprocess each, forced classic and persistent: the three results
are bitwise equal (compared by digest, so that nothing of a 128K-row output is kept between workloads).

Cache workloads.  The cache-decode pool holds more than 2^31 elements and its block table is permuted so that
sequence 0's last pages, the appended row among them, sit past element 2^31: the kernel's and the append's 64-bit
offsets are exercised.  FP8 pools are quantized as a caller would, with per-tensor scales from the data; one FP8
decode run rotates q and the appended keys (rotary_dim 64, NeoX) at positions near 256K: q_rot must equal the eager
fp32 rotation bit for bit, and the appended row the quantized rotated key.  Its twin qkv8_cache_decode builds the same
pools and quantizes q too (kCacheQkv8: both products on FP8 wgmma, checked against the FP8 budget).  The varlen-cache workload (kVarlenCache,
which has no split-KV) runs a 2048-row prefill chunk on a 128K cache and decode rows on caches near 200K, appending
every query row's key first.

Measured accumulators.  test_pv16_chain_through_the_forward runs the forward at softmax_scale = 0, where P = 1 and l
is an exact integer, so N O (fp32 output, N a power of two) is the PV wgmma's accumulator itself; against the exact
float64 prefix sums of V it gives the error per k-step that PV16_MEASURED_BOUND bounds.  The FP8 PV chain is measured
to 16384 k-steps by test_fwd_fp8.test_wgmma_fp8_primitives.

Peak device memory stays under about 20 GB (the cache-decode pools: 2 x 4.3 GB), freed between workloads."""
import hashlib
import os
import random
import subprocess
import sys
import tempfile
import time
from dataclasses import dataclass, field

import numpy as np
import pytest
import torch

import test_fwd_fp8 as F8
from test_fwd_float64_reference import PV16_MEASURED_BOUND, Verdict, assert_guarded, compare, guarded, reference
from test_kvcache_fp8 import FP8, bits, quantize
from test_kvcache_rotary import positions, rope, rope_tables

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PATTERNS = ["noise_mean", "sink_repeat"]
CHUNK = 2 ** 25                 # float64 elements of one score block (256 MB)


def _dt(kind):
    return torch.bfloat16 if kind == "bf16" else torch.float16


# ------------------------------------------------------------------ inputs ----------------------------------------------

def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def make_q(pattern, shape, g):
    """q (..., D) in float32: N(0, 0.5^2); sink_repeat: dimension 0 from U(0.5, 8), which sets each row's gap delta."""
    q = torch.empty(shape, device="cuda").normal_(0.0, 0.5, generator=g)
    if pattern == "sink_repeat":
        q[..., 0] = torch.empty(shape[:-1], device="cuda").uniform_(0.5, 8.0, generator=g)
    return q


def make_kv(pattern, n, Hkv, D, g, first):
    """k, v (n, Hkv, D) in float32 for keys [first, first + n) of one sequence.  sink_repeat: every key the same row
    per head (dimension 0 zero), the sequence's key 0 that row with dimension 0 = 8."""
    v = 1.0 + torch.empty((n, Hkv, D), device="cuda").normal_(0.0, 0.5, generator=g)
    if pattern == "noise_mean":
        return torch.empty((n, Hkv, D), device="cuda").normal_(0.0, 0.5, generator=g), v
    rep = torch.Generator(device="cuda").manual_seed(7)       # the same repeated row in every sequence and call
    row = torch.empty((1, Hkv, D), device="cuda").normal_(0.0, 0.5, generator=rep)
    row[..., 0] = 0.0
    k = row.expand(n, Hkv, D).clone()
    if first == 0 and n > 0:
        k[0, :, 0] = 8.0
    return k, v


def fp8_of(x):
    """A caller's per-tensor quantization: the largest magnitude maps to 448."""
    s = float(np.float32(float(x.abs().max()) / 448.0))
    return (x / s).clamp(-448, 448).to(FP8), s


def digest(*ts):
    h = hashlib.sha256()
    for t in ts:
        h.update(bits(t.contiguous()).cpu().numpy().tobytes() if t.dtype != torch.float32 else
                 t.contiguous().view(torch.int32).cpu().numpy().tobytes())
    return h.hexdigest()


# ------------------------------------------------------------------ checking sampled rows -------------------------------

def row_blocks(Sq, seed):
    """All rows of a short sequence; of a long one the first 256, the last 256 and 64 random blocks of 8 rows."""
    if Sq <= 1024:
        return [(0, Sq)]
    rng = random.Random(seed)
    return [(0, 256), (Sq - 256, Sq)] + [(r, r + 8) for r in (rng.randrange(256, Sq - 264) for _ in range(64))]


def check_seq(q, k, v, out, lse, causal, scale, kind, blocks, fp8=None, mutate=None):
    """One sequence: q (Hq, Sq, D), k / v (Hkv, Sk, D), out (Hq, Sq, D), lse (Hq, Sq) on the GPU; the rows of `blocks`
    of every head against the float64 reference.  fp8 = (q_scale, k_scale, v_scale) for kDenseFp8 (q, k, v codes),
    (1, k_scale, v_scale) for an FP8 cache.  `mutate`: reference() keywords of a wrong problem, or ("drop_tile", j0)."""
    Hq, Sq, _ = q.shape
    Hkv, Sk = k.shape[0], k.shape[1]
    g = Hq // Hkv
    verdict = Verdict()
    kw = dict(mutate or {})
    drop = kw.pop("drop_tile", None)
    if drop is not None:
        kw["drop"] = (drop, drop + 128)
    heads_mod = kw.get("heads") == "mod"
    for h in range(Hq):
        kh = h % Hkv if heads_mod else h // g
        kk, vv = k[kh:kh + 1][None], v[kh:kh + 1][None]
        for r0, r1 in blocks:
            step = max(1, CHUNK // max(Sk, 1))
            for a in range(r0, r1, step):
                b = min(r1, a + step)
                # rows [a, b) see keys [0, b + Sk - Sq) (+ shift) under the bottom-right causal mask
                kend = max(min(Sk, b + Sk - Sq), 0) if causal else Sk
                qq = q[h:h + 1, a:b][None]
                o, l = out[h:h + 1, a:b][None], lse[h:h + 1, a:b][None]
                rk = {x: y for x, y in kw.items() if x != "heads"}
                if fp8 is not None and fp8[0] != 1.0:
                    ref = F8.fp8_reference(qq.double() if qq.dtype != FP8 else qq.float().double() * fp8[0],
                                           kk[:, :, :kend], vv[:, :, :kend], causal, scale, fp8[1], fp8[2], **rk)
                    ok, ra, le, msg = F8.compare(o, l, ref, kind)
                    one = Verdict(ok, ra, float((l.double() - ref[1]).abs().max()), msg)
                else:
                    ks, vs = (fp8[1], fp8[2]) if fp8 is not None else (1.0, 1.0)
                    ref = reference(qq, kk[:, :, :kend], vv[:, :, :kend], causal, scale, ks, vs, **rk)
                    one = compare(o, l, ref, kind)
                verdict.add(one, f"head {h} rows [{a}, {b})")
                del ref
    return verdict


# ------------------------------------------------------------------ workloads -------------------------------------------

@dataclass
class W:
    name: str
    mode: str                    # dense, varlen, cache, varlen_cache
    pattern: str
    seed: int
    kw: dict = field(default_factory=dict)
    negative: tuple = ()         # checker-rejects mutations run on this workload's result


CACHE_LENS = [261887, 261888, 261889, 262143, 262144, 262145, 250000, 255999]   # page edges near 256K (page 256)
VC_LENS = [131072, 199935, 199936, 199937, 200191, 200192, 204800, 196608]     # a 128K prefill, decodes near 200K


def workloads():
    out = []
    for i, pat in enumerate(PATTERNS):
        s = 1000 * (i + 1)
        out += [
            W(f"dense_causal_prefill_{pat}", "dense", pat, s + 1,
              dict(B=1, Hq=8, Hkv=2, Sq=131072, Sk=131072, D=128, kind="bf16", causal=True, ns=1),
              ("causal offset -1", "causal offset +1", "kv head h % Hkv", "dropped tile") if i == 1 else ()),
            W(f"dense_long_keys_{pat}", "dense", pat, s + 2,
              dict(B=1, Hq=4, Hkv=1, Sq=256, Sk=262144, D=64, kind="fp16", causal=False, ns=1, f32=i == 0),
              ("dropped tile",) if i == 1 else ()),
            W(f"dense_long_keys_auto_{pat}", "dense", pat, s + 2,
              dict(B=1, Hq=4, Hkv=1, Sq=256, Sk=262144, D=64, kind="fp16", causal=False, ns=0, f32=i == 1,
                   min_splits=16),
              ("dropped split",) if i == 1 else ()),
            W(f"varlen_{pat}", "varlen", pat, s + 3,
              dict(lq=[131072, 1, 17, 300, 129, 2000, 64, 1000, 5], lk=[131072, 1, 40, 300, 700, 2000, 64, 1500, 900],
                   Hq=8, Hkv=2, D=128, kind="bf16", causal=True),
              ("causal offset +1", "kv head h % Hkv") if i == 0 else ()),
            W(f"cache_decode_{pat}", "cache", pat, s + 4,
              dict(lens=CACHE_LENS, Hq=32, Hkv=8, D=128, kind="bf16", page=256, ns=(0, 1, 16)),
              ("kv head h % Hkv", "dropped tile") if i == 1 else ()),
            W(f"varlen_cache_mixed_{pat}", "varlen_cache", pat, s + 7,
              dict(sq=[2048] + [1] * 7, lens=VC_LENS, Hq=32, Hkv=8, D=128, kind="bf16", page=256),
              ("kv head h % Hkv", "dropped tile") if i == 1 else ()),
            W(f"fp8_cache_decode_{pat}", "cache", pat, s + 5,
              dict(lens=CACHE_LENS, Hq=32, Hkv=8, D=128, kind="fp16", page=256, ns=(0,), kvfp8=True,
                   rotary=(64, False) if i == 0 else None)),
            W(f"qkv8_cache_decode_{pat}", "cache", pat, s + 5,        # the same pools, e4m3 q on FP8 wgmma
              dict(lens=CACHE_LENS, Hq=32, Hkv=8, D=128, kind="fp16", page=256, ns=(0,), kvfp8=True, qkv8=True)),
            W(f"fp8_dense_{pat}", "dense", pat, s + 6,
              dict(B=1, Hq=4, Hkv=2, Sq=256, Sk=131072, D=128, kind="bf16", causal=False, ns=1, fp8=True),
              ("kv head h % Hkv",) if i == 1 else ()),
        ]
    return out


WORKLOADS = workloads()
BY_NAME = {w.name: w for w in WORKLOADS}

MUTATE = {"causal offset -1": dict(shift=-1), "causal offset +1": dict(shift=1), "kv head h % Hkv": dict(heads="mod")}


def _mutation(what, Sk, splits):
    if what == "dropped tile":
        return dict(drop_tile=(Sk // 2) // 128 * 128)
    if what == "dropped split":
        per = -(-(-(-Sk // 128)) // splits) * 128
        return dict(drop=(per, 2 * per))
    return MUTATE[what]


def _run_dense(tfa, w, check):
    kw = w.kw
    B, Hq, Hkv, Sq, Sk, D, kind = (kw[x] for x in ("B", "Hq", "Hkv", "Sq", "Sk", "D", "kind"))
    g = _gen(w.seed)
    scale = D ** -0.5
    q = make_q(w.pattern, (B, Hq, Sq, D), g)
    k, v = make_kv(w.pattern, Sk, Hkv, D, g, 0)
    k, v = k.permute(1, 0, 2)[None].contiguous(), v.permute(1, 0, 2)[None].contiguous()
    qkw, f8 = {}, None
    if kw.get("fp8"):
        (q, qs), (k, ks), (v, vs) = fp8_of(q), fp8_of(k), fp8_of(v)
        qkw, f8 = dict(q_scale=qs, k_scale=ks, v_scale=vs, out_dtype=_dt(kind)), (qs, ks, vs)
    else:
        q, k, v = q.to(_dt(kind)), k.to(_dt(kind)), v.to(_dt(kind))
    f32 = kw.get("f32", False)
    ob, out = guarded((B, Hq, Sq, D), torch.float32 if f32 else _dt(kind))
    lb, lse = guarded((B, Hq, Sq), torch.float32)
    _, _, n = tfa.attn_fwd(q, k, v, kw["causal"], scale, num_splits=kw["ns"], out_fp32=f32, out=out, lse=lse,
                           return_splits=True, **qkw)
    variant = tfa.lib().tfa_internal_last_variant()
    torch.cuda.synchronize()
    assert n >= kw.get("min_splits", 1), f"{w.name}: {n} splits"
    assert_guarded(ob, out)
    assert_guarded(lb, lse)
    res = dict(digest=digest(out, lse), variant=variant, splits=n, items=-(-Sq // 128) * B * Hq * n)
    if check:
        blocks = row_blocks(Sq, w.seed)
        res["verdict"] = check_seq(q[0], k[0], v[0], out[0], lse[0], kw["causal"], scale, kind, blocks, f8)
        res["negative"] = {what: check_seq(q[0], k[0], v[0], out[0], lse[0], kw["causal"], scale, kind, blocks[:2], f8,
                                           _mutation(what, Sk, n)) for what in w.negative}
    return res


def _run_varlen(tfa, w, check):
    kw = w.kw
    lq, lk, Hq, Hkv, D, kind = (kw[x] for x in ("lq", "lk", "Hq", "Hkv", "D", "kind"))
    g = _gen(w.seed)
    scale = D ** -0.5
    q = make_q(w.pattern, (sum(lq), Hq, D), g).to(_dt(kind))
    parts = [make_kv(w.pattern, n, Hkv, D, g, 0) for n in lk]
    k = torch.cat([p[0] for p in parts]).to(_dt(kind))
    v = torch.cat([p[1] for p in parts]).to(_dt(kind))
    del parts
    cu = lambda ls: torch.tensor([0] + np.cumsum(ls).tolist(), dtype=torch.int32, device="cuda")
    ob, out = guarded((sum(lq), Hq, D), _dt(kind))
    lb, lse = guarded((Hq, sum(lq)), torch.float32)
    tfa.attn_varlen_fwd(q, k, v, cu(lq), cu(lk), max(lq), kw["causal"], scale, out=out, lse=lse)
    variant = tfa.lib().tfa_internal_last_variant()
    torch.cuda.synchronize()
    assert_guarded(ob, out)
    assert_guarded(lb, lse)
    res = dict(digest=digest(out, lse), variant=variant, items=-(-max(lq) // 128) * len(lq) * Hq)
    if check:
        verdict, neg = Verdict(), {what: Verdict() for what in w.negative}
        qo, ko = np.cumsum([0] + lq), np.cumsum([0] + lk)
        for i in range(len(lq)):
            a = lambda x, o, j: x[o[j]:o[j + 1]].permute(1, 0, 2)
            args = (a(q, qo, i), a(k, ko, i), a(v, ko, i), a(out, qo, i), lse[:, qo[i]:qo[i + 1]])
            blocks = row_blocks(lq[i], w.seed + i)
            verdict.add(check_seq(*args, kw["causal"], scale, kind, blocks), f"sequence {i}")
            if i == 0:
                for what in w.negative:
                    neg[what] = check_seq(*args, kw["causal"], scale, kind, blocks[:2], None, MUTATE[what])
        res["verdict"], res["negative"] = verdict, neg
    return res


def _cache_table(B, mbps, seed):
    """A permuted block table whose sequence 0 holds the pool's highest blocks for its last 4 pages."""
    nblk = B * mbps + 5
    ids = torch.randperm(nblk, generator=torch.Generator().manual_seed(seed)).tolist()
    top = list(range(nblk - 1, nblk - 5, -1))
    rest = [x for x in ids if x not in top][:B * mbps - 4]
    table = torch.tensor(rest[:mbps - 4] + top + rest[mbps - 4:], dtype=torch.int32).view(B, mbps)
    return table, nblk


def _make_pools(w, lens, Hkv, D, page, tab, nblk, dt, fp8, new=()):
    """Paged k / v pools, NaN (FP8: 0x7f) outside each sequence's keys [0, L).  An FP8 pool is quantized as a caller
    would: per-tensor scales map the largest magnitude of the cached keys / values and of the tensors `new` (k, v) to
    be appended to 448; the keys are drawn twice from the same seed, once for the scales and once to store them."""
    def chunks():
        g = _gen(w.seed + 1)
        for b, L in enumerate(lens):
            for j0 in range(0, L, 16384):
                yield (b, j0, *make_kv(w.pattern, min(16384, L - j0), Hkv, D, g, j0))
    ks = vs = 1.0
    if fp8:
        ka = max([float(x.abs().max()) for x in new[:1]], default=0.0)
        va = max([float(x.abs().max()) for x in new[1:]], default=0.0)
        for _, _, kk, vv in chunks():
            ka, va = max(ka, float(kk.abs().max())), max(va, float(vv.abs().max()))
        ks, vs = float(np.float32(ka / 448.0)), float(np.float32(va / 448.0))
    kp = torch.empty((nblk, page, Hkv, D), dtype=torch.uint8 if fp8 else dt, device="cuda")
    vp = torch.empty_like(kp)
    kp.fill_(0x7F if fp8 else float("nan"))
    vp.fill_(0x7F if fp8 else float("nan"))
    for b, j0, kk, vv in chunks():
        if fp8:
            kk = (kk / ks).clamp(-448, 448).to(FP8).view(torch.uint8)
            vv = (vv / vs).clamp(-448, 448).to(FP8).view(torch.uint8)
        else:
            kk, vv = kk.to(dt), vv.to(dt)
        pos = torch.arange(j0, j0 + kk.shape[0], device="cuda")
        blk, off = tab[b, pos // page].long(), pos % page
        kp[blk, off], vp[blk, off] = kk, vv
    if fp8:
        kp, vp = kp.view(FP8), vp.view(FP8)
    return kp, vp, ks, vs


def _check_appended(w, kp, vp, tab, page, seqs, rows, new, fp8, ks, vs):
    """The pool rows at positions rows[i] of sequence seqs[i] hold row i of the appended k / v (FP8: quantized)."""
    b = torch.tensor(seqs, device="cuda")
    pos = torch.tensor(rows, device="cuda")
    blk, off = tab[b, pos // page].long(), pos % page
    for pool, x, s in zip((kp, vp), new, (ks, vs)):
        got = pool[blk, off]
        want = quantize(x, s) if fp8 else x
        assert torch.equal(bits(got.view(torch.uint8) if fp8 else got),
                           bits(want.view(torch.uint8) if fp8 else want)), f"{w.name}: appended rows"


def _seq_kv(kp, vp, tab, page, b, K):
    """Keys [0, K) of sequence b read back from the pool, (Hkv, K, D) each."""
    idx = torch.arange(K, device="cuda")
    rows_b, rows_o = tab[b, idx // page].long(), idx % page
    return kp[rows_b, rows_o].permute(1, 0, 2), vp[rows_b, rows_o].permute(1, 0, 2)


def _run_cache(tfa, w, check):
    kw = w.kw
    lens, Hq, Hkv, D, kind, page = (kw[x] for x in ("lens", "Hq", "Hkv", "D", "kind", "page"))
    B = len(lens)
    g = _gen(w.seed)
    scale = D ** -0.5
    dt = _dt(kind)
    mbps = -(-(max(lens) + 1) // page) + 1
    cap = mbps * page
    table, nblk = _cache_table(B, mbps, w.seed)
    assert nblk * page * Hkv * D > 2 ** 31
    assert int(table[0, lens[0] // page]) * page * Hkv * D >= 2 ** 31, "sequence 0's appended row below element 2^31"
    fp8 = kw.get("kvfp8", False)
    tab = table.cuda()
    q = make_q(w.pattern, (B, 1, Hq, D), g)
    q, qs = fp8_of(q) if kw.get("qkv8") else (q.to(dt), 1.0)
    qkw = dict(q_scale=qs, out_dtype=dt) if kw.get("qkv8") else {}
    kn, vn = make_kv(w.pattern, B, Hkv, D, g, 1)
    kn, vn = kn[:, None].to(dt), vn[:, None].to(dt)
    kp, vp, ks, vs = _make_pools(w, lens, Hkv, D, page, tab, nblk, dt, fp8, (kn, vn))
    sl = torch.tensor(lens, dtype=torch.int32, device="cuda")
    rot, qa, kr = {}, q, kn
    if kw.get("rotary"):
        rd, il = kw["rotary"]
        seqlen_ro = cap + 64
        cos, sin = rope_tables(seqlen_ro, rd, kind)
        rot = dict(rotary_cos=cos, rotary_sin=sin, rotary_interleaved=il)
        qa = rope(q, positions(lens, cap, 1, 1, True, True, seqlen_ro), cos, sin, rd, il)
        kr = rope(kn, positions(lens, cap, 1, 1, True, False, seqlen_ro), cos, sin, rd, il)
        assert min(lens) >= 2 ** 17, "rotary at positions near 256K"
    res = dict(runs=[])
    for ns in kw["ns"]:
        ob, out = guarded((B, 1, Hq, D), dt)
        lb, lse = guarded((B, Hq, 1), torch.float32)
        q_rot = torch.full_like(q, float("nan")) if rot else None
        _, _, n = tfa.attn_kvcache_fwd(q, kp, vp, sl, tab, kn, vn, is_causal=True, scale=scale, num_splits=ns, out=out,
                                       lse=lse, return_splits=True, k_scale=ks, v_scale=vs, **qkw,
                                       **(dict(rot, q_rot=q_rot) if rot else {}))
        variant = tfa.lib().tfa_internal_last_variant()
        torch.cuda.synchronize()
        assert_guarded(ob, out)
        assert_guarded(lb, lse)
        if rot:
            assert torch.equal(bits(q_rot), bits(qa)), f"{w.name}: q_rot differs from the eager fp32 rotation"
        if ns == 0:
            sms = torch.cuda.get_device_properties(0).multi_processor_count
            assert n == 1 and B * Hq > sms // 2, f"{w.name}: the heuristic split {n} ways"
        _check_appended(w, kp, vp, tab, page, list(range(B)), lens, (kr[:, 0], vn[:, 0]), fp8, ks, vs)
        run = dict(ns=ns, splits=n, digest=digest(out, lse, *([q_rot] if rot else [])), variant=variant)
        if check:
            verdict, neg = Verdict(), {}
            f8 = (qs, ks, vs) if fp8 else None
            for b, L in enumerate(lens):
                kk, vv = _seq_kv(kp, vp, tab, page, b, L + 1)
                args = (qa[b].permute(1, 0, 2), kk, vv, out[b].permute(1, 0, 2), lse[b])
                verdict.add(check_seq(*args, True, scale, kind, [(0, 1)], f8), f"sequence {b}")
                if b == 0 and ns == kw["ns"][0]:
                    for what in w.negative:
                        neg[what] = check_seq(*args, True, scale, kind, [(0, 1)], f8, _mutation(what, L + 1, 1))
                del kk, vv
            run["verdict"], run["negative"] = verdict, neg
        res["runs"].append(run)
    res["digest"] = "/".join(r["digest"] for r in res["runs"])
    res["variant"] = res["runs"][0]["variant"]
    res["items"] = B * Hq
    return res


def _run_varlen_cache(tfa, w, check):
    """kVarlenCache: a packed batch of query rows against a paged cache, each sequence's rows appended first; no
    split-KV, so one CTA accumulates a row's whole key range."""
    kw = w.kw
    sq, lens, Hq, Hkv, D, kind, page = (kw[x] for x in ("sq", "lens", "Hq", "Hkv", "D", "kind", "page"))
    B, total = len(sq), sum(sq)
    g = _gen(w.seed)
    scale = D ** -0.5
    dt = _dt(kind)
    mbps = -(-max(L + n for L, n in zip(lens, sq)) // page) + 1
    table, nblk = _cache_table(B, mbps, w.seed)
    tab = table.cuda()
    q = make_q(w.pattern, (total, Hq, D), g).to(dt)
    kn, vn = make_kv(w.pattern, total, Hkv, D, g, 1)              # appended keys: never a sequence's key 0
    kn, vn = kn.to(dt), vn.to(dt)
    kp, vp, _, _ = _make_pools(w, lens, Hkv, D, page, tab, nblk, dt, False)
    sl = torch.tensor(lens, dtype=torch.int32, device="cuda")
    qo = np.cumsum([0] + sq)
    cu = torch.tensor(qo.tolist(), dtype=torch.int32, device="cuda")
    ob, out = guarded((total, Hq, D), dt)
    lb, lse = guarded((Hq, total), torch.float32)
    tfa.attn_varlen_kvcache_fwd(q, kp, vp, cu, max(sq), sl, tab, kn, vn, is_causal=True, scale=scale, out=out, lse=lse)
    variant = tfa.lib().tfa_internal_last_variant()
    torch.cuda.synchronize()
    assert_guarded(ob, out)
    assert_guarded(lb, lse)
    _check_appended(w, kp, vp, tab, page, [b for b, n in enumerate(sq) for _ in range(n)],
                    [L + i for L, n in zip(lens, sq) for i in range(n)], (kn, vn), False, 1.0, 1.0)
    res = dict(digest=digest(out, lse), variant=variant, items=-(-max(sq) // 128) * B * Hq)
    if check:
        verdict, neg = Verdict(), {}
        for b, (L, n) in enumerate(zip(lens, sq)):
            kk, vv = _seq_kv(kp, vp, tab, page, b, L + n)
            args = (q[qo[b]:qo[b + 1]].permute(1, 0, 2), kk, vv, out[qo[b]:qo[b + 1]].permute(1, 0, 2),
                    lse[:, qo[b]:qo[b + 1]])
            blocks = row_blocks(n, w.seed + b)
            verdict.add(check_seq(*args, True, scale, kind, blocks), f"sequence {b}")
            if b == 0:
                for what in w.negative:
                    neg[what] = check_seq(*args, True, scale, kind, blocks[:2], None, _mutation(what, L + n, 1))
            del kk, vv
        res["verdict"], res["negative"] = verdict, neg
    return res


RUN = {"dense": _run_dense, "varlen": _run_varlen, "cache": _run_cache, "varlen_cache": _run_varlen_cache}


def run_workload(tfa, w, check=True):
    try:
        return RUN[w.mode](tfa, w, check)
    finally:
        torch.cuda.empty_cache()


# ------------------------------------------------------------------ GPU ---------------------------------------------------

@pytest.fixture(scope="module")
def tfa(built):
    import tfa_ctypes
    tfa_ctypes.lib()
    return tfa_ctypes


@pytest.fixture(scope="module")
def auto_runs(tfa):
    t0 = time.time()
    torch.cuda.reset_peak_memory_stats()
    res = {w.name: run_workload(tfa, w) for w in WORKLOADS}
    print(f"\n[long context] {len(res)} workloads run and checked in {time.time() - t0:.0f} s, peak device memory "
          f"{torch.cuda.max_memory_allocated() / 2 ** 30:.1f} GiB")
    return res


def _verdicts(r):
    return [(f" ns {x['ns']} ({x['splits']} splits)", x) for x in r["runs"]] if "runs" in r else [("", r)]


@pytest.mark.gpu
@pytest.mark.parametrize("name", [w.name for w in WORKLOADS])
def test_long_context_within_budget_of_float64_reference(auto_runs, name):
    fails = []
    for label, r in _verdicts(auto_runs[name]):
        v = r["verdict"]
        print(f"\n[long context] {name}{label}: schedule {auto_runs[name]['variant']}, max err/budget {v.ratio:.3f}, "
              f"max |dLSE| {v.lse_err:.2e}")
        if not v.ok:
            fails.append(f"{label}: {v.msg}")
    assert not fails, f"{name}: " + "; ".join(fails)


@pytest.mark.gpu
@pytest.mark.parametrize("name", [w.name for w in WORKLOADS if w.negative])
def test_checker_rejects_long_context_result_against_wrong_reference(auto_runs, name):
    """The kernel's own result against a reference that drops one 128-key tile or one split, maps query head h to kv
    head h % Hkv, or moves the causal diagonal by one on the first rows: rejected (one key fewer moves LSE by only
    1 / N here, below the bound).  kDenseFp8 takes the head mapping only: its S-accumulation term eta widens the LSE
    bound past what one tile of 1024 moves."""
    tried = 0
    for label, r in _verdicts(auto_runs[name]):
        for what, v in r.get("negative", {}).items():
            tried += 1
            assert not v.ok, f"{name}{label}: {what} passes (ratio {v.ratio:.3f}, LSE {v.lse_err:.2e})"
    assert tried == len(BY_NAME[name].negative)


SCHEDULE_RUN = r'''
import os, sys, torch
sys.path.insert(0, os.path.join(os.environ["TFA_ROOT"], "tiny-flash-attention_b200"))
sys.path.insert(0, os.path.join(os.environ["TFA_ROOT"], "tests"))
import tfa_ctypes as tfa
from test_fwd_long_context import WORKLOADS, run_workload
res = {}
for w in WORKLOADS:
    r = run_workload(tfa, w, check=False)
    res[w.name] = dict(digest=r["digest"], variant=r["variant"])
torch.save(res, os.environ["TFA_OUT"])
'''


@pytest.mark.gpu
def test_long_context_bitwise_equal_under_both_schedules(auto_runs):
    outs = {}
    with tempfile.TemporaryDirectory() as tmp:
        for variant in ("classic", "persist"):
            path = os.path.join(tmp, variant + ".pt")
            env = dict(os.environ, TFA_ROOT=ROOT, TFA_OUT=path, TFA_KERNEL=variant)
            p = subprocess.run([sys.executable, "-c", SCHEDULE_RUN], env=env, capture_output=True, text=True,
                               timeout=1800)
            assert p.returncode == 0, p.stderr[-3000:]
            outs[variant] = torch.load(path)
    for name, r in auto_runs.items():
        for variant, code in (("classic", 0), ("persist", 4)):
            got = outs[variant][name]
            assert got["variant"] == code, (name, variant)
            assert got["digest"] == r["digest"], (name, variant)


@pytest.mark.gpu
def test_pv16_chain_through_the_forward(tfa):
    """softmax_scale = 0: P = 1 and l = N exactly, N a power of two, so N O (fp32 output) is the PV accumulator of one
    row over N / 16 k-steps.  Its error against the exact float64 sum of V, over the sum over the k-steps of |C before
    the step| + sum |v| of the step, stays within PV16_MEASURED_BOUND (bf16 and fp16, V of mean 0 and of mean 1)."""
    worst = {}
    for kind in ("bf16", "fp16"):
        for N in (16384, 65536, 262144):
            for mean in (0.0, 1.0):
                g = _gen(N + int(mean) + (kind == "fp16"))
                D, H = 64, 2
                q = torch.empty((1, H, 128, D), device="cuda").normal_(0, 0.5, generator=g).to(_dt(kind))
                k = torch.empty((1, H, N, D), device="cuda").normal_(0, 0.5, generator=g).to(_dt(kind))
                v = (mean + torch.empty((1, H, N, D), device="cuda").normal_(0, 0.5, generator=g)).to(_dt(kind))
                out, lse = tfa.attn_fwd(q, k, v, False, 0.0, num_splits=1, out_fp32=True)
                torch.cuda.synchronize()
                vd = v[0].double()                                          # (H, N, D)
                cs = vd.cumsum(1)
                before = torch.cat([torch.zeros_like(cs[:, :1]), cs[:, 15:-1:16]], 1)   # C before each k-step
                tot = before.abs().sum(1) + vd.abs().sum(1)                 # (H, D)
                assert torch.all(lse[0] == lse[0, 0, 0])
                err = (out[0].double() * N - cs[:, -1:]).abs() / tot[:, None]
                worst[(kind, N, mean)] = float(err.max())
                del q, k, v, vd, cs
                torch.cuda.empty_cache()
    print("\n[16-bit PV chain] worst |N O - sum V| / sum_steps(|C before| + sum|v|) per (kind, N, mean V): " +
          ", ".join(f"{x}: {y:.3e}" for x, y in worst.items()))
    assert max(worst.values()) <= PV16_MEASURED_BOUND, worst
