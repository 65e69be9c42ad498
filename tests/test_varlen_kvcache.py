"""A variable-length batch of queries against a (paged) KV cache: tfa_attn_varlen_kvcache_fwd /
attention_cutlass.flash_attention_v2_varlen_kvcache.

CPU: the entry point is declared and exported, every argument error comes back before any device work, the length rule
and the append destination match their definition exhaustively (negative lengths, n_b > capacity and out-of-range table
entries included), and the barrier-protocol model accepts the mode's item mix and still catches a store after the
release.
GPU: each sequence equals a one-sequence tfa_attn_kvcache_fwd call bit for bit (out, lse and the pools after the
append), the whole batch equals tfa_attn_varlen_fwd on the gathered cache, an all-decode batch equals one cache call,
mixed cases match the float64 oracle, NaN in unused slots changes nothing, the append and the forward write exactly
what they should, both schedules agree, the call replays from a CUDA graph with new lengths, offsets and tables, and it
is 1 / 2 launches."""
import ctypes
import os
import random
import subprocess
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

TFA_EINVAL_SEQLENS = -12
TFA_EINVAL_KVCACHE = -13


def declared_functions():
    import re
    src = open(os.path.join(ROOT, "include", "tfa_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return set(re.findall(r"\b(tfa_[a-z0-9_]+)\s*\(", src))


# ------------------------------------------------------------------ CPU ------------------------------------------------

def test_header_declares_and_library_exports_varlen_kvcache(built):
    import tfa_ctypes
    assert "tfa_attn_varlen_kvcache_fwd" in declared_functions()
    assert "tfa_attn_varlen_kvcache_args" in open(os.path.join(ROOT, "include", "tfa_b200.h")).read()
    L = ctypes.CDLL(tfa_ctypes.LIB_PATH)
    assert hasattr(L, "tfa_attn_varlen_kvcache_fwd")
    assert L.tfa_abi_version() == 2


def test_varlen_kvcache_argument_validation_without_device(built):
    """Host buffers only: every code must come back before anything touches a device (on a CPU-only box a call that
    got that far would fail with a CUDA error instead)."""
    import tfa_ctypes
    L = tfa_ctypes.lib()
    buf = ctypes.create_string_buffer(4096 + 16)
    base = (ctypes.addressof(buf) + 15) & ~15
    ints = base + 1024                                        # 16-byte aligned, so 4-byte aligned
    Hq, Hkv, D, page = 4, 2, 64, 256

    def mk(**kw):
        return tfa_ctypes.VarlenKvcacheArgs(
            kw.get("q", base), base, base, kw.get("k_new", None), kw.get("v_new", None), kw.get("out", base), None,
            kw.get("cu_q", ints), kw.get("seqlens", ints), kw.get("table", ints), kw.get("B", 2), kw.get("Hq", Hq),
            kw.get("Hkv", Hkv), kw.get("D", D), kw.get("total_q", 300), kw.get("max_q", 200), kw.get("nblk", 8),
            kw.get("page", page), kw.get("mbps", 4), kw.get("qss", Hq * D), kw.get("qsh", D), page * Hkv * D,
            kw.get("kss", Hkv * D), D, kw.get("bts", 4), kw.get("nss", Hkv * D), kw.get("nsh", D),
            kw.get("dtype", 0), 1, kw.get("scale", 0.1), 0, None)

    call = lambda **kw: L.tfa_attn_varlen_kvcache_fwd(ctypes.byref(mk(**kw)))
    new = dict(k_new=base, v_new=base)
    assert L.tfa_attn_varlen_kvcache_fwd(None) == -1          # TFA_EINVAL_PTR
    assert call(q=None) == -1 and call(q=base + 2) == -1 and call(out=base + 8) == -1
    assert call(k_new=base + 8, v_new=base) == -1 and call(k_new=base, v_new=base + 2) == -1
    assert call(D=96) == -2                                   # TFA_EINVAL_DIM
    assert call(B=0) == -3 and call(total_q=0) == -3 and call(Hq=0) == -3 and call(Hkv=0) == -3
    assert call(dtype=2) == -4                                # TFA_EINVAL_DTYPE
    assert call(qss=60) == -5 and call(qsh=12) == -5 and call(kss=30) == -5      # TFA_EINVAL_STRIDE
    assert call(nss=12, **new) == -5 and call(nsh=4, **new) == -5 and call(nss=-8, **new) == -5
    assert call(scale=-1.0) == -9 and call(scale=float("nan")) == -9             # TFA_EINVAL_SCALE
    assert call(Hkv=3) == -10                                 # TFA_EINVAL_HEADS
    S = TFA_EINVAL_SEQLENS
    assert call(cu_q=None) == S and call(cu_q=ints + 2) == S
    assert call(max_q=0) == S and call(max_q=-5) == S and call(max_q=301) == S  # not in [1, total_q]
    E = TFA_EINVAL_KVCACHE
    assert call(seqlens=None) == E and call(seqlens=ints + 2) == E
    assert call(table=ints + 1) == E
    assert call(page=200) == E and call(page=64) == E         # paged: multiple of 128
    assert call(mbps=0) == E and call(nblk=0) == E and call(page=0) == E
    assert call(bts=3) == E                                   # table rows overlap
    assert call(k_new=base) == E and call(v_new=base) == E    # one of the pair
    # contiguous cache (no table): one page of any size per sequence, block b
    assert call(table=None, page=300, mbps=2) == E and call(table=None, page=300, mbps=1, nblk=1) == E
    # a cache error comes before a shape error, as for tfa_attn_kvcache_fwd
    assert call(mbps=0, B=0) == E


def _h():
    import tfa_ctypes
    L = tfa_ctypes.lib()
    ip, ll, ci = ctypes.POINTER(ctypes.c_int), ctypes.c_longlong, ctypes.c_int
    L.tfa_internal_varlen_cache_lens.argtypes = [ci, ci, ci, ci, ip]
    L.tfa_internal_varlen_append_offset.argtypes = [ci, ip, ll, ci, ci, ci, ci, ci, ci, ci, ll, ll, ll]
    L.tfa_internal_varlen_append_offset.restype = ll
    return L


def lens_rule(raw, cap, n, append):
    """(L_b, K_b) of sequence b: its clamped cached length and the keys it attends."""
    if not append:
        k = min(max(raw, 0), cap)
        return k, k
    Lb = min(max(raw, 0), max(cap - n, 0))
    return Lb, min(Lb + n, cap)


def test_varlen_cache_lens_exhaustively(built):
    L = _h()
    out = (ctypes.c_int * 2)()
    for cap in (1, 128, 300, 1024):
        for n in sorted({0, 1, 7, cap - 1, cap, cap + 1, 2 * cap + 5}):
            for raw in list(range(-5, cap + 6)) + [cap + n, -2**31, 2**31 - 1]:
                for append in (0, 1):
                    L.tfa_internal_varlen_cache_lens(raw, cap, n, append, out)
                    Lb, Kb = lens_rule(raw, cap, n, append)
                    assert (out[0], out[1]) == (Lb, Kb), (cap, n, raw, append)
                    assert 0 <= Lb <= Kb <= cap
                    if append:
                        assert Kb - Lb == min(n, cap)         # every appended key that fits is attended


def test_varlen_append_offset_exhaustively(built):
    """Every appended token of every sequence and head: the element offset of its cache row through the table, or -1
    (dropped) when it does not fit the capacity or its entry is outside [0, num_blocks)."""
    L = _h()
    rng = random.Random(11)
    Hkv, D = 3, 64
    for page, mbps, B, nblk in ((128, 4, 5, 17), (256, 2, 4, 9), (128, 1, 3, 4)):
        cap = page * mbps
        cs_s, cs_h = Hkv * D + 8, D
        cs_b = page * cs_s
        stride = mbps + 1
        table = [rng.choice([-1, nblk, nblk + 7, -100] + list(range(nblk))) for _ in range(B * stride)]
        tarr = (ctypes.c_int * len(table))(*table)
        for n in (1, 5, 129, cap - 1, cap, cap + 3, 2 * cap):
            for raw in (-7, 0, 1, cap - n, cap, cap + 9, rng.randint(0, cap)):
                for b in range(B):
                    Lb, Kb = lens_rule(raw, cap, n, True)
                    for i in range(n):
                        key = Lb + i
                        for h in range(Hkv):
                            want = -1
                            if key < Kb:
                                blk = table[b * stride + key // page]
                                if 0 <= blk < nblk:
                                    want = blk * cs_b + (key % page) * cs_s + h * cs_h
                            got = L.tfa_internal_varlen_append_offset(raw, tarr, stride, b, i, h, page, cap, n, nblk,
                                                                      cs_b, cs_s, cs_h)
                            assert got == want, (page, n, raw, b, i, h)
        # contiguous: block b, page = capacity
        for n in (1, cap, cap + 2):
            for b in range(B):
                Lb, Kb = lens_rule(5, cap, n, True)
                for i in range(n):
                    got = L.tfa_internal_varlen_append_offset(5, None, 0, b, i, 1, cap, cap, n, B, cs_b * mbps, cs_s,
                                                              cs_h)
                    assert got == (b * cs_b * mbps + (Lb + i) * cs_s + cs_h if Lb + i < Kb else -1)


def _protocol_model():
    sys.path.insert(0, os.path.join(ROOT, "scripts"))
    import protocol_model as pm
    return pm


def test_protocol_model_varlen_cache_items():
    """Skipped items, tile-less items that are still written, and items with a V tail, in both ring depths."""
    pm = _protocol_model()
    kinds = set()
    for trial in range(400):
        rng = random.Random(90210 + trial)
        items, empty, vtail = pm.random_varlen_cache_items(rng)
        kinds |= {"skip" for i, n in enumerate(items) if n == 0 and i not in empty}
        kinds |= {"empty" for _ in empty} | {"vtail" for _ in vtail}
        pm.Sim(items, rng.choice([4, 8]), rng, empty, vtail).run()
    assert kinds == {"skip", "empty", "vtail"}


def test_protocol_model_catches_a_store_after_the_release_in_varlen_cache_items():
    """Mutation: the zeroing stores move after the warpgroup's release of the slot -> the producer may refill it
    under them, which the model must report on this mode's items too."""
    src = open(os.path.join(ROOT, "scripts", "protocol_model.py")).read()
    store = "            if item in self.vtail:                            # zero the V rows past the keys, then PV " \
            "reads the slot\n                yield from store_into(ev % N, (item, n - 1, \"V\"))\n"
    release = "            self.kv_empty[ev % N].arrive()\n            ent += 2 * n\n"
    assert store in src and release in src
    mutated = src.replace(store, "").replace(
        release, "            self.kv_empty[ev % N].arrive()\n            if item in self.vtail:\n"
                 "                yield from store_into(ev % N, (item, n - 1, \"V\"))\n            ent += 2 * n\n")
    ns = {"__name__": "mutated_model"}
    exec(compile(mutated, "mutated_model", "exec"), ns)
    caught = 0
    for trial in range(200):
        rng = random.Random(31 + trial)
        items, empty, vtail = ns["random_varlen_cache_items"](rng)
        try:
            ns["Sim"](items, 4, rng, empty, vtail).run()
        except AssertionError:
            caught += 1
    assert caught > 5


# ------------------------------------------------------------------ GPU ------------------------------------------------

@pytest.fixture(scope="module")
def tfa(built):
    import tfa_ctypes
    tfa_ctypes.lib()
    return tfa_ctypes


def _dt(kind):
    return torch.bfloat16 if kind == "bf16" else torch.float16


def offsets(ls):
    c = np.concatenate([[0], np.cumsum(ls)]).astype(int)
    return list(zip(c[:-1].tolist(), c[1:].tolist()))


def cu(ls):
    return torch.tensor(np.concatenate([[0], np.cumsum(ls)]), dtype=torch.int32, device="cuda")


def bits(t):
    return t.view(torch.int16)


class Problem:
    """Packed q (sum sq, Hq, D) and, with `new`, packed k_new / v_new (sum sq, Hkv, D); a pool (num_blocks, page, Hkv,
    D) behind a random permuted block table, or a contiguous (B, cap, Hkv, D) cache when page is None, whose first
    clamp(lens[b], 0, cap) keys of each sequence hold N(0, 0.5^2) data and every other slot `fill`."""

    def __init__(self, sq, lens, Hq, Hkv, D, kind, page, cap, seed=20, fill=float("nan"), new=True, spare=3):
        g = torch.Generator(device="cpu")
        g.manual_seed(seed)
        dt = _dt(kind)
        mk = lambda *s: torch.empty(s, dtype=torch.float32).normal_(0.0, 0.5, generator=g).to(dt)
        B, total = len(sq), sum(sq)
        self.sq, self.lens, self.cap, self.page, self.D, self.kind = sq, lens, cap, page, D, kind
        self.q = mk(total, Hq, D).cuda()
        self.kn = mk(total, Hkv, D).cuda() if new else None
        self.vn = mk(total, Hkv, D).cuda() if new else None
        if page is None:
            self.table, mbps, nblk = None, 1, B
            slots = [[b] for b in range(B)]
            shape = (B, cap, Hkv, D)
        else:
            mbps, nblk = cap // page, B * (cap // page) + spare
            perm = torch.randperm(nblk, generator=g)[:B * mbps].to(torch.int32).view(B, mbps)
            self.table = perm.cuda()
            slots = perm.tolist()
            shape = (nblk, page, Hkv, D)
        pools = []
        for _ in range(2):
            pool = torch.full(shape, fill, dtype=dt)
            for b in range(B):
                data = mk(cap, Hkv, D)
                data[min(max(lens[b], 0), cap):] = fill
                pool[torch.tensor(slots[b])] = data.view(len(slots[b]), -1, Hkv, D)
            pools.append(pool.cuda())
        self.k, self.v = pools
        self.seqlens = torch.tensor(lens, dtype=torch.int32, device="cuda")
        self.cu_q = cu(sq)
        self.max_q = max(sq)
        self.nblk = nblk

    def K(self, b, n=None):
        n = min(self.sq[b], self.max_q) if n is None else n
        return lens_rule(self.lens[b], self.cap, n, self.kn is not None)

    def run(self, tfa, causal, k=None, v=None, max_q=None, **kw):
        """The call under test on pools k / v (default: copies of the problem's), returning out, lse, k, v."""
        k = self.k.clone() if k is None else k
        v = self.v.clone() if v is None else v
        args = dict(k_new=self.kn, v_new=self.vn, is_causal=causal, scale=self.D ** -0.5)
        args.update(kw)
        out, lse = tfa.attn_varlen_kvcache_fwd(self.q, k, v, self.cu_q, self.max_q if max_q is None else max_q,
                                               self.seqlens, self.table, **args)
        return out, lse, k, v

    def per_sequence(self, tfa, causal, out_fp32=False):
        """One tfa_attn_kvcache_fwd call per sequence (B = 1, Sq = Snew = Sq_b, one split) on one copy of the pools:
        {b: (out (Sq_b, Hq, D), lse (Hq, Sq_b))}, and the pools after every append."""
        k, v = self.k.clone(), self.v.clone()
        res = {}
        for b, (q0, q1) in enumerate(offsets(self.sq)):
            if q1 == q0:
                continue
            if self.table is None:
                kc, vc, tab = k[b:b + 1], v[b:b + 1], None
            else:
                kc, vc, tab = k, v, self.table[b:b + 1]
            extra = {}
            if self.kn is not None:
                extra = dict(k_new=self.kn[q0:q1][None], v_new=self.vn[q0:q1][None])
            o, l = tfa.attn_kvcache_fwd(self.q[q0:q1][None], kc, vc, self.seqlens[b:b + 1], tab, is_causal=causal,
                                        scale=self.D ** -0.5, num_splits=1, out_fp32=out_fp32, **extra)
            res[b] = (o[0], l[0])
        return res, k, v

    def gather(self, pool, b, K):
        """Sequence b's first K keys of a pool as (K, Hkv, D)."""
        if self.table is None:
            return pool[b, :K]
        t = self.table[b].long()
        return pool[t].reshape(-1, *pool.shape[2:])[:K]


# (D, kind, Hq, Hkv, page, causal, new); page None: the contiguous cache
CASES = [
    (128, "bf16", 32, 8, 256, True, True),
    (128, "fp16", 8, 8, 128, True, False),
    (64, "fp16", 32, 8, None, True, True),
    (64, "bf16", 8, 8, 256, False, True),
    (128, "bf16", 32, 8, None, False, False),
    (64, "bf16", 32, 8, 128, True, True),
    (128, "fp16", 8, 8, 256, False, False),
    (64, "fp16", 8, 8, 128, True, False),
]
SQ = [129, 0, 1, 300, 127, 128, 1, 257, 5]


def case_lens(cap):
    """Cached lengths for SQ: 0, near the capacity (exactly full after the append, and past it), short caches under
    long query chunks (causal Sq_b > K_b without an append: key-less rows), negative."""
    return [0, 40, cap - 1, 3, cap - 127, 700, cap + 50, 100, -4]


@pytest.mark.gpu
@pytest.mark.parametrize("D,kind,Hq,Hkv,page,causal,new", CASES)
def test_varlen_kvcache_equals_per_sequence_cache_call_bitwise(tfa, D, kind, Hq, Hkv, page, causal, new):
    cap = 1100 if page is None else 1536
    P = Problem(SQ, case_lens(cap), Hq, Hkv, D, kind, page, cap, seed=D + Hq + int(causal), new=new)
    for f32 in (False, True):
        out, lse, k, v = P.run(tfa, causal, out_fp32=f32)
        ref, kr, vr = P.per_sequence(tfa, causal, out_fp32=f32)
        torch.cuda.synchronize()
        assert torch.equal(bits(k), bits(kr)) and torch.equal(bits(v), bits(vr))
        for b, (q0, q1) in enumerate(offsets(SQ)):
            if q1 == q0:
                continue
            assert torch.equal(out[q0:q1], ref[b][0]), (f32, b)
            assert torch.equal(lse[:, q0:q1], ref[b][1]), (f32, b)
        if causal and not new:                                   # a sequence with key-less rows is in the batch
            q0, q1 = offsets(SQ)[3]
            assert P.K(3)[1] == 3 and torch.isposinf(lse[:, q0:q0 + 297]).all()
            assert torch.count_nonzero(out[q0:q0 + 297]).item() == 0


@pytest.mark.gpu
@pytest.mark.parametrize("D,kind,page,causal,new", [(128, "bf16", 256, True, True), (64, "fp16", None, False, False),
                                                    (128, "fp16", 128, False, True), (64, "bf16", 128, True, False)])
def test_varlen_kvcache_equals_varlen_on_gathered_cache(tfa, D, kind, page, causal, new):
    """tfa_attn_varlen_fwd on K/V gathered from the pools after the append, with cu_seqlens_k built from K_b."""
    cap = 1100 if page is None else 1536
    lens = case_lens(cap)
    if causal and not new:
        lens[3] = 400                            # keep K_b >= Sq_b: rows without keys are covered above
    P = Problem(SQ, lens, 8, 2, D, kind, page, cap, seed=5, new=new)
    out, lse, k, v = P.run(tfa, causal)
    Ks = [P.K(b)[1] for b in range(len(SQ))]
    kg = torch.cat([P.gather(k, b, K) for b, K in enumerate(Ks)])
    vg = torch.cat([P.gather(v, b, K) for b, K in enumerate(Ks)])
    o2, l2 = tfa.attn_varlen_fwd(P.q, kg, vg, P.cu_q, cu(Ks), P.max_q, causal, D ** -0.5)
    torch.cuda.synchronize()
    assert torch.equal(out, o2) and torch.equal(lse, l2)


@pytest.mark.gpu
@pytest.mark.parametrize("new", [True, False])
def test_all_decode_batch_equals_one_cache_call(tfa, new):
    B, Hq, Hkv, D, page, cap = 24, 32, 8, 128, 256, 2048
    rng = random.Random(4)
    lens = [rng.randint(0, cap) for _ in range(B)]
    lens[0], lens[1] = 0, cap
    P = Problem([1] * B, lens, Hq, Hkv, D, "bf16", page, cap, seed=6, new=new)
    out, lse, k, v = P.run(tfa, True)
    k2, v2 = P.k.clone(), P.v.clone()
    extra = dict(k_new=P.kn[:, None], v_new=P.vn[:, None]) if new else {}
    o2, l2 = tfa.attn_kvcache_fwd(P.q[:, None], k2, v2, P.seqlens, P.table, is_causal=True, scale=D ** -0.5,
                                  num_splits=1, **extra)
    torch.cuda.synchronize()
    assert torch.equal(out, o2[:, 0]) and torch.equal(lse, l2[:, :, 0].t())
    assert torch.equal(bits(k), bits(k2)) and torch.equal(bits(v), bits(v2))


ORACLE = [
    # sq, lens, cap, page, causal, new, D, kind, Hq, Hkv
    ([300, 1, 0, 129, 64], [0, 900, 50, 1000, 10], 1024, 256, True, True, 128, "bf16", 8, 2),
    ([200, 3, 130], [5, 0, 64], 512, 128, True, False, 64, "fp16", 4, 1),     # causal Sq_b > K_b, K_b = 0
    ([300, 7, 129], [0, 100, 40], 200, None, True, True, 64, "bf16", 4, 2),   # Sq_b > capacity: keys dropped
    ([250, 1, 60], [1000, 3, 0], 1280, 128, False, True, 128, "fp16", 4, 4),
]


@pytest.mark.gpu
@pytest.mark.parametrize("sq,lens,cap,page,causal,new,D,kind,Hq,Hkv", ORACLE)
def test_varlen_kvcache_matches_oracle(tfa, sq, lens, cap, page, causal, new, D, kind, Hq, Hkv):
    from test_general_attn import check_lse, check_out16, check_out32, oracle_general
    P = Problem(sq, lens, Hq, Hkv, D, kind, page, cap, seed=3, new=new)
    o32, lse32, k, v = P.run(tfa, causal, out_fp32=True)
    o16, lse16, _, _ = P.run(tfa, causal)
    torch.cuda.synchronize()
    assert torch.equal(lse32, lse16)
    for b, (q0, q1) in enumerate(offsets(sq)):
        if q1 == q0:
            continue
        Sq, (Lb, K) = q1 - q0, P.K(b)
        if new:                                  # the appended keys that fit, from k_new
            fit = K - Lb
            assert torch.equal(bits(P.gather(k, b, K)[Lb:]), bits(P.kn[q0:q0 + fit]))
        n_empty = Sq if K == 0 else (min(Sq, max(0, Sq - K)) if causal else 0)
        got32, got16 = o32[q0:q1].permute(1, 0, 2)[None], o16[q0:q1].permute(1, 0, 2)[None]
        got_lse = lse32[:, q0:q1][None]
        if n_empty:
            assert torch.count_nonzero(got32[:, :, :n_empty]).item() == 0
            assert torch.count_nonzero(got16[:, :, :n_empty]).item() == 0
            assert torch.all(torch.isposinf(got_lse[:, :, :n_empty]))
        if n_empty == Sq:
            continue
        kk = P.gather(k, b, K).permute(1, 0, 2)[None]
        vv = P.gather(v, b, K).permute(1, 0, 2)[None]
        want32, want_lse = oracle_general(P.q[q0:q1].permute(1, 0, 2)[None], kk, vv, causal, D ** -0.5, kind,
                                          round_out=False)
        check_out32(got32, want32, causal)
        check_out16(got16, want32, kind)
        check_lse(got_lse, want_lse)


@pytest.mark.gpu
@pytest.mark.parametrize("D,kind,page", [(128, "bf16", 256), (64, "fp16", None)])
def test_nan_in_unused_cache_slots_changes_nothing(tfa, D, kind, page):
    cap = 768
    args = dict(sq=[129, 1, 0, 300, 2], lens=[300, 0, 10, 129, cap - 2], Hq=8, Hkv=2, D=D, kind=kind, page=page,
                cap=cap, seed=5)
    for new in (True, False):
        pz = Problem(fill=0.0, new=new, **args)
        pn = Problem(fill=float("nan"), new=new, **args)
        assert torch.isnan(pn.k).any() and torch.isnan(pn.v).any()
        for causal in (False, True):
            oz, lz, _, _ = pz.run(tfa, causal)
            on, ln, _, _ = pn.run(tfa, causal)
            torch.cuda.synchronize()
            assert torch.isfinite(on).all()
            assert torch.equal(oz, on) and torch.equal(lz, ln), (new, causal)


def scatter_append(P, pool, new, table, n_of):
    """What the append must do, in torch: token i of sequence b goes to key L_b + i through the table when it fits the
    capacity; a token whose entry lies outside [0, num_blocks) is dropped."""
    pool = pool.clone()
    tab = table.cpu().tolist() if table is not None else None
    for b, (q0, q1) in enumerate(offsets(P.sq)):
        n = n_of(b)
        Lb, Kb = P.K(b, n)
        for i in range(n):
            key = Lb + i
            if key >= Kb:
                continue
            if tab is None:
                pool[b, key] = new[q0 + i]
            else:
                blk = tab[b][key // P.page]
                if 0 <= blk < P.nblk:
                    pool[blk, key % P.page] = new[q0 + i]
    return pool


@pytest.mark.gpu
@pytest.mark.parametrize("f32", [False, True])
def test_exact_writes(tfa, f32):
    """The append writes exactly its tokens (an out-of-range table entry drops them); out / lse are written for the
    first max_seqlen_q rows of every sequence and nowhere else: rows past max_seqlen_q and guard regions either side
    of the buffers keep their NaN."""
    sq = [300, 0, 5, 200, 1, 150]
    max_q = 150
    lens = [0, 10, 1020, 256, -3, 700]
    Hq, Hkv, D, page, cap, G = 4, 2, 64, 128, 1024, 64
    P = Problem(sq, lens, Hq, Hkv, D, "bf16", page, cap, seed=12)
    P.max_q = max_q
    bad = P.table.clone()
    bad[3, 2] = -1                           # the append of sequence 3 (keys 256..405) crosses pages 2 and 3
    bad[3, 3] = P.nblk + 3
    tq = sum(sq)
    n_of = lambda b: min(sq[b], max_q)
    dt = torch.float32 if f32 else torch.bfloat16
    for tab in (P.table, bad):
        obuf = torch.full((G + tq * Hq * D + G,), float("nan"), dtype=dt, device="cuda")
        lbuf = torch.full((G + Hq * tq + G,), float("nan"), dtype=torch.float32, device="cuda")
        out, lse = obuf[G:G + tq * Hq * D].view(tq, Hq, D), lbuf[G:G + Hq * tq].view(Hq, tq)
        k, v = P.k.clone(), P.v.clone()
        P.table, keep = tab, P.table
        want_k, want_v = scatter_append(P, P.k, P.kn, tab, n_of), scatter_append(P, P.v, P.vn, tab, n_of)
        P.run(tfa, True, k=k, v=v, out=out, lse=lse, out_fp32=f32, max_q=max_q)
        P.table = keep
        torch.cuda.synchronize()
        assert torch.equal(bits(k), bits(want_k)) and torch.equal(bits(v), bits(want_v))
        assert torch.isnan(obuf[:G]).all() and torch.isnan(obuf[G + tq * Hq * D:]).all()
        assert torch.isnan(lbuf[:G]).all() and torch.isnan(lbuf[G + Hq * tq:]).all()
        for b, (q0, q1) in enumerate(offsets(sq)):
            n = n_of(b)
            assert not torch.isnan(out[q0:q0 + n]).any() and not torch.isnan(lse[:, q0:q0 + n]).any(), b
            assert torch.isnan(out[q0 + n:q1]).all() and torch.isnan(lse[:, q0 + n:q1]).all(), b
    # the rows that were computed are those of the sequences cut to their first max_seqlen_q rows
    sq2 = [min(s, max_q) for s in sq]
    P2 = Problem(sq2, lens, Hq, Hkv, D, "bf16", page, cap, seed=12)
    keep = [torch.cat([x[q0:q0 + n] for (q0, _), n in zip(offsets(sq), sq2)]) for x in (P.q, P.kn, P.vn)]
    P2.q, P2.kn, P2.vn = keep
    P2.k, P2.v, P2.table = P.k, P.v, P.table
    o1, l1, k1, _ = P.run(tfa, True, max_q=max_q)
    o2, l2, k2, _ = P2.run(tfa, True)
    torch.cuda.synchronize()
    assert torch.equal(bits(k1), bits(k2))
    for (q0, _), (p0, p1) in zip(offsets(sq), offsets(sq2)):
        assert torch.equal(o1[q0:q0 + p1 - p0], o2[p0:p1]) and torch.equal(l1[:, q0:q0 + p1 - p0], l2[:, p0:p1])


@pytest.mark.gpu
def test_varlen_kvcache_classic_and_persistent_agree_bitwise(tfa):
    code = r'''
import os, sys, torch
sys.path.insert(0, os.path.join(os.environ["TFA_ROOT"], "tiny-flash-attention_b200"))
sys.path.insert(0, os.path.join(os.environ["TFA_ROOT"], "tests"))
import tfa_ctypes as tfa
from test_varlen_kvcache import Problem, SQ, case_lens
res = []
for causal, new, page in ((True, True, 256), (False, False, None), (True, False, 128), (False, True, 128)):
    cap = 1100 if page is None else 1536
    P = Problem(SQ, case_lens(cap), 32, 8, 128, "bf16", page, cap, seed=9, new=new)
    o, lse, k, v = P.run(tfa, causal)
    res.append((o.cpu(), lse.cpu(), k.cpu().view(torch.int16), tfa.lib().tfa_internal_last_variant()))
torch.cuda.synchronize()
torch.save(res, os.environ["TFA_OUT"])
'''
    import tempfile
    outs = {}
    with tempfile.TemporaryDirectory() as tmp:
        for variant in ("classic", "persist"):
            path = os.path.join(tmp, variant + ".pt")
            env = dict(os.environ, TFA_ROOT=ROOT, TFA_OUT=path, TFA_KERNEL=variant)
            p = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=600)
            assert p.returncode == 0, p.stderr[-2000:]
            outs[variant] = torch.load(path)
    for (a, la, ka, va), (b, lb, kb, vb) in zip(outs["classic"], outs["persist"]):
        assert (va, vb) == (0, 4)
        assert torch.equal(a, b) and torch.equal(la, lb) and torch.equal(ka, kb)


@pytest.mark.gpu
def test_varlen_kvcache_cuda_graph_replays_with_new_offsets_lengths_and_table(tfa):
    """Capture one step (append + attention), then rewrite cu_seqlens_q (same total_q), cache_seqlens and the block
    table in place and replay: out, lse and the pools equal eager calls on the same state."""
    sq1, sq2 = [200, 1, 1, 54], [1, 129, 100, 26]
    lens1, lens2 = [300, 5, 1000, 0], [900, 0, 256, 1100]
    P = Problem(sq1, lens1, 8, 2, 128, "bf16", 256, 1280, seed=13, fill=0.0)   # the new table maps other pages
    k0, v0 = P.k.clone(), P.v.clone()
    k, v = P.k.clone(), P.v.clone()
    out = torch.empty((sum(sq1), 8, 128), dtype=torch.bfloat16, device="cuda")
    lse = torch.empty((8, sum(sq1)), dtype=torch.float32, device="cuda")
    step = lambda: P.run(tfa, True, k=k, v=v, out=out, lse=lse, max_q=256)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):                               # warm-up outside the capture
        step()
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        step()
    results = []
    for sq, lens, perm_seed in ((sq1, lens1, None), (sq2, lens2, 3)):
        if perm_seed is not None:
            gp = torch.Generator(device="cpu")
            gp.manual_seed(perm_seed)
            P.cu_q.copy_(cu(sq))
            P.seqlens.copy_(torch.tensor(lens, dtype=torch.int32))
            P.table.copy_(torch.randperm(P.nblk, generator=gp)[:P.table.numel()].to(torch.int32).view(P.table.shape))
        k.copy_(k0)
        v.copy_(v0)
        graph.replay()
        ke, ve = k0.clone(), v0.clone()
        eo, el = tfa.attn_varlen_kvcache_fwd(P.q, ke, ve, P.cu_q.clone(), 256, P.seqlens.clone(), P.table.clone(),
                                             P.kn, P.vn, is_causal=True, scale=128 ** -0.5)
        torch.cuda.synchronize()
        assert torch.equal(out, eo) and torch.equal(lse, el)
        assert torch.equal(bits(k), bits(ke)) and torch.equal(bits(v), bits(ve))
        results.append(out.clone())
    assert not torch.equal(results[0], results[1])


@pytest.mark.gpu
def test_varlen_kvcache_launch_counts(tfa):
    P = Problem([500, 0, 1, 129], [10, 0, 64, 129], 4, 2, 64, "fp16", 128, 768, seed=1)
    for new, want in ((False, 1), (True, 2)):
        kw = {} if new else dict(k_new=None, v_new=None)
        n0 = tfa.launch_count()
        P.run(tfa, True, **kw)
        assert tfa.launch_count() - n0 == want, new
    torch.cuda.synchronize()


@pytest.mark.gpu
def test_extension_varlen_kvcache_entry(built, tfa):
    import attention_cutlass as ac
    P = Problem([300, 1, 0, 129], [300, 1, 0, 640], 8, 2, 128, "bf16", 256, 1024, seed=17)
    scale = 128 ** -0.5
    k1, v1 = P.k.clone(), P.v.clone()
    out, lse = ac.flash_attention_v2_varlen_kvcache(P.q, k1, v1, P.cu_q, P.max_q, P.seqlens, P.table, P.kn, P.vn,
                                                    True, scale)
    want, wl, k2, v2 = P.run(tfa, True)
    torch.cuda.synchronize()
    assert out.shape == P.q.shape and out.dtype == torch.bfloat16 and lse.shape == (8, P.q.shape[0])
    assert lse.dtype == torch.float32
    assert torch.equal(out, want) and torch.equal(lse, wl) and torch.equal(bits(k1), bits(k2))
    # without an append, on a contiguous cache
    kc = torch.zeros((4, 700, 2, 128), dtype=torch.bfloat16, device="cuda")
    o3, l3 = ac.flash_attention_v2_varlen_kvcache(P.q, kc, kc, P.cu_q, P.max_q, P.seqlens, None, None, None, False,
                                                  scale)
    torch.cuda.synchronize()
    assert o3.shape == P.q.shape and torch.isfinite(o3).all()
    call = lambda **kw: ac.flash_attention_v2_varlen_kvcache(
        kw.get("q", P.q), kw.get("k", P.k), kw.get("v", P.v), kw.get("cu_q", P.cu_q), kw.get("max_q", P.max_q),
        kw.get("sl", P.seqlens), kw.get("table", P.table), kw.get("kn", None), kw.get("vn", None), True, scale)
    with pytest.raises(RuntimeError, match="int32"):
        call(cu_q=P.cu_q.long())
    with pytest.raises(RuntimeError, match="int32"):
        call(sl=P.seqlens.long())
    with pytest.raises(RuntimeError, match="device"):
        call(cu_q=P.cu_q.cpu())
    with pytest.raises(RuntimeError, match="B \\+ 1"):
        call(cu_q=P.cu_q[:1])
    with pytest.raises(RuntimeError, match="cache_seqlens"):
        call(sl=P.seqlens[:-1])
    with pytest.raises(RuntimeError, match="block_table"):
        call(table=P.table.long())
    with pytest.raises(RuntimeError, match="together"):
        call(kn=P.kn)
    with pytest.raises(RuntimeError, match="total_q, Hkv, D"):
        call(kn=P.kn[:-1], vn=P.vn[:-1])
    with pytest.raises(RuntimeError, match="multiple of K/V heads"):
        call(q=P.q[:, :3])
    with pytest.raises(RuntimeError, match="128"):
        call(k=P.k[:, :100], v=P.v[:, :100])
    with pytest.raises(RuntimeError, match="max_seqlen_q"):
        call(max_q=0)
    with pytest.raises(RuntimeError, match="3 dimensions"):
        call(q=P.q[None])
