"""Attention against a (paged) KV cache: tfa_attn_kvcache_fwd / attention_cutlass.flash_attention_v2_kvcache.

CPU: the entry point is declared and exported, every argument error comes back before any device work, the host-callable
page-lookup / append-index helpers match their definition exhaustively (out-of-range lengths and table entries
included), and the barrier-protocol model accepts the consumers' stores into a V slot and catches a store after the
release.
GPU: each sequence equals the dense tfa_attn_fwd on its gathered K/V bit for bit (where the dense path does the same
arithmetic), the contiguous cache equals the paged one, splits stay within the oracle's tolerances, NaN in unused cache
slots changes nothing, the append writes exactly its tokens, outputs stay inside their buffers, both schedules agree,
the call replays from a CUDA graph with new lengths and tables, and it is 1 / 2 / 3 launches."""
import ctypes
import os
import random
import subprocess
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

TFA_EINVAL_KVCACHE = -13


def declared_functions():
    import re
    src = open(os.path.join(ROOT, "include", "tfa_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return set(re.findall(r"\b(tfa_[a-z0-9_]+)\s*\(", src))


# ------------------------------------------------------------------ CPU ------------------------------------------------

def test_header_declares_and_library_exports_kvcache(built):
    import tfa_ctypes
    assert "tfa_attn_kvcache_fwd" in declared_functions()
    assert "TFA_EINVAL_KVCACHE (-13)" in open(os.path.join(ROOT, "include", "tfa_b200.h")).read()
    L = ctypes.CDLL(tfa_ctypes.LIB_PATH)
    assert hasattr(L, "tfa_attn_kvcache_fwd")


def test_kvcache_error_string(built):
    import tfa_ctypes
    msg = tfa_ctypes.lib().tfa_error_string(TFA_EINVAL_KVCACHE)
    assert msg.startswith(b"tfa:") and b"cache_seqlens" in msg and b"block_table" in msg and b"128" in msg


def test_kvcache_argument_validation_without_device(built):
    """Host buffers only: every code must come back before anything touches a device (on a CPU-only box a call that
    got that far would fail with a CUDA error instead)."""
    import tfa_ctypes
    L = tfa_ctypes.lib()
    buf = ctypes.create_string_buffer(4096 + 16)
    base = (ctypes.addressof(buf) + 15) & ~15
    ints = base + 1024                                        # 16-byte aligned, so 4-byte aligned
    Hq, Hkv, D, page = 4, 2, 64, 256

    def mk(**kw):
        return tfa_ctypes.KvcacheArgs(
            kw.get("q", base), base, base, kw.get("k_new", None), kw.get("v_new", None), kw.get("out", base), None,
            kw.get("seqlens", ints), kw.get("table", ints), kw.get("B", 2), kw.get("Hq", Hq), kw.get("Hkv", Hkv),
            kw.get("Sq", 1), kw.get("D", D), kw.get("nblk", 8), kw.get("page", page), kw.get("mbps", 4),
            kw.get("snew", 1), Hq * D, kw.get("qss", Hq * D), D, page * Hkv * D, kw.get("kss", Hkv * D), D,
            kw.get("bts", 4), Hkv * D, kw.get("nss", Hkv * D), D, kw.get("dtype", 0), 1, kw.get("scale", 0.1), 0,
            kw.get("splits", 1), None, 0, None)

    call = lambda **kw: L.tfa_attn_kvcache_fwd(ctypes.byref(mk(**kw)))
    assert L.tfa_attn_kvcache_fwd(None) == -1                 # TFA_EINVAL_PTR
    assert call(q=None) == -1 and call(q=base + 2) == -1 and call(out=base + 8) == -1
    assert call(k_new=base + 8, v_new=base) == -1
    assert call(D=96) == -2                                   # TFA_EINVAL_DIM
    assert call(B=0) == -3 and call(Sq=0) == -3 and call(Hq=0) == -3
    assert call(dtype=2) == -4                                # TFA_EINVAL_DTYPE
    assert call(qss=60) == -5 and call(kss=30) == -5          # TFA_EINVAL_STRIDE
    assert call(k_new=base, v_new=base, nss=12) == -5
    assert call(scale=-1.0) == -9 and call(scale=float("nan")) == -9              # TFA_EINVAL_SCALE
    assert call(Hkv=3) == -10                                 # TFA_EINVAL_HEADS
    E = TFA_EINVAL_KVCACHE
    assert call(seqlens=None) == E and call(seqlens=ints + 2) == E
    assert call(table=ints + 1) == E
    assert call(page=200) == E and call(page=64) == E         # paged: multiple of 128
    assert call(mbps=0) == E and call(nblk=0) == E and call(page=0) == E
    assert call(bts=3) == E                                   # table rows overlap
    assert call(k_new=base) == E and call(v_new=base) == E    # one of the pair
    assert call(k_new=base, v_new=base, snew=0) == E
    assert call(k_new=base, v_new=base, snew=4 * page + 1) == E                 # > capacity
    # contiguous cache (no table): one page of any size per sequence, block b
    assert call(table=None, page=300, mbps=2) == E and call(table=None, page=300, mbps=1, nblk=1) == E


def _h():
    import tfa_ctypes
    L = tfa_ctypes.lib()
    ip, ll, ci = ctypes.POINTER(ctypes.c_int), ctypes.c_longlong, ctypes.c_int
    L.tfa_internal_page_lookup.argtypes = [ip, ll, ci, ci, ci, ip]
    L.tfa_internal_cache_len.argtypes = [ci, ci, ci]
    L.tfa_internal_append_offset.argtypes = [ip, ip, ll, ci, ci, ci, ci, ci, ci, ci, ll, ll, ll]
    L.tfa_internal_append_offset.restype = ll
    return L


def test_cache_len_clamps_exhaustively(built):
    L = _h()
    for cap in (1, 128, 300, 1024):
        for snew in sorted({0, 1, 7, cap}):
            if snew > cap:
                continue
            for raw in list(range(-5, cap + 6)) + [-2**31, 2**31 - 1]:
                assert L.tfa_internal_cache_len(raw, cap, snew) == min(max(raw, 0), cap - snew), (cap, snew, raw)


def test_page_lookup_exhaustively(built):
    """Every key of every sequence, paged (page sizes 128 and 256, a strided table with out-of-range entries) and
    contiguous: the block is the table's entry as stored (hardware bounds-checks the loads), the row is key % page."""
    L = _h()
    rng = random.Random(3)
    out = (ctypes.c_int * 2)()
    for page, mbps, B in ((128, 5, 3), (256, 3, 4)):
        stride = mbps + 2
        table = [rng.randint(-3, B * mbps + 3) for _ in range(B * stride)]
        arr = (ctypes.c_int * len(table))(*table)
        for b in range(B):
            for key in range(mbps * page):
                L.tfa_internal_page_lookup(arr, stride, b, key, page, out)
                assert (out[0], out[1]) == (table[b * stride + key // page], key % page), (page, b, key)
    for cap in (1, 300):
        for b in range(3):
            for key in range(cap):
                L.tfa_internal_page_lookup(None, 0, b, key, cap, out)
                assert (out[0], out[1]) == (b, key)


def test_append_offset_exhaustively(built):
    """Every appended token of every sequence and head: the element offset of its cache row through the table, or -1
    (dropped) when the entry is outside [0, num_blocks); lengths outside [0, capacity - snew] are clamped."""
    L = _h()
    rng = random.Random(11)
    Hkv, D = 3, 64
    for page, mbps, B, nblk, snew in ((128, 4, 5, 17, 1), (256, 2, 4, 9, 5), (128, 3, 3, 9, 128 * 3)):
        cap = page * mbps
        cs_s, cs_h = Hkv * D + 8, D
        cs_b = page * cs_s
        stride = mbps + 1
        table = [rng.choice([-1, nblk, nblk + 7, -100] + list(range(nblk))) for _ in range(B * stride)]
        lens = [rng.choice([-7, 0, 1, cap - snew, cap, cap + 9, rng.randint(0, cap)]) for _ in range(B)]
        tarr = (ctypes.c_int * len(table))(*table)
        larr = (ctypes.c_int * B)(*lens)
        for b in range(B):
            Lb = min(max(lens[b], 0), cap - snew)
            for i in range(snew):
                key = Lb + i
                blk = table[b * stride + key // page]
                for h in range(Hkv):
                    want = blk * cs_b + (key % page) * cs_s + h * cs_h if 0 <= blk < nblk else -1
                    got = L.tfa_internal_append_offset(larr, tarr, stride, b, i, h, page, cap, snew, nblk, cs_b, cs_s,
                                                       cs_h)
                    assert got == want, (page, b, i, h)
        # contiguous: block b, page = capacity
        for b in range(B):
            Lb = min(max(lens[b], 0), cap - snew)
            for i in range(snew):
                got = L.tfa_internal_append_offset(larr, None, 0, b, i, 1, cap, cap, snew, B, cs_b * mbps, cs_s, cs_h)
                assert got == b * cs_b * mbps + (Lb + i) * cs_s + cs_h


def _protocol_model():
    sys.path.insert(0, os.path.join(ROOT, "scripts"))
    import protocol_model as pm
    return pm


def test_protocol_model_consumer_stores_into_v_slot():
    """KV-cache items: both warpgroups zero the tail of the last V tile between its kv_full and their release, mixed
    with items without tiles, in both ring depths."""
    pm = _protocol_model()
    for trial in range(400):
        rng = random.Random(777 + trial)
        items, empty, vtail = pm.random_cache_items(rng)
        pm.Sim(items, rng.choice([4, 8]), rng, empty, vtail).run()


def test_protocol_model_catches_a_store_after_the_release():
    """Mutation: the zeroing stores move after the warpgroup's release of the slot -> the producer may refill it
    under them, which the model must report."""
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
        items, empty, vtail = ns["random_cache_items"](rng)
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


def make_cache(lens, Sq, Hq, Hkv, D, kind, page, seed=20, fill=0.0, mbps=None, spare=3, snew=0):
    """q (B, Sq, Hq, D); a random permuted block table; a pool (num_blocks, page, Hkv, D) whose first K_b = lens[b]
    keys of each sequence hold N(0, 0.5^2) data and every other slot `fill`.  Returns q, k_pool, v_pool, table,
    seqlens (all on the GPU)."""
    g = torch.Generator(device="cpu")
    g.manual_seed(seed)
    dt = _dt(kind)
    B = len(lens)
    mk = lambda *s: torch.empty(s, dtype=torch.float32).normal_(0.0, 0.5, generator=g).to(dt)
    if mbps is None:
        mbps = max(1, -(-(max(lens) + snew) // page))
    nblk = B * mbps + spare
    perm = torch.randperm(nblk, generator=g)[:B * mbps].to(torch.int32).view(B, mbps)
    pools = []
    for _ in range(2):
        pool = torch.full((nblk, page, Hkv, D), fill, dtype=dt)
        for b in range(B):
            data = mk(mbps * page, Hkv, D)
            data[lens[b]:] = fill
            pool[perm[b].long()] = data.view(mbps, page, Hkv, D)
        pools.append(pool.cuda())
    q = mk(B, Sq, Hq, D).cuda()
    return q, pools[0], pools[1], perm.cuda(), torch.tensor(lens, dtype=torch.int32, device="cuda")


def gather(pool, table, b, K):
    """Sequence b's first K keys of a paged pool as a contiguous dense (1, Hkv, K, D) tensor."""
    mbps, page = table.shape[1], pool.shape[1]
    return pool[table[b].long()].reshape(mbps * page, *pool.shape[2:])[:K].permute(1, 0, 2)[None].contiguous()


def qseq(q, b):
    return q[b:b + 1].permute(0, 2, 1, 3).contiguous()        # (1, Hq, Sq, D)


def oseq(out, b):
    return out[b:b + 1].permute(0, 2, 1, 3)                   # (B, Sq, Hq, D) -> (1, Hq, Sq, D)


def check_keyless(out, lse, b, rows):
    assert torch.count_nonzero(oseq(out, b)[:, :, :rows]).item() == 0
    assert torch.all(torch.isposinf(lse[b, :, :rows]))


def check_vs_oracle(out, lse, q, kp, vp, table, b, K, causal, scale, kind):
    from test_general_attn import check_lse, check_out16, check_out32, oracle_general
    want32, want_lse = oracle_general(qseq(q, b), gather(kp, table, b, K), gather(vp, table, b, K), causal, scale, kind,
                                      round_out=False)
    got = oseq(out, b)
    if got.dtype == torch.float32:
        check_out32(got, want32, causal)
    else:
        check_out16(got, want32, kind)
    check_lse(lse[b:b + 1], want_lse)


BITWISE = [
    # D, kind, Hq, Hkv, page, Sq, causal
    (128, "bf16", 32, 8, 256, 1, False),
    (128, "fp16", 8, 8, 128, 4, True),
    (64, "bf16", 8, 1, 128, 200, True),
    (64, "fp16", 4, 1, 256, 1, True),
    (128, "bf16", 8, 2, 128, 200, False),
    (64, "bf16", 4, 4, 256, 4, False),
]
LENS = [300, 0, 128, 1, 1000, 256, 77]


@pytest.mark.gpu
@pytest.mark.parametrize("D,kind,Hq,Hkv,page,Sq,causal", BITWISE)
def test_kvcache_equals_dense_on_gathered_cache_bitwise(tfa, D, kind, Hq, Hkv, page, Sq, causal):
    """K_b multiples of 128 and not, and 0.  Causal with Sq > K_b as well: the first Sq - K_b rows see no key in both
    calls; the sequence is also checked against the oracle."""
    q, kp, vp, table, lens = make_cache(LENS, Sq, Hq, Hkv, D, kind, page)
    scale = D ** -0.5
    for f32 in (False, True):
        out, lse = tfa.attn_kvcache_fwd(q, kp, vp, lens, table, is_causal=causal, scale=scale, out_fp32=f32)
        for b, K in enumerate(LENS):
            if K == 0:
                check_keyless(out, lse, b, Sq)
                continue
            if causal and Sq > K:
                check_keyless(out, lse, b, Sq - K)
                check_vs_oracle(out, lse, q, kp, vp, table, b, K, causal, scale, kind)
            o_ref, l_ref = tfa.attn_fwd(qseq(q, b), gather(kp, table, b, K), gather(vp, table, b, K), causal, scale,
                                        num_splits=1, out_fp32=f32)
            assert torch.equal(oseq(out, b), o_ref), (f32, b, K)
            assert torch.equal(lse[b:b + 1], l_ref), (f32, b, K)
    torch.cuda.synchronize()


@pytest.mark.gpu
@pytest.mark.parametrize("causal", [False, True])
def test_contiguous_cache_equals_identity_table_and_dense(tfa, causal):
    lens = [500, 0, 129, 512]
    B, Sq, Hq, Hkv, D, page, mbps = 4, 4, 8, 2, 128, 128, 4
    q, kp, vp, _, sl = make_cache(lens, Sq, Hq, Hkv, D, "bf16", page, mbps=mbps, spare=0, seed=4)
    ident = torch.arange(B * mbps, dtype=torch.int32, device="cuda").view(B, mbps)
    kc, vc = kp.view(B, mbps * page, Hkv, D), vp.view(B, mbps * page, Hkv, D)
    o1, l1 = tfa.attn_kvcache_fwd(q, kp, vp, sl, ident, is_causal=causal)
    o2, l2 = tfa.attn_kvcache_fwd(q, kc, vc, sl, None, is_causal=causal)
    assert torch.equal(o1, o2) and torch.equal(l1, l2)
    # a contiguous capacity that is no multiple of 128 (TMA zero-fills the box past it)
    cap = 300
    kc3, vc3 = kc[:, :cap].contiguous(), vc[:, :cap].contiguous()
    sl3 = torch.tensor([300, 0, 129, 1], dtype=torch.int32, device="cuda")
    o3, l3 = tfa.attn_kvcache_fwd(q, kc3, vc3, sl3, None, is_causal=causal)
    for b, K in enumerate(sl3.tolist()):
        if K == 0:
            check_keyless(o3, l3, b, Sq)
            continue
        if causal and Sq > K:
            continue
        kd = kc3[b:b + 1, :K].permute(0, 2, 1, 3).contiguous()
        vd = vc3[b:b + 1, :K].permute(0, 2, 1, 3).contiguous()
        o_ref, l_ref = tfa.attn_fwd(qseq(q, b), kd, vd, causal, D ** -0.5, num_splits=1)
        assert torch.equal(oseq(o3, b), o_ref) and torch.equal(l3[b:b + 1], l_ref), b
    torch.cuda.synchronize()


SPLITS = [
    # lens, Sq, Hq, Hkv, D, kind, page, causal, num_splits
    ([4000, 0, 129, 2048], 1, 8, 2, 128, "bf16", 256, False, 5),
    ([4000, 77, 1000], 4, 4, 4, 64, "fp16", 128, True, 3),
    ([3000, 10], 200, 4, 1, 64, "bf16", 128, True, 4),
    ([8192], 1, 8, 1, 128, "fp16", 256, False, 0),          # automatic: one (batch, head) pair per 16 SMs
]


@pytest.mark.gpu
@pytest.mark.parametrize("lens,Sq,Hq,Hkv,D,kind,page,causal,ns", SPLITS)
def test_kvcache_split_kv_matches_oracle(tfa, lens, Sq, Hq, Hkv, D, kind, page, causal, ns):
    q, kp, vp, table, sl = make_cache(lens, Sq, Hq, Hkv, D, kind, page, seed=8, mbps=-(-max(lens) // page) + 2)
    scale = D ** -0.5
    o32, lse32, n = tfa.attn_kvcache_fwd(q, kp, vp, sl, table, is_causal=causal, scale=scale, num_splits=ns,
                                         out_fp32=True, return_splits=True)
    o16, lse16 = tfa.attn_kvcache_fwd(q, kp, vp, sl, table, is_causal=causal, scale=scale, num_splits=ns)
    torch.cuda.synchronize()
    assert n > 1
    assert torch.isfinite(o32).all() and torch.isfinite(o16).all()
    for b, K in enumerate(lens):
        rows = Sq if K == 0 else (max(0, Sq - K) if causal else 0)
        if rows:
            check_keyless(o32, lse32, b, rows)
            check_keyless(o16, lse16, b, rows)
        if K:
            check_vs_oracle(o32, lse32, q, kp, vp, table, b, K, causal, scale, kind)
            check_vs_oracle(o16, lse16, q, kp, vp, table, b, K, causal, scale, kind)


@pytest.mark.gpu
@pytest.mark.parametrize("ns", [1, 4])
@pytest.mark.parametrize("D,kind", [(128, "bf16"), (64, "fp16")])
def test_nan_in_unused_cache_slots_changes_nothing(tfa, ns, D, kind):
    """Unused slots of used pages and every unused page hold NaN: the output is finite and bitwise equal to the run
    whose unused slots hold zeros."""
    lens = [300, 0, 129, 1024, 1]
    args = dict(Sq=4, Hq=8, Hkv=2, D=D, kind=kind, page=256, seed=5, mbps=5, spare=4)
    q, kz, vz, table, sl = make_cache(lens, fill=0.0, **args)
    _, kn, vn, _, _ = make_cache(lens, fill=float("nan"), **args)
    assert torch.isnan(kn).any() and torch.isnan(vn).any()
    for causal in (False, True):
        for f32 in (False, True):
            oz, lz = tfa.attn_kvcache_fwd(q, kz, vz, sl, table, is_causal=causal, num_splits=ns, out_fp32=f32)
            on, ln = tfa.attn_kvcache_fwd(q, kn, vn, sl, table, is_causal=causal, num_splits=ns, out_fp32=f32)
            torch.cuda.synchronize()
            assert torch.isfinite(on).all()
            assert torch.equal(oz, on) and torch.equal(lz, ln), (causal, f32)


def scatter_append(pool, table, lens, new, page, nblk):
    """What the append must do, in torch: token i of sequence b goes to key clamp(L_b) + i through the table; a token
    whose entry lies outside [0, num_blocks) is dropped."""
    pool = pool.clone()
    mbps = table.shape[1]
    cap = mbps * page
    snew = new.shape[1]
    tab = table.cpu().tolist()
    for b, L in enumerate(lens):
        Lb = min(max(L, 0), cap - snew)
        for i in range(snew):
            key = Lb + i
            blk = tab[b][key // page]
            if 0 <= blk < nblk:
                pool[blk, key % page] = new[b, i]
    return pool


def bits(t):
    return t.view(torch.int16)


@pytest.mark.gpu
@pytest.mark.parametrize("snew,ns,page,kind", [(1, 1, 256, "bf16"), (4, 3, 128, "fp16"), (200, 1, 128, "bf16"),
                                               (3, 4, 256, "bf16")])
def test_append_writes_its_tokens_and_nothing_else(tfa, snew, ns, page, kind):
    """The pool after the call equals a torch scatter of k_new / v_new through the table, every other byte unchanged
    (NaN in unused slots included); the output equals a call on the pre-appended cache without k_new.  Lengths past
    the capacity or negative are clamped; a sequence with an out-of-range table entry drops those tokens."""
    Hq, Hkv, D = 8, 2, 128
    mbps = 4
    cap = mbps * page
    lens = [300, 0, cap, -9, 127, 2 * page - 1]
    q, kp, vp, table, _ = make_cache([min(max(L, 0), cap) for L in lens], 4, Hq, Hkv, D, kind, page, seed=12,
                                     fill=float("nan"), mbps=mbps)
    nblk = kp.shape[0]
    bad = table.clone()
    bad[5, 1] = -1                       # the append of sequence 5 crosses from page 1 into page 2
    bad[5, 2] = nblk + 3
    sl = torch.tensor(lens, dtype=torch.int32, device="cuda")
    g = torch.Generator(device="cpu")
    g.manual_seed(99)
    kn = torch.empty((6, snew, Hkv, D)).normal_(0, 0.5, generator=g).to(_dt(kind)).cuda()
    vn = torch.empty((6, snew, Hkv, D)).normal_(0, 0.5, generator=g).to(_dt(kind)).cuda()
    for tab in (table, bad):
        want_k = scatter_append(kp, tab, lens, kn, page, nblk)
        want_v = scatter_append(vp, tab, lens, vn, page, nblk)
        k1, v1 = kp.clone(), vp.clone()
        n0 = tfa.launch_count()
        out, lse = tfa.attn_kvcache_fwd(q, k1, v1, sl, tab, kn, vn, is_causal=True, num_splits=ns)
        assert tfa.launch_count() - n0 == (3 if ns > 1 else 2)
        torch.cuda.synchronize()
        assert torch.equal(bits(k1), bits(want_k)) and torch.equal(bits(v1), bits(want_v))
        if tab is bad:
            continue                     # reads through an out-of-range entry return zeros: no reference to compare
        # the same attention without the append, on the cache as the append left it
        seqlens_after = torch.tensor([min(max(L, 0), cap - snew) + snew for L in lens], dtype=torch.int32,
                                     device="cuda")
        o2, l2 = tfa.attn_kvcache_fwd(q, want_k, want_v, seqlens_after, tab, is_causal=True, num_splits=ns)
        torch.cuda.synchronize()
        assert torch.isfinite(out).all()
        assert torch.equal(out, o2) and torch.equal(lse, l2)


@pytest.mark.gpu
@pytest.mark.parametrize("f32,ns", [(False, 1), (True, 1), (False, 3)])
def test_kvcache_writes_every_row_and_nothing_else(tfa, f32, ns):
    """NaN-filled out / lse with guard regions on both sides: every row is written (K_b = 0 and key-less causal rows
    included), no guard byte changes."""
    lens = [200, 0, 129, 7, 700]
    Sq, Hq, D, G = 8, 4, 64, 64
    q, kp, vp, table, sl = make_cache(lens, Sq, Hq, 1, D, "bf16", 128, seed=5, fill=float("nan"))
    B = len(lens)
    n = B * Sq * Hq * D
    dt = torch.float32 if f32 else q.dtype
    obuf = torch.full((G + n + G,), float("nan"), dtype=dt, device="cuda")
    lbuf = torch.full((G + B * Hq * Sq + G,), float("nan"), dtype=torch.float32, device="cuda")
    out, lse = obuf[G:G + n].view(B, Sq, Hq, D), lbuf[G:G + B * Hq * Sq].view(B, Hq, Sq)
    tfa.attn_kvcache_fwd(q, kp, vp, sl, table, is_causal=True, out_fp32=f32, out=out, lse=lse, num_splits=ns)
    torch.cuda.synchronize()
    assert not torch.isnan(out).any() and not torch.isnan(lse).any()
    assert torch.isnan(obuf[:G]).all() and torch.isnan(obuf[G + n:]).all()
    assert torch.isnan(lbuf[:G]).all() and torch.isnan(lbuf[G + B * Hq * Sq:]).all()


@pytest.mark.gpu
def test_kvcache_classic_and_persistent_agree_bitwise(tfa):
    code = r'''
import os, sys, torch
sys.path.insert(0, os.path.join(os.environ["TFA_ROOT"], "tiny-flash-attention_b200"))
sys.path.insert(0, os.path.join(os.environ["TFA_ROOT"], "tests"))
import tfa_ctypes as tfa
from test_kvcache import make_cache
lens = [1000, 0, 129, 2049, 64, 300]
res = []
for causal, Sq, ns in ((True, 1, 1), (False, 4, 1), (True, 200, 1), (False, 1, 3)):
    q, kp, vp, table, sl = make_cache(lens, Sq, 8, 2, 128, "bf16", 256, seed=9, fill=float("nan"))
    o, lse = tfa.attn_kvcache_fwd(q, kp, vp, sl, table, is_causal=causal, num_splits=ns)
    res.append((o.cpu(), lse.cpu(), tfa.lib().tfa_internal_last_variant()))
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
    for (a, la, va), (b, lb, vb) in zip(outs["classic"], outs["persist"]):
        assert (va, vb) == (0, 4)
        assert torch.equal(a, b) and torch.equal(la, lb)


@pytest.mark.gpu
def test_kvcache_cuda_graph_replays_with_new_lengths_and_table(tfa):
    """Capture one decode step (append + attention + split-KV combine), then rewrite cache_seqlens and block_table in
    place and replay: out, lse and the cache equal eager calls on the same state."""
    lens1, lens2 = [300, 5, 1000, 129], [1000, 700, 0, 256]
    B, Hq, Hkv, D, page, mbps = 4, 8, 2, 128, 256, 5
    q, kp, vp, table, sl = make_cache(lens1, 1, Hq, Hkv, D, "bf16", page, seed=13, mbps=mbps)
    k0, v0 = kp.clone(), vp.clone()
    g = torch.Generator(device="cpu")
    g.manual_seed(5)
    kn = torch.empty((B, 1, Hkv, D)).normal_(0, 0.5, generator=g).to(torch.bfloat16).cuda()
    vn = torch.empty((B, 1, Hkv, D)).normal_(0, 0.5, generator=g).to(torch.bfloat16).cuda()
    out = torch.empty_like(q)
    lse = torch.empty((B, Hq, 1), dtype=torch.float32, device="cuda")
    step = lambda: tfa.attn_kvcache_fwd(q, kp, vp, sl, table, kn, vn, is_causal=True, num_splits=3, out=out, lse=lse)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):                               # warm-up outside the capture
        step()
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        step()

    def eager(lens_t, tab):
        kc, vc = k0.clone(), v0.clone()
        o, l = tfa.attn_kvcache_fwd(q, kc, vc, lens_t.clone(), tab.clone(), kn, vn, is_causal=True, num_splits=3)
        return o, l, kc, vc

    results = []
    for lens, perm_seed in ((lens1, None), (lens2, 3)):
        if perm_seed is not None:
            gp = torch.Generator(device="cpu")
            gp.manual_seed(perm_seed)
            sl.copy_(torch.tensor(lens, dtype=torch.int32))
            table.copy_(torch.randperm(kp.shape[0], generator=gp)[:B * mbps].to(torch.int32).view(B, mbps))
        kp.copy_(k0)
        vp.copy_(v0)
        graph.replay()
        want_o, want_l, want_k, want_v = eager(sl, table)
        torch.cuda.synchronize()
        assert torch.equal(out, want_o) and torch.equal(lse, want_l)
        assert torch.equal(bits(kp), bits(want_k)) and torch.equal(bits(vp), bits(want_v))
        results.append(out.clone())
    assert not torch.equal(results[0], results[1])


@pytest.mark.gpu
def test_kvcache_launch_counts(tfa):
    q, kp, vp, table, sl = make_cache([500, 0, 64, 129], 1, 4, 2, 64, "fp16", 128, seed=1, mbps=5)
    kn = torch.zeros((4, 1, 2, 64), dtype=torch.float16, device="cuda")
    for kw, want in ((dict(), 1), (dict(k_new=kn, v_new=kn), 2), (dict(num_splits=3), 2),
                     (dict(k_new=kn, v_new=kn, num_splits=3), 3)):
        n0 = tfa.launch_count()
        tfa.attn_kvcache_fwd(q, kp, vp, sl, table, is_causal=True, **kw)
        assert tfa.launch_count() - n0 == want, kw
    torch.cuda.synchronize()


@pytest.mark.gpu
def test_extension_kvcache_entry(built, tfa):
    import attention_cutlass as ac
    lens = [300, 1, 0, 640]
    q, kp, vp, table, sl = make_cache(lens, 2, 8, 2, 128, "bf16", 256, seed=17, fill=float("nan"), mbps=4)
    scale = 128 ** -0.5
    out, lse = ac.flash_attention_v2_kvcache(q, kp, vp, sl, table, None, None, True, scale, 1)
    want, wl = tfa.attn_kvcache_fwd(q, kp, vp, sl, table, is_causal=True, scale=scale)
    torch.cuda.synchronize()
    assert out.shape == q.shape and out.dtype == torch.bfloat16 and lse.shape == (4, 8, 2)
    assert torch.equal(out, want) and torch.equal(lse, wl)
    # a non-dense q (a strided view) is computed as its contiguous copy
    qv = torch.cat([q, q], dim=2)[:, :, :8]
    o2, l2 = ac.flash_attention_v2_kvcache(qv, kp, vp, sl, table, None, None, True, scale, 1)
    assert torch.equal(o2, out) and torch.equal(l2, lse)
    # contiguous cache + append + automatic splits
    kc = torch.zeros((4, 1024, 2, 128), dtype=torch.bfloat16, device="cuda")
    vc = torch.zeros_like(kc)
    kn = torch.ones((4, 1, 2, 128), dtype=torch.bfloat16, device="cuda")
    o3, l3 = ac.flash_attention_v2_kvcache(q, kc, vc, sl, None, kn, kn, False, scale, 0)
    torch.cuda.synchronize()
    assert torch.equal(kc[torch.arange(4), sl.long()], kn[:, 0]) and torch.isfinite(o3).all()
    with pytest.raises(RuntimeError, match="int32"):
        ac.flash_attention_v2_kvcache(q, kp, vp, sl.long(), table, None, None, True, scale, 1)
    with pytest.raises(RuntimeError, match="block_table"):
        ac.flash_attention_v2_kvcache(q, kp, vp, sl, table.long(), None, None, True, scale, 1)
    with pytest.raises(RuntimeError, match="together"):
        ac.flash_attention_v2_kvcache(q, kp, vp, sl, table, kn, None, True, scale, 1)
    with pytest.raises(RuntimeError, match="multiple of K/V heads"):
        ac.flash_attention_v2_kvcache(q[:, :, :3], kp, vp, sl, table, None, None, True, scale, 1)
    with pytest.raises(RuntimeError, match="128"):
        ac.flash_attention_v2_kvcache(q, kp[:, :100], vp[:, :100], sl, table, None, None, True, scale, 1)
