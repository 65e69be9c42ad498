"""Split-KV for the variable-length KV-cache calls: tfa_attn_varlen_kvcache_split_fwd /
tfa_attn_varlen_kvcache_qkv8_split_fwd and the num_splits keyword of the attention_cutlass varlen-cache bindings.

CPU: the header declares and the library exports the four symbols, every argument error comes back before any device
work in the documented order, the workspace size and the split count follow their definitions (the split count is the
dense problem's), the combine's packed row -> sequence rule matches its definition exhaustively (malformed offsets
included), and the bindings take num_splits=.
GPU: each sequence equals the dense-query cache call at the same num_splits bit for bit (16-bit and FP8 caches, rotary,
e4m3 q, a 16-bit q quantized in the append), one split and auto without a workspace equal the call without split, auto
with a workspace equals the count it reports, rows outside the computed ones keep their contents, a NaN workspace and
NaN in unused slots change nothing, a long decode in a mixed batch stays within the float64 budget, the call replays
from a CUDA graph, both schedules agree, and the launch counts are right."""
import ctypes
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from test_fwd_float64_reference import compare, reference
from test_kvcache_rotary import rope_tables
from test_varlen_kvcache import Problem, case_lens, cu, declared_functions, offsets

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FP8 = torch.float8_e4m3fn
NEW = ("tfa_attn_varlen_kvcache_split_fwd", "tfa_attn_varlen_kvcache_qkv8_split_fwd",
       "tfa_attn_varlen_kvcache_num_splits", "tfa_attn_varlen_kvcache_workspace_bytes")


# ------------------------------------------------------------------ CPU ------------------------------------------------

def test_header_declares_and_library_exports_split_calls(built):
    import tfa_ctypes
    decl = declared_functions()
    L = ctypes.CDLL(tfa_ctypes.LIB_PATH)
    for name in NEW:
        assert name in decl and hasattr(L, name), name
    assert "tfa_split_args" in open(os.path.join(ROOT, "include", "tfa_b200.h")).read()
    assert L.tfa_abi_version() == 2


def _host_args(tfa_ctypes, base, ints, **kw):
    Hq, Hkv, D, page = kw.get("Hq", 4), 2, kw.get("D", 64), 256
    return tfa_ctypes.VarlenKvcacheArgs(
        base, base, base, kw.get("k_new", None), kw.get("k_new", None), base, None, ints, ints, ints, kw.get("B", 2),
        Hq, Hkv, D, kw.get("total_q", 300), kw.get("max_q", 200), 8, page, kw.get("mbps", 4), Hq * D, D,
        page * Hkv * D, Hkv * D, D, 4, Hkv * D, D, 0, 1, kw.get("scale", 0.1), 0, None)


def test_split_argument_errors_without_device(built):
    """Host buffers only: every code comes back before anything touches a device.  A call whose arguments all pass
    reaches the device check (TFA_EARCH without a GPU); the workspace is checked after it."""
    import tfa_ctypes
    L = tfa_ctypes.lib()
    buf = ctypes.create_string_buffer(4096 + 16)
    base = (ctypes.addressof(buf) + 15) & ~15
    ints = base + 1024
    SA, QA = tfa_ctypes.SplitArgs, tfa_ctypes.QkvQuantArgs
    rot = tfa_ctypes.RotaryArgs(base, base, 4096, 64, 0, base)
    qa = QA(2, 0.5, 0.5, 0.5)

    def call(sp=SA(2, None, 0), rotary=None, **kw):
        return L.tfa_attn_varlen_kvcache_split_fwd(ctypes.byref(_host_args(tfa_ctypes, base, ints, **kw)),
                                                   rotary and ctypes.byref(rotary), None,
                                                   sp and ctypes.byref(sp))

    def call8(sp=SA(2, None, 0), q8=None, rotary=None, quant=qa, **kw):
        return L.tfa_attn_varlen_kvcache_qkv8_split_fwd(ctypes.byref(_host_args(tfa_ctypes, base, ints, **kw)),
                                                        rotary and ctypes.byref(rotary), quant and ctypes.byref(quant),
                                                        q8, sp and ctypes.byref(sp))

    assert L.tfa_attn_varlen_kvcache_split_fwd(None, None, None, ctypes.byref(SA(2, None, 0))) == -1
    assert call(sp=None) == -1 and call8(sp=None) == -1 and call8(quant=None) == -1
    assert call8(q8=base + 8) == -1                                     # misaligned q8
    assert call8(rotary=rot) == -14                                     # e4m3 q: nothing to rotate
    assert call(mbps=0, B=0) == -13                                     # the cache first, as the call without split
    assert call(D=96) == -2 and call(B=0) == -3 and call(scale=-1.0) == -9
    assert call(sp=SA(-1, None, 0)) == -3 and call8(sp=SA(-5, None, 0)) == -3   # num_splits < 0
    assert call(sp=SA(-1, None, 0), D=96) == -2                         # among the shape checks, in their order
    assert call(max_q=0) == -12 and call(max_q=0, sp=SA(-1, None, 0)) == -3
    assert call(rotary=rot) == -14                                      # rotary needs k_new
    assert call8(quant=QA(1, 0.5, 0.5, 0.5)) == -16
    # every argument passes: the device check (no GPU), or on an H100 the missing workspace, before any device work
    want = -11 if torch.cuda.is_available() else -7
    assert call(sp=SA(2, None, 0)) == want and call(sp=SA(3, base + 8, 1 << 20)) == want
    assert call8(sp=SA(2, base, 16)) == want                            # too small


def test_workspace_bytes_formula(built):
    import tfa_ctypes
    L = tfa_ctypes.lib()
    buf = ctypes.create_string_buffer(4096 + 16)
    base = (ctypes.addressof(buf) + 15) & ~15
    for Hq, D, total_q, B in ((4, 64, 300, 2), (32, 128, 1, 1), (8, 128, 70000, 5)):
        a = _host_args(tfa_ctypes, base, base, Hq=Hq, D=D, total_q=total_q, B=B)
        for n in (0, 1, 2, 3, 16, 1024):
            want = n * Hq * total_q * (D + 1) * 4 if n > 1 else 0
            assert L.tfa_attn_varlen_kvcache_workspace_bytes(ctypes.byref(a), n) == want, (Hq, D, total_q, n)
    assert L.tfa_attn_varlen_kvcache_workspace_bytes(None, 2) == 0


def test_num_splits_matches_the_dense_problem(built):
    """The split count of (B, Hq, max_seqlen_q, capacity, causal) under tfa_attn_num_splits, over a grid of shapes,
    clamped to the KV tiles of the capacity."""
    import tfa_ctypes
    L = tfa_ctypes.lib()
    buf = ctypes.create_string_buffer(4096 + 16)
    base = (ctypes.addressof(buf) + 15) & ~15
    seen = set()
    for B in (1, 3, 64):
        for Hq in (4, 32):
            for max_q in (1, 129, 1000):
                for mbps in (1, 3, 64, 512):
                    for causal in (0, 1):
                        for n in (0, 1, 2, 3, 8, 1024):
                            a = _host_args(tfa_ctypes, base, base, B=B, Hq=Hq, max_q=max_q, total_q=max_q * B,
                                           mbps=mbps)
                            a.is_causal = causal
                            cap = mbps * 256
                            d = tfa_ctypes.AttnArgs(None, None, None, None, None, B, Hq, 2, max_q, cap, 64, 0, 0, 0,
                                                    0, 0, 0, 0, causal, 0.1, 0, n, None, 0, None)
                            got = L.tfa_attn_varlen_kvcache_num_splits(ctypes.byref(a), n)
                            assert got == L.tfa_attn_num_splits(ctypes.byref(d)), (B, Hq, max_q, mbps, causal, n)
                            if n > 1:
                                nkv = -(-cap // 128)
                                t = -(-nkv // min(n, nkv))
                                assert got == (-(-nkv // t) if min(n, nkv) > 1 else 1)
                            seen.add(got)
    assert {1, 2, 3, 8} <= seen
    assert L.tfa_attn_varlen_kvcache_num_splits(None, 2) == 1


def packed_rule(cu_l, B, total, S, r):
    """The combine's row rule: the b with clamp(cu[b]) <= r < clamp(cu[b+1]) that an upper-bound binary search over
    cu[0..B] finds, and whether r is one of that sequence's first S rows."""
    c = lambda x: min(max(x, 0), total)
    lo, hi = 0, B + 1
    while lo < hi:
        mid = (lo + hi) // 2
        if c(cu_l[mid]) <= r:
            lo = mid + 1
        else:
            hi = mid
    b = lo - 1
    if b < 0 or b >= B:
        return False, b, -1
    return r - c(cu_l[b]) < S, b, r - c(cu_l[b])


def test_packed_row_sequence_rule_exhaustively(built):
    """Every packed row of well-formed and malformed offsets (decreasing, negative, past total_q): the row is merged
    exactly when it is one of the first min(Sq_b, S) rows of a sequence b whose rows hold it, and then with that
    sequence's b and i; the search reads only cu[0..B] (a guard entry holding a trap value is never seen)."""
    import tfa_ctypes
    L = tfa_ctypes.lib()
    L.tfa_internal_packed_row_seq.argtypes = [ctypes.POINTER(ctypes.c_int), ctypes.c_int, ctypes.c_int, ctypes.c_int,
                                              ctypes.c_int, ctypes.POINTER(ctypes.c_int)]
    rng = np.random.default_rng(7)
    cases = [([0, 3, 3, 10, 12], 12), ([0, 12], 12), ([2, 5, 9], 12), ([0, 5, 2, 9, 7, 12], 12),
             ([-4, 3, 20, 6], 12), ([5, 5, 5], 6), ([7, 1], 8), ([-9, -2, 0, 40], 16), ([0, 1, 2, 3, 4, 5, 6], 6)]
    for _ in range(200):
        B = int(rng.integers(1, 9))
        total = int(rng.integers(1, 40))
        cases.append((rng.integers(-5, total + 6, size=B + 1).tolist(), total))
    out = (ctypes.c_int * 2)()
    for cu_l, total in cases:
        B = len(cu_l) - 1
        arr = (ctypes.c_int * (B + 2))(*(cu_l + [-2 ** 31]))            # the guard entry past cu[B]
        for S in (1, 2, 3, total):
            for r in range(total):
                got = L.tfa_internal_packed_row_seq(arr, B, total, S, r, out)
                ok, b, i = packed_rule(cu_l, B, total, S, r)
                assert bool(got) == ok, (cu_l, total, S, r)
                if ok:
                    assert (out[0], out[1]) == (b, i)
                    c = lambda x: min(max(x, 0), total)
                    assert c(cu_l[b]) <= r < c(cu_l[b + 1]) and i < S   # inside sequence b's computed rows
                    if all(x <= y for x, y in zip(cu_l, cu_l[1:])) and cu_l[0] >= 0:
                        assert sum(c(cu_l[k]) <= r < c(cu_l[k + 1]) for k in range(B)) == 1
                elif all(x <= y for x, y in zip(cu_l, cu_l[1:])):
                    # well-formed offsets: a row not merged is in no sequence or past its first S rows
                    c = lambda x: min(max(x, 0), total)
                    assert not any(c(cu_l[k]) <= r < c(cu_l[k]) + min(c(cu_l[k + 1]) - c(cu_l[k]), S)
                                   for k in range(B))


def test_bindings_accept_num_splits(built):
    """CPU tensors stop at the CUDA check: a binding that did not take num_splits= would raise TypeError."""
    import attention_cutlass as ac
    q = torch.zeros((4, 2, 64), dtype=torch.bfloat16)
    kc = torch.zeros((1, 128, 2, 64), dtype=torch.bfloat16)
    k8, q8 = kc.to(FP8), q.to(FP8)
    c = torch.tensor([0, 4], dtype=torch.int32)
    sl = torch.zeros(1, dtype=torch.int32)
    calls = [
        lambda: ac.flash_attention_v2_varlen_kvcache(q, kc, kc, c, 4, sl, None, None, None, True, 0.1, num_splits=2),
        lambda: ac.flash_attention_v2_varlen_kvcache_rotary(q, kc, kc, c, 4, sl, None, q[:, :1], q[:, :1], kc[0, :, 0],
                                                            kc[0, :, 0], False, True, 0.1, num_splits=0),
        lambda: ac.flash_attention_v2_varlen_kvcache_fp8(q, k8, k8, c, 4, sl, None, None, None, 1.0, 1.0, True, 0.1,
                                                         num_splits=3),
        lambda: ac.flash_attention_v2_varlen_kvcache_qkv8(q8, k8, k8, c, 4, sl, None, None, None, 1.0, 1.0, 1.0, True,
                                                          0.1, torch.bfloat16, num_splits=8),
        lambda: ac.flash_attention_v2_varlen_kvcache_qkv8_q16(q, k8, k8, c, 4, sl, None, None, None, 1.0, 1.0, 1.0,
                                                              True, 0.1, num_splits=1024),
    ]
    for f in calls:
        with pytest.raises(RuntimeError, match="CUDA"):
            f()


# ------------------------------------------------------------------ GPU ------------------------------------------------

@pytest.fixture(scope="module")
def tfa(built):
    import tfa_ctypes
    tfa_ctypes.lib()
    return tfa_ctypes


def bits(t):
    return t.view({1: torch.uint8, 2: torch.int16, 4: torch.int32}[t.element_size()])


def to_fp8(t, s):
    return (t.float() / s).clamp(-448, 448).to(FP8)            # NaN stays NaN (code 0x7f)


KS, VS, QS = 0.0123, 0.00731, 0.0171


def make_variant(variant, sq, lens, Hq, Hkv, D, kind, page, cap, seed, new=True, fill=float("nan")):
    """Problem P of test_varlen_kvcache turned into `variant`, and the keyword arguments both calls take for it."""
    P = Problem(sq, lens, Hq, Hkv, D, kind, page, cap, seed=seed, new=new, fill=fill)
    kw = {}
    if variant in ("fp8", "rotary_fp8", "qkv8", "q16", "q16_rotary"):
        P.k, P.v = to_fp8(P.k, KS), to_fp8(P.v, VS)
        kw.update(k_scale=KS, v_scale=VS)
    if variant.startswith("rotary") or variant == "q16_rotary":
        cos, sin = rope_tables(cap + 64, 64 if D == 128 else D, kind)
        kw.update(rotary_cos=cos, rotary_sin=sin, rotary_interleaved=(D == 64))
    if variant == "qkv8":
        P.q = to_fp8(P.q, QS)
        kw.update(q_scale=QS, out_dtype=torch.bfloat16 if kind == "bf16" else torch.float16)
    if variant.startswith("q16"):
        kw.update(q8_scale=QS)
    return P, kw


def per_sequence(tfa, P, causal, ns, kw, out_fp32=False):
    """The dense-query cache call per sequence (B = 1, Sq = Snew = n_b, num_splits = ns) on one copy of the pools:
    {b: (out (n_b, Hq, D), lse (Hq, n_b), splits)} and the pools after every append."""
    k, v = P.k.clone(), P.v.clone()
    res = {}
    for b, (q0, q1) in enumerate(offsets(P.sq)):
        n = min(q1 - q0, P.max_q)
        if n == 0:
            continue
        kc, vc, tab = (k[b:b + 1], v[b:b + 1], None) if P.table is None else (k, v, P.table[b:b + 1])
        extra = dict(k_new=P.kn[q0:q0 + n][None], v_new=P.vn[q0:q0 + n][None]) if P.kn is not None else {}
        o, l, got = tfa.attn_kvcache_fwd(P.q[q0:q0 + n][None], kc, vc, P.seqlens[b:b + 1], tab, is_causal=causal,
                                         scale=P.D ** -0.5, num_splits=ns, out_fp32=out_fp32, return_splits=True,
                                         **extra, **kw)
        res[b] = (o[0], l[0], got)
    return res, k, v


def run(tfa, P, causal, kw, **extra):
    k, v = P.k.clone(), P.v.clone()
    out, lse, n = tfa.attn_varlen_kvcache_fwd(P.q, k, v, P.cu_q, P.max_q, P.seqlens, P.table, P.kn, P.vn,
                                              is_causal=causal, scale=P.D ** -0.5, return_splits=True, **kw, **extra)
    return out, lse, n, k, v


# (D, kind, Hq, Hkv, page, causal, new, variant); page None: the contiguous cache
CASES = [
    (128, "bf16", 32, 8, 256, True, True, "plain"),
    (64, "fp16", 8, 8, None, True, False, "plain"),          # K_b = 0 and causal key-less rows (n_b > K_b)
    (128, "fp16", 8, 8, 128, False, True, "plain"),
    (64, "bf16", 32, 8, 128, False, False, "plain"),
    (128, "bf16", 16, 4, 256, True, True, "fp8"),
    (64, "fp16", 16, 4, None, False, False, "fp8"),
    (128, "fp16", 16, 4, 256, True, True, "rotary"),
    (64, "bf16", 16, 4, 128, False, True, "rotary_fp8"),
    (128, "bf16", 16, 4, 256, True, True, "qkv8"),
    (64, "fp16", 16, 4, 128, False, False, "qkv8"),
    (64, "fp16", 16, 4, 128, False, True, "q16"),
    (128, "bf16", 16, 4, 256, True, True, "q16_rotary"),
]
SQ = [129, 0, 1, 300, 127, 128, 1, 257, 5]


@pytest.mark.gpu
@pytest.mark.parametrize("D,kind,Hq,Hkv,page,causal,new,variant", CASES)
def test_split_equals_per_sequence_dense_call_bitwise(tfa, D, kind, Hq, Hkv, page, causal, new, variant):
    """At num_splits 2, 3, 8 and one clamped to the capacity's tiles, each sequence's out and lse (and the pools) equal
    the dense-query cache call on that sequence alone at the same num_splits.  The batch holds Sq_b = 0, K_b = 0 or
    key-less causal rows (without an append), K_b = capacity, K_b not a multiple of 128, and splits wholly past K_b."""
    cap = 1100 if page is None else 1536
    nkv = -(-cap // 128)
    P, kw = make_variant(variant, SQ, case_lens(cap), Hq, Hkv, D, kind, page, cap, seed=D + Hq + int(causal), new=new)
    for ns in (2, 3, 8, 64):
        f32 = ns == 3 and variant == "plain"
        out, lse, n, k, v = run(tfa, P, causal, kw, num_splits=ns, out_fp32=f32)
        ref, kr, vr = per_sequence(tfa, P, causal, ns, kw, out_fp32=f32)
        torch.cuda.synchronize()
        t = -(-nkv // min(ns, nkv))
        assert n == -(-nkv // t) and all(r[2] == n for r in ref.values()), (ns, n)
        assert torch.equal(bits(k), bits(kr)) and torch.equal(bits(v), bits(vr)), ns
        for b, (q0, q1) in enumerate(offsets(SQ)):
            if b in ref:
                assert torch.equal(bits(out[q0:q1]), bits(ref[b][0])), (ns, b)
                assert torch.equal(bits(lse[:, q0:q1]), bits(ref[b][1])), (ns, b)
        if causal and not new:
            q0, _ = offsets(SQ)[3]
            assert torch.isposinf(lse[:, q0:q0 + 297]).all() and torch.count_nonzero(out[q0:q0 + 297]).item() == 0


@pytest.mark.gpu
@pytest.mark.parametrize("variant", ["plain", "rotary_fp8", "qkv8", "q16_rotary"])
def test_one_split_and_auto_without_workspace_equal_the_call_without_split(tfa, variant):
    """num_splits = 1 (through the attention_cutlass binding, which always takes the split entry point) and auto with
    no workspace: out, lse and the pools bit-identical to the call without split, with its launch count."""
    D, kind, page, cap = 128, "bf16", 256, 4096
    P, kw = make_variant(variant, [1, 1, 3, 1], [4000, 100, 2049, 0], 8, 2, D, kind, page, cap, seed=3)
    out0, lse0, _, k0, v0 = run(tfa, P, True, kw)
    torch.cuda.synchronize()
    n0 = tfa.launch_count()
    outa, lsea, _, ka, va = run(tfa, P, True, kw, num_splits=0, workspace=torch.empty(0, device="cuda"))
    torch.cuda.synchronize()
    assert tfa.launch_count() - n0 == 2                             # the append and the forward, no combine
    for a, b in ((outa, out0), (lsea, lse0), (ka, k0), (va, v0)):
        assert torch.equal(bits(a), bits(b))
    if variant == "plain":
        import attention_cutlass as ac
        k1, v1 = P.k.clone(), P.v.clone()
        o1, l1 = ac.flash_attention_v2_varlen_kvcache(P.q, k1, v1, P.cu_q, P.max_q, P.seqlens, P.table, P.kn, P.vn,
                                                      True, D ** -0.5, num_splits=1)
        torch.cuda.synchronize()
        assert torch.equal(bits(o1), bits(out0)) and torch.equal(lse0, l1)
        assert torch.equal(bits(k1), bits(k0)) and torch.equal(bits(v1), bits(v0))


@pytest.mark.gpu
@pytest.mark.parametrize("variant", ["plain", "fp8", "q16"])
def test_auto_with_workspace_equals_the_count_it_reports(tfa, variant):
    """An all-decode step of 4 sequences x 8 heads fills 32 of the SMs: auto splits, into the count
    tfa_attn_varlen_kvcache_num_splits reports, bit-identical to asking for that count; the binding agrees."""
    D, kind, page, cap = 128, "bf16", 256, 8192
    P, kw = make_variant(variant, [1, 1, 1, 1], [8000, 1, 3000, 8191], 8, 2, D, kind, page, cap, seed=4)
    outa, lsea, na, ka, va = run(tfa, P, True, kw, num_splits=0)
    oute, lsee, ne, ke, ve = run(tfa, P, True, kw, num_splits=na)
    torch.cuda.synchronize()
    assert na > 1 and ne == na
    for a, b in ((outa, oute), (lsea, lsee), (ka, ke), (va, ve)):
        assert torch.equal(bits(a), bits(b))
    if variant == "plain":
        import attention_cutlass as ac
        k1, v1 = P.k.clone(), P.v.clone()
        o1, l1 = ac.flash_attention_v2_varlen_kvcache(P.q, k1, v1, P.cu_q, P.max_q, P.seqlens, P.table, P.kn, P.vn,
                                                      True, D ** -0.5, num_splits=0)
        torch.cuda.synchronize()
        assert torch.equal(bits(o1), bits(outa)) and torch.equal(l1, lsea)


@pytest.mark.gpu
@pytest.mark.parametrize("f32", [False, True])
def test_exact_writes_and_nan_workspace(tfa, f32):
    """Sentinel-filled out / lse keep their sentinels on rows past a sequence's first max_seqlen_q rows and on rows in
    no sequence (before cu[0], after cu[B]); a NaN-filled workspace and NaN in unused cache slots change nothing."""
    sq = [1, 250, 0, 37, 1]
    total, pre, post = sum(sq) + 9, 4, 5
    P = Problem(sq, [1000, 30, 5, 2000, 0], 8, 2, 128, "bf16", 256, 2304, seed=5, new=False)
    Pz = Problem(sq, [1000, 30, 5, 2000, 0], 8, 2, 128, "bf16", 256, 2304, seed=5, new=False, fill=0.0)
    for Q in (P, Pz):                       # rows in no sequence around the packed batch
        Q.q = torch.cat([torch.full((pre, 8, 128), float("nan"), dtype=torch.bfloat16, device="cuda"), Q.q,
                         torch.full((post, 8, 128), float("nan"), dtype=torch.bfloat16, device="cuda")])
        Q.cu_q = Q.cu_q + pre
        Q.max_q = 200                       # sequence 1 computes its first 200 rows only
    odt = torch.float32 if f32 else torch.bfloat16
    computed = torch.zeros(total, dtype=torch.bool, device="cuda")
    for (q0, q1) in offsets(sq):
        computed[pre + q0:pre + q0 + min(q1 - q0, 200)] = True
    results = {}
    for Q, ws_fill in ((P, float("nan")), (Pz, 0.0)):
        for ns in (3, 9):
            o = torch.full((total, 8, 128), -7.25, dtype=odt, device="cuda")
            l = torch.full((8, total), 123.5, dtype=torch.float32, device="cuda")
            ws = torch.full((ns * 8 * total * 129,), ws_fill, dtype=torch.float32, device="cuda")
            out, lse, got, _, _ = run(tfa, Q, True, {}, num_splits=ns, out=o, lse=l, out_fp32=f32, workspace=ws)
            torch.cuda.synchronize()
            assert got == ns
            assert (out[~computed] == -7.25).all() and (lse[:, ~computed] == 123.5).all()
            assert not (lse[:, computed] == 123.5).any() and torch.isfinite(out[computed]).all()
            results.setdefault(ns, []).append((out[computed].clone(), lse[:, computed].clone()))
    for (o1, l1), (o2, l2) in results.values():
        assert torch.equal(bits(o1), bits(o2)) and torch.equal(l1, l2)


@pytest.mark.gpu
def test_long_decodes_in_a_mixed_batch_within_float64_budget(tfa):
    """Two decodes at 65K-131K cached keys and a 300-token prefill chunk, split 16 ways: every sequence within the
    bound tests/test_fwd_float64_reference.py derives."""
    sq, lens = [1, 300, 1], [70001, 5000, 131000]
    cap = 131072 + 256
    Hq, Hkv, D = 8, 2, 128
    P = Problem(sq, lens, Hq, Hkv, D, "bf16", 256, cap, seed=17)
    out, lse, n, k, v = run(tfa, P, True, {}, num_splits=16)
    torch.cuda.synchronize()
    assert n == 16
    for b, (q0, q1) in enumerate(offsets(sq)):
        K = P.K(b)[1]
        kb, vb = P.gather(k, b, K), P.gather(v, b, K)
        ref = reference(P.q[q0:q1].permute(1, 0, 2)[None], kb.permute(1, 0, 2)[None], vb.permute(1, 0, 2)[None], True,
                        D ** -0.5)
        verdict = compare(out[q0:q1].permute(1, 0, 2)[None], lse[:, q0:q1][None], ref, "bf16")
        print(f"\n[float64 reference] sequence {b}: K {K}, max err/budget {verdict.ratio:.3f}, "
              f"max |dLSE| {verdict.lse_err:.2e}")
        assert verdict.ok, f"sequence {b}: {verdict.msg}"


@pytest.mark.gpu
def test_split_cuda_graph_replays_with_new_offsets_lengths_and_table(tfa):
    """Capture append + forward + combine with a caller-owned workspace, rewrite cu_seqlens_q (same total_q),
    cache_seqlens and the table in place and replay: out, lse and the pools equal eager calls on the same state."""
    sq1, sq2 = [200, 1, 1, 54], [1, 129, 100, 26]
    lens1, lens2 = [300, 5, 1000, 0], [900, 0, 256, 1100]
    P = Problem(sq1, lens1, 8, 2, 128, "bf16", 256, 1280, seed=13, fill=0.0)
    k0, v0 = P.k.clone(), P.v.clone()
    k, v = P.k.clone(), P.v.clone()
    out = torch.empty((sum(sq1), 8, 128), dtype=torch.bfloat16, device="cuda")
    lse = torch.empty((8, sum(sq1)), dtype=torch.float32, device="cuda")
    ws = torch.empty((4 * 8 * sum(sq1) * 129,), dtype=torch.float32, device="cuda")
    step = lambda: P.run(tfa, True, k=k, v=v, out=out, lse=lse, max_q=256, num_splits=4, workspace=ws)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
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
                                             P.kn, P.vn, is_causal=True, scale=128 ** -0.5, num_splits=4)
        torch.cuda.synchronize()
        assert torch.equal(out, eo) and torch.equal(lse, el)
        assert torch.equal(bits(k), bits(ke)) and torch.equal(bits(v), bits(ve))
        results.append(out.clone())
    assert not torch.equal(results[0], results[1])


@pytest.mark.gpu
def test_split_classic_and_persistent_agree_bitwise(tfa):
    code = r'''
import os, sys, torch
sys.path.insert(0, os.path.join(os.environ["TFA_ROOT"], "tiny-flash-attention_b200"))
sys.path.insert(0, os.path.join(os.environ["TFA_ROOT"], "tests"))
import tfa_ctypes as tfa
from test_varlen_kvcache import Problem, SQ, case_lens
res = []
for causal, new, page, ns in ((True, True, 256, 3), (False, False, None, 8), (True, False, 128, 64)):
    cap = 1100 if page is None else 1536
    P = Problem(SQ, case_lens(cap), 32, 8, 128, "bf16", page, cap, seed=9, new=new)
    o, lse, k, v = P.run(tfa, causal, num_splits=ns)
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
def test_split_launch_counts(tfa):
    for variant, new, ns, want in (("plain", False, 1, 1), ("plain", True, 1, 2), ("plain", False, 3, 2),
                                   ("plain", True, 3, 3), ("rotary", True, 3, 3), ("q16", False, 3, 3),
                                   ("qkv8", True, 3, 3)):
        P, kw = make_variant(variant, [500, 0, 1, 129], [10, 0, 64, 129], 4, 2, 64, "fp16", 128, 768, seed=1,
                             new=new)
        n0 = tfa.launch_count()
        run(tfa, P, True, kw, num_splits=ns, workspace=torch.empty(3 * 4 * 630 * 65, device="cuda"))
        assert tfa.launch_count() - n0 == want, (variant, new, ns)
    torch.cuda.synchronize()
