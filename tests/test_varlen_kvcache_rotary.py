"""Rotary position embedding in the variable-length KV-cache call: tfa_attn_varlen_kvcache_rotary_fwd /
attention_cutlass.flash_attention_v2_varlen_kvcache_rotary / flash_attention_v2_varlen_kvcache_fp8(rotary_cos=...) /
tfa_ctypes.attn_varlen_kvcache_fwd(rotary_cos=...).

CPU: the entry point is declared and exported, every argument error comes back before any device work and in the
documented order, the host-callable position rule matches its definition exhaustively (negative lengths, lengths past
the capacity and n_b > capacity included), and the existing variable-length cache bindings still take their old
positional calls.
GPU: out, lse and both pools equal rotating q / k_new in eager torch fp32 and making the unrotated call (16-bit and FP8
caches); each sequence equals the dense-query rotary call on that sequence alone; a short sequence near the capacity
next to a long one is rotated at its own positions; NaN in q_rot, unused cache slots and cos / sin rows past
seqlen_ro - 1 changes nothing; a float64 reference agrees; the call is 2 launches and replays from a CUDA graph with new
offsets, lengths and tables; the extension equals the ctypes call."""
import ctypes
import os

import pytest
import torch

from test_kvcache_rotary import rope, rope_tables
from test_varlen_kvcache import Problem, bits, declared_functions, lens_rule, offsets, scatter_append

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FP8 = torch.float8_e4m3fn

TFA_EINVAL_PTR = -1
TFA_EINVAL_DIM = -2
TFA_EARCH = -7
TFA_EINVAL_SCALE = -9
TFA_EINVAL_SEQLENS = -12
TFA_EINVAL_KVCACHE = -13
TFA_EINVAL_ROTARY = -14
TFA_EINVAL_KVQUANT = -15


# ------------------------------------------------------------------ CPU ------------------------------------------------

def test_header_declares_and_library_exports_varlen_kvcache_rotary(built):
    import tfa_ctypes
    assert "tfa_attn_varlen_kvcache_rotary_fwd" in declared_functions()
    header = open(os.path.join(ROOT, "include", "tfa_b200.h")).read()
    assert "#define TFA_ABI_VERSION 2" in header
    L = ctypes.CDLL(tfa_ctypes.LIB_PATH)
    assert hasattr(L, "tfa_attn_varlen_kvcache_rotary_fwd")
    assert L.tfa_abi_version() == 2


def test_varlen_rotary_argument_validation_order_without_device(built):
    """Host buffers only: every code comes back before anything touches a device, in the documented order -- cache,
    shapes, cu_seqlens_q / max_seqlen_q, rotary, FP8 (quantization args, then s'), device."""
    import tfa_ctypes
    L = tfa_ctypes.lib()
    buf = ctypes.create_string_buffer(8192 + 16)
    base = (ctypes.addressof(buf) + 15) & ~15
    ints = base + 1024
    tabs = base + 2048                                        # 16-byte aligned cos / sin / q_rot stand-ins
    Hq, Hkv, D, page, mbps = 4, 2, 64, 256, 4
    cap = page * mbps

    def va(**kw):
        return tfa_ctypes.VarlenKvcacheArgs(
            base, base, base, kw.get("k_new", base), kw.get("v_new", base), base, None, kw.get("cu_q", ints),
            kw.get("seqlens", ints), ints, 2, Hq, Hkv, kw.get("D", D), 300, kw.get("max_q", 200), 8, page, mbps,
            Hq * D, D, page * Hkv * D, kw.get("kss", Hkv * D), D, 4, Hkv * D, D, 0, kw.get("causal", 1),
            kw.get("scale", 0.1), 0, None)

    def ro(**kw):
        return tfa_ctypes.RotaryArgs(kw.get("cos", tabs), kw.get("sin", tabs + 512), kw.get("seqlen_ro", cap),
                                     kw.get("rd", D), kw.get("il", 0), kw.get("q_rot", tabs + 1024))

    def qa(**kw):
        return tfa_ctypes.KvQuantArgs(kw.get("dt", 2), kw.get("ks", 0.5), kw.get("vs", 0.5))

    def call(a=None, r=None, q=None):
        return L.tfa_attn_varlen_kvcache_rotary_fwd(ctypes.byref(a or va()), ctypes.byref(r or ro()),
                                                    ctypes.byref(q) if q is not None else None)

    bad_ro, bad_q = ro(rd=15), qa(dt=0)
    for q in (None, qa()):
        qp = ctypes.byref(q) if q is not None else None
        assert L.tfa_attn_varlen_kvcache_rotary_fwd(None, ctypes.byref(ro()), qp) == TFA_EINVAL_PTR
        assert L.tfa_attn_varlen_kvcache_rotary_fwd(ctypes.byref(va()), None, qp) == TFA_EINVAL_PTR
    # 1. the cache arguments, before everything else
    assert call(va(seqlens=None, D=96, max_q=0), bad_ro, bad_q) == TFA_EINVAL_KVCACHE
    assert call(va(k_new=base, v_new=None), bad_ro, bad_q) == TFA_EINVAL_KVCACHE
    # 2. the shapes, strides and scale
    assert call(va(D=96, max_q=0), bad_ro, bad_q) == TFA_EINVAL_DIM
    assert call(va(scale=-1.0, max_q=0), bad_ro, bad_q) == TFA_EINVAL_SCALE
    # 3. cu_seqlens_q / max_seqlen_q
    assert call(va(max_q=0), bad_ro, bad_q) == TFA_EINVAL_SEQLENS
    assert call(va(cu_q=ints + 2), bad_ro, bad_q) == TFA_EINVAL_SEQLENS
    # 4. the rotary arguments, with or without a (bad) FP8 block
    E = TFA_EINVAL_ROTARY
    for q in (None, qa(), bad_q):
        for rd in (15, 17, 24, 40, 0, -16, D + 16, 2 * D, 8):
            assert call(r=ro(rd=rd), q=q) == E, (rd, q)
        for name in ("cos", "sin", "q_rot"):
            assert call(r=ro(**{name: None}), q=q) == E, name
            for off in (2, 8):
                assert call(r=ro(**{name: tabs + 2048 + off}), q=q) == E, (name, off)
        assert call(r=ro(seqlen_ro=cap - 1), q=q) == E and call(r=ro(seqlen_ro=0), q=q) == E
        assert call(va(k_new=None, v_new=None), q=q) == E        # rotary rotates the appended keys: required
        assert call(va(k_new=None, v_new=None), ro(il=1), q) == E
    # 5. the FP8 arguments: the quantization block, then the effective scale s' = fp32(softmax_scale * k_scale)
    K = TFA_EINVAL_KVQUANT
    for q in (qa(dt=0), qa(dt=1), qa(ks=0.0), qa(vs=-1.0), qa(ks=float("nan")), qa(vs=float("inf"))):
        assert call(q=q) == K
        assert call(va(scale=1e38), q=q) == K
    assert call(va(kss=Hkv * D + 8), q=qa()) == K              # a 16-bit stride that is not a multiple of 16
    assert call(va(scale=1e38), q=qa(ks=100.0)) == TFA_EINVAL_SCALE             # s' overflows
    assert call(va(scale=1e-30), q=qa(ks=1e-20)) == TFA_EINVAL_SCALE            # s' underflows to uniform attention
    # the FP8 call without rotary keeps the same codes
    fp8_call = lambda a, q: L.tfa_attn_varlen_kvcache_fp8_fwd(ctypes.byref(a), ctypes.byref(q))
    assert fp8_call(va(), qa(dt=0)) == K and fp8_call(va(scale=1e38), qa(ks=100.0)) == TFA_EINVAL_SCALE
    assert fp8_call(va(scale=1e-30), qa(ks=1e-20)) == TFA_EINVAL_SCALE
    # 6. the device: reached only when every argument passed (asked on a machine without one only: with a GPU the call
    # would go on to launch on these host buffers)
    if not torch.cuda.is_available():
        assert call() == TFA_EARCH and call(q=qa()) == TFA_EARCH


def pos_rule(raw, cap, n, i, causal, is_query, seqlen_ro):
    """The header's rule: L_b from the varlen cache lengths of n appended keys, then L_b + i (keys; causal queries) or
    L_b (non-causal queries), clamped to seqlen_ro - 1."""
    Lb, _ = lens_rule(raw, cap, n, True)
    return min(Lb if (is_query and not causal) else Lb + i, seqlen_ro - 1)


def test_seq_rotary_pos_exhaustively(built):
    import tfa_ctypes
    L = tfa_ctypes.lib()
    L.tfa_internal_seq_rotary_pos.argtypes = [ctypes.c_int] * 7
    L.tfa_internal_seq_rotary_pos.restype = ctypes.c_int
    L.tfa_internal_rotary_pos.argtypes = [ctypes.c_int] * 5
    L.tfa_internal_rotary_pos.restype = ctypes.c_int
    L.tfa_internal_cache_len.argtypes = [ctypes.c_int] * 3
    L.tfa_internal_cache_len.restype = ctypes.c_int
    f = L.tfa_internal_seq_rotary_pos
    checked = 0
    for cap, ns in ((1, None), (2, None), (7, None), (33, None), (130, (0, 1, 2, 64, 129, 130, 131, 135, 261))):
        ns = range(0, cap + 4) if ns is None else ns
        raws = list(range(-3, cap + 5)) + [2 * cap + 7, -2**31, 2**31 - 1]
        for seqlen_ro in sorted({cap, cap + 1, cap + 33}):
            for n in ns:
                for raw in raws:
                    for i in range(0, n + 2):
                        for causal in (0, 1):
                            for is_q in (0, 1):
                                got = f(raw, cap, n, i, causal, is_q, seqlen_ro)
                                assert got == pos_rule(raw, cap, n, i, causal, is_q, seqlen_ro), \
                                    (cap, seqlen_ro, n, raw, i, causal, is_q)
                                checked += 1
                    # every position a call reads lies in the table; a kept key sits in its own, in-capacity slot
                    Lb, Kb = lens_rule(raw, cap, n, True)
                    for i in range(min(n, cap)):
                        assert f(raw, cap, n, i, 1, 0, seqlen_ro) == Lb + i < Kb <= cap
                    if 0 < n <= cap:               # the dense-query call's rule for Sq = Snew = n
                        Ld = L.tfa_internal_cache_len(raw, cap, n)
                        for i in range(n):
                            for causal in (0, 1):
                                for is_q in (0, 1):
                                    assert f(raw, cap, n, i, causal, is_q, seqlen_ro) == \
                                        L.tfa_internal_rotary_pos(Ld, i, causal, is_q, seqlen_ro)
    assert checked > 1_000_000


def test_existing_varlen_cache_bindings_accept_old_positional_calls(built):
    """CPU tensors stop at the first device check: a signature that no longer took the old positional call would raise
    TypeError instead.  The FP8 binding also takes the new keyword arguments, and the rotary binding exists."""
    import attention_cutlass as ac
    q = torch.zeros((4, 2, 64), dtype=torch.bfloat16)
    kc = torch.zeros((1, 128, 2, 64), dtype=torch.bfloat16)
    k8 = kc.to(FP8)
    cu = torch.tensor([0, 4], dtype=torch.int32)
    sl = torch.zeros(1, dtype=torch.int32)
    with pytest.raises(RuntimeError, match="CUDA"):
        ac.flash_attention_v2_varlen_kvcache(q, kc, kc, cu, 4, sl, None, None, None, True, 0.1)
    with pytest.raises(RuntimeError, match="CUDA"):
        ac.flash_attention_v2_varlen_kvcache_fp8(q, k8, k8, cu, 4, sl, None, None, None, 1.0, 1.0, True, 0.1)
    with pytest.raises(RuntimeError, match="CUDA"):
        ac.flash_attention_v2_varlen_kvcache_fp8(q, k8, k8, cu, 4, sl, None, q[:, :1], q[:, :1], 1.0, 1.0, True, 0.1,
                                                 rotary_cos=kc[0, :, 0], rotary_sin=kc[0, :, 0],
                                                 rotary_interleaved=True)
    with pytest.raises(RuntimeError, match="CUDA"):
        ac.flash_attention_v2_varlen_kvcache_rotary(q, kc, kc, cu, 4, sl, None, q[:, :1], q[:, :1], kc[0, :, 0],
                                                    kc[0, :, 0], False, True, 0.1)
    doc = ac.flash_attention_v2_varlen_kvcache_fp8.__doc__
    assert "rotary_cos: torch.Tensor | None = None" in doc and "rotary_interleaved: bool = False" in doc


# ------------------------------------------------------------------ GPU ------------------------------------------------

@pytest.fixture(scope="module")
def tfa(built):
    import tfa_ctypes
    tfa_ctypes.lib()
    return tfa_ctypes


def packed_positions(sq, lens, cap, max_q, causal, is_query, seqlen_ro, n_of=None):
    """(total_q,) table rows of the header's rule for every packed row; rows past a sequence's n_b get 0 (they are
    neither computed nor appended).  n_of(b) replaces n_b (the wrong rule, for the trap test)."""
    pos = [0] * sum(sq)
    for b, (q0, q1) in enumerate(offsets(sq)):
        n = min(q1 - q0, max_q)
        m = n if n_of is None else n_of(b)
        for i in range(n):
            pos[q0 + i] = pos_rule(lens[b], cap, m, i, causal, is_query, seqlen_ro)
    return torch.tensor(pos, dtype=torch.long, device="cuda")


def rope_packed(x, pos, cos, sin, rd, il, ftype=torch.float32):
    return rope(x[None], pos[None], cos, sin, rd, il, ftype)[0]


def fp8_pools(P):
    """P's pools as e4m3 codes (the data rounded, NaN slots as 0x7f in K and 0xff in V)."""
    k8 = P.k.float().clamp(-448, 448).to(FP8)
    v8 = P.v.float().clamp(-448, 448).to(FP8)
    v8.view(torch.uint8)[torch.isnan(P.v)] = 0xFF
    return k8, v8


class Rot:
    """A Problem with rotary tables of seqlen_ro = cap + extra rows (followed by `guard` NaN rows)."""

    def __init__(self, P, rd, il, extra=64, guard=0, fp8=False, scales=(0.5, 0.25)):
        self.P, self.rd, self.il = P, rd, il
        self.seqlen_ro = P.cap + extra
        self.cos, self.sin = rope_tables(self.seqlen_ro, rd, P.kind, guard=guard)
        self.fp8 = fp8
        self.k0, self.v0 = fp8_pools(P) if fp8 else (P.k, P.v)
        self.q_kw = dict(k_scale=scales[0], v_scale=scales[1]) if fp8 else {}

    def fused(self, tfa, causal, max_q=None, k=None, v=None, **kw):
        P = self.P
        k = self.k0.clone() if k is None else k
        v = self.v0.clone() if v is None else v
        out, lse, _, _ = P.run(tfa, causal, k=k, v=v, max_q=max_q, rotary_cos=self.cos, rotary_sin=self.sin,
                               rotary_interleaved=self.il, **self.q_kw, **kw)
        return out, lse, k, v

    def rotated(self, causal, max_q=None, n_of=None):
        P = self.P
        mq = P.max_q if max_q is None else max_q
        qp = packed_positions(P.sq, P.lens, P.cap, mq, causal, True, self.seqlen_ro, n_of)
        kp = packed_positions(P.sq, P.lens, P.cap, mq, causal, False, self.seqlen_ro, n_of)
        return (rope_packed(P.q, qp, self.cos, self.sin, self.rd, self.il),
                rope_packed(P.kn, kp, self.cos, self.sin, self.rd, self.il))

    def unfused(self, tfa, causal, max_q=None):
        """Rotate in eager torch fp32 at the header's positions, then the unrotated call on fresh pools."""
        P = self.P
        qr, kr = self.rotated(causal, max_q)
        k, v = self.k0.clone(), self.v0.clone()
        mq = P.max_q if max_q is None else max_q
        out, lse = tfa.attn_varlen_kvcache_fwd(qr, k, v, P.cu_q, mq, P.seqlens, P.table, kr, P.vn, is_causal=causal,
                                               scale=P.D ** -0.5, **self.q_kw)
        return out, lse, k, v, qr

    def per_sequence(self, tfa, causal, max_q=None):
        """The dense-query rotary call on one sequence at a time (B = 1, Sq = Snew = n_b, one split), on one copy of
        the pools: {b: (out, lse)} and the pools after every append."""
        P = self.P
        mq = P.max_q if max_q is None else max_q
        k, v = self.k0.clone(), self.v0.clone()
        res = {}
        for b, (q0, q1) in enumerate(offsets(P.sq)):
            n = min(q1 - q0, mq)
            if n == 0:
                continue
            if P.table is None:
                kc, vc, tab = k[b:b + 1], v[b:b + 1], None
            else:
                kc, vc, tab = k, v, P.table[b:b + 1]
            o, l = tfa.attn_kvcache_fwd(P.q[q0:q0 + n][None], kc, vc, P.seqlens[b:b + 1], tab,
                                        P.kn[q0:q0 + n][None], P.vn[q0:q0 + n][None], is_causal=causal,
                                        scale=P.D ** -0.5, num_splits=1, rotary_cos=self.cos, rotary_sin=self.sin,
                                        rotary_interleaved=self.il, **self.q_kw)
            res[b] = (o[0], l[0])
        return res, k, v


# (D, kind, rotary_dim, interleaved, causal, page, Hq, Hkv); page None: the contiguous cache
CASES = [
    (128, "bf16", 128, False, True, 256, 32, 8),
    (128, "fp16", 64, True, False, 128, 8, 2),
    (64, "fp16", 64, False, True, None, 8, 8),
    (64, "bf16", 32, True, True, 128, 32, 8),
    (128, "bf16", 16, True, False, None, 8, 2),
    (64, "bf16", 64, True, False, 256, 4, 1),
]
SQ = [129, 0, 1, 300, 127, 128, 1, 257, 5]


def case_lens(cap):
    """0, near the capacity (exactly full after the append, and past it), short, negative."""
    return [0, 40, cap - 1, 3, cap - 127, 700, cap + 50, 100, -4]


def _problem(D, kind, page, Hq, Hkv, seed, sq=SQ, lens=None, fill=float("nan")):
    cap = 1100 if page is None else 1536
    return Problem(sq, case_lens(cap) if lens is None else lens, Hq, Hkv, D, kind, page, cap, seed=seed, fill=fill)


@pytest.mark.gpu
@pytest.mark.parametrize("fp8", [False, True])
@pytest.mark.parametrize("D,kind,rd,il,causal,page,Hq,Hkv", CASES)
def test_varlen_rotary_equals_unfused_torch_rotation_bitwise(tfa, D, kind, rd, il, causal, page, Hq, Hkv, fp8):
    """out, lse, q_rot's rows and both whole pools (byte for byte on an FP8 cache) equal rotating q / k_new in eager
    torch fp32 and calling the unrotated variable-length cache call on the same starting pools."""
    P = _problem(D, kind, page, Hq, Hkv, seed=D + Hq + int(causal) + 7 * int(fp8))
    R = Rot(P, rd, il, fp8=fp8)
    q_in, kn_in = P.q.clone(), P.kn.clone()
    q_rot = torch.full_like(P.q, float("nan"))
    o1, l1, k1, v1 = R.fused(tfa, causal, q_rot=q_rot)
    o2, l2, k2, v2, qr = R.unfused(tfa, causal)
    torch.cuda.synchronize()
    for b, (q0, q1) in enumerate(offsets(P.sq)):
        assert torch.equal(bits(q_rot[q0:q1]), bits(qr[q0:q1])), b
    assert torch.equal(o1, o2) and torch.equal(l1, l2)
    assert torch.equal(k1.view(torch.uint8), k2.view(torch.uint8))
    assert torch.equal(v1.view(torch.uint8), v2.view(torch.uint8))
    assert torch.equal(bits(P.q), bits(q_in)) and torch.equal(bits(P.kn), bits(kn_in))
    assert torch.isfinite(o1).all()


@pytest.mark.gpu
@pytest.mark.parametrize("fp8", [False, True])
@pytest.mark.parametrize("D,kind,rd,il,causal,page,Hq,Hkv", CASES[:4])
def test_varlen_rotary_equals_dense_rotary_call_per_sequence(tfa, D, kind, rd, il, causal, page, Hq, Hkv, fp8):
    """Each sequence's out and lse, and the pools after all appends, equal the dense-query rotary call
    (tfa_attn_kvcache_rotary_fwd, FP8: tfa_attn_kvcache_fp8_fwd with rotary) on that sequence alone with
    Sq = Snew = n_b and one split.  max_seqlen_q below the longest sequence cuts it to its first rows."""
    P = _problem(D, kind, page, Hq, Hkv, seed=3 + D + int(fp8))
    R = Rot(P, rd, il, fp8=fp8)
    for max_q in (None, 200):
        o1, l1, k1, v1 = R.fused(tfa, causal, max_q=max_q)
        ref, k2, v2 = R.per_sequence(tfa, causal, max_q=max_q)
        torch.cuda.synchronize()
        assert torch.equal(k1.view(torch.uint8), k2.view(torch.uint8))
        assert torch.equal(v1.view(torch.uint8), v2.view(torch.uint8))
        for b, (o, l) in ref.items():
            q0 = offsets(P.sq)[b][0]
            n = o.shape[0]
            assert torch.equal(o1[q0:q0 + n], o), (max_q, b)
            assert torch.equal(l1[:, q0:q0 + n], l), (max_q, b)


@pytest.mark.gpu
@pytest.mark.parametrize("fp8", [False, True])
@pytest.mark.parametrize("il", [False, True])
def test_short_sequence_near_the_capacity_is_rotated_at_its_own_positions(tfa, il, fp8):
    """Sequence 1 (3 rows) sits 5 keys below the capacity next to a sequence of max_seqlen_q = 200 rows: its L_b is
    capacity - 5, while a rule taking L_b from max_seqlen_q would give capacity - 200.  The call equals the header's
    rule and differs from the other one."""
    cap, page = 512, 128
    sq, lens = [200, 3, 1], [10, cap - 5, 100]
    P = Problem(sq, lens, 8, 2, 128, "bf16", page, cap, seed=21)
    R = Rot(P, 128, il, fp8=fp8)
    q_rot = torch.empty_like(P.q)
    o1, l1, k1, v1 = R.fused(tfa, True, q_rot=q_rot)
    o2, l2, k2, v2, qr = R.unfused(tfa, True)
    wrong_q, wrong_k = R.rotated(True, n_of=lambda b: max(sq))
    torch.cuda.synchronize()
    assert lens_rule(lens[1], cap, 3, True)[0] == cap - 5 and lens_rule(lens[1], cap, 200, True)[0] == cap - 200
    assert torch.equal(bits(q_rot), bits(qr)) and torch.equal(o1, o2) and torch.equal(l1, l2)
    assert torch.equal(k1.view(torch.uint8), k2.view(torch.uint8))
    assert torch.equal(v1.view(torch.uint8), v2.view(torch.uint8))
    assert not torch.equal(bits(q_rot[200:203]), bits(wrong_q[200:203]))
    _, wk = R.rotated(True)
    assert not torch.equal(bits(wk[200:203]), bits(wrong_k[200:203]))


@pytest.mark.gpu
@pytest.mark.parametrize("fp8", [False, True])
def test_sequence_longer_than_the_capacity_drops_keys(tfa, fp8):
    """Malformed: n_b = 300 rows against a 256-key contiguous cache, with seqlen_ro = capacity.  The first 256 keys
    are kept at positions 0..255, the rest dropped; causal query positions past the table clamp to its last row."""
    cap = 256
    sq, lens = [300, 5, 40], [7, 100, 0]
    P = Problem(sq, lens, 8, 2, 64, "fp16", None, cap, seed=23, fill=float("nan"))
    R = Rot(P, 64, False, extra=0, guard=16, fp8=fp8)
    q_rot = torch.empty_like(P.q)
    o1, l1, k1, v1 = R.fused(tfa, True, q_rot=q_rot)
    o2, l2, k2, v2, qr = R.unfused(tfa, True)
    torch.cuda.synchronize()
    assert int(packed_positions(sq, lens, cap, 300, True, True, cap).max()) == cap - 1
    assert torch.equal(bits(q_rot), bits(qr)) and torch.equal(o1, o2) and torch.equal(l1, l2)
    assert torch.equal(k1.view(torch.uint8), k2.view(torch.uint8))
    assert torch.isfinite(o1).all()
    if not fp8:
        _, kr = R.rotated(True)
        want = scatter_append(P, P.k, kr, None, lambda b: sq[b])
        assert torch.equal(bits(k1), bits(want))


@pytest.mark.gpu
@pytest.mark.parametrize("fp8", [False, True])
@pytest.mark.parametrize("D,kind,page", [(128, "bf16", 256), (64, "fp16", None)])
def test_nan_in_q_rot_unused_slots_and_table_tail_changes_nothing(tfa, D, kind, page, fp8):
    """q_rot pre-filled with NaN inside NaN guards, NaN in every unused cache slot (FP8 codes 0x7f in K, 0xff in V) and
    NaN cos / sin rows after seqlen_ro = capacity rows: results equal a run with zeros there.  Rows past
    max_seqlen_q keep the out / lse they held, no store leaves out, lse or q_rot, and q_rot keeps NaN in the rows of
    no sequence's first n_b."""
    sq, max_q, G = [300, 1, 0, 129, 2], 150, 64
    args = dict(sq=sq, lens=[300, 0, 10, 129, 768 - 2], Hq=8, Hkv=2, D=D, kind=kind, page=page, cap=768, seed=5)
    pz = Problem(fill=0.0, **args)
    pn = Problem(fill=float("nan"), **args)
    rz = Rot(pz, D, True, extra=0, fp8=fp8)
    rn = Rot(pn, D, True, extra=0, guard=16, fp8=fp8)
    if fp8:
        assert (rn.k0.view(torch.uint8) == 0x7F).any() and (rn.v0.view(torch.uint8) == 0xFF).any()
    tq, Hq = sum(sq), 8
    n = tq * Hq * D
    for causal in (False, True):
        obuf = torch.full((G + n + G,), float("nan"), dtype=pn.q.dtype, device="cuda")
        qbuf = torch.full((G + n + G,), float("nan"), dtype=pn.q.dtype, device="cuda")
        lbuf = torch.full((G + Hq * tq + G,), float("nan"), dtype=torch.float32, device="cuda")
        out, q_rot = obuf[G:G + n].view(tq, Hq, D), qbuf[G:G + n].view(tq, Hq, D)
        lse = lbuf[G:G + Hq * tq].view(Hq, tq)
        rn.fused(tfa, causal, max_q=max_q, out=out, lse=lse, q_rot=q_rot)
        oz, lz, kz, _ = rz.fused(tfa, causal, max_q=max_q)
        torch.cuda.synchronize()
        for buf, m in ((obuf, n), (qbuf, n), (lbuf, Hq * tq)):
            assert torch.isnan(buf[:G]).all() and torch.isnan(buf[G + m:]).all()
        for b, (q0, q1) in enumerate(offsets(sq)):
            k = min(q1 - q0, max_q)
            assert torch.equal(out[q0:q0 + k], oz[q0:q0 + k]) and torch.equal(lse[:, q0:q0 + k], lz[:, q0:q0 + k])
            assert torch.isfinite(out[q0:q0 + k]).all() and torch.isfinite(q_rot[q0:q0 + k]).all()
            assert torch.isnan(out[q0 + k:q1]).all() and torch.isnan(lse[:, q0 + k:q1]).all()
            assert torch.isnan(q_rot[q0 + k:q1]).all()


@pytest.mark.gpu
@pytest.mark.parametrize("name,sq,lens,cap,page,causal,D,kind,rd,il,fp8", [
    ("mixed", [300, 1, 0, 129, 64], [0, 900, 50, 1000, 10], 1024, 256, True, 128, "bf16", 128, False, False),
    ("prefill", [250, 1, 60], [1000, 3, 0], 1280, 128, False, 64, "fp16", 32, True, False),
    ("fp8", [200, 3, 130], [5, 0, 64], 512, None, True, 128, "bf16", 64, False, True),
])
def test_varlen_rotary_within_float64_reference_budget(tfa, name, sq, lens, cap, page, causal, D, kind, rd, il, fp8):
    """out (16-bit and fp32) and lse against the float64 reference of test_fwd_float64_reference on each sequence's
    rotated queries and the keys the pools hold after the call."""
    from test_fwd_float64_reference import compare, reference
    P = Problem(sq, lens, 8, 2, D, kind, page, cap, seed=31)
    R = Rot(P, rd, il, fp8=fp8)
    q_rot = torch.empty_like(P.q)
    o32, l32, k, v = R.fused(tfa, causal, q_rot=q_rot, out_fp32=True)
    o16, l16, _, _ = R.fused(tfa, causal)
    qr, _ = R.rotated(causal)
    torch.cuda.synchronize()
    assert torch.equal(l32, l16)
    ks, vs = (0.5, 0.25) if fp8 else (1.0, 1.0)
    for b, (q0, q1) in enumerate(offsets(sq)):
        if q1 == q0:
            continue
        assert torch.equal(bits(q_rot[q0:q1]), bits(qr[q0:q1]))
        _, K = P.K(b)
        kk = P.gather(k, b, K).permute(1, 0, 2)[None]
        vv = P.gather(v, b, K).permute(1, 0, 2)[None]
        ref = reference(q_rot[q0:q1].permute(1, 0, 2)[None], kk, vv, causal, D ** -0.5, k_scale=ks, v_scale=vs)
        for o in (o32, o16):
            verdict = compare(o[q0:q1].permute(1, 0, 2)[None], l32[:, q0:q1][None], ref, kind)
            assert verdict.ok, (name, b, o.dtype, verdict.msg)


@pytest.mark.gpu
@pytest.mark.parametrize("fp8", [False, True])
def test_varlen_rotary_cuda_graph_replays_with_new_offsets_lengths_and_table(tfa, fp8):
    """Capture one rotary step (rotary append + attention), rewrite cu_seqlens_q (same total_q), cache_seqlens and the
    block table in place and replay: out, lse, q_rot and the pools equal eager calls on the same state."""
    sq1, sq2 = [200, 1, 1, 54], [1, 129, 100, 26]
    lens1, lens2 = [300, 5, 1000, 0], [900, 0, 256, 1100]
    P = Problem(sq1, lens1, 8, 2, 128, "bf16", 256, 1280, seed=13, fill=0.0)
    R = Rot(P, 128, False, fp8=fp8)
    k, v = R.k0.clone(), R.v0.clone()
    tq = sum(sq1)
    out = torch.empty((tq, 8, 128), dtype=torch.bfloat16, device="cuda")
    lse = torch.empty((8, tq), dtype=torch.float32, device="cuda")
    q_rot = torch.empty_like(P.q)
    step = lambda: R.fused(tfa, True, max_q=256, k=k, v=v, out=out, lse=lse, q_rot=q_rot)
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
            P.cu_q.copy_(torch.tensor([0] + torch.tensor(sq).cumsum(0).tolist(), dtype=torch.int32))
            P.seqlens.copy_(torch.tensor(lens, dtype=torch.int32))
            P.table.copy_(torch.randperm(P.nblk, generator=gp)[:P.table.numel()].to(torch.int32).view(P.table.shape))
            P.sq, P.lens = sq, lens
        k.copy_(R.k0)
        v.copy_(R.v0)
        graph.replay()
        eq = torch.empty_like(P.q)
        eo, el, ek, ev = R.fused(tfa, True, max_q=256, q_rot=eq)
        uo, ul, uk, _, qr = R.unfused(tfa, True, max_q=256)
        torch.cuda.synchronize()
        assert torch.equal(out, eo) and torch.equal(lse, el) and torch.equal(bits(q_rot), bits(eq))
        assert torch.equal(k.view(torch.uint8), ek.view(torch.uint8))
        assert torch.equal(v.view(torch.uint8), ev.view(torch.uint8))
        assert torch.equal(out, uo) and torch.equal(bits(q_rot), bits(qr))
        results.append(q_rot.clone())
    assert not torch.equal(results[0], results[1])


@pytest.mark.gpu
def test_varlen_rotary_launch_count(tfa):
    P = Problem([500, 0, 1, 129], [10, 0, 64, 129], 4, 2, 64, "fp16", 128, 768, seed=1)
    for fp8 in (False, True):
        R = Rot(P, 32, False, fp8=fp8)
        n0 = tfa.launch_count()
        R.fused(tfa, True)
        assert tfa.launch_count() - n0 == 2, fp8
    torch.cuda.synchronize()


@pytest.mark.gpu
def test_extension_varlen_rotary_entries_equal_ctypes(built, tfa):
    import attention_cutlass as ac
    P = Problem([300, 1, 0, 129], [300, 1, 0, 640], 8, 2, 128, "bf16", 256, 1024, seed=17, fill=0.0)
    scale = 128 ** -0.5
    for il in (False, True):
        R = Rot(P, 64, il)
        k1, v1 = P.k.clone(), P.v.clone()
        out, lse = ac.flash_attention_v2_varlen_kvcache_rotary(P.q, k1, v1, P.cu_q, P.max_q, P.seqlens, P.table, P.kn,
                                                               P.vn, R.cos, R.sin, il, True, scale)
        want, wl, wk, wv = R.fused(tfa, True)
        torch.cuda.synchronize()
        assert out.shape == P.q.shape and lse.shape == (8, P.q.shape[0])
        assert torch.equal(out, want) and torch.equal(lse, wl)
        assert torch.equal(bits(k1), bits(wk)) and torch.equal(bits(v1), bits(wv))
        R8 = Rot(P, 64, il, fp8=True)
        k8, v8 = R8.k0.clone(), R8.v0.clone()
        o8, l8 = ac.flash_attention_v2_varlen_kvcache_fp8(P.q, k8, v8, P.cu_q, P.max_q, P.seqlens, P.table, P.kn, P.vn,
                                                          0.5, 0.25, True, scale, rotary_cos=R8.cos,
                                                          rotary_sin=R8.sin, rotary_interleaved=il)
        w8, wl8, wk8, wv8 = R8.fused(tfa, True)
        torch.cuda.synchronize()
        assert torch.equal(o8, w8) and torch.equal(l8, wl8)
        assert torch.equal(k8.view(torch.uint8), wk8.view(torch.uint8))
        assert torch.equal(v8.view(torch.uint8), wv8.view(torch.uint8))
    R = Rot(P, 64, False)
    call = lambda **kw: ac.flash_attention_v2_varlen_kvcache_rotary(
        P.q, P.k.clone(), P.v.clone(), P.cu_q, P.max_q, P.seqlens, P.table, kw.get("kn", P.kn), kw.get("vn", P.vn),
        kw.get("cos", R.cos), kw.get("sin", R.sin), False, True, scale)
    with pytest.raises(RuntimeError, match="k_new"):
        call(kn=None, vn=None)
    with pytest.raises(RuntimeError, match="dtype"):
        call(cos=R.cos.float(), sin=R.sin.float())
    with pytest.raises(RuntimeError, match="seqlen_ro"):
        call(cos=R.cos[:P.cap - 1], sin=R.sin[:P.cap - 1])
    with pytest.raises(RuntimeError, match="rotary_dim"):
        call(cos=R.cos[:, :4].contiguous(), sin=R.sin[:, :4].contiguous())
    with pytest.raises(RuntimeError, match="together"):
        ac.flash_attention_v2_varlen_kvcache_fp8(P.q, P.k.to(FP8), P.v.to(FP8), P.cu_q, P.max_q, P.seqlens, P.table,
                                                 P.kn, P.vn, 0.5, 0.25, True, scale, rotary_cos=R.cos)
