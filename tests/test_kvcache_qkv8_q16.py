"""The e4m3-query cache calls fed from a 16-bit q: tfa_attn_kvcache_qkv8_q16_fwd / tfa_attn_varlen_kvcache_qkv8_q16_fwd,
attention_cutlass.flash_attention_v2_kvcache_qkv8_q16 / flash_attention_v2_varlen_kvcache_qkv8_q16 and the q8_scale
routing of tfa_ctypes.attn_kvcache_fwd / attn_varlen_kvcache_fwd.

The oracle is the composition of merged calls: the widening FP8-cache call (with rotary when the case has it) on a copy
of the pools gives rot(q) and the reference pools; torch quantizes rot(q) (or q) with q_scale; the e4m3-query call runs
on those pools without an append, at the lengths the append leaves.  The new call must match all three bit for bit.

CPU: the header declares both calls, the library exports them, and every argument error comes back before any device
work in the documented order, ending in TFA_EARCH without a GPU.
GPU: bit-identity with the oracle (out, lse, pools, q8) over head dims, output dtypes, GQA, page sizes, query and
append lengths, rotary layouts and cache lengths; saturating and subnormal quotients; the varlen call on mixed batches;
split-KV; both schedules; CUDA-graph replay; launch counts; guard regions; the bindings and the routing errors."""
import ctypes
import os
import subprocess
import sys

import pytest
import torch

from test_kvcache_qkv8 import bits, cache_lens_dense, cache_lens_varlen, make_pools

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "tfa_b200.h")

FP8 = torch.float8_e4m3fn
TFA_FP8_E4M3 = 2
CALLS = ("tfa_attn_kvcache_qkv8_q16_fwd", "tfa_attn_varlen_kvcache_qkv8_q16_fwd")
E_PTR, E_DIM, E_DTYPE, E_STRIDE, E_ARCH, E_SCALE, E_HEADS = -1, -2, -4, -5, -7, -9, -10
E_SEQLENS, E_KVCACHE, E_ROTARY, E_QKVQUANT = -12, -13, -14, -16


# ------------------------------------------------------------------ CPU ------------------------------------------------

def test_header_declares_and_library_exports_q16_calls(built):
    import tfa_ctypes
    from test_kvcache_fp8 import declared_functions
    src = " ".join(open(HEADER).read().split())
    assert ("int tfa_attn_kvcache_qkv8_q16_fwd(const tfa_attn_kvcache_args* args, const tfa_rotary_args* rotary "
            "/* NULL: none */, const tfa_qkv_quant_args* quant, void* q8);") in src
    assert ("int tfa_attn_varlen_kvcache_qkv8_q16_fwd(const tfa_attn_varlen_kvcache_args* args, const tfa_rotary_args* "
            "rotary /* NULL: none */, const tfa_qkv_quant_args* quant, void* q8);") in src
    assert "#define TFA_ABI_VERSION 2" in src
    names = declared_functions()
    L = ctypes.CDLL(tfa_ctypes.LIB_PATH)
    for fn in CALLS:
        assert fn in names and hasattr(L, fn)


def _buffers():
    buf = ctypes.create_string_buffer(8192 + 16)
    base = (ctypes.addressof(buf) + 15) & ~15
    return buf, base, base + 1024, base + 4096


def _quant(kw, qs=0.02):
    import tfa_ctypes
    return tfa_ctypes.QkvQuantArgs(kw.get("qdt", TFA_FP8_E4M3), kw.get("qs", qs), kw.get("ks", 0.5), kw.get("vs", 2.0))


def _rotary(kw, base):
    import tfa_ctypes
    if not kw.get("rot", False):
        return None
    return tfa_ctypes.RotaryArgs(kw.get("cos", base), base, kw.get("seqlen_ro", 1024), kw.get("rd", 32), 0,
                                 kw.get("q_rot", None))


def test_kvcache_q16_argument_checks_and_their_order(built):
    """Host buffers only.  q8 first (with args and quant), then the cache, the 16-bit problem, rotary without q_rot,
    the quantization against q8's layout (a 16-bit q whose strides are multiples of 8 but not 16 is fine), s', the
    device."""
    import tfa_ctypes
    L = tfa_ctypes.lib()
    buf, base, ints, q8 = _buffers()
    Hq, Hkv, D, page = 4, 2, 64, 256

    def mk(**kw):
        kn = base if kw.get("append", kw.get("rot", False)) else None
        return tfa_ctypes.KvcacheArgs(
            kw.get("q", base), base, base, kn, kn, kw.get("out", base), None, kw.get("seqlens", ints),
            kw.get("table", ints), kw.get("B", 2), Hq, kw.get("Hkv", Hkv), 1, kw.get("D", D), 8, page, 4, 1,
            kw.get("qsb", Hq * D), kw.get("qss", Hq * D), kw.get("qsh", D), kw.get("ksb", page * Hkv * D),
            kw.get("kss", Hkv * D), kw.get("ksh", D), 4, Hkv * D, Hkv * D, D, kw.get("dtype", 0), 1,
            kw.get("scale", 0.1), kw.get("f32", 0), 1, None, 0, None)

    def call(**kw):
        r = _rotary(kw, base)
        return L.tfa_attn_kvcache_qkv8_q16_fwd(ctypes.byref(mk(**kw)), ctypes.byref(r) if r else None,
                                               ctypes.byref(_quant(kw)), kw.get("q8", q8))

    quant = _quant({})
    assert L.tfa_attn_kvcache_qkv8_q16_fwd(None, None, ctypes.byref(quant), q8) == E_PTR
    assert L.tfa_attn_kvcache_qkv8_q16_fwd(ctypes.byref(mk()), None, None, q8) == E_PTR
    assert call(q8=None) == E_PTR and call(q8=q8 + 8) == E_PTR and call(q8=q8 + 1) == E_PTR
    assert call(q8=None, seqlens=None) == E_PTR and call(q8=q8 + 8, D=96, qdt=0) == E_PTR
    # the cache arguments
    assert call(seqlens=None) == E_KVCACHE and call(seqlens=None, D=96) == E_KVCACHE
    assert call(seqlens=None, rot=True, cos=None) == E_KVCACHE
    # the 16-bit problem: q's strides in multiples of 8, dtype bf16 / fp16
    assert call(q=None) == E_PTR and call(out=base + 8) == E_PTR
    assert call(D=96) == E_DIM and call(dtype=2) == E_DTYPE and call(qss=60) == E_STRIDE and call(qsh=68) == E_STRIDE
    assert call(scale=-1.0) == E_SCALE and call(Hkv=3) == E_HEADS
    assert call(D=96, rot=True, cos=None) == E_DIM and call(qss=60, qdt=0) == E_STRIDE
    # rotary, q_rot not checked; rotary needs k_new
    assert call(rot=True, cos=None) == E_ROTARY and call(rot=True, cos=base + 8) == E_ROTARY
    assert call(rot=True, rd=24) == E_ROTARY and call(rot=True, rd=80) == E_ROTARY
    assert call(rot=True, seqlen_ro=1023) == E_ROTARY
    assert call(rot=True, append=False) == E_ROTARY and call(rot=True, cos=None, qdt=0) == E_ROTARY
    # the quantization: q8's layout is contiguous, so the caller's q strides do not matter; the caches' do
    assert call(qdt=0) == E_QKVQUANT and call(qdt=1) == E_QKVQUANT and call(qs=0.0) == E_QKVQUANT
    for bad in (-1.0, float("nan"), float("inf")):
        assert call(qs=bad) == E_QKVQUANT and call(ks=bad) == E_QKVQUANT and call(vs=bad) == E_QKVQUANT
    assert call(kss=Hkv * D + 8) == E_QKVQUANT and call(ksh=D + 8) == E_QKVQUANT
    assert call(ksb=page * Hkv * D + 8) == E_QKVQUANT
    assert call(rot=True, qs=0.0) == E_QKVQUANT
    # s' = fp32(fp32(scale * q_scale) * k_scale)
    assert call(scale=1.0e38, qs=1.0, ks=10.0) == E_SCALE and call(scale=1e-30, qs=1e-10, ks=1e-10) == E_SCALE
    if not torch.cuda.is_available():
        assert call() == E_ARCH and call(f32=1) == E_ARCH
        assert call(qss=Hq * D + 8, qsb=Hq * D + 8, qsh=D + 8) == E_ARCH   # multiples of 8, not of 16: accepted
        assert call(rot=True) == E_ARCH and call(rot=True, q_rot=base + 8) == E_ARCH   # q_rot is not read
        assert call(append=True) == E_ARCH and call(append=False) == E_ARCH          # quantize-only: no k_new needed


def test_varlen_kvcache_q16_argument_checks_and_their_order(built):
    import tfa_ctypes
    L = tfa_ctypes.lib()
    buf, base, ints, q8 = _buffers()
    Hq, Hkv, D, page = 4, 2, 64, 128

    def mk(**kw):
        kn = base if kw.get("append", kw.get("rot", False)) else None
        return tfa_ctypes.VarlenKvcacheArgs(
            base, base, base, kn, kn, base, None, kw.get("cu", ints), kw.get("seqlens", ints), ints, 2, Hq, Hkv,
            kw.get("D", D), 8, kw.get("maxq", 4), 8, page, 4, kw.get("qss", Hq * D), kw.get("qsh", D),
            page * Hkv * D, kw.get("kss", Hkv * D), D, 4, Hkv * D, D, kw.get("dtype", 1), 1, kw.get("scale", 0.1), 0,
            None)

    def call(**kw):
        kw.setdefault("seqlen_ro", 512)
        r = _rotary(kw, base)
        return L.tfa_attn_varlen_kvcache_qkv8_q16_fwd(ctypes.byref(mk(**kw)), ctypes.byref(r) if r else None,
                                                      ctypes.byref(_quant(kw, 0.5)), kw.get("q8", q8))

    assert L.tfa_attn_varlen_kvcache_qkv8_q16_fwd(None, None, None, q8) == E_PTR
    assert L.tfa_attn_varlen_kvcache_qkv8_q16_fwd(ctypes.byref(mk()), None, None, q8) == E_PTR
    assert call(q8=None) == E_PTR and call(q8=q8 + 4) == E_PTR and call(q8=None, cu=None) == E_PTR
    assert call(seqlens=None) == E_KVCACHE and call(seqlens=None, cu=None) == E_KVCACHE
    assert call(D=96) == E_DIM and call(dtype=2) == E_DTYPE and call(D=96, cu=None) == E_DIM
    assert call(qss=Hq * D + 4) == E_STRIDE
    assert call(cu=None) == E_SEQLENS and call(maxq=9) == E_SEQLENS and call(cu=None, rot=True, cos=None) == E_SEQLENS
    assert call(rot=True, cos=None) == E_ROTARY and call(rot=True, append=False) == E_ROTARY
    assert call(rot=True, seqlen_ro=511) == E_ROTARY and call(rot=True, rd=16, cos=None, qdt=1) == E_ROTARY
    assert call(qdt=1) == E_QKVQUANT and call(qs=0.0) == E_QKVQUANT and call(ks=float("nan")) == E_QKVQUANT
    assert call(kss=Hkv * D + 8) == E_QKVQUANT
    assert call(scale=1.0e38, qs=1.0, ks=10.0) == E_SCALE
    if not torch.cuda.is_available():
        assert call() == E_ARCH and call(qss=Hq * D + 8) == E_ARCH and call(qsh=D + 8) == E_ARCH
        assert call(rot=True) == E_ARCH and call(append=True) == E_ARCH


# ------------------------------------------------------------------ GPU ------------------------------------------------

@pytest.fixture(scope="module")
def tfa(built):
    import tfa_ctypes
    tfa_ctypes.lib()
    return tfa_ctypes


QS, KS, VS = 0.0213, 0.0171, 0.0119


def _dt(kind):
    return {"bf16": torch.bfloat16, "fp16": torch.float16, "f32": torch.bfloat16}[kind]


def quantize(x, scale):
    return (x.float() / scale).clamp(-448, 448).to(FP8)


def rope_tables(seqlen_ro, rotary_dim, dt):
    """cos / sin (seqlen_ro, rotary_dim / 2) in dt, base 10000."""
    inv = 10000.0 ** (-torch.arange(0, rotary_dim, 2, dtype=torch.float64) / rotary_dim)
    ang = torch.arange(seqlen_ro, dtype=torch.float64)[:, None] * inv[None]
    return ang.cos().to(dt).cuda(), ang.sin().to(dt).cuda()


def _rot_kw(rotary, rotary_dim, cap, dt):
    if rotary == "none":
        return {}
    cos, sin = rope_tables(cap + 7, rotary_dim, dt)
    return dict(rotary_cos=cos, rotary_sin=sin, rotary_interleaved=rotary == "gptj")


def dense_oracle(tfa, q, kp, vp, sl, table, cap, kn, vn, rkw, causal, scale, kind, num_splits=1):
    """(out, lse, k pool, v pool, q8) of the composition of merged calls."""
    k1, v1 = kp.clone(), vp.clone()
    if rkw:
        qr = torch.empty(q.shape, dtype=q.dtype, device="cuda")
        tfa.attn_kvcache_fwd(q, k1, v1, sl, table, kn, vn, is_causal=causal, scale=scale, k_scale=KS, v_scale=VS,
                             q_rot=qr, **rkw)
    else:
        qr = q
        if kn is not None:
            tfa.attn_kvcache_fwd(q, k1, v1, sl, table, kn, vn, is_causal=causal, scale=scale, k_scale=KS, v_scale=VS)
    q8 = quantize(qr, QS)
    snew = kn.shape[1] if kn is not None else 0
    lens = [cache_lens_dense(x, cap, snew) if snew else min(max(x, 0), cap) for x in sl.tolist()]
    sl2 = torch.tensor(lens, dtype=torch.int32, device="cuda")
    o, l = tfa.attn_kvcache_fwd(q8, k1, v1, sl2, table, is_causal=causal, scale=scale, num_splits=num_splits,
                                out_fp32=kind == "f32", q_scale=QS, k_scale=KS, v_scale=VS, out_dtype=q.dtype)
    return o, l, k1, v1, q8


def dense_new(tfa, q, kp, vp, sl, table, kn, vn, rkw, causal, scale, kind, num_splits=1, q8=None):
    k2, v2 = kp.clone(), vp.clone()
    if q8 is None:
        q8 = torch.full(q.shape, 0x7F, dtype=torch.uint8, device="cuda").view(FP8)
    o, l = tfa.attn_kvcache_fwd(q, k2, v2, sl, table, kn, vn, is_causal=causal, scale=scale, num_splits=num_splits,
                                out_fp32=kind == "f32", q8_scale=QS, k_scale=KS, v_scale=VS, q8=q8, **rkw)
    return o, l, k2, v2, q8


def assert_same(got, want, rows=None):
    names = ("out", "lse", "k pool", "v pool", "q8")
    for name, a, b in zip(names, got, want):
        if name == "q8" and rows is not None:
            a, b = a[rows], b[rows]
        assert torch.equal(bits(a.contiguous()), bits(b.contiguous())), name


DENSE = [
    # D, out kind, Hq, Hkv, page (None: contiguous), Sq, causal, Snew, rotary, rotary_dim
    (128, "bf16", 32, 8, 256, 1, True, 1, "neox", 128),
    (128, "bf16", 32, 8, 256, 1, False, 0, "none", 0),
    (128, "fp16", 8, 8, 128, 4, True, 4, "gptj", 128),
    (128, "f32", 8, 1, None, 129, True, 0, "none", 0),
    (64, "bf16", 8, 1, 128, 129, False, 3, "neox", 32),
    (64, "fp16", 8, 8, None, 4, False, 1, "gptj", 64),
    (64, "f32", 32, 8, 256, 1, True, 1, "none", 0),
    (128, "fp16", 8, 1, 128, 129, True, 129, "neox", 64),
    (64, "bf16", 32, 8, 128, 4, True, 4, "none", 0),
    (128, "f32", 8, 8, 128, 4, False, 2, "gptj", 96),
    (128, "bf16", 8, 2, 256, 129, True, 1, "gptj", 128),      # Sq > Snew near the capacity
    (64, "fp16", 16, 2, 256, 1, True, 0, "none", 0),
]


@pytest.mark.gpu
@pytest.mark.parametrize("D,kind,Hq,Hkv,page,Sq,causal,snew,rotary,rd", DENSE)
def test_dense_query_call_equals_the_composition_bitwise(tfa, D, kind, Hq, Hkv, page, Sq, causal, snew, rotary, rd):
    """Lengths 0, 1, 129, non-multiples of 128 and the full capacity; NaN codes in every slot past K_b."""
    contiguous = page is None
    mbps = 1000 if contiguous else 1024 // page
    lens = [300, 0, 1000 if contiguous else 1024, 1, 129, 77]
    kp, vp, table, cap = make_pools(lens, Hkv, D, page or 1, mbps, seed=70 + D + Sq, contiguous=contiguous,
                                    fill=0xFF if Sq % 2 else 0x7F)
    B = len(lens)
    g = torch.Generator().manual_seed(Sq + snew + D)
    dt = _dt(kind)
    q = torch.empty((B, Sq, Hq, D)).normal_(0, 0.5, generator=g).to(dt).cuda()
    kn = vn = None
    if snew:
        kn = torch.empty((B, snew, Hkv, D)).normal_(0, 0.5, generator=g).to(dt).cuda()
        vn = torch.empty((B, snew, Hkv, D)).normal_(0, 0.5, generator=g).to(dt).cuda()
    sl = torch.tensor(lens, dtype=torch.int32, device="cuda")
    rkw = _rot_kw(rotary, rd, cap, dt)
    scale = D ** -0.5
    want = dense_oracle(tfa, q, kp, vp, sl, table, cap, kn, vn, rkw, causal, scale, kind)
    got = dense_new(tfa, q, kp, vp, sl, table, kn, vn, rkw, causal, scale, kind)
    torch.cuda.synchronize()
    assert got[0].dtype == (torch.float32 if kind == "f32" else dt) and got[0].stride() == q.stride()
    assert_same(got, want)
    assert torch.isfinite(got[0]).all()


@pytest.mark.gpu
@pytest.mark.parametrize("kind,rotary", [("bf16", "none"), ("fp16", "neox"), ("bf16", "gptj")])
def test_saturating_and_subnormal_quotients_match_torch(tfa, kind, rotary):
    """q / q_scale beyond +-448 saturates, below e4m3's smallest normal it rounds to subnormals or to zero: q8 equals
    torch's quantization of q (rot(q)) bit for bit, and the results the oracle's."""
    B, Sq, Hq, Hkv, D, page = 2, 3, 4, 2, 128, 128
    lens = [200, 17]
    kp, vp, table, cap = make_pools(lens, Hkv, D, page, 2, seed=4)
    dt = _dt(kind)
    g = torch.Generator().manual_seed(12)
    mag = torch.empty((B, Sq, Hq, D)).uniform_(0, 1, generator=g)
    sign = torch.where(torch.rand((B, Sq, Hq, D), generator=g) < 0.5, -1.0, 1.0)
    big = QS * (300 + mag * 2000)                            # quotients from 300 to 2300: most saturate
    tiny = QS * mag * 2.0 ** -6                              # quotients below 2^-6: subnormals and zeros
    q = (sign * torch.where(torch.arange(D) % 2 == 0, big, tiny)).to(dt).cuda()
    kn = torch.empty((B, Sq, Hkv, D)).normal_(0, 0.5, generator=g).to(dt).cuda()
    sl = torch.tensor(lens, dtype=torch.int32, device="cuda")
    rkw = _rot_kw(rotary, 64, cap, dt)                       # dimensions [64, 128) pass through unrotated
    want = dense_oracle(tfa, q, kp, vp, sl, table, cap, kn, kn, rkw, True, 1e-3, kind)
    got = dense_new(tfa, q, kp, vp, sl, table, kn, kn, rkw, True, 1e-3, kind)
    torch.cuda.synchronize()
    assert_same(got, want)
    codes = bits(got[4]) & 0x7F
    assert bool((codes == 0x7E).any()) and bool((codes == 0).any()) and bool(((codes > 0) & (codes < 8)).any())
    if rotary == "none":
        assert torch.equal(bits(got[4]), bits(quantize(q, QS)))


def varlen_oracle(tfa, q, kp, vp, cu, maxq, sl, table, cap, kn, vn, rkw, causal, scale, kind, seq_rows):
    k1, v1 = kp.clone(), vp.clone()
    if rkw:
        qr = torch.empty(q.shape, dtype=q.dtype, device="cuda")
        tfa.attn_varlen_kvcache_fwd(q, k1, v1, cu, maxq, sl, table, kn, vn, is_causal=causal, scale=scale, k_scale=KS,
                                    v_scale=VS, q_rot=qr, **rkw)
    else:
        qr = q
        if kn is not None:
            tfa.attn_varlen_kvcache_fwd(q, k1, v1, cu, maxq, sl, table, kn, vn, is_causal=causal, scale=scale,
                                        k_scale=KS, v_scale=VS)
    q8 = quantize(qr, QS)
    lens = [cache_lens_varlen(x, cap, n, kn is not None) for x, n in zip(sl.tolist(), seq_rows)]
    sl2 = torch.tensor(lens, dtype=torch.int32, device="cuda")
    o, l = tfa.attn_varlen_kvcache_fwd(q8, k1, v1, cu, maxq, sl2, table, is_causal=causal, scale=scale,
                                       out_fp32=kind == "f32", q_scale=QS, k_scale=KS, v_scale=VS, out_dtype=q.dtype)
    return o, l, k1, v1, q8


@pytest.mark.gpu
@pytest.mark.parametrize("kind,causal,append,D,rotary", [
    ("bf16", True, True, 128, "neox"), ("fp16", False, True, 64, "gptj"), ("bf16", True, False, 128, "none"),
    ("f32", True, True, 128, "none"), ("fp16", True, True, 128, "gptj")])
def test_varlen_call_equals_the_composition_bitwise(tfa, kind, causal, append, D, rotary):
    """Mixed prefill chunks and decodes, a sequence with Sq_b = 0, an end offset past total_q, and q8 pre-filled with
    NaN codes: only the rows of a sequence are compared, and nothing else leaks into out or lse."""
    seq_q = [3, 1, 200, 0, 1, 129]
    lens = [300, 5, 129, 40, 0, 1024]
    Hq, Hkv, page, mbps = 8, 2, 128, 8
    kp, vp, table, cap = make_pools(lens, Hkv, D, page, mbps, seed=50)
    total = sum(seq_q)
    dt = _dt(kind)
    g = torch.Generator().manual_seed(51)
    q = torch.empty((total, Hq, D)).normal_(0, 0.5, generator=g).to(dt).cuda()
    kn = torch.empty((total, Hkv, D)).normal_(0, 0.5, generator=g).to(dt).cuda() if append else None
    vn = torch.empty((total, Hkv, D)).normal_(0, 0.5, generator=g).to(dt).cuda() if append else None
    starts = [0] + torch.tensor(seq_q).cumsum(0).tolist()
    cu = torch.tensor(starts[:-1] + [total + 50], dtype=torch.int32, device="cuda")
    rows = list(seq_q)                                      # the last offset is clamped to total_q: same rows
    maxq = max(seq_q)
    sl = torch.tensor(lens, dtype=torch.int32, device="cuda")
    rkw = _rot_kw(rotary, D, cap, dt)
    scale = D ** -0.5
    want = varlen_oracle(tfa, q, kp, vp, cu, maxq, sl, table, cap, kn, vn, rkw, causal, scale, kind, rows)
    k2, v2 = kp.clone(), vp.clone()
    q8 = torch.full(q.shape, 0x7F, dtype=torch.uint8, device="cuda").view(FP8)
    o, l = tfa.attn_varlen_kvcache_fwd(q, k2, v2, cu, maxq, sl, table, kn, vn, is_causal=causal, scale=scale,
                                       out_fp32=kind == "f32", q8_scale=QS, k_scale=KS, v_scale=VS, q8=q8, **rkw)
    torch.cuda.synchronize()
    assert o.dtype == (torch.float32 if kind == "f32" else dt)
    assert_same((o, l, k2, v2, q8), want, rows=slice(0, total))
    assert torch.isfinite(o).all()


@pytest.mark.gpu
@pytest.mark.parametrize("num_splits,rotary", [(3, "neox"), (0, "none"), (3, "none"), (0, "gptj")])
def test_split_kv_equals_the_composition_with_the_same_splits(tfa, num_splits, rotary):
    Hq, Hkv, D, page, mbps, Sq = 8, 2, 128, 256, 8, 2
    lens = [2048, 1500, 0, 700, 129]
    kp, vp, table, cap = make_pools(lens, Hkv, D, page, mbps, seed=61)
    g = torch.Generator().manual_seed(62)
    q = torch.empty((len(lens), Sq, Hq, D)).normal_(0, 0.5, generator=g).to(torch.bfloat16).cuda()
    kn = torch.empty((len(lens), Sq, Hkv, D)).normal_(0, 0.5, generator=g).to(torch.bfloat16).cuda()
    sl = torch.tensor(lens, dtype=torch.int32, device="cuda")
    rkw = _rot_kw(rotary, D, cap, torch.bfloat16)
    want = dense_oracle(tfa, q, kp, vp, sl, table, cap, kn, kn, rkw, True, D ** -0.5, "bf16", num_splits)
    got = dense_new(tfa, q, kp, vp, sl, table, kn, kn, rkw, True, D ** -0.5, "bf16", num_splits)
    torch.cuda.synchronize()
    assert_same(got, want)
    _, _, n = tfa.attn_kvcache_fwd(q, kp.clone(), vp.clone(), sl, table, kn, kn, is_causal=True, num_splits=num_splits,
                                   q8_scale=QS, k_scale=KS, v_scale=VS, return_splits=True, **rkw)
    assert n > 1


SCHEDULES = r'''
import os, sys, torch
sys.path.insert(0, os.path.join(os.environ["TFA_ROOT"], "tiny-flash-attention_b200"))
sys.path.insert(0, os.path.join(os.environ["TFA_ROOT"], "tests"))
import tfa_ctypes as tfa
from test_kvcache_qkv8 import make_pools
from test_kvcache_qkv8_q16 import QS, KS, VS, rope_tables
lens = [1000, 0, 129, 2047, 64, 300]
res = []
g = torch.Generator().manual_seed(9)
cos, sin = rope_tables(2048, 128, torch.bfloat16)
for causal, Sq, ns, rot in ((True, 1, 1, True), (False, 4, 1, False), (True, 200, 1, True), (False, 1, 3, True)):
    kp, vp, table, _ = make_pools(lens, 2, 128, 256, 8, seed=9)
    q = torch.empty((len(lens), Sq, 8, 128)).normal_(0, 0.5, generator=g).to(torch.bfloat16).cuda()
    kn = torch.empty((len(lens), Sq, 2, 128)).normal_(0, 0.5, generator=g).to(torch.bfloat16).cuda()
    sl = torch.tensor(lens, dtype=torch.int32, device="cuda")
    rkw = dict(rotary_cos=cos, rotary_sin=sin) if rot else {}
    q8 = torch.empty(q.shape, dtype=torch.float8_e4m3fn, device="cuda")
    o, l = tfa.attn_kvcache_fwd(q, kp, vp, sl, table, kn, kn, is_causal=causal, num_splits=ns, q8_scale=QS,
                                k_scale=KS, v_scale=VS, q8=q8, **rkw)
    res.append((o.cpu(), l.cpu(), q8.view(torch.uint8).cpu(), kp.view(torch.uint8).cpu(),
                tfa.lib().tfa_internal_last_variant()))
qv = torch.empty((300, 8, 128)).normal_(0, 0.5, generator=g).to(torch.float16).cuda()
cu = torch.tensor([0, 1, 1, 201, 202, 203, 300], dtype=torch.int32, device="cuda")
kp, vp, table, _ = make_pools(lens, 2, 128, 256, 8, seed=9)
o, l = tfa.attn_varlen_kvcache_fwd(qv, kp, vp, cu, 200, sl, table, qv[:, :2], qv[:, 2:4], is_causal=True, q8_scale=QS,
                                   k_scale=KS, v_scale=VS, rotary_cos=cos.half(), rotary_sin=sin.half())
res.append((o.cpu(), l.cpu(), o.cpu(), kp.view(torch.uint8).cpu(), tfa.lib().tfa_internal_last_variant()))
torch.cuda.synchronize()
torch.save(res, os.environ["TFA_OUT"])
'''


@pytest.mark.gpu
def test_classic_and_persistent_agree_bitwise(tfa):
    import tempfile
    outs = {}
    with tempfile.TemporaryDirectory() as tmp:
        for variant in ("classic", "persist"):
            path = os.path.join(tmp, variant + ".pt")
            env = dict(os.environ, TFA_ROOT=ROOT, TFA_OUT=path, TFA_KERNEL=variant)
            p = subprocess.run([sys.executable, "-c", SCHEDULES], env=env, capture_output=True, text=True, timeout=600)
            assert p.returncode == 0, p.stderr[-2000:]
            outs[variant] = torch.load(path)
    for ra, rb in zip(outs["classic"], outs["persist"]):
        assert (ra[-1], rb[-1]) == (0, 4)
        for a, b in zip(ra[:-1], rb[:-1]):
            assert torch.equal(bits(a), bits(b))


@pytest.mark.gpu
@pytest.mark.parametrize("rotary", ["neox", "none"])
def test_cuda_graph_replays_with_new_q_lengths_and_table(tfa, rotary):
    lens1, lens2 = [300, 5, 1000, 129], [1000, 700, 0, 256]
    B, Hq, Hkv, D, page, mbps = 4, 8, 2, 128, 256, 5
    kp, vp, table, cap = make_pools(lens1, Hkv, D, page, mbps, seed=13)
    k0, v0 = kp.clone(), vp.clone()
    g = torch.Generator().manual_seed(5)
    q = torch.empty((B, 1, Hq, D)).normal_(0, 0.5, generator=g).to(torch.bfloat16).cuda()
    kn = torch.empty((B, 1, Hkv, D)).normal_(0, 0.5, generator=g).to(torch.bfloat16).cuda()
    vn = torch.empty((B, 1, Hkv, D)).normal_(0, 0.5, generator=g).to(torch.bfloat16).cuda()
    sl = torch.tensor(lens1, dtype=torch.int32, device="cuda")
    out = torch.empty(q.shape, dtype=torch.bfloat16, device="cuda")
    lse = torch.empty((B, Hq, 1), dtype=torch.float32, device="cuda")
    q8 = torch.empty(q.shape, dtype=FP8, device="cuda")
    rkw = _rot_kw(rotary, D, cap, torch.bfloat16)
    kw = dict(is_causal=True, num_splits=3, q8_scale=QS, k_scale=KS, v_scale=VS, **rkw)
    step = lambda: tfa.attn_kvcache_fwd(q, kp, vp, sl, table, kn, vn, out=out, lse=lse, q8=q8, **kw)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        step()
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        step()
    results = []
    for lens, seed in ((lens1, None), (lens2, 3)):
        if seed is not None:
            gp = torch.Generator().manual_seed(seed)
            sl.copy_(torch.tensor(lens, dtype=torch.int32))
            table.copy_(torch.randperm(kp.shape[0], generator=gp)[:B * mbps].to(torch.int32).view(B, mbps))
            q.copy_(torch.empty(q.shape).normal_(0, 0.5, generator=gp).to(torch.bfloat16))
        kp.copy_(k0)
        vp.copy_(v0)
        graph.replay()
        want = dense_oracle(tfa, q, k0, v0, sl.clone(), table.clone(), cap, kn, vn, rkw, True, D ** -0.5, "bf16", 3)
        torch.cuda.synchronize()
        assert_same((out, lse, kp, vp, q8), want)
        results.append(out.clone())
    assert not torch.equal(results[0], results[1])


@pytest.mark.gpu
def test_launch_counts_and_guard_regions(tfa):
    B, Hq, Hkv, D = 4, 4, 2, 64
    lens = [500, 0, 64, 129]
    kp, vp, table, cap = make_pools(lens, Hkv, D, 128, 5, seed=1)
    g = torch.Generator().manual_seed(2)
    q = torch.empty((B, 1, Hq, D)).normal_(0, 0.5, generator=g).to(torch.float16).cuda()
    sl = torch.tensor(lens, dtype=torch.int32, device="cuda")
    kn = torch.empty((B, 1, Hkv, D)).normal_(0, 0.5, generator=g).to(torch.float16).cuda()
    rkw = _rot_kw("neox", D, cap, torch.float16)
    kw = dict(is_causal=True, q8_scale=QS, k_scale=KS, v_scale=VS)
    for extra, want in ((dict(), 2), (dict(k_new=kn, v_new=kn), 2), (dict(k_new=kn, v_new=kn, **rkw), 2),
                        (dict(num_splits=3), 3), (dict(k_new=kn, v_new=kn, num_splits=3, **rkw), 3)):
        n0 = tfa.launch_count()
        tfa.attn_kvcache_fwd(q, kp, vp, sl, table, **kw, **extra)
        assert tfa.launch_count() - n0 == want, extra
    cu = torch.tensor([0, 1, 1, 2, 3], dtype=torch.int32, device="cuda")
    qv = q[:, 0].contiguous()
    knv = kn[:, 0][:3].contiguous()
    for extra in (dict(), dict(k_new=knv, v_new=knv), dict(k_new=knv, v_new=knv, **rkw)):
        n0 = tfa.launch_count()
        tfa.attn_varlen_kvcache_fwd(qv[:3], kp, vp, cu, 1, sl, table, **kw, **extra)
        assert tfa.launch_count() - n0 == 2, extra
    # guard regions around out, lse, q8 and the pools
    big = torch.full((6, *q.shape[1:]), 7.0, dtype=torch.float16, device="cuda")
    lbig = torch.full((6, Hq, 1), 7.0, dtype=torch.float32, device="cuda")
    qbig = torch.full((6, *q.shape[1:]), 0x5A, dtype=torch.uint8, device="cuda")
    pk = torch.full((kp.shape[0] + 2, *kp.shape[1:]), 0x5A, dtype=torch.uint8, device="cuda")
    pv = pk.clone()
    pk[1:-1] = kp.view(torch.uint8)
    pv[1:-1] = vp.view(torch.uint8)
    for ns in (1, 3):
        tfa.attn_kvcache_fwd(q, pk[1:-1].view(FP8), pv[1:-1].view(FP8), sl, table, kn, kn, num_splits=ns,
                             out=big[1:5], lse=lbig[1:5], q8=qbig[1:5].view(FP8), **kw, **rkw)
        torch.cuda.synchronize()
        assert torch.all(big[0] == 7) and torch.all(big[5] == 7) and torch.all(lbig[0] == 7) and torch.all(lbig[5] == 7)
        assert torch.all(qbig[0] == 0x5A) and torch.all(qbig[5] == 0x5A) and not torch.all(qbig[1:5] == 0x5A)
        for p in (pk, pv):
            assert torch.all(p[0] == 0x5A) and torch.all(p[-1] == 0x5A)
    ov = torch.full((5, Hq, D), 7.0, dtype=torch.float16, device="cuda")
    lv = torch.full((Hq * 3 + 2,), 7.0, dtype=torch.float32, device="cuda")
    qv8 = torch.full((5, Hq, D), 0x5A, dtype=torch.uint8, device="cuda")
    tfa.attn_varlen_kvcache_fwd(qv[:3], kp, vp, cu, 1, sl, table, knv, knv, out=ov[1:4], lse=lv[1:-1].view(Hq, 3),
                                q8=qv8[1:4].view(FP8), **kw, **rkw)
    torch.cuda.synchronize()
    assert torch.all(ov[0] == 7) and torch.all(ov[4] == 7) and lv[0] == 7 and lv[-1] == 7
    assert torch.all(qv8[0] == 0x5A) and torch.all(qv8[4] == 0x5A)


@pytest.mark.gpu
def test_extension_entries_equal_the_c_calls_and_routing_errors(built, tfa):
    import attention_cutlass as ac
    lens = [300, 1, 0, 640]
    B, Sq, Hq, Hkv, D = 4, 2, 8, 2, 128
    kp, vp, table, cap = make_pools(lens, Hkv, D, 256, 4, seed=17, fill=0xFF)
    g = torch.Generator().manual_seed(17)
    q = torch.empty((B, Sq, Hq, D)).normal_(0, 0.5, generator=g).to(torch.float16).cuda()
    kn = torch.empty((B, Sq, Hkv, D)).normal_(0, 0.5, generator=g).to(torch.float16).cuda()
    sl = torch.tensor(lens, dtype=torch.int32, device="cuda")
    scale = D ** -0.5
    cos, sin = rope_tables(cap, 64, torch.float16)
    for rot in (dict(), dict(rotary_cos=cos, rotary_sin=sin, rotary_interleaved=True)):
        k1, v1, k2, v2 = kp.clone(), vp.clone(), kp.clone(), vp.clone()
        out, lse = ac.flash_attention_v2_kvcache_qkv8_q16(q, k1, v1, sl, table, kn, kn, QS, KS, VS, True, scale, 1,
                                                          **rot)
        want, wl = tfa.attn_kvcache_fwd(q, k2, v2, sl, table, kn, kn, is_causal=True, scale=scale, q8_scale=QS,
                                        k_scale=KS, v_scale=VS, **rot)
        torch.cuda.synchronize()
        assert out.shape == q.shape and out.dtype == torch.float16 and lse.shape == (B, Hq, Sq)
        assert torch.equal(bits(out), bits(want)) and torch.equal(lse, wl)
        assert torch.equal(bits(k1), bits(k2)) and torch.equal(bits(v1), bits(v2))
        cu = torch.tensor([0, 2, 3, 3, 5], dtype=torch.int32, device="cuda")
        qv = q.reshape(B * Sq, Hq, D)[:5].contiguous()
        knv = kn.reshape(B * Sq, Hkv, D)[:5].contiguous()
        o2, l2 = ac.flash_attention_v2_varlen_kvcache_qkv8_q16(qv, k1, v1, cu, 2, sl, table, knv, knv, QS, KS, VS,
                                                               True, scale, **rot)
        w2, wl2 = tfa.attn_varlen_kvcache_fwd(qv, k2, v2, cu, 2, sl, table, knv, knv, is_causal=True, scale=scale,
                                              q8_scale=QS, k_scale=KS, v_scale=VS, **rot)
        torch.cuda.synchronize()
        assert o2.dtype == torch.float16 and torch.equal(bits(o2), bits(w2)) and torch.equal(l2, wl2)
        assert torch.equal(bits(k1), bits(k2)) and torch.equal(bits(v1), bits(v2))
    o0, l0 = ac.flash_attention_v2_kvcache_qkv8_q16(q, kp, vp, sl, table, None, None, QS, KS, VS, False, scale, 0)
    w0, wl0 = tfa.attn_kvcache_fwd(q, kp, vp, sl, table, is_causal=False, scale=scale, num_splits=0, q8_scale=QS,
                                   k_scale=KS, v_scale=VS)
    torch.cuda.synchronize()
    assert torch.equal(bits(o0), bits(w0)) and torch.equal(l0, wl0)
    # the extension's argument errors
    with pytest.raises(RuntimeError, match="float8_e4m3fn"):
        ac.flash_attention_v2_kvcache_qkv8_q16(q, kp.half(), vp.half(), sl, table, None, None, QS, KS, VS, True, scale,
                                               1)
    with pytest.raises(RuntimeError, match="rotary needs k_new"):
        ac.flash_attention_v2_kvcache_qkv8_q16(q, kp, vp, sl, table, None, None, QS, KS, VS, True, scale, 1,
                                               rotary_cos=cos, rotary_sin=sin)
    with pytest.raises(RuntimeError, match="q_scale, k_scale and v_scale"):
        ac.flash_attention_v2_kvcache_qkv8_q16(q, kp, vp, sl, table, None, None, 0.0, KS, VS, True, scale, 1)
    # ctypes routing errors of q8_scale: a float8 q, a 16-bit cache, a q_scale / out_dtype beside it
    q8 = quantize(q, QS)
    with pytest.raises(ValueError, match="q8_scale"):
        tfa.attn_kvcache_fwd(q8, kp, vp, sl, table, q8_scale=QS, k_scale=KS, v_scale=VS, out_dtype=torch.float16)
    with pytest.raises(ValueError, match="q8_scale"):
        tfa.attn_varlen_kvcache_fwd(q8[:, 0], kp, vp, cu, 1, sl, table, q8_scale=QS, k_scale=KS, v_scale=VS,
                                    out_dtype=torch.float16)
    with pytest.raises(TypeError, match="q8_scale"):
        tfa.attn_kvcache_fwd(q, kp.half(), vp.half(), sl, table, q8_scale=QS)
    with pytest.raises(TypeError, match="q8_scale"):
        tfa.attn_varlen_kvcache_fwd(q[:, 0], kp.half(), vp.half(), cu, 1, sl, table, q8_scale=QS)
    with pytest.raises(ValueError, match="float8_e4m3fn q"):
        tfa.attn_kvcache_fwd(q, kp, vp, sl, table, q8_scale=QS, q_scale=0.5, k_scale=KS, v_scale=VS)
