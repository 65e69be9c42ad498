"""Attention against an FP8 (e4m3) KV cache: tfa_attn_kvcache_fp8_fwd / tfa_attn_varlen_kvcache_fp8_fwd and
attention_cutlass.flash_attention_v2_kvcache_fp8 / flash_attention_v2_varlen_kvcache_fp8.

CPU: the entry points are declared and exported, the error string exists, every argument error comes back before any
device work, and the barrier-protocol model with the converter role passes and catches two misplaced converter steps.
GPU: out and lse equal the 16-bit cache call on the widened cache bit for bit (softmax scale s' = scale * k_scale, out
times a power-of-two v_scale), general scales stay within the oracle's tolerances, the appends store exactly torch's
clamp-and-cast codes and nothing else, rotary pools are the quantized 16-bit rotary pools, NaN codes in unused slots
change nothing, the variable-length call equals per-sequence calls, split-KV, both schedules, CUDA-graph replay, launch
counts, guard regions and the extension entry points."""
import ctypes
import os
import random
import subprocess
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

TFA_EINVAL_KVQUANT = -15
TFA_FP8_E4M3 = 2


def declared_functions():
    import re
    src = open(os.path.join(ROOT, "include", "tfa_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return set(re.findall(r"\b(tfa_[a-z0-9_]+)\s*\(", src))


# ------------------------------------------------------------------ CPU ------------------------------------------------

def test_header_declares_and_library_exports_fp8_calls(built):
    import tfa_ctypes
    names = declared_functions()
    hdr = open(os.path.join(ROOT, "include", "tfa_b200.h")).read()
    assert "TFA_EINVAL_KVQUANT (-15)" in hdr and "#define TFA_FP8_E4M3 2" in hdr and "TFA_ABI_VERSION 2" in hdr
    L = ctypes.CDLL(tfa_ctypes.LIB_PATH)
    for fn in ("tfa_attn_kvcache_fp8_fwd", "tfa_attn_varlen_kvcache_fp8_fwd"):
        assert fn in names and hasattr(L, fn)
    msg = tfa_ctypes.lib().tfa_error_string(TFA_EINVAL_KVQUANT)
    assert msg.startswith(b"tfa:") and b"FP8" in msg and b"k_scale" in msg and b"16" in msg


def _buffers():
    buf = ctypes.create_string_buffer(4096 + 16)
    base = (ctypes.addressof(buf) + 15) & ~15
    return buf, base, base + 1024


def test_kvcache_fp8_argument_validation_without_device(built):
    """Host buffers only: every code must come back before anything touches a device.  The 16-bit call's checks come
    first, in their order; then the quantization arguments."""
    import tfa_ctypes
    L = tfa_ctypes.lib()
    buf, base, ints = _buffers()
    Hq, Hkv, D, page = 4, 2, 64, 256

    def mk(**kw):
        return tfa_ctypes.KvcacheArgs(
            kw.get("q", base), base, base, kw.get("k_new", None), kw.get("v_new", None), kw.get("out", base), None,
            kw.get("seqlens", ints), kw.get("table", ints), kw.get("B", 2), kw.get("Hq", Hq), kw.get("Hkv", Hkv),
            kw.get("Sq", 1), kw.get("D", D), kw.get("nblk", 8), kw.get("page", page), kw.get("mbps", 4),
            kw.get("snew", 1), Hq * D, kw.get("qss", Hq * D), D, kw.get("ksb", page * Hkv * D),
            kw.get("kss", Hkv * D), kw.get("ksh", D), kw.get("bts", 4), Hkv * D, kw.get("nss", Hkv * D), D,
            kw.get("dtype", 0), 1, kw.get("scale", 0.1), 0, kw.get("splits", 1), None, 0, None)

    def quant(**kw):
        return tfa_ctypes.KvQuantArgs(kw.get("cdt", TFA_FP8_E4M3), kw.get("ks", 0.5), kw.get("vs", 2.0))

    def call(rot=None, **kw):
        return L.tfa_attn_kvcache_fp8_fwd(ctypes.byref(mk(**kw)), ctypes.byref(rot) if rot else None,
                                          ctypes.byref(quant(**kw)))

    assert L.tfa_attn_kvcache_fp8_fwd(None, None, ctypes.byref(quant())) == -1
    assert L.tfa_attn_kvcache_fp8_fwd(ctypes.byref(mk()), None, None) == -1
    # the 16-bit call's errors, through the new entry point
    assert call(q=None) == -1 and call(out=base + 8) == -1
    assert call(D=96) == -2 and call(B=0) == -3
    assert call(dtype=2) == -4                                # q's dtype: bf16 / fp16 only
    assert call(qss=60) == -5 and call(kss=30) == -5
    assert call(scale=-1.0) == -9 and call(Hkv=3) == -10
    assert call(seqlens=None) == -13 and call(page=64) == -13 and call(k_new=base) == -13
    # rotary errors
    rot = tfa_ctypes.RotaryArgs(base, base, page * 4, 32, 0, base)
    assert call(rot=rot, k_new=base, v_new=base, cdt=0) == TFA_EINVAL_KVQUANT   # valid rotary: the next check runs
    assert call(rot=tfa_ctypes.RotaryArgs(None, base, page * 4, 32, 0, base), k_new=base, v_new=base) == -14
    assert call(rot=tfa_ctypes.RotaryArgs(base, base, page * 4, 24, 0, base), k_new=base, v_new=base) == -14
    assert call(rot=rot) == -14                               # rotary without k_new
    # quantization arguments
    E = TFA_EINVAL_KVQUANT
    assert call(cdt=0) == E and call(cdt=1) == E and call(cdt=3) == E
    for bad in (0.0, -1.0, float("nan"), float("inf"), -float("inf")):
        assert call(ks=bad) == E and call(vs=bad) == E, bad
    assert call(kss=Hkv * D + 8) == E and call(ksh=D + 8) == E and call(ksb=page * Hkv * D + 8) == E
    # a rotary error comes before a quantization error, a cache error before both
    assert call(rot=rot, cdt=0) == -14 and call(seqlens=None, cdt=0) == -13
    # s' = scale * k_scale must stay finite and must not underflow (uniform attention in disguise)
    assert call(scale=3.0e38, ks=10.0) == -9
    assert call(scale=1e-30, ks=1e-20) == -9 and call(scale=1e-20, ks=1e-19) == -9
    big = 3.3e38               # finite scales above 3e38 pass their own check; s' then overflows or underflows
    assert call(ks=big, scale=1.0) == -9 and call(vs=big, scale=1e-30, ks=1e-20) == -9


def test_varlen_kvcache_fp8_argument_validation_without_device(built):
    import tfa_ctypes
    L = tfa_ctypes.lib()
    buf, base, ints = _buffers()
    Hq, Hkv, D, page = 4, 2, 64, 128

    def mk(**kw):
        return tfa_ctypes.VarlenKvcacheArgs(
            base, base, base, None, None, base, None, kw.get("cu", ints), kw.get("seqlens", ints), ints, 2, Hq, Hkv,
            kw.get("D", D), 8, kw.get("maxq", 4), 8, page, 4, Hq * D, D, page * Hkv * D, kw.get("kss", Hkv * D), D,
            4, 0, 0, kw.get("dtype", 1), 1, 0.1, 0, None)

    def call(**kw):
        q = tfa_ctypes.KvQuantArgs(kw.get("cdt", TFA_FP8_E4M3), kw.get("ks", 1.0), kw.get("vs", 1.0))
        return L.tfa_attn_varlen_kvcache_fp8_fwd(ctypes.byref(mk(**kw)), ctypes.byref(q))

    assert L.tfa_attn_varlen_kvcache_fp8_fwd(None, None) == -1
    assert call(D=96) == -2 and call(dtype=2) == -4 and call(seqlens=None) == -13
    assert call(cu=None) == -12 and call(maxq=9) == -12
    E = TFA_EINVAL_KVQUANT
    assert call(cdt=1) == E and call(ks=0.0) == E and call(vs=float("nan")) == E and call(kss=Hkv * D + 8) == E
    assert call(cu=None, cdt=1) == -12


def _protocol_model():
    sys.path.insert(0, os.path.join(ROOT, "scripts"))
    import protocol_model as pm
    return pm


def test_protocol_model_with_the_converter():
    """Both FP8 modes' items (skipped, tile-less but written, last tile past the keys), ring depths 4 / 8, raw ring
    depths 2 / 4."""
    pm = _protocol_model()
    for trial in range(400):
        rng = random.Random(4242 + trial)
        items, empty, vtail, nraw = pm.random_fp8_cache_items(rng, varlen=trial % 2 == 1)
        pm.Sim(items, rng.choice([4, 8]), rng, empty, vtail, fp8=True, nraw=nraw).run()


CONV_STORES = '                    self.kv_buf[slot] = "converting"\n                    yield lambda: True\n'
CONV_KV_FULL = "                    self.kv_full[slot].arrive()               # after the last store (and its proxy fence)"
CONV_EMPTY_WAIT = "                    yield lambda s=slot, p=((ent // N) & 1) ^ 1: self.kv_empty[s].done(p)\n" \
                  "                    # widen"


def _caught(mutated, seeds=200):
    ns = {"__name__": "mutated_model"}
    exec(compile(mutated, "mutated_model", "exec"), ns)
    caught = 0
    for trial in range(seeds):
        rng = random.Random(91 + trial)
        items, empty, vtail, nraw = ns["random_fp8_cache_items"](rng, trial % 2 == 1)
        try:
            ns["Sim"](items, 4, rng, empty, vtail, fp8=True, nraw=nraw).run()
        except AssertionError:
            caught += 1
    return caught


def test_protocol_model_catches_kv_full_before_the_last_store():
    """Mutation: the converter arrives on kv_full while its stores into the slot are still in flight -> a softmax
    warpgroup may issue its wgmma on a half-written slot, which the model must report."""
    src = open(os.path.join(ROOT, "scripts", "protocol_model.py")).read()
    assert CONV_STORES in src and CONV_KV_FULL in src
    mutated = src.replace(CONV_KV_FULL, "                    pass").replace(
        CONV_STORES, '                    self.kv_buf[slot] = "converting"\n                    self.kv_full[slot].arrive()\n'
                     '                    yield lambda: True\n')
    assert _caught(mutated) > 5


def test_protocol_model_catches_a_store_before_the_kv_empty_wait():
    src = open(os.path.join(ROOT, "scripts", "protocol_model.py")).read()
    assert CONV_EMPTY_WAIT in src
    # the converter no longer waits for the consumers to release the slot before widening into it
    mutated = src.replace(CONV_EMPTY_WAIT, "                    # widen")
    assert _caught(mutated) > 5


# ------------------------------------------------------------------ GPU ------------------------------------------------

@pytest.fixture(scope="module")
def tfa(built):
    import tfa_ctypes
    tfa_ctypes.lib()
    return tfa_ctypes


FP8 = torch.float8_e4m3fn
FINITE = [c for c in range(256) if c not in (0x7F, 0xFF)]


def _dt(kind):
    return torch.bfloat16 if kind == "bf16" else torch.float16


def quantize(x, scale):
    """torch's reference for the append: an IEEE fp32 division (on the CPU: torch's CUDA division by a scalar multiplies
    by its reciprocal), round to nearest-even, saturate to +-448."""
    q = (x.cpu().float() / torch.tensor(scale, dtype=torch.float32)).clamp(-448, 448).to(FP8)
    return q.to(x.device)


def make_fp8_cache(lens, Sq, Hq, Hkv, D, kind, page, seed=20, fill=0, mbps=None, spare=3, snew=0, contiguous=False):
    """q (B, Sq, Hq, D); a permuted block table (or None for a contiguous cache); e4m3 pools whose first lens[b] keys of
    each sequence hold every finite code (random order) and every other slot the byte `fill`."""
    g = torch.Generator(device="cpu")
    g.manual_seed(seed)
    B = len(lens)
    if mbps is None:
        mbps = max(1, -(-(max(lens) + snew) // page))
    if contiguous:
        mbps, page, nblk = 1, mbps * page, B
        perm = torch.arange(B, dtype=torch.int32).view(B, 1)
    else:
        nblk = B * mbps + spare
        perm = torch.randperm(nblk, generator=g)[:B * mbps].to(torch.int32).view(B, mbps)
    codes = torch.tensor(FINITE, dtype=torch.uint8)
    pools = []
    for _ in range(2):
        pool = torch.full((nblk, page, Hkv, D), fill, dtype=torch.uint8)
        for b in range(B):
            data = codes[torch.randint(0, len(FINITE), (mbps * page, Hkv, D), generator=g)]
            data[lens[b]:] = fill
            pool[perm[b].long()] = data.view(mbps, page, Hkv, D)
        pools.append(pool.view(FP8).cuda())
    q = torch.empty((B, Sq, Hq, D)).normal_(0.0, 0.5, generator=g).to(_dt(kind)).cuda()
    table = None if contiguous else perm.cuda()
    return q, pools[0], pools[1], table, torch.tensor(lens, dtype=torch.int32, device="cuda")


def bits(t):
    return t.view(torch.uint8) if t.element_size() == 1 else t.view(torch.int16 if t.element_size() == 2 else torch.int32)


WIDEN = [
    # D, kind, Hq, Hkv, page (None: contiguous), Sq, causal
    (128, "bf16", 32, 8, 256, 1, False),
    (128, "fp16", 8, 8, 128, 4, True),
    (64, "bf16", 8, 1, 128, 200, True),
    (64, "fp16", 4, 1, 256, 1, True),
    (128, "bf16", 8, 2, None, 200, False),
    (64, "fp16", 4, 4, None, 4, False),
]
LENS = [300, 0, 128, 1, 1000, 256, 77]


@pytest.mark.gpu
@pytest.mark.parametrize("D,kind,Hq,Hkv,page,Sq,causal", WIDEN)
def test_fp8_equals_16bit_call_on_widened_cache_bitwise(tfa, D, kind, Hq, Hkv, page, Sq, causal):
    """Every finite code, power-of-two v_scale: out = 16-bit call(k8, v8 widened, s') * v_scale, lse equal."""
    q, kp, vp, table, lens = make_fp8_cache(LENS, Sq, Hq, Hkv, D, kind, page or 128, contiguous=page is None,
                                            mbps=8 if page is None else None)
    dt = _dt(kind)
    scale, k_scale, v_scale = D ** -0.5, 0.0371, 0.25
    s_eff = float(torch.tensor(scale, dtype=torch.float32) * torch.tensor(k_scale, dtype=torch.float32))
    for f32 in (False, True):
        out, lse = tfa.attn_kvcache_fwd(q, kp, vp, lens, table, is_causal=causal, scale=scale, out_fp32=f32,
                                        k_scale=k_scale, v_scale=v_scale)
        o16, l16 = tfa.attn_kvcache_fwd(q, kp.to(dt), vp.to(dt), lens, table, is_causal=causal, scale=s_eff,
                                        out_fp32=f32)
        torch.cuda.synchronize()
        assert torch.equal(lse, l16), f32
        assert torch.equal(bits(out), bits(o16 * v_scale)), f32


@pytest.mark.gpu
@pytest.mark.parametrize("kind,causal,Sq,ns", [("bf16", False, 1, 1), ("fp16", True, 4, 1), ("bf16", True, 1, 3),
                                               ("bf16", False, 200, 1), ("fp16", False, 1, 0)])
def test_fp8_general_scales_match_oracle(tfa, kind, causal, Sq, ns):
    """k_scale / v_scale that are no powers of two, split-KV included: a float64 oracle on the dequantized cache."""
    from test_kvcache import check_vs_oracle
    lens = [300, 1000, 129, 2049] if ns != 1 else [300, 1000, 129, 77]
    q, kp, vp, table, sl = make_fp8_cache(lens, Sq, 8, 2, 128, kind, 256, seed=7)
    ks, vs = 0.0123, 0.00731
    scale = 128 ** -0.5
    out, lse = tfa.attn_kvcache_fwd(q, kp, vp, sl, table, is_causal=causal, scale=scale, num_splits=ns, k_scale=ks,
                                    v_scale=vs)
    kd, vd = kp.float() * ks, vp.float() * vs
    for b, K in enumerate(lens):
        check_vs_oracle(out, lse, q, kd, vd, table, b, K, causal, scale, kind)


SPECIAL = [448.0, -448.0, 464.0, 465.0, -465.0, float("inf"), -float("inf"), 0.0, -0.0, 2.0 ** -9, -(2.0 ** -9),
           3 * 2.0 ** -9, 2.0 ** -10, 2.0 ** -11, 0.0013, 1000.0, 300.0, 1.0625]


def _appended(table, lens, snew, cap, page, nblk):
    """[(b, i, block, row)] of every appended token kept, per the cache's length rule."""
    res = []
    for b, raw in enumerate(lens):
        L = min(max(raw, 0), cap - snew)
        for i in range(snew):
            key = L + i
            blk = int(table[b, key // page]) if table is not None else b
            if 0 <= blk < nblk:
                res.append((b, i, blk, key % page if table is not None else key))
    return res


@pytest.mark.gpu
@pytest.mark.parametrize("kind,snew,page", [("bf16", 1, 128), ("fp16", 5, 256), ("bf16", 130, None)])
def test_fp8_append_stores_torch_codes_and_nothing_else(tfa, kind, snew, page):
    lens = [300, 0, 1000, 511, -4, 9999]
    B, Hq, Hkv, D = len(lens), 8, 2, 128
    mbps = 4
    q, kp, vp, table, _ = make_fp8_cache([min(max(x, 0), 1000) for x in lens], 1, Hq, Hkv, D, kind, page or 256,
                                         seed=3, mbps=mbps, contiguous=page is None, fill=0x7f)
    pg = kp.shape[1]
    cap = pg * (1 if page is None else mbps)
    nblk = kp.shape[0]
    if table is not None:
        table[1, 0] = -1                                      # out-of-range entries drop their tokens
        table[3, 1] = nblk + 5
    sl = torch.tensor(lens, dtype=torch.int32, device="cuda")
    g = torch.Generator(device="cpu")
    g.manual_seed(8)
    dt = _dt(kind)
    kn = torch.empty((B, snew, Hkv, D)).normal_(0, 3.0, generator=g)
    sp = torch.tensor(SPECIAL)
    kn.view(-1)[: kn.numel() // 2] = sp[torch.randint(0, len(SPECIAL), (kn.numel() // 2,), generator=g)]
    ks, vs = 0.75, 1.0
    kn = (kn * ks).to(dt).cuda()
    vn = torch.flip(kn, dims=[0]).contiguous()
    k0, v0 = kp.clone(), vp.clone()
    tfa.attn_kvcache_fwd(q, kp, vp, sl, table, kn, vn, is_causal=True, k_scale=ks, v_scale=vs)
    torch.cuda.synchronize()
    wk, wv = k0.clone(), v0.clone()
    tab = table.cpu() if table is not None else None
    for b, i, blk, row in _appended(tab, lens, snew, cap, pg, nblk):
        wk[blk, row] = quantize(kn[b, i], ks)
        wv[blk, row] = quantize(vn[b, i], vs)
    assert torch.equal(bits(kp), bits(wk)) and torch.equal(bits(vp), bits(wv))


@pytest.mark.gpu
@pytest.mark.parametrize("interleaved", [False, True])
def test_fp8_rotary_pools_and_output(tfa, interleaved):
    """The pools equal the 16-bit rotary call's appended keys quantized; out equals the FP8 call without k_new on that
    pool with the rotary call's q_rot."""
    lens = [300, 0, 700, 129]
    B, Sq, Hq, Hkv, D, page, mbps, snew = 4, 2, 8, 2, 128, 256, 4, 2
    kind, dt = "bf16", torch.bfloat16
    q, kp, vp, table, sl = make_fp8_cache(lens, Sq, Hq, Hkv, D, kind, page, seed=12, mbps=mbps)
    cap = page * mbps
    g = torch.Generator(device="cpu")
    g.manual_seed(2)
    kn = torch.empty((B, snew, Hkv, D)).normal_(0, 1, generator=g).to(dt).cuda()
    vn = torch.empty((B, snew, Hkv, D)).normal_(0, 1, generator=g).to(dt).cuda()
    ang = torch.arange(cap)[:, None] * (10000.0 ** (-torch.arange(0, 64, 2) / 64))[None]
    cos, sin = ang.cos().to(dt).cuda(), ang.sin().to(dt).cuda()
    ks, vs = 0.02, 0.5
    k16, v16 = kp.to(dt), vp.to(dt)
    q_rot16 = torch.empty_like(q)
    tfa.attn_kvcache_fwd(q, k16, v16, sl, table, kn, vn, is_causal=True, rotary_cos=cos, rotary_sin=sin,
                         rotary_interleaved=interleaved, q_rot=q_rot16)
    k8, v8 = kp.clone(), vp.clone()
    q_rot = torch.empty_like(q)
    out, lse = tfa.attn_kvcache_fwd(q, k8, v8, sl, table, kn, vn, is_causal=True, rotary_cos=cos, rotary_sin=sin,
                                    rotary_interleaved=interleaved, q_rot=q_rot, k_scale=ks, v_scale=vs)
    torch.cuda.synchronize()
    assert torch.equal(q_rot, q_rot16)
    wk, wv = kp.clone(), vp.clone()
    for b, i, blk, row in _appended(table.cpu(), lens, snew, cap, page, kp.shape[0]):
        wk[blk, row] = quantize(k16[blk, row], ks)
        wv[blk, row] = quantize(v16[blk, row], vs)
    assert torch.equal(bits(k8), bits(wk)) and torch.equal(bits(v8), bits(wv))
    lens2 = torch.tensor([min(max(x, 0), cap - snew) + snew for x in lens], dtype=torch.int32, device="cuda")
    o2, l2 = tfa.attn_kvcache_fwd(q_rot, k8, v8, lens2, table, is_causal=True, k_scale=ks, v_scale=vs)
    torch.cuda.synchronize()
    assert torch.equal(out, o2) and torch.equal(lse, l2)


@pytest.mark.gpu
@pytest.mark.parametrize("D,kind,ns", [(128, "bf16", 1), (64, "fp16", 1), (128, "fp16", 3)])
def test_fp8_nan_codes_in_unused_slots_change_nothing(tfa, D, kind, ns):
    lens = [300, 0, 129, 1000]
    outs = []
    for fill in (0x7f, 0xff, 0):
        q, kp, vp, table, sl = make_fp8_cache(lens, 4, 8, 2, D, kind, 256, seed=5, fill=fill)
        o, l = tfa.attn_kvcache_fwd(q, kp, vp, sl, table, is_causal=False, num_splits=ns, k_scale=0.1, v_scale=0.3)
        outs.append((o, l))
    torch.cuda.synchronize()
    assert torch.isfinite(outs[0][0]).all() and torch.isfinite(outs[1][0]).all()
    for o, l in outs[:2]:
        assert torch.equal(o, outs[2][0]) and torch.equal(l, outs[2][1])


@pytest.mark.gpu
@pytest.mark.parametrize("kind,causal,append", [("bf16", True, True), ("fp16", False, True), ("bf16", True, False)])
def test_fp8_varlen_equals_per_sequence_calls(tfa, kind, causal, append):
    """Mixed prefill and decode rows; out, lse and the pools equal one FP8 cache call per sequence, bit for bit."""
    seq_q = [3, 1, 200, 0, 1]
    lens = [300, 5, 129, 40, 0]
    B, Hq, Hkv, D, page, mbps = len(seq_q), 8, 2, 128, 128, 4
    dt = _dt(kind)
    _, kp, vp, table, sl = make_fp8_cache(lens, 1, Hq, Hkv, D, kind, page, seed=21, mbps=mbps)
    total = sum(seq_q)
    g = torch.Generator(device="cpu")
    g.manual_seed(6)
    q = torch.empty((total, Hq, D)).normal_(0, 0.5, generator=g).to(dt).cuda()
    kn = torch.empty((total, Hkv, D)).normal_(0, 0.5, generator=g).to(dt).cuda() if append else None
    vn = torch.empty((total, Hkv, D)).normal_(0, 0.5, generator=g).to(dt).cuda() if append else None
    cu = torch.tensor([0] + list(torch.tensor(seq_q).cumsum(0)), dtype=torch.int32, device="cuda")
    ks, vs = 0.05, 0.125
    k1, v1 = kp.clone(), vp.clone()
    out, lse = tfa.attn_varlen_kvcache_fwd(q, k1, v1, cu, max(seq_q), sl, table, kn, vn, is_causal=causal,
                                           k_scale=ks, v_scale=vs)
    k2, v2 = kp.clone(), vp.clone()
    for b, n in enumerate(seq_q):
        if n == 0:
            continue
        r0 = int(cu[b])
        qb = q[r0:r0 + n][None]
        kw = dict(k_new=kn[r0:r0 + n][None], v_new=vn[r0:r0 + n][None]) if append else {}
        ob, lb = tfa.attn_kvcache_fwd(qb, k2, v2, sl[b:b + 1], table[b:b + 1], is_causal=causal, k_scale=ks,
                                      v_scale=vs, **kw)
        assert torch.equal(out[r0:r0 + n], ob[0]), b
        assert torch.equal(lse[:, r0:r0 + n], lb[0]), b
    torch.cuda.synchronize()
    assert torch.equal(bits(k1), bits(k2)) and torch.equal(bits(v1), bits(v2))


@pytest.mark.gpu
def test_fp8_classic_and_persistent_agree_bitwise(tfa):
    code = r'''
import os, sys, torch
sys.path.insert(0, os.path.join(os.environ["TFA_ROOT"], "tiny-flash-attention_b200"))
sys.path.insert(0, os.path.join(os.environ["TFA_ROOT"], "tests"))
import tfa_ctypes as tfa
from test_kvcache_fp8 import make_fp8_cache
lens = [1000, 0, 129, 2049, 64, 300]
res = []
for causal, Sq, ns in ((True, 1, 1), (False, 4, 1), (True, 200, 1), (False, 1, 3)):
    q, kp, vp, table, sl = make_fp8_cache(lens, Sq, 8, 2, 128, "bf16", 256, seed=9, fill=0x7f)
    o, lse = tfa.attn_kvcache_fwd(q, kp, vp, sl, table, is_causal=causal, num_splits=ns, k_scale=0.1, v_scale=0.7)
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
def test_fp8_cuda_graph_replays_with_new_lengths_and_table(tfa):
    lens1, lens2 = [300, 5, 1000, 129], [1000, 700, 0, 256]
    B, Hq, Hkv, D, page, mbps = 4, 8, 2, 128, 256, 5
    q, kp, vp, table, sl = make_fp8_cache(lens1, 1, Hq, Hkv, D, "bf16", page, seed=13, mbps=mbps)
    k0, v0 = kp.clone(), vp.clone()
    g = torch.Generator(device="cpu")
    g.manual_seed(5)
    kn = torch.empty((B, 1, Hkv, D)).normal_(0, 0.5, generator=g).to(torch.bfloat16).cuda()
    vn = torch.empty((B, 1, Hkv, D)).normal_(0, 0.5, generator=g).to(torch.bfloat16).cuda()
    out = torch.empty_like(q)
    lse = torch.empty((B, Hq, 1), dtype=torch.float32, device="cuda")
    kw = dict(is_causal=True, num_splits=3, k_scale=0.01, v_scale=0.02)
    step = lambda: tfa.attn_kvcache_fwd(q, kp, vp, sl, table, kn, vn, out=out, lse=lse, **kw)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        step()
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        step()
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
        kc, vc = k0.clone(), v0.clone()
        want_o, want_l = tfa.attn_kvcache_fwd(q, kc, vc, sl.clone(), table.clone(), kn, vn, **kw)
        torch.cuda.synchronize()
        assert torch.equal(out, want_o) and torch.equal(lse, want_l)
        assert torch.equal(bits(kp), bits(kc)) and torch.equal(bits(vp), bits(vc))
        results.append(out.clone())
    assert not torch.equal(results[0], results[1])


@pytest.mark.gpu
def test_fp8_launch_counts_and_guard_regions(tfa):
    q, kp, vp, table, sl = make_fp8_cache([500, 0, 64, 129], 1, 4, 2, 64, "fp16", 128, seed=1, mbps=5)
    kn = torch.zeros((4, 1, 2, 64), dtype=torch.float16, device="cuda")
    cos = torch.ones((5 * 128, 16), dtype=torch.float16, device="cuda")
    rot = dict(k_new=kn, v_new=kn, rotary_cos=cos, rotary_sin=cos)
    for kw, want in ((dict(), 1), (dict(k_new=kn, v_new=kn), 2), (dict(num_splits=3), 2),
                     (dict(k_new=kn, v_new=kn, num_splits=3), 3), (rot, 2), (dict(rot, num_splits=3), 3)):
        n0 = tfa.launch_count()
        tfa.attn_kvcache_fwd(q, kp, vp, sl, table, is_causal=True, k_scale=0.5, v_scale=0.5, **kw)
        assert tfa.launch_count() - n0 == want, kw
    # a 16-bit cache takes no scales
    k16 = kp.to(torch.float16)
    with pytest.raises(ValueError, match="float8_e4m3fn"):
        tfa.attn_kvcache_fwd(q, k16, k16, sl, table, is_causal=True, k_scale=0.5)
    with pytest.raises(ValueError, match="float8_e4m3fn"):
        tfa.attn_varlen_kvcache_fwd(q[:, 0].contiguous(), k16, k16, torch.tensor([0, 1, 2, 3, 4], dtype=torch.int32,
                                    device="cuda"), 1, sl, table, v_scale=2.0)
    # guard regions: out and lse inside larger sentinel buffers
    big = torch.full((6, *q.shape[1:]), 7.0, dtype=q.dtype, device="cuda")
    lbig = torch.full((6, 4, 1), 7.0, dtype=torch.float32, device="cuda")
    for ns in (1, 3):
        o, l = tfa.attn_kvcache_fwd(q, kp, vp, sl, table, is_causal=True, num_splits=ns, k_scale=0.5, v_scale=0.5,
                                    out=big[1:5], lse=lbig[1:5])
        torch.cuda.synchronize()
        assert torch.all(big[0] == 7) and torch.all(big[5] == 7) and torch.all(lbig[0] == 7) and torch.all(lbig[5] == 7)
    n0 = tfa.launch_count()
    cu = torch.tensor([0, 1, 1, 2, 3], dtype=torch.int32, device="cuda")
    qv = q[:, 0].contiguous()
    tfa.attn_varlen_kvcache_fwd(qv, kp, vp, cu, 1, sl, table, kn[:, 0][:3], kn[:, 0][:3], k_scale=0.5, v_scale=0.5)
    assert tfa.launch_count() - n0 == 2
    torch.cuda.synchronize()


@pytest.mark.gpu
def test_extension_fp8_entries(built, tfa):
    import attention_cutlass as ac
    lens = [300, 1, 0, 640]
    q, kp, vp, table, sl = make_fp8_cache(lens, 2, 8, 2, 128, "bf16", 256, seed=17, fill=0xff, mbps=4)
    scale, ks, vs = 128 ** -0.5, 0.03, 0.6
    out, lse = ac.flash_attention_v2_kvcache_fp8(q, kp, vp, sl, table, None, None, ks, vs, True, scale, 1)
    want, wl = tfa.attn_kvcache_fwd(q, kp, vp, sl, table, is_causal=True, scale=scale, k_scale=ks, v_scale=vs)
    torch.cuda.synchronize()
    assert out.shape == q.shape and out.dtype == torch.bfloat16 and lse.shape == (4, 8, 2)
    assert torch.equal(out, want) and torch.equal(lse, wl)
    cu = torch.tensor([0, 2, 3, 3, 5], dtype=torch.int32, device="cuda")
    qv = q.reshape(8, 8, 128)[:5].contiguous()
    o2, l2 = ac.flash_attention_v2_varlen_kvcache_fp8(qv, kp, vp, cu, 2, sl, table, None, None, ks, vs, True, scale)
    w2, wl2 = tfa.attn_varlen_kvcache_fwd(qv, kp, vp, cu, 2, sl, table, is_causal=True, scale=scale, k_scale=ks,
                                          v_scale=vs)
    torch.cuda.synchronize()
    assert torch.equal(o2, w2) and torch.equal(l2, wl2)
    # the 16-bit entry points keep rejecting an FP8 cache, the FP8 ones a 16-bit cache
    with pytest.raises(RuntimeError, match="same dtype"):
        ac.flash_attention_v2_kvcache(q, kp, vp, sl, table, None, None, True, scale, 1)
    with pytest.raises(RuntimeError, match="float8_e4m3fn"):
        ac.flash_attention_v2_kvcache_fp8(q, kp.to(torch.bfloat16), vp.to(torch.bfloat16), sl, table, None, None, ks,
                                          vs, True, scale, 1)
    with pytest.raises(RuntimeError, match="float8_e4m3fn"):
        ac.flash_attention_v2_varlen_kvcache_fp8(qv, kp.view(torch.uint8), vp.view(torch.uint8), cu, 2, sl, table,
                                                 None, None, ks, vs, True, scale)
    with pytest.raises(RuntimeError, match="k_scale and v_scale"):
        ac.flash_attention_v2_kvcache_fp8(q, kp, vp, sl, table, None, None, 0.0, vs, True, scale, 1)
    with pytest.raises(RuntimeError, match="k_scale and v_scale"):
        ac.flash_attention_v2_varlen_kvcache_fp8(qv, kp, vp, cu, 2, sl, table, None, None, ks, float("inf"), True,
                                                 scale)
    with pytest.raises(RuntimeError, match="together"):
        ac.flash_attention_v2_kvcache_fp8(q, kp, vp, sl, table, None, None, ks, vs, True, scale, 1,
                                          rotary_cos=torch.ones((1024, 32), dtype=q.dtype, device="cuda"))
