"""e4m3 queries against an FP8 (e4m3) KV cache, both products on FP8 tensor cores: tfa_attn_kvcache_qkv8_fwd /
tfa_attn_varlen_kvcache_qkv8_fwd, attention_cutlass.flash_attention_v2_kvcache_qkv8 /
flash_attention_v2_varlen_kvcache_qkv8 and the float8 q routing of tfa_ctypes.attn_kvcache_fwd /
attn_varlen_kvcache_fwd.

CPU: the header declares both calls, the library exports them, the error string exists, every argument error comes back
before any device work in the documented order (ending in TFA_EARCH without a GPU), and the barrier-protocol model runs
the kDenseFp8 protocol on the cache modes' item lists and still catches the two misplaced converter steps there.
GPU: each sequence's out and lse equal tfa_attn_fp8_fwd() on that sequence alone (its q rows, its first K_b cached keys
gathered) bit for bit, for the dense-query and the varlen call; the appends leave the pools of tfa_attn_kvcache_fp8_fwd();
NaN codes in unused slots change nothing; split-KV, both schedules, CUDA-graph replay, launch counts, guard regions and
the bindings."""
import ctypes
import os
import random
import subprocess
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "tfa_b200.h")
sys.path.insert(0, os.path.join(ROOT, "scripts"))

TFA_EINVAL_QKVQUANT = -16
TFA_FP8_E4M3 = 2
FP8 = torch.float8_e4m3fn
CALLS = ("tfa_attn_kvcache_qkv8_fwd", "tfa_attn_varlen_kvcache_qkv8_fwd")


# ------------------------------------------------------------------ CPU ------------------------------------------------

def test_header_declares_and_library_exports_qkv8_calls(built):
    import tfa_ctypes
    from test_kvcache_fp8 import declared_functions
    src = open(HEADER).read()
    assert "int tfa_attn_kvcache_qkv8_fwd(const tfa_attn_kvcache_args* args, const tfa_qkv_quant_args* quant);" in src
    assert ("int tfa_attn_varlen_kvcache_qkv8_fwd(const tfa_attn_varlen_kvcache_args* args, "
            "const tfa_qkv_quant_args* quant);") in src
    assert "#define TFA_ABI_VERSION 2" in src
    names = declared_functions()
    L = ctypes.CDLL(tfa_ctypes.LIB_PATH)
    for fn in CALLS:
        assert fn in names and hasattr(L, fn)
    msg = tfa_ctypes.lib().tfa_error_string(TFA_EINVAL_QKVQUANT)
    assert msg.startswith(b"tfa:") and b"q_scale" in msg and b"16" in msg


def _buffers():
    buf = ctypes.create_string_buffer(4096 + 16)
    base = (ctypes.addressof(buf) + 15) & ~15
    return buf, base, base + 1024


def test_kvcache_qkv8_argument_checks_and_their_order(built):
    """Host buffers only: every code comes back before anything touches a device.  The cache checks first, then the
    16-bit call's (dtype = the output's), then the quantization, then s', then the device."""
    import tfa_ctypes
    L = tfa_ctypes.lib()
    buf, base, ints = _buffers()
    Hq, Hkv, D, page = 4, 2, 64, 256

    def mk(**kw):
        return tfa_ctypes.KvcacheArgs(
            kw.get("q", base), base, base, kw.get("k_new", None), kw.get("v_new", None), kw.get("out", base), None,
            kw.get("seqlens", ints), kw.get("table", ints), kw.get("B", 2), Hq, kw.get("Hkv", Hkv), 1,
            kw.get("D", D), 8, page, 4, 1, kw.get("qsb", Hq * D), kw.get("qss", Hq * D), kw.get("qsh", D),
            kw.get("ksb", page * Hkv * D), kw.get("kss", Hkv * D), kw.get("ksh", D), 4, Hkv * D, Hkv * D, D,
            kw.get("dtype", 0), 1, kw.get("scale", 0.1), kw.get("f32", 0), 1, None, 0, None)

    def call(**kw):
        quant = tfa_ctypes.QkvQuantArgs(kw.get("qdt", TFA_FP8_E4M3), kw.get("qs", 0.02), kw.get("ks", 0.5),
                                        kw.get("vs", 2.0))
        return L.tfa_attn_kvcache_qkv8_fwd(ctypes.byref(mk(**kw)), ctypes.byref(quant))

    assert L.tfa_attn_kvcache_qkv8_fwd(None, ctypes.byref(tfa_ctypes.QkvQuantArgs(2, 1.0, 1.0, 1.0))) == -1
    assert L.tfa_attn_kvcache_qkv8_fwd(ctypes.byref(mk()), None) == -1
    # the cache arguments first
    assert call(seqlens=None) == -13 and call(seqlens=None, D=96) == -13 and call(seqlens=None, qdt=0) == -13
    assert call(k_new=base) == -13
    # then the 16-bit call's checks; dtype is the output's (bf16 / fp16)
    assert call(q=None) == -1 and call(out=base + 8) == -1
    assert call(D=96) == -2 and call(B=0) == -3 and call(dtype=2) == -4
    assert call(qss=60) == -5 and call(kss=30) == -5
    assert call(scale=-1.0) == -9 and call(Hkv=3) == -10
    assert call(D=96, qdt=0) == -2 and call(dtype=2, qs=0.0) == -4
    # then the quantization: dtype code, scales, q and cache strides in multiples of 16
    E = TFA_EINVAL_QKVQUANT
    assert call(qdt=0) == E and call(qdt=1) == E and call(qdt=3) == E
    for bad in (0.0, -1.0, float("nan"), float("inf"), -float("inf")):
        assert call(qs=bad) == E and call(ks=bad) == E and call(vs=bad) == E, bad
    assert call(qss=Hq * D + 8) == E and call(qsh=D + 8) == E and call(qsb=Hq * D + 8) == E
    assert call(kss=Hkv * D + 8) == E and call(ksh=D + 8) == E and call(ksb=page * Hkv * D + 8) == E
    assert call(qdt=0, scale=1.0e38, qs=1.0, ks=10.0) == E
    # then s' = fp32(fp32(scale * q_scale) * k_scale): finite, and no underflow below FLT_MIN
    assert call(scale=1.0e38, qs=1.0, ks=10.0) == -9
    assert call(scale=1e-30, qs=1e-10, ks=1e-10) == -9 and call(scale=1e-20, qs=1.0, ks=1e-19) == -9
    if not torch.cuda.is_available():
        assert call() == -7 and call(f32=1) == -7


def test_varlen_kvcache_qkv8_argument_checks_and_their_order(built):
    import tfa_ctypes
    L = tfa_ctypes.lib()
    buf, base, ints = _buffers()
    Hq, Hkv, D, page = 4, 2, 64, 128

    def mk(**kw):
        return tfa_ctypes.VarlenKvcacheArgs(
            base, base, base, None, None, base, None, kw.get("cu", ints), kw.get("seqlens", ints), ints, 2, Hq, Hkv,
            kw.get("D", D), 8, kw.get("maxq", 4), 8, page, 4, kw.get("qss", Hq * D), D, page * Hkv * D,
            kw.get("kss", Hkv * D), D, 4, 0, 0, kw.get("dtype", 1), 1, kw.get("scale", 0.1), 0, None)

    def call(**kw):
        quant = tfa_ctypes.QkvQuantArgs(kw.get("qdt", TFA_FP8_E4M3), kw.get("qs", 0.5), kw.get("ks", 1.0),
                                        kw.get("vs", 1.0))
        return L.tfa_attn_varlen_kvcache_qkv8_fwd(ctypes.byref(mk(**kw)), ctypes.byref(quant))

    assert L.tfa_attn_varlen_kvcache_qkv8_fwd(None, None) == -1
    assert L.tfa_attn_varlen_kvcache_qkv8_fwd(ctypes.byref(mk()), None) == -1
    assert call(seqlens=None) == -13 and call(seqlens=None, cu=None) == -13
    assert call(D=96) == -2 and call(dtype=2) == -4 and call(D=96, cu=None) == -2
    assert call(cu=None) == -12 and call(maxq=9) == -12 and call(cu=None, qdt=1) == -12
    E = TFA_EINVAL_QKVQUANT
    assert call(qdt=1) == E and call(qs=0.0) == E and call(ks=float("nan")) == E and call(vs=-2.0) == E
    assert call(qss=Hq * D + 8) == E and call(kss=Hkv * D + 8) == E
    assert call(scale=1.0e38, qs=1.0, ks=10.0) == -9
    if not torch.cuda.is_available():
        assert call() == -7


def test_protocol_model_on_the_cache_items():
    """The kDenseFp8 protocol on kCacheQkv8 / kVarlenCacheQkv8 item lists: items skipped by every role, tile-less items
    whose rows are written, items whose last tile has keys past K_b; every depth combination of the generator."""
    import protocol_model as pm
    kinds = set()
    for trial in range(400):
        rng = random.Random(5150 + trial)
        items, empty, vtail, depths = pm.random_qkv8_cache_items(rng, varlen=trial % 2 == 1)
        kinds |= {"skipped" for i, n in enumerate(items) if n == 0 and i not in empty}
        kinds |= {"empty" for _ in empty} | {"tail" for _ in vtail}
        pm.DenseFp8Sim(items, *depths, rng, empty).run()
    assert kinds == {"skipped", "empty", "tail"}


MODEL_SRC = open(os.path.join(ROOT, "scripts", "protocol_model.py")).read()
WAIT_EMPTY = "                yield lambda s=vs, p=((tile // V) & 1) ^ 1: self.vt_empty[s].done(p)\n"
STORE = "                yield from self._store_vt(w, vs, rs, tag)\n"
ARRIVE = "                self.vt_full[vs].arrive()                     # after the last store (and its proxy fence)\n"


def _caught(old, new, trials=80):
    assert MODEL_SRC.count(old) == 1
    ns = {"__name__": "mutated_model"}
    exec(compile(MODEL_SRC.replace(old, new), "mutated_model", "exec"), ns)
    caught = 0
    for trial in range(trials):
        rng = random.Random(6262 + trial)
        items, empty, _, depths = ns["random_qkv8_cache_items"](rng, trial % 2 == 1)
        try:
            ns["DenseFp8Sim"](items, *depths, rng, empty).run()
        except AssertionError:
            caught += 1
    return caught


def test_protocol_model_catches_vt_full_before_the_last_store_on_cache_items():
    assert _caught(STORE + ARRIVE, ARRIVE + STORE) > 10


def test_protocol_model_catches_a_store_before_the_vt_empty_wait_on_cache_items():
    assert _caught(WAIT_EMPTY + STORE, STORE + WAIT_EMPTY) > 10


# ------------------------------------------------------------------ GPU ------------------------------------------------

@pytest.fixture(scope="module")
def tfa(built):
    import tfa_ctypes
    tfa_ctypes.lib()
    return tfa_ctypes


QS, KS, VS = 0.0213, 0.0171, 0.0119


def _dt(kind):
    return {"bf16": torch.bfloat16, "fp16": torch.float16, "f32": torch.bfloat16}[kind]


def bits(t):
    return t.view(torch.uint8) if t.element_size() == 1 else t.view(torch.int16 if t.element_size() == 2 else torch.int32)


def e4m3(g, scale, *shape):
    """N(0, 0.5^2) quantized as a caller would: (x / s).clamp(-448, 448).to(float8_e4m3fn)."""
    return (torch.empty(shape).normal_(0.0, 0.5, generator=g) / scale).clamp(-448, 448).to(FP8)


def make_pools(lens, Hkv, D, page, mbps, seed, fill=0x7F, contiguous=False, spare=3):
    """e4m3 pools whose first lens[b] keys of each sequence hold quantized normals and every other slot the byte
    `fill`; a permuted block table, or None for a contiguous (B, capacity) cache.  Returns (k, v, table, capacity)."""
    g = torch.Generator().manual_seed(seed)
    B = len(lens)
    if contiguous:
        mbps, page, nblk = 1, mbps * page if page else mbps, B
        perm = torch.arange(B, dtype=torch.int32).view(B, 1)
    else:
        nblk = B * mbps + spare
        perm = torch.randperm(nblk, generator=g)[:B * mbps].to(torch.int32).view(B, mbps)
    pools = []
    for s in (KS, VS):
        pool = torch.full((nblk, page, Hkv, D), fill, dtype=torch.uint8)
        for b in range(B):
            data = e4m3(g, s, mbps * page, Hkv, D).view(torch.uint8)
            data[max(lens[b], 0):] = fill
            pool[perm[b].long()] = data.view(mbps, page, Hkv, D)
        pools.append(pool.view(FP8).cuda())
    return pools[0], pools[1], None if contiguous else perm.cuda(), mbps * page


def gather(pool, table, b, K):
    """Keys [0, K) of sequence b as a contiguous (1, Hkv, K, D) tensor."""
    idx = torch.arange(K, device=pool.device)
    page = pool.shape[1]
    if table is None:
        rows = pool[b, :K]
    else:
        rows = pool[table[b].long()[idx // page], idx % page]
    return rows.permute(1, 0, 2)[None].contiguous()


def fp8_alone(tfa, qb, kp, vp, table, b, K, causal, scale, kind, num_splits=1):
    """tfa_attn_fp8_fwd on sequence b alone: qb (Sq, Hq, D) e4m3, its first K cached keys; (out (Sq, Hq, D), lse
    (Hq, Sq)), or out = 0 / lse = +inf without keys."""
    Sq, Hq, D = qb.shape
    odt = torch.float32 if kind == "f32" else _dt(kind)
    if K == 0:
        return (torch.zeros((Sq, Hq, D), dtype=odt, device="cuda"),
                torch.full((Hq, Sq), float("inf"), device="cuda"))
    o, l = tfa.attn_fwd(qb.permute(1, 0, 2)[None].contiguous(), gather(kp, table, b, K), gather(vp, table, b, K),
                        causal, scale, num_splits=num_splits, out_fp32=kind == "f32", q_scale=QS, k_scale=KS,
                        v_scale=VS, out_dtype=_dt(kind))
    return o[0].permute(1, 0, 2), l[0]


def cache_lens_dense(raw, cap, snew):
    L = min(max(raw, 0), cap - snew)
    return L + snew


def cache_lens_varlen(raw, cap, n, append):
    kept = min(n, cap) if append else 0
    L = min(max(raw, 0), cap - kept)
    return L + kept


DENSE = [
    # D, out kind, Hq, Hkv, page (None: contiguous), Sq, causal, Snew
    (128, "bf16", 32, 8, 256, 1, False, 0),
    (128, "bf16", 32, 8, 256, 1, True, 1),
    (128, "fp16", 8, 8, 128, 4, True, 4),
    (128, "f32", 8, 1, None, 129, True, 0),
    (64, "bf16", 8, 1, 128, 129, False, 3),
    (64, "fp16", 8, 8, None, 4, False, 1),
    (64, "f32", 32, 8, 256, 1, True, 0),
    (128, "fp16", 8, 1, 128, 129, True, 129),
    (64, "bf16", 32, 8, 128, 4, True, 0),
    (128, "f32", 8, 8, 128, 4, False, 2),
]


@pytest.mark.gpu
@pytest.mark.parametrize("D,kind,Hq,Hkv,page,Sq,causal,snew", DENSE)
def test_dense_query_call_equals_fp8_forward_per_sequence_bitwise(tfa, D, kind, Hq, Hkv, page, Sq, causal, snew):
    """Lengths 0, non-multiples of 128 and the full capacity; NaN codes in every slot past K_b."""
    mbps = 1000 if page is None else 1024 // page
    contiguous = page is None
    cap = 1000 if contiguous else 1024
    lens = [300, 0, cap, 1, 129, 77]
    kp, vp, table, cap = make_pools(lens, Hkv, D, page or 1, mbps, seed=40 + D + Sq, contiguous=contiguous)
    B = len(lens)
    g = torch.Generator().manual_seed(Sq + snew)
    q = e4m3(g, QS, B, Sq, Hq, D).cuda()
    kw = {}
    if snew:
        kw = dict(k_new=(torch.empty((B, snew, Hkv, D)).normal_(0, 0.5, generator=g)).to(_dt(kind)).cuda(),
                  v_new=(torch.empty((B, snew, Hkv, D)).normal_(0, 0.5, generator=g)).to(_dt(kind)).cuda())
    sl = torch.tensor(lens, dtype=torch.int32, device="cuda")
    scale = D ** -0.5
    out, lse = tfa.attn_kvcache_fwd(q, kp, vp, sl, table, is_causal=causal, scale=scale, out_fp32=kind == "f32",
                                    q_scale=QS, k_scale=KS, v_scale=VS, out_dtype=_dt(kind), **kw)
    assert out.dtype == (torch.float32 if kind == "f32" else _dt(kind)) and out.stride() == q.stride()
    for b in range(B):
        K = cache_lens_dense(lens[b], cap, snew)
        ob, lb = fp8_alone(tfa, q[b], kp, vp, table, b, K, causal, scale, kind)
        torch.cuda.synchronize()
        assert torch.equal(bits(out[b]), bits(ob.contiguous())), (b, K)
        assert torch.equal(bits(lse[b]), bits(lb)), (b, K)


def _varlen_case(seq_q, lens, Hq, Hkv, D, page, mbps, seed, kind, append):
    kp, vp, table, cap = make_pools(lens, Hkv, D, page, mbps, seed=seed)
    total = sum(seq_q)
    g = torch.Generator().manual_seed(seed + 1)
    q = e4m3(g, QS, total, Hq, D).cuda()
    kn = torch.empty((total, Hkv, D)).normal_(0, 0.5, generator=g).to(_dt(kind)).cuda() if append else None
    vn = torch.empty((total, Hkv, D)).normal_(0, 0.5, generator=g).to(_dt(kind)).cuda() if append else None
    starts = [0] + list(torch.tensor(seq_q).cumsum(0).tolist())
    return kp, vp, table, cap, q, kn, vn, starts


@pytest.mark.gpu
@pytest.mark.parametrize("kind,causal,append,D", [("bf16", True, True, 128), ("fp16", False, True, 64),
                                                  ("bf16", True, False, 128), ("f32", True, True, 128)])
def test_varlen_call_equals_fp8_forward_per_sequence_bitwise(tfa, kind, causal, append, D):
    """Mixed prefill chunks and decodes, a sequence with Sq_b = 0 and one whose end offset lies past total_q (clamped);
    the pools equal those of the varlen FP8-cache call with a 16-bit q."""
    seq_q = [3, 1, 200, 0, 1, 129]
    lens = [300, 5, 129, 40, 0, 1024]
    Hq, Hkv, page, mbps = 8, 2, 128, 8
    kp, vp, table, cap, q, kn, vn, starts = _varlen_case(seq_q, lens, Hq, Hkv, D, page, mbps, 50, kind, append)
    total = starts[-1]
    cu_list = starts[:-1] + [total + 50]                      # clamped to total_q by the kernels
    cu = torch.tensor(cu_list, dtype=torch.int32, device="cuda")
    sl = torch.tensor(lens, dtype=torch.int32, device="cuda")
    scale = D ** -0.5
    k1, v1 = kp.clone(), vp.clone()
    out, lse = tfa.attn_varlen_kvcache_fwd(q, k1, v1, cu, max(seq_q), sl, table, kn, vn, is_causal=causal, scale=scale,
                                           out_fp32=kind == "f32", q_scale=QS, k_scale=KS, v_scale=VS,
                                           out_dtype=_dt(kind))
    for b, n in enumerate(seq_q):
        if n == 0:
            continue
        r0 = starts[b]
        K = cache_lens_varlen(lens[b], cap, n, append)
        ob, lb = fp8_alone(tfa, q[r0:r0 + n], k1, v1, table, b, K, causal, scale, kind)
        torch.cuda.synchronize()
        assert torch.equal(bits(out[r0:r0 + n]), bits(ob.contiguous())), (b, K)
        assert torch.equal(bits(lse[:, r0:r0 + n].contiguous()), bits(lb)), (b, K)
    if append:
        k2, v2 = kp.clone(), vp.clone()
        q16 = torch.zeros((total, Hq, D), dtype=_dt(kind), device="cuda")
        tfa.attn_varlen_kvcache_fwd(q16, k2, v2, cu, max(seq_q), sl, table, kn, vn, is_causal=causal, k_scale=KS,
                                    v_scale=VS)
        torch.cuda.synchronize()
        assert torch.equal(bits(k1), bits(k2)) and torch.equal(bits(v1), bits(v2))


@pytest.mark.gpu
@pytest.mark.parametrize("kind,snew,page", [("bf16", 1, 128), ("fp16", 5, 256), ("bf16", 130, None)])
def test_append_leaves_the_fp8_cache_calls_pools(tfa, kind, snew, page):
    """Out-of-range table entries, negative and oversized cache_seqlens: the pools equal those after
    tfa_attn_kvcache_fp8_fwd with the same k_new / v_new / scales, and no slot outside the appended ones changes."""
    from test_kvcache_fp8 import _appended
    lens = [300, 0, 1000, 511, -4, 9999]
    B, Hq, Hkv, D, mbps = len(lens), 8, 2, 128, 4
    kp, vp, table, cap = make_pools([min(max(x, 0), 1000) for x in lens], Hkv, D, page or 256, mbps, seed=3,
                                    contiguous=page is None)
    nblk, pg = kp.shape[0], kp.shape[1]
    if table is not None:
        table[1, 0] = -1
        table[3, 1] = nblk + 5
    sl = torch.tensor(lens, dtype=torch.int32, device="cuda")
    g = torch.Generator().manual_seed(8)
    kn = (torch.empty((B, snew, Hkv, D)).normal_(0, 3.0, generator=g) * KS).to(_dt(kind)).cuda()
    vn = torch.flip(kn, dims=[0]).contiguous()
    q8 = e4m3(g, QS, B, 1, Hq, D).cuda()
    k0, v0 = kp.clone(), vp.clone()
    tfa.attn_kvcache_fwd(q8, kp, vp, sl, table, kn, vn, is_causal=True, q_scale=QS, k_scale=KS, v_scale=VS,
                         out_dtype=_dt(kind))
    k2, v2 = k0.clone(), v0.clone()
    tfa.attn_kvcache_fwd(q8.to(_dt(kind)), k2, v2, sl, table, kn, vn, is_causal=True, k_scale=KS, v_scale=VS)
    torch.cuda.synchronize()
    assert torch.equal(bits(kp), bits(k2)) and torch.equal(bits(vp), bits(v2))
    tab = table.cpu() if table is not None else None
    touched = torch.zeros(kp.shape[:2], dtype=torch.bool)
    for _, _, blk, row in _appended(tab, lens, snew, cap, pg, nblk):
        touched[blk, row] = True
    keep = ~touched.cuda()
    assert torch.equal(bits(kp)[keep], bits(k0)[keep]) and torch.equal(bits(vp)[keep], bits(v0)[keep])
    assert not torch.equal(bits(kp), bits(k0))


@pytest.mark.gpu
@pytest.mark.parametrize("D,kind,ns", [(128, "bf16", 1), (64, "fp16", 1), (128, "fp16", 4)])
def test_nan_codes_in_unused_slots_change_nothing(tfa, D, kind, ns):
    """0x7f / 0xff in every slot past K_b, the rest of the last page included, against zeros there."""
    lens = [300, 0, 129, 1000]
    g = torch.Generator().manual_seed(11)
    q = e4m3(g, QS, 4, 4, 8, D).cuda()
    qv = e4m3(g, QS, 7, 8, D).cuda()
    cu = torch.tensor([0, 3, 3, 4, 7], dtype=torch.int32, device="cuda")
    outs = []
    for fill in (0x7F, 0xFF, 0):
        kp, vp, table, _ = make_pools(lens, 2, D, 256, 4, seed=5, fill=fill)
        sl = torch.tensor(lens, dtype=torch.int32, device="cuda")
        kw = dict(q_scale=QS, k_scale=KS, v_scale=VS, out_dtype=_dt(kind))
        o, l = tfa.attn_kvcache_fwd(q, kp, vp, sl, table, is_causal=False, num_splits=ns, **kw)
        o2, l2 = tfa.attn_varlen_kvcache_fwd(qv, kp, vp, cu, 3, sl, table, is_causal=True, **kw)
        outs.append((o, l, o2, l2))
    torch.cuda.synchronize()
    for r in outs[:2]:
        assert torch.isfinite(r[0]).all() and torch.isfinite(r[2]).all()
        for a, b in zip(r, outs[2]):
            assert torch.equal(bits(a), bits(b))


@pytest.mark.gpu
@pytest.mark.parametrize("D,kind,causal", [(128, "bf16", False), (64, "fp16", True), (128, "f32", True)])
def test_split_kv(tfa, D, kind, causal):
    """Every K_b at the capacity: num_splits = 4 equals tfa_attn_fp8_fwd(num_splits = 4) bit for bit.  Ragged lengths:
    num_splits = 4 within the float64 budget of the FP8 forward."""
    from test_fwd_fp8 import compare, deq, fp8_reference
    Hq, Hkv, page, mbps, Sq = 8, 2, 256, 8, 4
    cap = page * mbps
    scale = D ** -0.5
    g = torch.Generator().manual_seed(D)
    for lens, exact in (([cap] * 3, True), ([1500, 0, 700, 129], False)):
        kp, vp, table, _ = make_pools(lens, Hkv, D, page, mbps, seed=60)
        B = len(lens)
        q = e4m3(g, QS, B, Sq, Hq, D).cuda()
        sl = torch.tensor(lens, dtype=torch.int32, device="cuda")
        out, lse, n = tfa.attn_kvcache_fwd(q, kp, vp, sl, table, is_causal=causal, scale=scale, num_splits=4,
                                           out_fp32=kind == "f32", return_splits=True, q_scale=QS, k_scale=KS,
                                           v_scale=VS, out_dtype=_dt(kind))
        assert n == 4
        for b, K in enumerate(lens):
            if exact:
                ob, lb = fp8_alone(tfa, q[b], kp, vp, table, b, K, causal, scale, kind, num_splits=4)
                torch.cuda.synchronize()
                assert torch.equal(bits(out[b]), bits(ob.contiguous())) and torch.equal(bits(lse[b]), bits(lb)), b
            elif K == 0:
                assert bool((out[b] == 0).all()) and bool(torch.isposinf(lse[b]).all())
            else:
                qd = deq(q[b].permute(1, 0, 2)[None], QS)
                ref = fp8_reference(qd, gather(kp, table, b, K), gather(vp, table, b, K), causal, scale, KS, VS)
                ok, r, le, msg = compare(out[b].permute(1, 0, 2)[None], lse[b][None], ref,
                                         "bf16" if kind == "f32" else kind)
                assert ok, (b, msg)


SCHEDULES = r'''
import os, sys, torch
sys.path.insert(0, os.path.join(os.environ["TFA_ROOT"], "tiny-flash-attention_b200"))
sys.path.insert(0, os.path.join(os.environ["TFA_ROOT"], "tests"))
import tfa_ctypes as tfa
from test_kvcache_qkv8 import QS, KS, VS, e4m3, make_pools
lens = [1000, 0, 129, 2047, 64, 300]
res = []
g = torch.Generator().manual_seed(9)
for causal, Sq, ns in ((True, 1, 1), (False, 4, 1), (True, 200, 1), (False, 1, 3)):
    kp, vp, table, _ = make_pools(lens, 2, 128, 256, 8, seed=9)
    q = e4m3(g, QS, len(lens), Sq, 8, 128).cuda()
    sl = torch.tensor(lens, dtype=torch.int32, device="cuda")
    o, l = tfa.attn_kvcache_fwd(q, kp, vp, sl, table, is_causal=causal, num_splits=ns, q_scale=QS, k_scale=KS,
                                v_scale=VS, out_dtype=torch.bfloat16)
    res.append((o.cpu(), l.cpu(), tfa.lib().tfa_internal_last_variant()))
qv = e4m3(g, QS, 300, 8, 128).cuda()
cu = torch.tensor([0, 1, 1, 201, 202, 203, 300], dtype=torch.int32, device="cuda")
o, l = tfa.attn_varlen_kvcache_fwd(qv, kp, vp, cu, 200, sl, table, is_causal=True, q_scale=QS, k_scale=KS, v_scale=VS,
                                   out_dtype=torch.float16)
res.append((o.cpu(), l.cpu(), tfa.lib().tfa_internal_last_variant()))
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
    for (a, la, va), (b, lb, vb) in zip(outs["classic"], outs["persist"]):
        assert (va, vb) == (0, 4)
        assert torch.equal(bits(a), bits(b)) and torch.equal(bits(la), bits(lb))


@pytest.mark.gpu
def test_cuda_graph_replays_with_new_lengths_and_table(tfa):
    lens1, lens2 = [300, 5, 1000, 129], [1000, 700, 0, 256]
    B, Hq, Hkv, D, page, mbps = 4, 8, 2, 128, 256, 5
    kp, vp, table, _ = make_pools(lens1, Hkv, D, page, mbps, seed=13)
    k0, v0 = kp.clone(), vp.clone()
    g = torch.Generator().manual_seed(5)
    q = e4m3(g, QS, B, 1, Hq, D).cuda()
    kn = torch.empty((B, 1, Hkv, D)).normal_(0, 0.5, generator=g).to(torch.bfloat16).cuda()
    vn = torch.empty((B, 1, Hkv, D)).normal_(0, 0.5, generator=g).to(torch.bfloat16).cuda()
    sl = torch.tensor(lens1, dtype=torch.int32, device="cuda")
    out = torch.empty(q.shape, dtype=torch.bfloat16, device="cuda")
    lse = torch.empty((B, Hq, 1), dtype=torch.float32, device="cuda")
    kw = dict(is_causal=True, num_splits=3, q_scale=QS, k_scale=KS, v_scale=VS, out_dtype=torch.bfloat16)
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
            gp = torch.Generator().manual_seed(perm_seed)
            sl.copy_(torch.tensor(lens, dtype=torch.int32))
            table.copy_(torch.randperm(kp.shape[0], generator=gp)[:B * mbps].to(torch.int32).view(B, mbps))
        kp.copy_(k0)
        vp.copy_(v0)
        graph.replay()
        kc, vc = k0.clone(), v0.clone()
        want_o, want_l = tfa.attn_kvcache_fwd(q, kc, vc, sl.clone(), table.clone(), kn, vn, **kw)
        torch.cuda.synchronize()
        assert torch.equal(bits(out), bits(want_o)) and torch.equal(lse, want_l)
        assert torch.equal(bits(kp), bits(kc)) and torch.equal(bits(vp), bits(vc))
        results.append(out.clone())
    assert not torch.equal(results[0], results[1])


@pytest.mark.gpu
def test_launch_counts_guard_regions_and_routing(tfa):
    B, Hq, Hkv, D = 4, 4, 2, 64
    kp, vp, table, _ = make_pools([500, 0, 64, 129], Hkv, D, 128, 5, seed=1)
    g = torch.Generator().manual_seed(2)
    q = e4m3(g, QS, B, 1, Hq, D).cuda()
    sl = torch.tensor([500, 0, 64, 129], dtype=torch.int32, device="cuda")
    kn = torch.zeros((B, 1, Hkv, D), dtype=torch.float16, device="cuda")
    kw = dict(is_causal=True, q_scale=QS, k_scale=KS, v_scale=VS, out_dtype=torch.float16)
    for extra, want in ((dict(), 1), (dict(k_new=kn, v_new=kn), 2), (dict(num_splits=3), 2),
                        (dict(k_new=kn, v_new=kn, num_splits=3), 3)):
        n0 = tfa.launch_count()
        tfa.attn_kvcache_fwd(q, kp, vp, sl, table, **kw, **extra)
        assert tfa.launch_count() - n0 == want, extra
    cu = torch.tensor([0, 1, 1, 2, 3], dtype=torch.int32, device="cuda")
    qv = q[:, 0].contiguous()
    for extra, want in ((dict(), 1), (dict(k_new=kn[:, 0][:3], v_new=kn[:, 0][:3]), 2)):
        n0 = tfa.launch_count()
        tfa.attn_varlen_kvcache_fwd(qv[:3], kp, vp, cu, 1, sl, table, **kw, **extra)
        assert tfa.launch_count() - n0 == want, extra
    # guard regions around out, lse and the pools
    big = torch.full((6, *q.shape[1:]), 7.0, dtype=torch.float16, device="cuda")
    lbig = torch.full((6, Hq, 1), 7.0, dtype=torch.float32, device="cuda")
    pk = torch.full((kp.shape[0] + 2, *kp.shape[1:]), 0x5A, dtype=torch.uint8, device="cuda")
    pv = pk.clone()
    pk[1:-1] = kp.view(torch.uint8)
    pv[1:-1] = vp.view(torch.uint8)
    for ns in (1, 3):
        tfa.attn_kvcache_fwd(q, pk[1:-1].view(FP8), pv[1:-1].view(FP8), sl, table, kn, kn, num_splits=ns,
                             out=big[1:5], lse=lbig[1:5], **kw)
        torch.cuda.synchronize()
        assert torch.all(big[0] == 7) and torch.all(big[5] == 7) and torch.all(lbig[0] == 7) and torch.all(lbig[5] == 7)
        for p in (pk, pv):
            assert torch.all(p[0] == 0x5A) and torch.all(p[-1] == 0x5A)
    ov = torch.full((5, Hq, D), 7.0, dtype=torch.float16, device="cuda")
    lv = torch.full((Hq * 3 + 2,), 7.0, dtype=torch.float32, device="cuda")
    tfa.attn_varlen_kvcache_fwd(qv[:3], kp, vp, cu, 1, sl, table, out=ov[1:4], lse=lv[1:-1].view(Hq, 3), **kw)
    torch.cuda.synchronize()
    assert torch.all(ov[0] == 7) and torch.all(ov[4] == 7) and lv[0] == 7 and lv[-1] == 7
    # routing errors: a float8 q needs a float8 cache, takes no rotary, and k_new in out_dtype
    k16 = kp.to(torch.float16)
    with pytest.raises(TypeError, match="float8_e4m3fn cache"):
        tfa.attn_kvcache_fwd(q, k16, k16, sl, table, **kw)
    with pytest.raises(TypeError, match="float8_e4m3fn cache"):
        tfa.attn_varlen_kvcache_fwd(qv[:3], k16, k16, cu, 1, sl, table, **kw)
    cos = torch.ones((5 * 128, 16), dtype=torch.float16, device="cuda")
    with pytest.raises(ValueError, match="rotary"):
        tfa.attn_kvcache_fwd(q, kp, vp, sl, table, kn, kn, rotary_cos=cos, rotary_sin=cos, **kw)
    with pytest.raises(ValueError, match="rotary"):
        tfa.attn_varlen_kvcache_fwd(qv[:3], kp, vp, cu, 1, sl, table, kn[:, 0][:3], kn[:, 0][:3], rotary_cos=cos,
                                    rotary_sin=cos, **kw)
    with pytest.raises(TypeError, match="out_dtype"):
        tfa.attn_kvcache_fwd(q, kp, vp, sl, table, kn.bfloat16(), kn.bfloat16(), **kw)
    with pytest.raises(ValueError, match="float8_e4m3fn q"):
        tfa.attn_kvcache_fwd(q.to(torch.float16), kp, vp, sl, table, is_causal=True, q_scale=0.5, k_scale=KS)


@pytest.mark.gpu
def test_extension_entries_equal_the_c_calls(built, tfa):
    import attention_cutlass as ac
    lens = [300, 1, 0, 640]
    B, Sq, Hq, Hkv, D = 4, 2, 8, 2, 128
    kp, vp, table, _ = make_pools(lens, Hkv, D, 256, 4, seed=17, fill=0xFF)
    g = torch.Generator().manual_seed(17)
    q = e4m3(g, QS, B, Sq, Hq, D).cuda()
    kn = torch.empty((B, Sq, Hkv, D)).normal_(0, 0.5, generator=g).to(torch.float16).cuda()
    sl = torch.tensor(lens, dtype=torch.int32, device="cuda")
    scale = 128 ** -0.5
    k1, v1, k2, v2 = kp.clone(), vp.clone(), kp.clone(), vp.clone()
    out, lse = ac.flash_attention_v2_kvcache_qkv8(q, k1, v1, sl, table, kn, kn, QS, KS, VS, True, scale, 1,
                                                  torch.float16)
    want, wl = tfa.attn_kvcache_fwd(q, k2, v2, sl, table, kn, kn, is_causal=True, scale=scale, q_scale=QS, k_scale=KS,
                                    v_scale=VS, out_dtype=torch.float16)
    torch.cuda.synchronize()
    assert out.shape == q.shape and out.dtype == torch.float16 and lse.shape == (B, Hq, Sq)
    assert torch.equal(bits(out), bits(want)) and torch.equal(lse, wl)
    assert torch.equal(bits(k1), bits(k2)) and torch.equal(bits(v1), bits(v2))
    o0, l0 = ac.flash_attention_v2_kvcache_qkv8(q, k1, v1, sl, table, None, None, QS, KS, VS, False, scale, 0,
                                                torch.bfloat16)
    w0, wl0 = tfa.attn_kvcache_fwd(q, k1, v1, sl, table, is_causal=False, scale=scale, num_splits=0, q_scale=QS,
                                   k_scale=KS, v_scale=VS, out_dtype=torch.bfloat16)
    torch.cuda.synchronize()
    assert torch.equal(bits(o0), bits(w0)) and torch.equal(l0, wl0)
    cu = torch.tensor([0, 2, 3, 3, 5], dtype=torch.int32, device="cuda")
    qv = q.reshape(B * Sq, Hq, D)[:5].contiguous()
    knv = kn.reshape(B * Sq, Hkv, D)[:5].contiguous()
    o2, l2 = ac.flash_attention_v2_varlen_kvcache_qkv8(qv, k1, v1, cu, 2, sl, table, knv, knv, QS, KS, VS, True, scale,
                                                       torch.float16)
    w2, wl2 = tfa.attn_varlen_kvcache_fwd(qv, k2, v2, cu, 2, sl, table, knv, knv, is_causal=True, scale=scale,
                                          q_scale=QS, k_scale=KS, v_scale=VS, out_dtype=torch.float16)
    torch.cuda.synchronize()
    assert o2.dtype == torch.float16 and torch.equal(bits(o2), bits(w2)) and torch.equal(l2, wl2)
    assert torch.equal(bits(k1), bits(k2)) and torch.equal(bits(v1), bits(v2))
    with pytest.raises(RuntimeError, match="float8_e4m3fn"):
        ac.flash_attention_v2_kvcache_qkv8(q, kp.to(torch.bfloat16), vp.to(torch.bfloat16), sl, table, None, None, QS,
                                           KS, VS, True, scale, 1, torch.bfloat16)
    with pytest.raises(RuntimeError, match="out_dtype"):
        ac.flash_attention_v2_kvcache_qkv8(q, kp, vp, sl, table, None, None, QS, KS, VS, True, scale, 1, torch.float32)
    with pytest.raises(RuntimeError, match="out_dtype"):
        ac.flash_attention_v2_kvcache_qkv8(q, kp, vp, sl, table, kn, kn, QS, KS, VS, True, scale, 1, torch.bfloat16)
    with pytest.raises(RuntimeError, match="q_scale, k_scale and v_scale"):
        ac.flash_attention_v2_varlen_kvcache_qkv8(qv, kp, vp, cu, 2, sl, table, None, None, 0.0, KS, VS, True, scale,
                                                  torch.float16)
