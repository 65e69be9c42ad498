"""The FP8 variable-length forward: tfa_attn_varlen_fp8_fwd / attention_cutlass.flash_attention_v2_varlen_fp8 -- packed
e4m3 q, k and v addressed through cu_seqlens, both products on e4m3 wgmma.

CPU: the entry point is declared and exported, every argument error comes back before any device work in the documented
order, the extension rejects wrong element types and devices, and the barrier-protocol model accepts packed items
without tiles.
GPU: each packed sequence equals tfa_attn_fp8_fwd on that sequence alone bit for bit, and a seeded mix is within the
float64 budget of tests/test_fwd_fp8.py; NaN codes in the neighbouring sequences' K and V change nothing; exactly the
rows of every sequence are written; both schedules agree; the call is one launch and replays from a CUDA graph with new
lengths; the extension and ctypes entry points agree."""
import ctypes
import os
import random
import subprocess
import sys
import tempfile

import numpy as np
import pytest
import torch

from test_fwd_fp8 import _dt, compare, deq, fp8_reference
from test_kvcache_fp8 import FP8, bits
from test_varlen import declared_functions, offsets

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SCALES = (0.0213, 0.0171, 0.0119)
TFA_EINVAL_SEQLENS, TFA_EINVAL_QKVQUANT, TFA_EINVAL_SCALE = -12, -16, -9


# ------------------------------------------------------------------ CPU ------------------------------------------------

@pytest.fixture(scope="module")
def tfa(built):
    import tfa_ctypes
    tfa_ctypes.lib()
    return tfa_ctypes


def test_header_declares_and_library_exports_varlen_fp8(tfa):
    src = open(os.path.join(ROOT, "include", "tfa_b200.h")).read()
    assert "tfa_attn_varlen_fp8_fwd" in declared_functions()
    assert "int tfa_attn_varlen_fp8_fwd(const tfa_attn_varlen_args* args, const tfa_qkv_quant_args* quant);" in src
    assert "#define TFA_ABI_VERSION 2" in src
    assert hasattr(ctypes.CDLL(tfa.LIB_PATH), "tfa_attn_varlen_fp8_fwd")


def test_varlen_fp8_argument_checks_and_their_order(tfa):
    """Host buffers only: every code must come back before anything touches a device.  tfa_attn_varlen_fwd's checks
    in its order, then TFA_EINVAL_QKVQUANT, then TFA_EINVAL_SCALE for s'."""
    L = tfa.lib()
    buf = ctypes.create_string_buffer(4096 + 16)
    base = (ctypes.addressof(buf) + 15) & ~15
    cu = base + 1024
    Hq, Hkv, D = 4, 2, 64
    nan, inf = float("nan"), float("inf")

    def call(qkw=None, **kw):
        a = tfa.VarlenArgs(
            kw.get("q", base), base, base, base, None, kw.get("cu_q", cu), kw.get("cu_k", cu), 2, Hq, Hkv,
            kw.get("D", D), 300, 400, kw.get("max_q", 200), kw.get("qss", Hq * D), D, kw.get("kss", Hkv * D), D,
            kw.get("dtype", 0), 1, kw.get("scale", 0.125), 0, None)
        qd = dict(qkv_dtype=2, q_scale=0.02, k_scale=0.03, v_scale=0.01)
        qd.update(qkw or {})
        quant = tfa.QkvQuantArgs(qd["qkv_dtype"], qd["q_scale"], qd["k_scale"], qd["v_scale"])
        return L.tfa_attn_varlen_fp8_fwd(ctypes.byref(a), ctypes.byref(quant))

    assert L.tfa_attn_varlen_fp8_fwd(None, None) == -1
    cases = [
        (dict(q=None), {}, -1), (dict(D=96), {}, -2), (dict(dtype=2), {}, -4), (dict(qss=260), {}, -5),
        (dict(scale=nan), {}, -9),
        (dict(cu_q=None), {}, TFA_EINVAL_SEQLENS), (dict(cu_k=None), {}, TFA_EINVAL_SEQLENS),
        (dict(cu_q=cu + 2), {}, TFA_EINVAL_SEQLENS), (dict(cu_k=cu + 1), {}, TFA_EINVAL_SEQLENS),
        (dict(max_q=0), {}, TFA_EINVAL_SEQLENS), (dict(max_q=301), {}, TFA_EINVAL_SEQLENS),
        # the quantization's checks: strides that are multiples of 8 but not of 16, scales, the element type
        (dict(kss=Hkv * D + 8), {}, TFA_EINVAL_QKVQUANT), (dict(qss=Hq * D + 8), {}, TFA_EINVAL_QKVQUANT),
        ({}, dict(q_scale=0.0), TFA_EINVAL_QKVQUANT), ({}, dict(k_scale=nan), TFA_EINVAL_QKVQUANT),
        ({}, dict(v_scale=inf), TFA_EINVAL_QKVQUANT), ({}, dict(qkv_dtype=0), TFA_EINVAL_QKVQUANT),
        # s' = fp32(fp32(softmax_scale q_scale) k_scale) overflows, or underflows below FLT_MIN
        (dict(scale=1e30), dict(q_scale=1e10, k_scale=1.0), TFA_EINVAL_SCALE),
        (dict(scale=1e-20), dict(q_scale=1e-10, k_scale=1e-10), TFA_EINVAL_SCALE),
        # order
        (dict(D=96, cu_q=None), dict(q_scale=0.0), -2),
        (dict(cu_q=None), dict(q_scale=0.0), TFA_EINVAL_SEQLENS),
        (dict(max_q=0, kss=Hkv * D + 8), {}, TFA_EINVAL_SEQLENS),
        (dict(scale=1e30, kss=Hkv * D + 8), dict(q_scale=1e10), TFA_EINVAL_QKVQUANT),
        (dict(scale=1e30), dict(q_scale=1e10, v_scale=0.0), TFA_EINVAL_QKVQUANT),
    ]
    for kw, qkw, want in cases:
        got = call(qkw, **kw)
        assert got == want, (kw, qkw, got, want)


def test_extension_rejects_wrong_types_and_devices(built):
    """Checked before any device work, so this runs without a GPU: 16-bit q, an output dtype that is not 16-bit, and
    q / k / v on different devices each raise RuntimeError."""
    import attention_cutlass as ac
    dev = "cuda" if torch.cuda.is_available() else "cpu"
    q8 = torch.zeros((64, 2, 64), dtype=FP8, device=dev)
    cu = torch.tensor([0, 64], dtype=torch.int32, device=dev)
    args = lambda q, k, v, od: (q, k, v, cu, cu, 64, *SCALES, True, 0.125, od)
    with pytest.raises(RuntimeError, match="float8_e4m3fn"):
        ac.flash_attention_v2_varlen_fp8(*args(q8.to(torch.bfloat16), q8, q8, torch.bfloat16))
    with pytest.raises(RuntimeError, match="float8_e4m3fn"):
        ac.flash_attention_v2_varlen_fp8(*args(q8, q8.to(torch.float16), q8, torch.float16))
    for od in (torch.float32, FP8, torch.float8_e5m2):
        with pytest.raises(RuntimeError, match="out_dtype"):
            ac.flash_attention_v2_varlen_fp8(*args(q8, q8, q8, od))
    other = torch.zeros((64, 2, 64), dtype=FP8, device="meta")
    with pytest.raises(RuntimeError, match="same device"):
        ac.flash_attention_v2_varlen_fp8(*args(q8, other, q8, torch.bfloat16))
    with pytest.raises(RuntimeError, match="same device"):
        ac.flash_attention_v2_varlen_fp8(*args(q8, q8, other, torch.bfloat16))


def test_protocol_model_runs_packed_fp8_items():
    """kVarlenFp8 items in DenseFp8Sim: items past a sequence's end (skipped by every role), items inside it without a
    key (written, no barrier) and items with tiles, at every ring-depth combination random_varlen_fp8 draws."""
    sys.path.insert(0, os.path.join(ROOT, "scripts"))
    import protocol_model as pm
    for trial in range(400):
        rng = random.Random(31337 + trial)
        items, empty, depths = pm.random_varlen_fp8(rng)
        pm.DenseFp8Sim(items, *depths, rng, empty).run()
    pm.DenseFp8Sim([0, 3, 0, 0, 2, 0], 2, 1, 1, random.Random(3), empty=[2, 5]).run()


# ------------------------------------------------------------------ GPU ------------------------------------------------

EDGES = [0, 1, 63, 64, 127, 128, 129, 255, 257]


def make_fp8_batch(lq, lk, Hq, Hkv, D, seed):
    """Packed e4m3 q (sum lq, Hq, D), k / v (sum lk, Hkv, D), quantized from N(0, 0.5^2) as a caller would, and their
    int32 cu_seqlens, on the GPU."""
    g = torch.Generator().manual_seed(seed)
    mk = lambda s, *shape: (torch.empty(shape).normal_(0.0, 0.5, generator=g) / s).clamp(-448, 448).to(FP8).cuda()
    q, k, v = mk(SCALES[0], sum(lq), Hq, D), mk(SCALES[1], sum(lk), Hkv, D), mk(SCALES[2], sum(lk), Hkv, D)
    cu = lambda ls: torch.tensor(np.concatenate([[0], np.cumsum(ls)]), dtype=torch.int32, device="cuda")
    return q, k, v, cu(lq), cu(lk)


def seq(x, c0, c1):
    """Rows [c0, c1) of a packed (total, H, D) tensor as a contiguous (1, H, S, D) one (a view-free copy of the codes)."""
    return x[c0:c1].permute(1, 0, 2).unsqueeze(0).contiguous()


def varlen(tfa, q, k, v, cu_q, cu_k, max_q, causal, kind, f32=False, **kw):
    return tfa.attn_varlen_fwd(q, k, v, cu_q, cu_k, max_q, causal, q.shape[-1] ** -0.5, out_fp32=f32,
                               q_scale=SCALES[0], k_scale=SCALES[1], v_scale=SCALES[2], out_dtype=_dt(kind), **kw)


BITWISE = [
    # causal, D, kind, Hq, Hkv, keys: "same" Sk_b = Sq_b, "more" Sk_b > Sq_b, "fewer" Sk_b < Sq_b (causal: key-less rows)
    (True, 128, "bf16", 4, 4, "more"),
    (True, 64, "fp16", 8, 2, "fewer"),
    (False, 128, "fp16", 8, 2, "same"),
    (False, 64, "bf16", 2, 2, "more"),
    (True, 128, "bf16", 8, 2, "fewer"),
    (True, 64, "bf16", 4, 1, "same"),
]


def _keys(lq, keys, rng):
    if keys == "same":
        return lq[:]
    if keys == "more":
        return [s + rng.choice([1, 63, 64, 129, 300]) for s in lq]
    return [max(0, s - rng.choice([1, 64, 100, 200])) for s in lq]


@pytest.mark.gpu
@pytest.mark.parametrize("causal,D,kind,Hq,Hkv,keys", BITWISE)
def test_varlen_fp8_equals_per_sequence_fp8_bitwise(tfa, causal, D, kind, Hq, Hkv, keys):
    """Every packed sequence's out and lse equal tfa_attn_fp8_fwd on that sequence alone (num_splits = 1), bit for bit,
    in 16-bit and fp32 output; sequences with no key are 0 / +inf."""
    rng = random.Random(D + Hq + int(causal))
    lq = EDGES[:]
    rng.shuffle(lq)
    lk = _keys(lq, keys, rng)
    q, k, v, cu_q, cu_k = make_fp8_batch(lq, lk, Hq, Hkv, D, seed=20 + D)
    for f32 in (False, True):
        out, lse = varlen(tfa, q, k, v, cu_q, cu_k, max(lq), causal, kind, f32)
        assert out.dtype == (torch.float32 if f32 else _dt(kind))
        for (q0, q1), (k0, k1) in zip(offsets(lq), offsets(lk)):
            if q1 == q0:
                continue
            if k1 == k0:
                assert torch.count_nonzero(out[q0:q1]).item() == 0 and torch.isposinf(lse[:, q0:q1]).all()
                continue
            o_ref, l_ref = tfa.attn_fwd(seq(q, q0, q1), seq(k, k0, k1), seq(v, k0, k1), causal, D ** -0.5,
                                        num_splits=1, out_fp32=f32, q_scale=SCALES[0], k_scale=SCALES[1],
                                        v_scale=SCALES[2], out_dtype=_dt(kind))
            assert torch.equal(bits(out[q0:q1]), bits(o_ref[0].permute(1, 0, 2))), (f32, q0, q1, k0, k1)
            assert torch.equal(bits(lse[:, q0:q1]), bits(l_ref[0])), (f32, q0, q1, k0, k1)
    torch.cuda.synchronize()


FLOAT64 = [
    # lq, lk, causal, D, kind, Hq, Hkv, f32
    ([300, 0, 200, 64, 129, 5, 1000], [100, 50, 0, 64, 500, 5, 1300], True, 128, "bf16", 8, 2, False),
    ([500, 77, 0, 1, 260, 2049], [200, 0, 10, 300, 260, 2049], True, 64, "fp16", 4, 1, True),
    ([300, 0, 200, 64, 129, 700], [100, 50, 0, 64, 500, 3000], False, 64, "bf16", 4, 4, False),
    ([257, 255, 128, 63], [4096, 255, 1, 63], False, 128, "fp16", 4, 2, True),
]


@pytest.mark.gpu
@pytest.mark.parametrize("lq,lk,causal,D,kind,Hq,Hkv,f32", FLOAT64)
def test_varlen_fp8_within_budget_of_float64_reference(tfa, lq, lk, causal, D, kind, Hq, Hkv, f32):
    """Each sequence within compare()'s float64 budget, every element, no pass fraction; key-less rows are 0 / +inf."""
    q, k, v, cu_q, cu_k = make_fp8_batch(lq, lk, Hq, Hkv, D, seed=3 + D)
    out, lse = varlen(tfa, q, k, v, cu_q, cu_k, max(lq), causal, kind, f32)
    torch.cuda.synchronize()
    worst = 0.0
    for (q0, q1), (k0, k1) in zip(offsets(lq), offsets(lk)):
        if q1 == q0:
            continue
        got_o, got_l = out[q0:q1].permute(1, 0, 2)[None], lse[:, q0:q1][None]
        if k1 == k0:
            assert torch.count_nonzero(got_o).item() == 0 and torch.isposinf(got_l).all()
            continue
        ref = fp8_reference(deq(seq(q, q0, q1), SCALES[0]), seq(k, k0, k1), seq(v, k0, k1), causal, D ** -0.5,
                            SCALES[1], SCALES[2])
        ok, r, le, msg = compare(got_o, got_l, ref, kind)
        assert ok, f"sequence rows [{q0}, {q1}): {msg}"
        worst = max(worst, r)
    print(f"\n[varlen fp8 float64] max err/budget {worst:.3f}")


@pytest.mark.gpu
@pytest.mark.parametrize("causal,D", [(True, 128), (False, 64)])
def test_varlen_fp8_nan_codes_in_neighbours_change_nothing(tfa, causal, D):
    """Every K and V byte outside a sequence's own rows set to the NaN codes 0x7f / 0xff: that sequence's out and lse
    keep every bit.  The keys a TMA box pulls in from a neighbour get -inf scores and zero V^T entries."""
    lq, lk = [129, 300, 1, 200, 64, 255], [129, 500, 40, 64, 257, 1]
    q, k, v, cu_q, cu_k = make_fp8_batch(lq, lk, 4, 2, D, seed=11)
    o1, l1 = varlen(tfa, q, k, v, cu_q, cu_k, max(lq), causal, "bf16")
    sq, sk = offsets(lq), offsets(lk)
    for victim in range(len(lq)):
        (a, b), (c, d) = sq[victim], sk[victim]
        k2, v2 = k.clone(), v.clone()
        for t, code in ((k2, 0x7F), (v2, 0xFF)):
            raw = t.view(torch.uint8)
            raw[:c] = code
            raw[d:] = code ^ 0x80                              # the other NaN code past the sequence
        o2, l2 = varlen(tfa, q, k2, v2, cu_q, cu_k, max(lq), causal, "bf16")
        torch.cuda.synchronize()
        assert torch.equal(bits(o1[a:b]), bits(o2[a:b])) and torch.equal(bits(l1[:, a:b]), bits(l2[:, a:b])), victim


@pytest.mark.gpu
@pytest.mark.parametrize("f32", [False, True])
def test_varlen_fp8_writes_exactly_its_rows(tfa, f32):
    """Sentinel-filled out / lse with guard regions: every row of [cu_q[b], cu_q[b] + min(Sq_b, max_seqlen_q)) is
    written and nothing else -- not the guards, not rows past max_seqlen_q of a sequence that has more (sequences with
    Sq_b = 0, Sk_b = 0 and causal Sq_b > Sk_b included)."""
    lq, lk = [200, 0, 129, 7, 300, 150], [64, 90, 0, 7, 700, 150]
    Hq, D, G, max_q = 4, 64, 64, 170
    q, k, v, cu_q, cu_k = make_fp8_batch(lq, lk, Hq, 1, D, seed=5)
    tq = sum(lq)
    dt = torch.float32 if f32 else torch.bfloat16
    obuf = torch.full((G + tq + G, Hq, D), float("nan"), dtype=dt, device="cuda")
    lbuf = torch.full((G + Hq * tq + G,), float("nan"), dtype=torch.float32, device="cuda")
    out, lse = obuf[G:G + tq], lbuf[G:G + Hq * tq].view(Hq, tq)
    varlen(tfa, q, k, v, cu_q, cu_k, max_q, True, "bf16", f32, out=out, lse=lse)
    torch.cuda.synchronize()
    written = torch.zeros(tq, dtype=torch.bool, device="cuda")
    for q0, q1 in offsets(lq):
        written[q0:q0 + min(q1 - q0, max_q)] = True
    assert not torch.isnan(out[written]).any() and not torch.isnan(lse[:, written]).any()
    assert torch.isnan(out[~written]).all() and torch.isnan(lse[:, ~written]).all()
    assert torch.isnan(obuf[:G]).all() and torch.isnan(obuf[G + tq:]).all()
    assert torch.isnan(lbuf[:G]).all() and torch.isnan(lbuf[G + Hq * tq:]).all()


SCHED = r'''
import os, sys, torch
sys.path.insert(0, os.path.join(os.environ["TFA_ROOT"], "tiny-flash-attention_b200"))
sys.path.insert(0, os.path.join(os.environ["TFA_ROOT"], "tests"))
import tfa_ctypes as tfa
from test_varlen_fp8 import make_fp8_batch, varlen
lq, lk = [1000, 0, 129, 2049, 64, 300, 1], [1000, 30, 0, 2100, 20, 300, 257]
res = []
for causal, D in ((True, 128), (False, 128), (True, 64)):
    q, k, v, cu_q, cu_k = make_fp8_batch(lq, lk, 8, 2, D, seed=9)
    o, lse = varlen(tfa, q, k, v, cu_q, cu_k, max(lq), causal, "bf16")
    res.append((o.cpu(), lse.cpu(), tfa.lib().tfa_internal_last_variant()))
torch.cuda.synchronize()
torch.save(res, os.environ["TFA_OUT"])
'''


@pytest.mark.gpu
def test_varlen_fp8_classic_and_persistent_agree_bitwise(tfa):
    outs = {}
    with tempfile.TemporaryDirectory() as tmp:
        for variant in ("classic", "persist"):
            path = os.path.join(tmp, variant + ".pt")
            env = dict(os.environ, TFA_ROOT=ROOT, TFA_OUT=path, TFA_KERNEL=variant)
            p = subprocess.run([sys.executable, "-c", SCHED], env=env, capture_output=True, text=True, timeout=600)
            assert p.returncode == 0, p.stderr[-2000:]
            outs[variant] = torch.load(path)
    for (a, la, va), (b, lb, vb) in zip(outs["classic"], outs["persist"]):
        assert (va, vb) == (0, 4)
        assert torch.equal(bits(a), bits(b)) and torch.equal(bits(la), bits(lb))


@pytest.mark.gpu
def test_varlen_fp8_is_one_launch_and_replays_from_a_cuda_graph(tfa):
    """One launch per call (16-bit and fp32 output); capture one call, rewrite cu_seqlens in place (same totals and
    max), replay: equals a fresh eager call bit for bit."""
    lq1, lk1 = [100, 300, 50, 250], [400, 300, 50, 100]
    lq2, lk2 = [300, 100, 250, 50], [50, 100, 400, 300]
    q, k, v, cu_q, cu_k = make_fp8_batch(lq1, lk1, 4, 2, 128, seed=13)
    for causal in (True, False):
        n0 = tfa.launch_count()
        varlen(tfa, q, k, v, cu_q, cu_k, 300, causal, "fp16")
        varlen(tfa, q, k, v, cu_q, cu_k, 300, causal, "fp16", True)
        assert tfa.launch_count() - n0 == 2
    out = torch.empty(q.shape, dtype=torch.bfloat16, device="cuda")
    lse = torch.empty((4, q.shape[0]), dtype=torch.float32, device="cuda")
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):                               # warm-up outside the capture
        varlen(tfa, q, k, v, cu_q, cu_k, 300, True, "bf16", out=out, lse=lse)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        varlen(tfa, q, k, v, cu_q, cu_k, 300, True, "bf16", out=out, lse=lse)
    g.replay()
    want1, wl1 = varlen(tfa, q, k, v, cu_q.clone(), cu_k.clone(), 300, True, "bf16")
    torch.cuda.synchronize()
    assert torch.equal(bits(out), bits(want1)) and torch.equal(bits(lse), bits(wl1))
    c2q, c2k = make_fp8_batch(lq2, lk2, 1, 1, 64, seed=1)[3:]
    cu_q.copy_(c2q)
    cu_k.copy_(c2k)
    g.replay()
    want2, wl2 = varlen(tfa, q, k, v, c2q, c2k, 300, True, "bf16")
    torch.cuda.synchronize()
    assert not torch.equal(bits(want1), bits(want2))
    assert torch.equal(bits(out), bits(want2)) and torch.equal(bits(lse), bits(wl2))


@pytest.mark.gpu
def test_varlen_fp8_extension_and_ctypes_agree(tfa):
    """q, k and v as views of one packed (total, 3, H, D) e4m3 tensor, no copy: the extension entry, the ctypes entry
    and the ctypes entry on contiguous copies give the same bits."""
    import attention_cutlass as ac
    lq = [300, 1, 129, 640, 0, 64]
    H, D = 4, 128
    g = torch.Generator().manual_seed(17)
    qkv = (torch.empty((sum(lq), 3, H, D)).normal_(0, 0.5, generator=g) / 0.02).clamp(-448, 448).to(FP8).cuda()
    cu = torch.tensor(np.concatenate([[0], np.cumsum(lq)]), dtype=torch.int32, device="cuda")
    q, k, v = qkv.unbind(1)
    assert q.data_ptr() - qkv.data_ptr() == 0 and k.stride(0) == 3 * H * D
    for causal, od in ((True, torch.bfloat16), (False, torch.float16)):
        out, lse = ac.flash_attention_v2_varlen_fp8(q, k, v, cu, cu, max(lq), *SCALES, causal, D ** -0.5, od)
        out2, lse2 = tfa.attn_varlen_fwd(q, k, v, cu, cu, max(lq), causal, D ** -0.5, q_scale=SCALES[0],
                                         k_scale=SCALES[1], v_scale=SCALES[2], out_dtype=od)
        out3, lse3 = ac.flash_attention_v2_varlen_fp8(q=q.contiguous(), k=k.contiguous(), v=v.contiguous(),
                                                      cu_seqlens_q=cu, cu_seqlens_k=cu, max_seqlen_q=max(lq),
                                                      q_scale=SCALES[0], k_scale=SCALES[1], v_scale=SCALES[2],
                                                      is_causal=causal, softmax_scale=D ** -0.5, out_dtype=od)
        torch.cuda.synchronize()
        assert out.shape == (sum(lq), H, D) and out.dtype == od and lse.shape == (H, sum(lq))
        for o, l in ((out2, lse2), (out3, lse3)):
            assert torch.equal(bits(out), bits(o)) and torch.equal(bits(lse), bits(l))
    with pytest.raises(RuntimeError, match="int32"):
        ac.flash_attention_v2_varlen_fp8(q, k, v, cu.long(), cu, max(lq), *SCALES, True, 0.1, torch.bfloat16)
    with pytest.raises(RuntimeError, match="device"):
        ac.flash_attention_v2_varlen_fp8(q, k, v, cu.cpu(), cu.cpu(), max(lq), *SCALES, True, 0.1, torch.bfloat16)
    with pytest.raises(RuntimeError, match="max_seqlen_q"):
        ac.flash_attention_v2_varlen_fp8(q, k, v, cu, cu, 0, *SCALES, True, 0.1, torch.bfloat16)
    with pytest.raises(RuntimeError, match="code -16"):
        ac.flash_attention_v2_varlen_fp8(q, k, v, cu, cu, max(lq), 0.0, 1.0, 1.0, True, 0.1, torch.bfloat16)
    # ctypes: 16-bit calls take no scales (ValueError, as attn_fwd); q, k and v are all e4m3 or none
    qb = q.to(torch.bfloat16)
    with pytest.raises(ValueError):
        tfa.attn_varlen_fwd(qb, qb, qb, cu, cu, max(lq), True, 0.1, q_scale=0.5)
    with pytest.raises(TypeError):
        tfa.attn_varlen_fwd(q, qb, qb, cu, cu, max(lq), True, 0.1)
