"""The FP8 attention forward (tfa_attn_fp8_fwd: e4m3 Q, K and V, both products on e4m3 wgmma) against a float64
reference, within a per-element budget derived from its arithmetic.

Reference: reference() of test_fwd_float64_reference on the dequantized inputs, q_scale * float(Q8) (float64, exact),
with k_scale / v_scale, softmax scale softmax_scale.  For row i and its visible keys j, p_j = exp(s_j - max), l = sum p_j.

Budget, per output element (b, h, i, d):
  * P rounded to e4m3 (3 mantissa bits, subnormal spacing 2^-9): the kernel holds P' = p e^(m - m') against a running
    max m' <= m, rounds it to nearest with an error of at most max(2^-4 P', min(P', 2^-10)), and sums l from the
    unrounded fp32 P'.  In reference units (divide by e^(m - m') >= 1) that is at most e_j = max(2^-4 p_j,
    min(p_j, 2^-10)): the lazy-rescale factor only shrinks the absolute term.  O moves by at most
        E_P = sum_j e_j |v_jd| / l.
  * S accumulation: e4m3 products are exact, but the H100's FP8 wgmma does not accumulate at full fp32 precision (it
    is reported to retain about 14 bits: DeepSeek-V3 technical report, arXiv:2412.19437, section 3.3.2).  The bound
    is this wgmma's own measured worst case: test_wgmma_fp8_primitives found |C - exact| up to 1.31e-3 (2^-9.6) of
    sum |a b| for chains from zero of up to 128 (1.16e-3 for the 128-deep SS chain, 6.6e-4 at 64 deep) on an H100
    80GB HBM3 (700 W), and asserts every such chain stays within ACC_MEASURED_BOUND = 2^-9 (1.5x that).  The budget
    takes twice the asserted bound, EPS_ACC = 2^-8, plus 2^-22 for the two fp32 roundings of
    s' = fp32(fp32(softmax_scale q_scale) k_scale).  So every logit moves by at most
    eta_ij = softmax_scale * EPS_ACC * sum_d |q_id k_jd|; with eta_i = max_j eta_ij every softmax weight moves by a
    factor within e^(+-2 eta_i), and O by at most (e^(2 eta_i) - 1) A, A = sum_j p_j |v_jd| / l.
  * O accumulation: O += P8 V8 runs on e4m3 wgmma too, 4 k-steps of 32 keys per KV tile, all into one accumulator
    over the row's whole key range (a split's).  The bound is again this wgmma's measured worst case:
    test_wgmma_fp8_primitives issues RS chains of up to 16384 k-steps (524288 keys) into an accumulator that starts
    at zero or at a large C0, and measures |C - exact| against the sum over the k-steps of |C before the step| + sum
    |a b| of the step: up to 4.04e-4 on the H100 above (3.79e-4 up to 512 k-steps: the measure barely grows with the
    chain).  It asserts PV_MEASURED_BOUND = 2^-11 (1.21x that), and the budget
    takes EPS_PV = 2 PV_MEASURED_BOUND.  |C before k-step i| is at most the sum of P8 |v| over the keys before it, and
    P8 <= p_j + e_j; so with n = ceil(Sk / 32) k-steps and key j in step j // 32, in reference units
        E_PV = EPS_PV sum_j (n - j // 32) (p_j + e_j) |v_jd| / l,
    an upper bound also for split-KV (each split restarts from zero) and for causal rows (masked keys add zeros).
  * 2^-14 A + 1e-6 for ex2.approx, the other fp32 arithmetic, 1/l and the split-KV combine, as for the 16-bit kernel.
  * A 16-bit output adds half an ulp of the largest value it can round (|O_ref| + the terms above).
LSE: l sums the unrounded P, so only the logits' error reaches it: |dLSE| <= eta_i + 1e-4 + 2e-6 |LSE_ref|
+ L_SUM, l's own rounding (test_fwd_float64_reference); L_SUM A joins O's budget for the same reason.
Key-less rows: exactly out = 0 and lse = +inf.  No pass fraction."""
import math
import os
import subprocess
import sys
import tempfile

import pytest
import torch

from test_fwd_float64_reference import L_SUM, OUT_EMIN, OUT_P, lse_bound, mutations, reference
from test_kvcache_fp8 import FINITE, FP8, bits

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "tfa_b200.h")
EPS_ACC = 2.0 ** -8 + 2.0 ** -22
ACC_MEASURED_BOUND = 2.0 ** -9      # per chain of up to 128: 1.5x the worst measured, half the budget's EPS_ACC
PV_MEASURED_BOUND = 2.0 ** -11      # per k-step of an RS chain, relative to |C before| + sum |a b|: 1.21x the worst
                                    # measured (4.04e-4 over 16384 k-steps, H100 80GB HBM3 at 700 W), half of EPS_PV
EPS_PV = 2 * PV_MEASURED_BOUND


# ------------------------------------------------------------------ budget ----------------------------------------------

def fp8_reference(q, k, v, causal, scale, ks, vs, **mut):
    """reference() of the dequantized problem (q already dequantized, float64), plus the budget's per-row eta and the
    e4m3 rounding term E_P."""
    o, lse, a, _, _ = reference(q, k, v, causal, scale, ks, vs, **mut)
    wide = lambda t: (t.float() if t.dtype == FP8 else t).to(torch.float64)
    kd, vd = wide(k) * ks, wide(v) * vs
    Hq, Hkv = q.shape[1], kd.shape[1]
    h = torch.arange(Hq, device=q.device) // (Hq // Hkv)
    kd, vd = kd[:, h], vd[:, h]
    Sq, Sk = q.shape[2], kd.shape[2]
    i = torch.arange(Sq, device=q.device)[:, None]
    j = torch.arange(Sk, device=q.device)[None, :]
    vis = (j <= i + (Sk - Sq)) if causal else torch.ones((Sq, Sk), dtype=torch.bool, device=q.device)
    s = (q @ kd.transpose(-1, -2) * scale).masked_fill(~vis, -math.inf)
    m = s.amax(-1, keepdim=True)
    m = torch.where(torch.isinf(m), torch.zeros_like(m), m)
    p = torch.exp(s - m)
    l = p.sum(-1, keepdim=True)
    inv = torch.where(l > 0, 1.0 / l, torch.zeros_like(l))
    e = torch.maximum(2.0 ** -4 * p, torch.minimum(p, torch.full_like(p, 2.0 ** -10)))
    ep = (e @ vd.abs()) * inv
    n = -(-Sk // 32)
    w = (n - torch.arange(Sk, device=q.device) // 32).to(torch.float64)
    epv = EPS_PV * (((p + e) * w) @ vd.abs()) * inv
    eta = ((q.abs() @ kd.abs().transpose(-1, -2)) * (scale * EPS_ACC)).masked_fill(~vis, 0.0).amax(-1)
    return o, lse, a, ep + epv, eta


def budget(ref, kind, out16):
    o_ref, _, a, ep, eta = ref           # ep: E_P + E_PV
    b = ep + torch.expm1(2 * eta)[..., None] * a + 2.0 ** -14 * a + L_SUM * a + 1e-6
    if out16:
        x = o_ref.abs() + b
        _, ex = torch.frexp(x)
        ex = torch.where(x > 0, ex.clamp(min=OUT_EMIN[kind]), torch.full_like(ex, OUT_EMIN[kind]))
        b = b + 0.5 * torch.ldexp(torch.ones_like(x), ex - OUT_P[kind])
    return b


def compare(out, lse, ref, kind):
    """(ok, max err / budget, max |dLSE| - bound, message)."""
    o_ref, l_ref = ref[0], ref[1]
    o, l = out.to(torch.float64), lse.to(torch.float64)
    keyless = torch.isinf(l_ref)
    if keyless.any() and not (bool((o[keyless] == 0).all()) and bool(torch.isposinf(l[keyless]).all())):
        return False, math.inf, math.inf, "a row without keys is not 0 / +inf"
    b = budget(ref, kind, out.dtype != torch.float32)
    ratio = torch.nan_to_num((o - o_ref).abs() / b, nan=math.inf).masked_fill(keyless[..., None], 0.0)
    lb = ref[4] + lse_bound(l_ref.masked_fill(keyless, 0.0))
    lex = (torch.nan_to_num((l - l_ref).abs(), nan=math.inf) - lb).masked_fill(keyless, -1.0)
    r, le = float(ratio.max()), float(lex.max())
    if r > 1.0:
        return False, r, le, f"O over budget: ratio {r:.3f}"
    if le > 0:
        return False, r, le, f"LSE over its bound by {le:.3e}"
    return True, r, le, ""


def _dt(kind):
    return torch.bfloat16 if kind == "bf16" else torch.float16


def make_fp8(B, Hq, Hkv, Sq, Sk, D, seed, scales=(0.0213, 0.0171, 0.0119), device="cpu"):
    """Normal(0, 0.5) inputs quantized as a caller would, (x / s).clamp(-448, 448).to(float8_e4m3fn)."""
    g = torch.Generator().manual_seed(seed)
    mk = lambda s, *shape: (torch.empty(shape).normal_(0.0, 0.5, generator=g) / s).clamp(-448, 448).to(FP8)
    qs, ks, vs = scales
    return mk(qs, B, Hq, Sq, D).to(device), mk(ks, B, Hkv, Sk, D).to(device), mk(vs, B, Hkv, Sk, D).to(device)


def deq(q8, qs):
    return q8.float().to(torch.float64) * qs


# ------------------------------------------------------------------ CPU: contract --------------------------------------

@pytest.fixture(scope="module")
def tfa(built):
    import tfa_ctypes
    tfa_ctypes.lib()
    return tfa_ctypes


def test_header_declares_the_fp8_call():
    src = open(HEADER).read()
    assert "#define TFA_EINVAL_QKVQUANT (-16)" in src
    assert "int tfa_attn_fp8_fwd(const tfa_attn_args* args, const tfa_qkv_quant_args* quant);" in src
    assert "float q_scale, k_scale, v_scale;" in src
    assert "#define TFA_ABI_VERSION 2" in src


def test_error_string_of_qkvquant(tfa):
    msg = tfa.lib().tfa_error_string(-16).decode()
    assert "FP8 attention" in msg and "q_scale" in msg and "16" in msg


def _args(tfa, **kw):
    """A valid FP8 call's arguments on fake, aligned device addresses: every check passes, none touches memory."""
    d = dict(q=0x10000, k=0x20000, v=0x30000, out=0x40000, lse=0x50000, B=2, Hq=4, Hkv=2, Sq=300, Sk=500, D=128,
             qsb=4 * 300 * 128, qsh=300 * 128, qss=128, ksb=2 * 500 * 128, ksh=500 * 128, kss=128, dtype=0,
             causal=1, scale=0.0883, f32=0, ns=1, ws=None, wsb=0)
    d.update(kw)
    return tfa.AttnArgs(d["q"], d["k"], d["v"], d["out"], d["lse"], d["B"], d["Hq"], d["Hkv"], d["Sq"], d["Sk"],
                        d["D"], d["qsb"], d["qsh"], d["qss"], d["ksb"], d["ksh"], d["kss"], d["dtype"], d["causal"],
                        d["scale"], d["f32"], d["ns"], d["ws"], d["wsb"], None)


def _call(tfa, args, quant=None, **qkw):
    import ctypes
    qd = dict(qkv_dtype=2, q_scale=0.02, k_scale=0.03, v_scale=0.01)
    qd.update(qkw)
    quant = quant or tfa.QkvQuantArgs(qd["qkv_dtype"], qd["q_scale"], qd["k_scale"], qd["v_scale"])
    return tfa.lib().tfa_attn_fp8_fwd(ctypes.byref(args), ctypes.byref(quant))


def test_argument_checks_and_their_order(tfa):
    """Each check alone, then pairs that show which runs first: the 16-bit call's checks in tfa_attn_fwd's order,
    then TFA_EINVAL_QKVQUANT, then TFA_EINVAL_SCALE for s'.  A valid call gets as far as the device check."""
    import ctypes
    inf, nan = float("inf"), float("nan")
    L = tfa.lib()
    assert L.tfa_attn_fp8_fwd(None, None) == -1
    assert L.tfa_attn_fp8_fwd(ctypes.byref(_args(tfa)), None) == -1
    cases = [
        (dict(q=0), {}, -1), (dict(out=0x40008), {}, -1), (dict(D=96), {}, -2), (dict(Sq=0), {}, -3),
        (dict(Hq=3), {}, -10), (dict(dtype=2), {}, -4), (dict(scale=-1.0), {}, -9), (dict(scale=nan), {}, -9),
        (dict(qss=136, qsh=300 * 136, qsb=4 * 300 * 136 + 4), {}, -5), (dict(ns=-1), {}, -3),
        # the quantization's own checks
        ({}, dict(qkv_dtype=0), -16), ({}, dict(q_scale=0.0), -16), ({}, dict(k_scale=-1.0), -16),
        ({}, dict(v_scale=inf), -16), ({}, dict(q_scale=nan), -16),
        (dict(qss=136, qsh=300 * 136, qsb=4 * 300 * 136), {}, -16), (dict(ksh=500 * 128 + 8), {}, -16),
        (dict(ksb=2 * 500 * 128 + 8), {}, -16),
        # s' = fp32(fp32(softmax_scale q_scale) k_scale): overflow, underflow below FLT_MIN
        (dict(scale=1e30), dict(q_scale=1e10, k_scale=1.0), -9),
        (dict(scale=1e-20), dict(q_scale=1e-10, k_scale=1e-10), -9),
        (dict(scale=1e-30), dict(q_scale=1e-3, k_scale=1e-6), -9),
        # order: the 16-bit checks come first, then the quantization's, then s'
        (dict(D=96), dict(qkv_dtype=0), -2), (dict(dtype=2), dict(v_scale=0.0), -4),
        (dict(qss=136, qsh=300 * 136, qsb=4 * 300 * 136 + 4), dict(qkv_dtype=0), -5),
        (dict(scale=1e30, qss=136, qsh=300 * 136, qsb=4 * 300 * 136), dict(q_scale=1e10), -16),
        (dict(scale=1e30), dict(q_scale=1e10, k_scale=0.0), -16),
    ]
    for akw, qkw, want in cases:
        got = _call(tfa, _args(tfa, **akw), **qkw)
        assert got == want, (akw, qkw, got, want)
    # valid scales, softmax_scale = 0 (uniform attention) included, pass every argument check; two splits asked for
    # without a workspace then stop the call before any device work: TFA_EINVAL_WORKSPACE, or TFA_EARCH without an H100
    for akw, qkw in (({}, {}), (dict(scale=0.0), {}), (dict(scale=1e-20), dict(q_scale=1e-5, k_scale=1e5))):
        got = _call(tfa, _args(tfa, ns=2, **akw), **qkw)
        assert got in (-11, -7), (akw, qkw, got)


def test_pi_is_a_bijection_and_packer_matches_converter(tfa):
    """pi permutes each 32-key block; for every thread tq, A register r and byte x, the accumulator element the packer
    puts there (row half, key 8 i + 2 tq + e) is the A column's key in the converter's V^T order."""
    L = tfa.lib()
    pi = [L.tfa_internal_fp8_p_key(c) for c in range(32)]
    assert sorted(pi) == list(range(32))
    assert all(pi[16 + c] == 16 + pi[c] for c in range(16))
    vt = [L.tfa_internal_fp8_vt_key(p) for p in range(128)]
    assert sorted(vt) == list(range(128))
    assert all(vt[p] == 32 * (p // 32) + pi[p % 32] for p in range(128))
    for kk in range(4):
        for tq in range(4):
            for r in range(4):
                for x in range(4):
                    j = L.tfa_internal_fp8_pack_src(r, x)
                    assert 0 <= j < 16
                    half, e, i = (j >> 1) & 1, j & 1, j >> 2
                    assert half == (r & 1)                              # a0 / a2 row g, a1 / a3 row g + 8
                    key = 32 * kk + 8 * i + 2 * tq + e                   # accumulator element s[16 kk + j]
                    col = 16 * (r >> 1) + 4 * tq + x                     # A column of register r, byte x
                    assert key == vt[32 * kk + col], (kk, tq, r, x)
    # every accumulator element of a k-step is packed exactly once per thread
    assert sorted(L.tfa_internal_fp8_pack_src(r, x) for r in range(4) for x in range(4)) == list(range(16))


def _emulate(q, k8, v8, causal, scale, ks, vs, stale):
    """The kernel's arithmetic in float64 but for the e4m3 rounding of P: P' against a max `stale` below the row's
    (e^stale <= 2^8, the lazy-rescale bound), rounded to e4m3; l from the unrounded P'."""
    kd, vd = k8.float().double() * ks, v8.float().double() * vs
    Hq, Hkv = q.shape[1], kd.shape[1]
    h = torch.arange(Hq) // (Hq // Hkv)
    kd, vd = kd[:, h], vd[:, h]
    Sq, Sk = q.shape[2], kd.shape[2]
    vis = (torch.arange(Sk)[None] <= torch.arange(Sq)[:, None] + Sk - Sq) if causal else torch.ones(Sq, Sk).bool()
    s = (q @ kd.transpose(-1, -2) * scale).masked_fill(~vis, -math.inf)
    m = s.amax(-1, keepdim=True) - stale
    m = torch.where(torch.isinf(m), torch.zeros_like(m), m)
    p = torch.exp(s - m)
    l = p.sum(-1, keepdim=True)
    p8 = p.float().to(FP8).double()
    o = torch.where(l > 0, (p8 @ vd) / l, torch.zeros_like(l))
    lse = torch.where(l[..., 0] > 0, m[..., 0] + torch.log(l[..., 0]), torch.full_like(l[..., 0], math.inf))
    return o, lse


@pytest.mark.parametrize("stale", [0.0, 3.0, 5.5])
@pytest.mark.parametrize("Hq,Hkv,Sq,Sk,D,causal", [(4, 2, 200, 300, 128, True), (4, 1, 160, 96, 64, True),
                                                   (2, 2, 64, 700, 64, False)])
def test_budget_covers_e4m3_p_emulation(Hq, Hkv, Sq, Sk, D, causal, stale):
    q8, k8, v8 = make_fp8(1, Hq, Hkv, Sq, Sk, D, seed=Sq + Sk)
    qs, ks, vs = 0.0213, 0.0171, 0.0119
    q = deq(q8, qs)
    scale = D ** -0.5
    o, lse = _emulate(q, k8, v8, causal, scale, ks, vs, stale)
    ref = fp8_reference(q, k8, v8, causal, scale, ks, vs)
    for kind in ("bf16", "fp16"):
        ok, r, _, msg = compare(o.to(_dt(kind)), lse.float(), ref, kind)
        assert ok, msg
    ok, r, _, msg = compare(o.float(), lse.float(), ref, "bf16")
    assert ok and r > 0.05, (msg, r)          # the budget is not loose by orders of magnitude


# per-sequence shapes of the GPU cases: Hq, Hkv, Sq, Sk, D, kind, causal, split_keys
MUTATION_SHAPES = [(4, 2, 300, 300, 128, "bf16", True, None), (4, 2, 160, 96, 64, "fp16", True, None),
                   (4, 2, 300, 300, 128, "bf16", True, 128), (4, 2, 48, 5, 64, "bf16", False, None)]


@pytest.mark.parametrize("Hq,Hkv,Sq,Sk,D,kind,causal,split_keys", MUTATION_SHAPES)
def test_checker_rejects_wrong_results(Hq, Hkv, Sq, Sk, D, kind, causal, split_keys):
    """The exact result of a wrong problem, rounded to the output, fails: causal +-1, kv head h % Hkv, one key short
    (the key range cut short), a dropped split; the right one passes."""
    q8, k8, v8 = make_fp8(1, Hq, Hkv, Sq, Sk, D, seed=7 * Sq + Sk)
    qs, ks, vs = 0.0213, 0.0171, 0.0119
    q = deq(q8, qs)
    scale = D ** -0.5
    ref = fp8_reference(q, k8, v8, causal, scale, ks, vs)
    dt = _dt(kind)
    assert compare(ref[0].to(dt), ref[1].float(), ref, kind)[0]
    for what, mut in mutations(Hq, Hkv, Sq, causal, split_keys):
        if mut == "drop_last":
            wrong = reference(q, k8[:, :, :-1], v8[:, :, :-1], causal, scale, ks, vs)
        else:
            wrong = reference(q, k8, v8, causal, scale, ks, vs, **mut)
        ok, r, le, _ = compare(wrong[0].to(dt), wrong[1].float(), ref, kind)
        assert not ok, f"{what} passes (ratio {r:.3f}, LSE excess {le:.2e})"


# ------------------------------------------------------------------ GPU: primitives -------------------------------------

def _codes(g, *shape):
    c = torch.tensor(FINITE, dtype=torch.uint8)
    return c[torch.randint(0, len(FINITE), shape, generator=g)]


def _step_magnitudes(a, b, c0, chain, mode):
    """For C = C0 + chain x A B issued as chain x K/32 k-steps of 32: the exact result and the sum over the k-steps of
    |C before the step| + sum |a b| of the step (float64, per element)."""
    K = a.shape[1]
    bt = b.T if mode == 0 else b
    parts = [a[:, 32 * s:32 * s + 32] @ bt[32 * s:32 * s + 32] for s in range(K // 32)]
    mags = [a[:, 32 * s:32 * s + 32].abs() @ bt[32 * s:32 * s + 32].abs() for s in range(K // 32)]
    c, tot = c0.clone(), torch.zeros_like(c0)
    for _ in range(chain):
        for pt, mg in zip(parts, mags):
            tot += c.abs() + mg
            c += pt
    return c, tot


@pytest.mark.gpu
def test_wgmma_fp8_primitives(tfa):
    """SS (Q K^T, K = 64 with the 64-byte swizzle and K = 128 with the 128-byte one) and RS (P V, P packed in
    fp8_p_key order against the converter's V^T, N = 64 and 128) against exact products.  Two accumulation errors
    are measured: S's, a chain of D / 32 k-steps from zero, relative to sum |a b|; and O's, up to 16384 k-steps (the
    keys of 524288) into one accumulator from a large nonzero C0, relative to the sum over the k-steps of |C before the
    step| + sum |a b| of the step.  The budget's EPS_ACC and EPS_PV are twice the bounds asserted here."""
    L = tfa.lib()
    g = torch.Generator().manual_seed(5)
    worst_s, worst_pv = {}, {}
    for mode, N, K in ((0, 128, 64), (0, 128, 128), (1, 64, 128), (1, 128, 128)):
        for trial in range(4):
            a = _codes(g, 128, K)
            b = _codes(g, N, K) if mode == 0 else _codes(g, 128, N)
            if trial == 2:                         # dynamic range: 448 against 2^-9-sized terms in every row
                a[:, 0] = 0x7E
                a[:, 1:] = torch.randint(1, 8, (128, K - 1), generator=g).to(torch.uint8)
            if mode == 1 and trial >= 1:           # P is nonnegative in the forward
                a = a & 0x7F
            af, bf = a.view(FP8).double(), b.view(FP8).double()
            chains = [(1, 0.0)] if mode == 0 else [(1, 0.0), (16, 1e4), (128, -3e5), (128, 0.0)]
            if mode == 1 and trial < 2:            # a 128K-key row: 4096 x 4 = 16384 k-steps
                chains += [(1024, 1e4), (4096, 0.0)]
            for chain, c0s in chains:
                c0 = torch.empty(128, N, dtype=torch.float64).uniform_(-1, 1, generator=g) * c0s
                c0 = c0.float().double()
                c = c0.float().cuda()
                ad, bd = a.cuda(), b.cuda()
                assert L.tfa_selftest_wgmma_fp8(ad.data_ptr(), bd.data_ptr(), c.data_ptr(), N, K, mode, chain,
                                                None) == 0
                torch.cuda.synchronize()
                assert not torch.isnan(c).any()
                exact, tot = _step_magnitudes(af, bf, c0, chain, mode)
                err = (c.cpu().double() - exact).abs()
                if chain == 1 and c0s == 0.0:
                    mag = af.abs() @ (bf.abs().T if mode == 0 else bf.abs())
                    key = (mode, N, K)
                    worst_s[key] = max(worst_s.get(key, 0.0), float((err / mag.clamp(min=1e-30)).max()))
                if mode == 1:
                    key = (N, chain, c0s)
                    worst_pv[key] = max(worst_pv.get(key, 0.0), float((err / tot.clamp(min=1e-30)).max()))
    print("\n[fp8 wgmma] chains from zero, worst |C - exact| / sum|a b| per (mode, N, K): " +
          ", ".join(f"{k}: {v:.3e}" for k, v in worst_s.items()))
    print("[fp8 wgmma] RS chains, worst |C - exact| / sum_steps(|C_before| + sum|a b|) per (N, chain, |C0|): " +
          ", ".join(f"{k}: {v:.3e}" for k, v in worst_pv.items()))
    # accumulation roundings, not a layout mistake (which would be of the order of one product)
    assert max(worst_s.values()) <= ACC_MEASURED_BOUND, worst_s
    assert max(worst_pv.values()) <= PV_MEASURED_BOUND, worst_pv


# ------------------------------------------------------------------ GPU: against float64 ---------------------------------

# B, Hq, Hkv, Sq, Sk, D, kind, causal, out_fp32, num_splits
CASES = [
    (4, 16, 4, 1024, 1024, 128, "bf16", True, False, 1),      # 512 items: persistent CTAs walk several
    (2, 8, 2, 700, 1500, 64, "fp16", False, True, 1),         # Sq < Sk, GQA, fp32 out
    (2, 8, 4, 900, 600, 64, "bf16", True, False, 1),          # Sq > Sk: key-less rows
    (1, 4, 2, 129, 2048, 128, "fp16", True, False, 5),        # split-KV
    (1, 4, 1, 200, 1100, 128, "bf16", False, True, 3),        # split-KV, fp32 out, MQA
    (1, 4, 2, 700, 300, 128, "bf16", True, False, 3),         # split-KV with empty splits (rows above the diagonal)
    (3, 4, 2, 257, 191, 64, "fp16", False, False, 1),         # S not a multiple of 128
    (2, 4, 4, 63, 65, 128, "fp16", True, True, 1),
    (1, 4, 2, 8192, 8192, 128, "bf16", True, False, 1),       # long key ranges: O accumulates up to 256 k-steps
    (1, 4, 1, 256, 16384, 64, "fp16", False, True, 1),        # 512 k-steps into one accumulator
]
SCALES = (0.0213, 0.0171, 0.0119)

RUN = r'''
import os, sys, torch
sys.path.insert(0, os.path.join(os.environ["TFA_ROOT"], "tiny-flash-attention_b200"))
sys.path.insert(0, os.path.join(os.environ["TFA_ROOT"], "tests"))
import tfa_ctypes as tfa
from test_fwd_fp8 import CASES, run_case
res = [run_case(tfa, i) for i in range(len(CASES))]
torch.save([(o.cpu(), l.cpu(), v) for o, l, v in res], os.environ["TFA_OUT"])
'''


def run_case(tfa, idx):
    B, Hq, Hkv, Sq, Sk, D, kind, causal, f32, ns = CASES[idx]
    q8, k8, v8 = make_fp8(B, Hq, Hkv, Sq, Sk, D, seed=100 + idx, device="cuda")
    out, lse = tfa.attn_fwd(q8, k8, v8, causal, D ** -0.5, num_splits=ns, out_fp32=f32, q_scale=SCALES[0],
                            k_scale=SCALES[1], v_scale=SCALES[2], out_dtype=_dt(kind))
    torch.cuda.synchronize()
    return out, lse, tfa.lib().tfa_internal_last_variant()


@pytest.fixture(scope="module")
def schedule_runs(tfa):
    """Every case under the forced classic and persistent schedules, one subprocess each."""
    outs = {}
    with tempfile.TemporaryDirectory() as tmp:
        for variant in ("classic", "persist"):
            path = os.path.join(tmp, variant + ".pt")
            env = dict(os.environ, TFA_ROOT=ROOT, TFA_OUT=path, TFA_KERNEL=variant)
            p = subprocess.run([sys.executable, "-c", RUN], env=env, capture_output=True, text=True, timeout=1200)
            assert p.returncode == 0, p.stderr[-3000:]
            outs[variant] = torch.load(path)
    return outs


@pytest.mark.gpu
@pytest.mark.parametrize("idx", range(len(CASES)))
def test_fp8_within_budget_of_float64_reference(tfa, schedule_runs, idx):
    B, Hq, Hkv, Sq, Sk, D, kind, causal, f32, ns = CASES[idx]
    q8, k8, v8 = make_fp8(B, Hq, Hkv, Sq, Sk, D, seed=100 + idx, device="cuda")
    ref = fp8_reference(deq(q8, SCALES[0]), k8, v8, causal, D ** -0.5, SCALES[1], SCALES[2])
    if causal and Sq > Sk:
        assert torch.isinf(ref[1]).any()
    for variant, code in (("classic", 0), ("persist", 4)):
        out, lse, got = schedule_runs[variant][idx]
        assert got == code
        assert out.dtype == (torch.float32 if f32 else _dt(kind))
        ok, r, le, msg = compare(out.cuda(), lse.cuda(), ref, kind)
        print(f"\n[fp8 float64] case {idx} {variant}: max err/budget {r:.3f}, LSE margin {le:.2e}")
        assert ok, f"case {idx} {variant}: {msg}"


@pytest.mark.gpu
def test_fp8_bitwise_equal_under_both_schedules(schedule_runs):
    for idx in range(len(CASES)):
        (o0, l0, _), (o1, l1, _) = schedule_runs["classic"][idx], schedule_runs["persist"][idx]
        assert torch.equal(bits(o0), bits(o1)) and torch.equal(bits(l0), bits(l1)), idx


@pytest.mark.gpu
def test_fp8_extension_entry_point(built):
    import attention_cutlass as ac
    q8, k8, v8 = make_fp8(1, 4, 2, 300, 400, 128, seed=3, device="cuda")
    out, lse = ac.flash_attention_v2_fp8(q8, k8, v8, *SCALES, True, 128 ** -0.5, torch.float16, 1)
    ref = fp8_reference(deq(q8, SCALES[0]), k8, v8, True, 128 ** -0.5, SCALES[1], SCALES[2])
    assert out.dtype == torch.float16
    ok, _, _, msg = compare(out, lse, ref, "fp16")
    assert ok, msg
    with pytest.raises(RuntimeError):
        ac.flash_attention_v2_fp8(q8.float().half(), k8, v8, *SCALES, True, 0.1, torch.float16, 1)
