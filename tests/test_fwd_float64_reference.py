"""Every sm_90a forward mode against a float64 reference, within a per-element error budget derived from the kernel's
arithmetic.

Reference (`reference`): torch float64 on the tensors' device, per sequence: GQA with kv head h // (Hq / Hkv), the
bottom-right causal mask j <= i + Sk - Sq.  Besides O and LSE it returns, for the visible keys j of row i with
p_j = exp(s_j - max) and l = sum p_j,
    A   = sum_j p_j |v_jd| / l                  (the attention-weighted mean of |V|)
    Sub = sum_{j: p_j < 2^-14} |v_jd| / l.
Rows with no visible key have O = 0 and LSE = +inf.  FP8 caches enter dequantized, k_scale * float(K8) and
v_scale * float(V8), which float64 holds exactly.

Budget (`budget`).  The kernel rounds P to 16 bits before the PV wgmma, with a relative error of at most u_P (2^-8 for
bf16, 2^-11 for fp16), and sums l from the unrounded fp32 P; so O moves by at most u_P * A, whatever reference max P
was taken against (a stale max only scales P and l alike).  fp16 P has subnormals below 2^-14, each off by up to 2^-25
absolute; against a stale max P is larger, so a P the kernel holds as subnormal is subnormal in the reference too and
its error, divided by the kernel's larger l, is at most 2^-25 |v| / l.  2^-14 * A + 1e-6 covers ex2.approx, the fp32
accumulations, 1/l and the split-KV combine.  Two terms depend on the key count and are negligible below a few
thousand keys:
  * The row sum l (u = 2^-24).  Each thread sums a tile's 16 pairs of fp32 P into a fresh partial (a pair add and at
    most 15 adds: 16 u of the partial), adds the partial into l with Kahan's compensated add (2 u of l plus a term of
    n_tiles u^2), subtracts the compensation at the end (u) and sums its quad by two shuffles (2 u); each lazy
    rescale multiplies l by alpha (u of l, which in the final max's units never exceeds the final l).  So l is within
    (21 + rescales) u + n_tiles u^2 of its exact sum whatever the key count; L_SUM = 32 u covers up to 10 rescales and
    10^6 tiles, and enters both the LSE bound and O's budget (as L_SUM A).  A running sum of one fp32 add per pair,
    as the kernel once had, drifts by up to n_tiles u and breaks the LSE bound at 128K equal keys
    (test_fwd_softmax_range.test_row_sum_order_keeps_lse_bound_on_a_constant_tail).
  * The 16-bit PV chain.  O += P V accumulates 16 keys per wgmma k-step into one fp32 accumulator over the row's whole
    key range (a split's).  test_fwd_long_context.test_pv16_chain_through_the_forward measures the error per k-step
    relative to |C before the step| + sum |a b| of the step and asserts PV16_MEASURED_BOUND; with EPS_PV16 twice that,
    n = ceil(Sk / 16) k-steps and key j in step j // 16,
        E_PV16 = EPS_PV16 sum_j (n - j // 16) p_j |v_jd| / l,
    shaped like the FP8 budget's E_PV and an upper bound for split-KV and causal rows in the same way.
A 16-bit output adds half an ulp of the largest value it can round:
    budget = u_P A + [fp16] 2^-25 Sub + 2^-14 A + L_SUM A + E_PV16 + 1e-6 + [16-bit out] 1/2 ulp_out(|O_ref| + u_P A).
Every element must be within budget, with no pass fraction; LSE within 1e-4 + 2e-6 |LSE_ref| + L_SUM; key-less rows
exactly 0 / +inf.  One key more or less in a row of N keys moves LSE by about 1/N, which the LSE bound sees up to
N ~ 10^4.

CPU: the reference equals the numpy float64 oracle; the budget holds for the C oracle's emulation of 16-bit P on the
lazy-rescale stress inputs; the checker rejects a causal offset of +-1, the kv head h % Hkv, a sequence one key short
and a dropped split-KV partial at the shapes the GPU tests run.
GPU: about a dozen seeded workloads, each at least 3 work items per SM, covering every mode (dense, varlen, cache,
varlen-cache, FP8, rotary), run under the automatic schedule and, in one subprocess per schedule, forced classic and
persistent: bitwise equal across the three, within budget, out / lse written into NaN guard buffers, appends and q_rot
exact.  Tile-edge sweeps of the dense, split-KV, varlen, varlen-cache and cache calls; and per mode, the checker
rejects the kernel's result against a deliberately wrong reference."""
import math
import os
import random
import subprocess
import sys
import tempfile
from dataclasses import dataclass, field

import numpy as np
import pytest
import torch

from test_general_attn import make_inputs
from test_kvcache import _dt, gather, make_cache, scatter_append
from test_kvcache_fp8 import FINITE, FP8, bits, make_fp8_cache, quantize
from test_kvcache_rotary import new_tokens, positions, rope, rope_tables
from test_varlen import make_batch, offsets, seq

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

U_P = {"bf16": 2.0 ** -8, "fp16": 2.0 ** -11}       # unit roundoff of the 16-bit P
OUT_P = {"bf16": 8, "fp16": 11}                      # significand bits of the 16-bit output
OUT_EMIN = {"bf16": -125, "fp16": -13}               # frexp exponent of the smallest normal (ulp floor below it)
SUBNORMAL_P = 2.0 ** -14
PV16_MEASURED_BOUND = 2.0 ** -22    # per k-step of the 16-bit PV chain, relative to |C before| + sum |a b|: 1.67x the
                                    # worst measured (1.43e-7, fp16, 262144 keys, V of mean 1; H100 80GB HBM3 at 700 W)
EPS_PV16 = 2 * PV16_MEASURED_BOUND
L_SUM = 32 * 2.0 ** -24              # relative rounding of the kernel's row sum l, at any key count (see the docstring)


def lse_bound(lse_ref):
    """|LSE - LSE_ref| allowed on rows with a key (lse_ref finite): fast logf and the fp32 LSE, plus l's rounding."""
    return 1e-4 + 2e-6 * lse_ref.abs() + L_SUM


# ------------------------------------------------------------------ reference and budget -------------------------------

def reference(q, k, v, causal, scale, k_scale=1.0, v_scale=1.0, shift=0, heads="group", drop=None):
    """float64 (O, LSE, A, Sub, E_PV16) of q (B, Hq, Sq, D) against k / v (B, Hkv, Sk, D), on q's device.  The rest are the
    checker's mutations: `shift` moves the causal diagonal, heads="mod" maps query head h to kv head h % Hkv, `drop`
    = (j0, j1) hides keys [j0, j1)."""
    wide = lambda t: (t.float() if t.dtype == FP8 else t).to(torch.float64)
    q = q.to(torch.float64)
    k = wide(k) * k_scale
    v = wide(v) * v_scale
    B, Hq, Sq, D = q.shape
    Hkv, Sk = k.shape[1], k.shape[2]
    dev = q.device
    h = torch.arange(Hq, device=dev)
    h = h // (Hq // Hkv) if heads == "group" else h % Hkv
    k, v = k[:, h], v[:, h]
    i = torch.arange(Sq, device=dev)[:, None]
    j = torch.arange(Sk, device=dev)[None, :]
    vis = torch.ones((Sq, Sk), dtype=torch.bool, device=dev)
    if causal:
        vis &= j <= i + (Sk - Sq + shift)
    if drop is not None:
        vis &= ~((j >= drop[0]) & (j < drop[1]))
    if Sk == 0:
        z = torch.zeros_like(q)
        return z, torch.full((B, Hq, Sq), math.inf, dtype=torch.float64, device=dev), z, z, z
    s = (q @ k.transpose(-1, -2) * scale).masked_fill(~vis, -math.inf)
    m = s.amax(-1, keepdim=True)
    m = torch.where(torch.isinf(m), torch.zeros_like(m), m)
    p = torch.exp(s - m)
    l = p.sum(-1, keepdim=True)
    inv = torch.where(l > 0, 1.0 / l, torch.zeros_like(l))
    av = v.abs()
    o = (p @ v) * inv
    a = (p @ av) * inv
    sub = (((p < SUBNORMAL_P) & vis).to(torch.float64) @ av) * inv
    n = -(-Sk // 16)                                       # 16-bit PV k-steps of 16 keys
    pv16 = EPS_PV16 * ((p * (n - j // 16).to(torch.float64)) @ av) * inv
    lse = torch.where(l[..., 0] > 0, m[..., 0] + torch.log(l[..., 0]), torch.full_like(l[..., 0], math.inf))
    return o, lse, a, sub, pv16


def budget(o_ref, a, sub, kind, out16, pv16=0.0):
    u = U_P[kind]
    b = u * a + 2.0 ** -14 * a + L_SUM * a + pv16 + 1e-6
    if kind == "fp16":
        b = b + 2.0 ** -25 * sub
    if out16:
        x = o_ref.abs() + u * a
        _, e = torch.frexp(x)                                  # x = m 2^e, m in [0.5, 1): ulp(x) = 2^(e - p)
        e = torch.where(x > 0, e.clamp(min=OUT_EMIN[kind]), torch.full_like(e, OUT_EMIN[kind]))
        b = b + 0.5 * torch.ldexp(torch.ones_like(x), e - OUT_P[kind])
    return b


@dataclass
class Verdict:
    ok: bool = True
    ratio: float = 0.0            # largest |O - O_ref| / budget over rows with a key
    lse_err: float = 0.0          # largest |LSE - LSE_ref| over rows with a key
    msg: str = ""

    def add(self, other, where):
        self.ratio = max(self.ratio, other.ratio)
        self.lse_err = max(self.lse_err, other.lse_err)
        if not other.ok and self.ok:
            self.ok, self.msg = False, f"{where}: {other.msg}"


def compare(out, lse, ref, kind):
    """out (1, Hq, S, D) (16-bit in q's dtype, or fp32), lse (1, Hq, S) against reference() of the same rows."""
    o_ref, l_ref, a, sub, pv16 = ref
    o, l = out.to(torch.float64), lse.to(torch.float64)
    keyless = torch.isinf(l_ref)
    v = Verdict()
    if keyless.any():
        if not (bool((o[keyless] == 0).all()) and bool(torch.isposinf(l[keyless]).all())):
            return Verdict(False, math.inf, math.inf, "a row without keys is not 0 / +inf")
    b = budget(o_ref, a, sub, kind, out.dtype != torch.float32, pv16)
    ratio = torch.nan_to_num((o - o_ref).abs() / b, nan=math.inf).masked_fill(keyless[..., None], 0.0)
    lerr = torch.nan_to_num((l - l_ref).abs(), nan=math.inf).masked_fill(keyless, 0.0)
    lexcess = lerr - lse_bound(l_ref.masked_fill(keyless, 0.0))
    v.ratio, v.lse_err = float(ratio.max()) if ratio.numel() else 0.0, float(lerr.max()) if lerr.numel() else 0.0
    if v.ratio > 1.0:
        at = np.unravel_index(int(ratio.argmax()), tuple(ratio.shape))
        v.ok, v.msg = False, f"O over budget: ratio {v.ratio:.3f} at (b, h, row, d) = {tuple(int(x) for x in at)}"
    elif lexcess.numel() and float(lexcess.max()) > 0:
        at = np.unravel_index(int(lexcess.argmax()), tuple(lexcess.shape))
        v.ok, v.msg = False, f"LSE off by {v.lse_err:.3e} at (b, h, row) = {tuple(int(x) for x in at)}"
    return v


# ------------------------------------------------------------------ CPU: the reference and the budget ------------------

def _rand(g, *shape, scale=1.0):
    return torch.empty(shape, dtype=torch.float64).normal_(0.0, 0.5, generator=g) * scale


@pytest.mark.parametrize("B,Hq,Hkv,Sq,Sk,D,causal", [
    (2, 4, 2, 5, 7, 16, True),
    (1, 6, 3, 9, 4, 8, True),            # Sq > Sk causal: rows 0..4 see no key
    (2, 4, 4, 3, 1, 8, False),           # Sk = 1
    (1, 4, 1, 3, 1, 8, True),            # Sk = 1 causal: only the last row sees it
    (2, 6, 2, 17, 33, 32, False),
])
def test_reference_equals_numpy_float64_oracle(B, Hq, Hkv, Sq, Sk, D, causal):
    from oracle import oracle as orc
    g = torch.Generator().manual_seed(Sq * 31 + Sk)
    q, k, v = _rand(g, B, Hq, Sq, D, scale=30.0), _rand(g, B, Hkv, Sk, D), _rand(g, B, Hkv, Sk, D)
    scale = D ** -0.5
    o, lse, a, sub, _ = reference(q, k, v, causal, scale)
    want_o, want_lse = orc.numpy_attention_general(q.numpy(), k.numpy(), v.numpy(), causal, scale)
    want_a, _ = orc.numpy_attention_general(q.numpy(), k.numpy(), np.abs(v.numpy()), causal, scale)
    assert np.abs(o.numpy() - want_o).max() <= 1e-12 and np.abs(a.numpy() - want_a).max() <= 1e-12
    inf = np.isinf(want_lse)
    assert np.array_equal(np.isposinf(lse.numpy()), inf)
    assert np.abs(lse.numpy()[~inf] - want_lse[~inf]).max() <= 1e-12
    if causal and Sq > Sk:
        assert inf.any() and np.all(o.numpy()[inf] == 0)
    # Sub by its definition, one row at a time
    kr, vr = k.repeat_interleave(Hq // Hkv, 1), v.repeat_interleave(Hq // Hkv, 1)
    for bb in range(B):
        for h in range(Hq):
            for i in range(Sq):
                n = min(Sk, i + Sk - Sq + 1) if causal else Sk
                if n <= 0:
                    assert float(sub[bb, h, i].abs().max()) == 0
                    continue
                s = (kr[bb, h, :n] @ q[bb, h, i]) * scale
                p = torch.exp(s - s.max())
                want = (vr[bb, h, :n].abs() * (p < SUBNORMAL_P)[:, None]).sum(0) / p.sum()
                assert torch.allclose(sub[bb, h, i], want, rtol=1e-12, atol=0)
    if Sk >= 4:
        assert float(sub.max()) > 0                     # q x 30 leaves some p below 2^-14


STRESS = [
    # pattern, Hq, Hkv, Sq, Sk, D, causal
    ("spread", 2, 2, 512, 512, 128, False),
    ("late_outlier", 2, 2, 512, 512, 64, True),
    ("staircase_up", 2, 2, 768, 768, 128, False),
    ("staircase_under", 2, 2, 768, 768, 64, True),
    ("spread", 4, 2, 256, 1536, 128, True),
]


@pytest.mark.parametrize("kind", ["bf16", "fp16"])
@pytest.mark.parametrize("pattern,Hq,Hkv,Sq,Sk,D,causal", STRESS)
def test_budget_covers_16bit_p_emulation(monkeypatch, pattern, Hq, Hkv, Sq, Sk, D, causal, kind):
    """The C oracle rounds P to 16 bits as the kernel does (fp32 everywhere else, fp32 output): within budget on the
    inputs built to drive the lazy rescale, where P runs against stale maxima and fp16 P goes subnormal."""
    from oracle import oracle as orc
    from test_lazy_rescale import make_case
    monkeypatch.setattr(torch.Tensor, "cuda", lambda self, *a, **kw: self)     # make_case's inputs, on the CPU
    q, k, v, scale = make_case(pattern, 1, Hq, Hkv, Sq, Sk, D, kind)
    mode = orc.ROUND_BF16 if kind == "bf16" else orc.ROUND_FP16
    o, lse = orc.attn_general(q.float().numpy(), k.float().numpy(), v.float().numpy(), causal, scale, mode, False)
    ref = reference(q, k, v, causal, scale)
    verdict = compare(torch.from_numpy(o), torch.from_numpy(lse), ref, kind)
    assert verdict.ok, verdict.msg
    assert verdict.ratio > 0.05                         # the budget is not loose by orders of magnitude


# the GPU workloads' per-sequence shapes (fewer heads): name, Hq, Hkv, Sq, Sk, D, kind, causal, split_keys, fp8
MUTATION_SHAPES = [
    ("dense causal", 4, 2, 1000, 1000, 128, "bf16", True, None, False),
    ("dense GQA Sq != Sk", 4, 2, 700, 1500, 64, "fp16", False, None, False),
    ("dense causal split-KV", 4, 2, 2048, 2048, 128, "bf16", True, 512, False),
    ("dense causal Sq > Sk", 4, 2, 900, 600, 64, "bf16", True, None, False),
    ("varlen", 4, 2, 1000, 1200, 128, "bf16", True, None, False),
    ("cache decode split-KV", 32, 8, 1, 1500, 128, "bf16", True, 512, False),
    ("cache Sq 200", 8, 2, 200, 900, 64, "fp16", True, None, False),
    ("varlen-cache prefill", 8, 2, 512, 1500, 128, "bf16", True, None, False),
    ("fp8 decode", 8, 2, 1, 1500, 128, "bf16", False, None, True),
    ("fp8 d64 split-KV", 16, 4, 4, 1100, 64, "fp16", True, 384, True),
]


def mutations(Hq, Hkv, Sq, causal, split_keys):
    """The wrong references a kernel bug could amount to, for one shape (those that change nothing there left out)."""
    out = []
    if causal:
        out += [("causal offset -1", dict(shift=-1))] + ([("causal offset +1", dict(shift=1))] if Sq > 1 else [])
    if Hkv > 1 and Hq // Hkv > 1:
        out.append(("kv head h % Hkv", dict(heads="mod")))
    out.append(("one key short", "drop_last"))
    if split_keys:
        out.append(("split partial dropped", dict(drop=(split_keys, 2 * split_keys))))
    return out


def _fp8_values(g, *shape):
    codes = torch.tensor(FINITE, dtype=torch.uint8)
    return codes[torch.randint(0, len(FINITE), shape, generator=g)].view(FP8)


@pytest.mark.parametrize("name,Hq,Hkv,Sq,Sk,D,kind,causal,split_keys,fp8", MUTATION_SHAPES, ids=[m[0] for m in
                                                                                               MUTATION_SHAPES])
def test_checker_rejects_wrong_results_at_gpu_shapes(name, Hq, Hkv, Sq, Sk, D, kind, causal, split_keys, fp8):
    """A result that is exact for a wrong problem (rounded to the 16-bit output, where the budget is widest) fails;
    the exact result of the right problem, rounded the same way, passes."""
    g = torch.Generator().manual_seed(Sq + Sk)
    dt = _dt(kind)
    q = _rand(g, 1, Hq, Sq, D).to(dt)
    ks, vs = (0.0123, 0.00731) if fp8 else (1.0, 1.0)
    if fp8:
        k, v = _fp8_values(g, 1, Hkv, Sk, D), _fp8_values(g, 1, Hkv, Sk, D)
    else:
        k, v = _rand(g, 1, Hkv, Sk, D).to(dt), _rand(g, 1, Hkv, Sk, D).to(dt)
    scale = D ** -0.5
    ref = reference(q, k, v, causal, scale, ks, vs)
    assert compare(ref[0].to(dt), ref[1].float(), ref, kind).ok
    for what, mut in mutations(Hq, Hkv, Sq, causal, split_keys):
        if mut == "drop_last":
            wrong = reference(q, k[:, :, :-1], v[:, :, :-1], causal, scale, ks, vs)
        else:
            wrong = reference(q, k, v, causal, scale, ks, vs, **mut)
        verdict = compare(wrong[0].to(dt), wrong[1].float(), ref, kind)
        assert not verdict.ok, f"{name}: {what} passes (ratio {verdict.ratio:.3f}, LSE {verdict.lse_err:.2e})"


# ------------------------------------------------------------------ GPU: at-scale workloads ----------------------------

@pytest.fixture(scope="module")
def tfa(built):
    import tfa_ctypes
    tfa_ctypes.lib()
    return tfa_ctypes


GUARD = 512


def guarded(shape, dtype):
    """A NaN-filled buffer with GUARD elements on both sides, and the view of its middle in `shape`."""
    n = math.prod(shape)
    buf = torch.full((GUARD + n + GUARD,), float("nan"), dtype=dtype, device="cuda")
    return buf, buf[GUARD:GUARD + n].view(shape)


def assert_guarded(buf, view):
    assert not torch.isnan(view).any(), "a row of out / lse was not written"
    assert torch.isnan(buf[:GUARD]).all() and torch.isnan(buf[GUARD + view.numel():]).all(), "a guard element changed"


@dataclass
class W:
    name: str
    mode: str                    # dense, varlen, cache, varlen_cache
    seed: int
    kw: dict = field(default_factory=dict)


def _decode_lens(seed, B, page, hi):
    """Lengths of a decode batch: 0, 1 and page +- 1 around one and two pages, the rest random in [0, hi]."""
    rng = random.Random(seed)
    edges = [0, 1, page - 1, page, page + 1, 2 * page - 1, 2 * page, 2 * page + 1]
    return edges + [rng.randint(0, hi) for _ in range(B - len(edges))]


def _short_varlen(seed):
    rng = random.Random(seed)
    lq = [rng.choice([0, 0, 1, 1, 2, 5, 64, 127, 129, 300, 1000]) for _ in range(48)]
    lk = [rng.choice([0, 1, 3, 64, 128, 200, 700, 1100]) if n else rng.choice([0, 50]) for n in lq]
    lq[0], lk[0] = 1000, 1000
    return lq, lk


VC_SQ = [512] * 4 + [1] * 60

WORKLOADS = [
    W("dense_causal_b8", "dense", 101, dict(B=8, Hq=16, Hkv=4, Sq=1000, Sk=1000, D=128, kind="bf16", causal=True)),
    W("dense_gqa_noncausal", "dense", 102, dict(B=6, Hq=16, Hkv=2, Sq=700, Sk=1500, D=64, kind="fp16", causal=False,
                                                f32=True)),
    W("dense_causal_splits", "dense", 103, dict(B=2, Hq=8, Hkv=2, Sq=2048, Sk=2048, D=128, kind="bf16", causal=True,
                                                ns=4)),
    W("dense_causal_sq_gt_sk", "dense", 104, dict(B=6, Hq=16, Hkv=8, Sq=900, Sk=600, D=64, kind="bf16", causal=True)),
    W("varlen_short", "varlen", 105, dict(seqs=_short_varlen(105), Hq=8, Hkv=2, D=128, kind="bf16", causal=True)),
    W("cache_decode", "cache", 106, dict(lens=_decode_lens(106, 64, 256, 1500), Sq=1, Hq=32, Hkv=8, D=128, kind="bf16",
                                         page=256, causal=True, snew=1)),
    W("cache_decode_splits", "cache", 107, dict(lens=_decode_lens(107, 64, 256, 1500), Sq=1, Hq=32, Hkv=8, D=128,
                                                kind="fp16", page=256, causal=True, snew=1, ns=3)),
    W("cache_sq4_causal", "cache", 108, dict(lens=_decode_lens(108, 16, 128, 900), Sq=4, Hq=32, Hkv=8, D=128,
                                             kind="bf16", page=128, causal=True)),
    W("cache_sq200_causal", "cache", 109, dict(lens=[0, 1, 199, 200, 201, 900, 555, 128], Sq=200, Hq=32, Hkv=8, D=64,
                                               kind="fp16", page=128, causal=True)),
    W("varlen_cache_mixed", "varlen_cache", 110, dict(sq=VC_SQ, lens=_decode_lens(110, 64, 256, 1500), Hq=32, Hkv=8,
                                                      D=128, kind="bf16", page=256, causal=True, append=True)),
    W("fp8_decode", "cache", 111, dict(lens=_decode_lens(111, 64, 256, 1500), Sq=1, Hq=32, Hkv=8, D=128, kind="bf16",
                                       page=256, causal=True, snew=1, fp8=(0.0123, 0.00731))),
    W("fp8_varlen_cache_mixed", "varlen_cache", 112, dict(sq=VC_SQ, lens=_decode_lens(112, 64, 256, 1500), Hq=32,
                                                          Hkv=8, D=128, kind="fp16", page=256, causal=True, append=True,
                                                          fp8=(0.0371, 0.0093))),
    W("fp8_rotary_decode", "cache", 113, dict(lens=_decode_lens(113, 64, 256, 1500), Sq=1, Hq=16, Hkv=4, D=128,
                                              kind="bf16", page=256, causal=True, snew=1, fp8=(0.0123, 0.00731),
                                              rotary=(128, False))),
    W("fp8_d64_splits", "cache", 114, dict(lens=_decode_lens(114, 32, 128, 1000), Sq=4, Hq=16, Hkv=4, D=64,
                                           kind="fp16", page=128, causal=True, snew=4, ns=3, fp8=(0.0217, 0.0113))),
    W("rotary_neox_decode", "cache", 115, dict(lens=_decode_lens(115, 48, 256, 1200), Sq=1, Hq=16, Hkv=4, D=128,
                                               kind="bf16", page=256, causal=True, snew=1, rotary=(64, False))),
    W("rotary_gptj_decode", "cache", 116, dict(lens=_decode_lens(116, 48, 128, 1200), Sq=1, Hq=16, Hkv=2, D=64,
                                               kind="fp16", page=128, causal=False, snew=1, rotary=(64, True))),
]
BY_NAME = {w.name: w for w in WORKLOADS}


def _run_dense(tfa, w, kw):
    B, Hq, Hkv, Sq, Sk, D, kind, causal = (kw[x] for x in ("B", "Hq", "Hkv", "Sq", "Sk", "D", "kind", "causal"))
    f32 = kw.get("f32", False)
    q, k, v = make_inputs(B, Hq, Hkv, Sq, Sk, D, kind, seed=w.seed)
    ob, out = guarded((B, Hq, Sq, D), torch.float32 if f32 else q.dtype)
    lb, lse = guarded((B, Hq, Sq), torch.float32)
    _, _, n = tfa.attn_fwd(q, k, v, causal, D ** -0.5, num_splits=kw.get("ns", 1), out_fp32=f32, out=out, lse=lse,
                           return_splits=True)
    variant = tfa.lib().tfa_internal_last_variant()
    torch.cuda.synchronize()
    assert_guarded(ob, out)
    assert_guarded(lb, lse)
    seqs = [(q[b:b + 1], k[b:b + 1], v[b:b + 1], out[b:b + 1], lse[b:b + 1]) for b in range(B)]
    return dict(out=out, lse=lse, q_rot=None, variant=variant, items=-(-Sq // 128) * B * Hq * n, seqs=seqs)


def _run_varlen(tfa, w, kw):
    (lq, lk), Hq, Hkv, D, kind, causal = (kw[x] for x in ("seqs", "Hq", "Hkv", "D", "kind", "causal"))
    q, k, v, cu_q, cu_k = make_batch(lq, lk, Hq, Hkv, D, kind, seed=w.seed)
    tq = sum(lq)
    ob, out = guarded((tq, Hq, D), q.dtype)
    lb, lse = guarded((Hq, tq), torch.float32)
    tfa.attn_varlen_fwd(q, k, v, cu_q, cu_k, max(lq), causal, D ** -0.5, out=out, lse=lse)
    variant = tfa.lib().tfa_internal_last_variant()
    torch.cuda.synchronize()
    assert_guarded(ob, out)
    assert_guarded(lb, lse)
    seqs = [(seq(q, q0, q1), seq(k, k0, k1), seq(v, k0, k1), out[q0:q1].permute(1, 0, 2)[None], lse[:, q0:q1][None])
            for (q0, q1), (k0, k1) in zip(offsets(lq), offsets(lk)) if q1 > q0]
    return dict(out=out, lse=lse, q_rot=None, variant=variant, items=-(-max(lq) // 128) * len(lq) * Hq, seqs=seqs)


def _cache_pools(kw, lens, Sq, snew, seed):
    """q, k / v pools, table, seqlens; FP8 pools hold every finite code, unused slots NaN (0x7f for FP8)."""
    args = (lens, Sq, kw["Hq"], kw["Hkv"], kw["D"], kw["kind"], kw["page"])
    if kw.get("fp8"):
        return make_fp8_cache(*args, seed=seed, fill=0x7f, snew=snew)
    return make_cache(*args, seed=seed, fill=float("nan"), snew=snew)


def _append(pool, table, lens, new, page, fp8_scale):
    """The pool after appending `new` (B, n, Hkv, D) through the table: 16-bit rows verbatim, FP8 rows quantized."""
    if fp8_scale is None:
        return scatter_append(pool, table, lens, new, page, pool.shape[0])
    got = scatter_append(pool.view(torch.uint8), table, lens, quantize(new, fp8_scale).view(torch.uint8), page,
                         pool.shape[0])
    return got.view(FP8)


def _gather(pool, table, b, K):
    if pool.dtype == FP8:
        return gather(pool.view(torch.uint8), table, b, K).view(FP8)
    return gather(pool, table, b, K)


def _run_cache(tfa, w, kw):
    lens, Sq, Hq, D, kind, page, causal = (kw[x] for x in ("lens", "Sq", "Hq", "D", "kind", "page", "causal"))
    snew, fp8, rotary = kw.get("snew", 0), kw.get("fp8"), kw.get("rotary")
    ks, vs = fp8 or (1.0, 1.0)
    B = len(lens)
    q, kp, vp, table, sl = _cache_pools(kw, lens, Sq, snew, w.seed)
    cap = table.shape[1] * page
    kn, vn = new_tokens(B, snew, kw["Hkv"], D, kind, w.seed + 1) if snew else (None, None)
    rot = {}
    if rotary:
        rd, il = rotary
        seqlen_ro = cap + 64
        cos, sin = rope_tables(seqlen_ro, rd, kind)
        q_rot = torch.full_like(q, float("nan"))
        rot = dict(rotary_cos=cos, rotary_sin=sin, rotary_interleaved=il, q_rot=q_rot)
    k1, v1 = kp.clone(), vp.clone()
    ob, out = guarded(tuple(q.shape), q.dtype)
    lb, lse = guarded((B, Hq, Sq), torch.float32)
    _, _, n = tfa.attn_kvcache_fwd(q, k1, v1, sl, table, kn, vn, is_causal=causal, scale=D ** -0.5,
                                   num_splits=kw.get("ns", 1), out=out, lse=lse, return_splits=True, k_scale=ks,
                                   v_scale=vs, **rot)
    variant = tfa.lib().tfa_internal_last_variant()
    torch.cuda.synchronize()
    assert_guarded(ob, out)
    assert_guarded(lb, lse)
    qa = q
    if rotary:
        qa = rope(q, positions(lens, cap, snew, Sq, causal, True, seqlen_ro), cos, sin, rd, il)
        assert torch.equal(bits(q_rot), bits(qa)), "q_rot differs from the eager fp32 rotation"
        kn = rope(kn, positions(lens, cap, snew, snew, causal, False, seqlen_ro), cos, sin, rd, il)
    if snew:
        assert torch.equal(bits(k1), bits(_append(kp, table, lens, kn, page, fp8 and ks))), "appended K rows"
        assert torch.equal(bits(v1), bits(_append(vp, table, lens, vn, page, fp8 and vs))), "appended V rows"
    else:
        assert torch.equal(bits(k1), bits(kp)) and torch.equal(bits(v1), bits(vp))
    Ks = [min(max(L, 0), cap - snew) + snew for L in lens]
    seqs = [(qa[b:b + 1].permute(0, 2, 1, 3), _gather(k1, table, b, K), _gather(v1, table, b, K),
             out[b:b + 1].permute(0, 2, 1, 3), lse[b:b + 1]) for b, K in enumerate(Ks)]
    return dict(out=out, lse=lse, q_rot=q_rot if rotary else None, variant=variant,
                items=-(-Sq // 128) * B * Hq * n, seqs=seqs, ks=ks, vs=vs)


def _run_varlen_cache(tfa, w, kw):
    sq, lens, Hq, Hkv, D, kind, page, causal = (kw[x] for x in ("sq", "lens", "Hq", "Hkv", "D", "kind", "page",
                                                                 "causal"))
    append, fp8 = kw.get("append", False), kw.get("fp8")
    ks, vs = fp8 or (1.0, 1.0)
    B, total = len(sq), sum(sq)
    _, kp, vp, table, sl = _cache_pools(kw, lens, 1, max(sq) if append else 0, w.seed)
    g = torch.Generator().manual_seed(w.seed + 2)
    mk = lambda *s: torch.empty(s).normal_(0.0, 0.5, generator=g).to(_dt(kind)).cuda()
    q = mk(total, Hq, D)
    kn, vn = (mk(total, Hkv, D), mk(total, Hkv, D)) if append else (None, None)
    cu = torch.tensor([0] + np.cumsum(sq).tolist(), dtype=torch.int32, device="cuda")
    k1, v1 = kp.clone(), vp.clone()
    ob, out = guarded((total, Hq, D), q.dtype)
    lb, lse = guarded((Hq, total), torch.float32)
    tfa.attn_varlen_kvcache_fwd(q, k1, v1, cu, max(sq), sl, table, kn, vn, is_causal=causal, scale=D ** -0.5, out=out,
                                lse=lse, k_scale=ks, v_scale=vs)
    variant = tfa.lib().tfa_internal_last_variant()
    torch.cuda.synchronize()
    assert_guarded(ob, out)
    assert_guarded(lb, lse)
    wk, wv = kp, vp
    seqs = []
    for b, ((r0, r1), L) in enumerate(zip(offsets(sq), lens)):
        n = r1 - r0
        if append and n:
            wk = _append(wk, table[b:b + 1], [L], kn[r0:r1][None], page, fp8 and ks)
            wv = _append(wv, table[b:b + 1], [L], vn[r0:r1][None], page, fp8 and vs)
        if n:
            K = L + (n if append else 0)
            seqs.append((q[r0:r1].permute(1, 0, 2)[None], _gather(k1, table, b, K), _gather(v1, table, b, K),
                         out[r0:r1].permute(1, 0, 2)[None], lse[:, r0:r1][None]))
    assert torch.equal(bits(k1), bits(wk)) and torch.equal(bits(v1), bits(wv)), "appended rows"
    return dict(out=out, lse=lse, q_rot=None, variant=variant, items=-(-max(sq) // 128) * B * Hq, seqs=seqs, ks=ks,
                vs=vs)


RUN = {"dense": _run_dense, "varlen": _run_varlen, "cache": _run_cache, "varlen_cache": _run_varlen_cache}


def run_workload(tfa, w):
    """Regenerate workload w's inputs from its seed, run it, check its guard regions, appends and q_rot; returns the
    results and, per sequence, (q, k, v, out, lse) as (1, H, S, D) views for the reference."""
    r = RUN[w.mode](tfa, w, w.kw)
    r.setdefault("ks", 1.0)
    r.setdefault("vs", 1.0)
    r.update(kind=w.kw["kind"], causal=w.kw["causal"], scale=w.kw["D"] ** -0.5)
    return r


def portable(r):
    return {x: (r[x].cpu() if r[x] is not None else None) for x in ("out", "lse", "q_rot")} | {"variant": r["variant"]}


def check_workload(r, mutate=None):
    """Every sequence of a run against the reference, or with `mutate` against a wrong one (see mutations())."""
    verdict = Verdict()
    drop_seq = next(i for i, s in enumerate(r["seqs"]) if s[1].shape[2] >= 2)
    for i, (q, k, v, out, lse) in enumerate(r["seqs"]):
        kw = {}
        if mutate == "drop_last":
            if i == drop_seq:
                k, v = k[:, :, :-1], v[:, :, :-1]
        elif mutate is not None:
            kw = mutate
        ref = reference(q, k, v, r["causal"], r["scale"], r["ks"], r["vs"], **kw)
        verdict.add(compare(out, lse, ref, r["kind"]), f"sequence {i} (Sq {q.shape[2]}, K {k.shape[2]})")
    return verdict


@pytest.fixture(scope="module")
def auto_runs(tfa):
    return {w.name: run_workload(tfa, w) for w in WORKLOADS}


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.mark.gpu
@pytest.mark.parametrize("name", [w.name for w in WORKLOADS])
def test_workload_within_budget_of_float64_reference(auto_runs, name):
    r = auto_runs[name]
    sms = _sms()
    assert r["items"] >= 3 * sms, f"{r['items']} work items for {sms} SMs: fewer than 3 per persistent CTA"
    verdict = check_workload(r)
    print(f"\n[float64 reference] {name}: {r['items']} items on {sms} SMs, schedule {r['variant']}, "
          f"max err/budget {verdict.ratio:.3f}, max |dLSE| {verdict.lse_err:.2e}")
    assert verdict.ok, f"{name}: {verdict.msg}"


SCHEDULE_RUN = r'''
import os, sys, torch
sys.path.insert(0, os.path.join(os.environ["TFA_ROOT"], "tiny-flash-attention_b200"))
sys.path.insert(0, os.path.join(os.environ["TFA_ROOT"], "tests"))
import tfa_ctypes as tfa
from test_fwd_float64_reference import WORKLOADS, portable, run_workload
res = {}
for w in WORKLOADS:
    res[w.name] = portable(run_workload(tfa, w))
    torch.cuda.empty_cache()
torch.save(res, os.environ["TFA_OUT"])
'''


@pytest.mark.gpu
def test_workloads_bitwise_equal_under_both_schedules(auto_runs):
    """One subprocess per forced schedule runs every workload (each run checks its own appends, q_rot and guard
    regions): out, lse and q_rot equal the automatic choice's bit for bit."""
    outs = {}
    with tempfile.TemporaryDirectory() as tmp:
        for variant in ("classic", "persist"):
            path = os.path.join(tmp, variant + ".pt")
            env = dict(os.environ, TFA_ROOT=ROOT, TFA_OUT=path, TFA_KERNEL=variant)
            p = subprocess.run([sys.executable, "-c", SCHEDULE_RUN], env=env, capture_output=True, text=True,
                               timeout=1200)
            assert p.returncode == 0, p.stderr[-3000:]
            outs[variant] = torch.load(path)
    for name, r in auto_runs.items():
        want = portable(r)
        for variant, code in (("classic", 0), ("persist", 4)):
            got = outs[variant][name]
            assert got["variant"] == code, (name, variant)
            for x in ("out", "lse", "q_rot"):
                if want[x] is None:
                    assert got[x] is None
                else:
                    assert torch.equal(bits(got[x]), bits(want[x])), (name, variant, x)


NEGATIVE = ["dense_causal_b8", "varlen_short", "cache_sq200_causal", "varlen_cache_mixed", "fp8_d64_splits",
            "fp8_varlen_cache_mixed"]


@pytest.mark.gpu
@pytest.mark.parametrize("name", NEGATIVE)
def test_checker_rejects_kernel_result_against_wrong_reference(auto_runs, name):
    """The kernel's own result, against a reference that is wrong by one key or one head mapping: rejected.  Only the
    reference changes."""
    r = auto_runs[name]
    kw = BY_NAME[name].kw
    assert kw["causal"] and kw["Hkv"] > 1 and kw["Hq"] // kw["Hkv"] > 1
    for what, mut in (("causal offset +1", dict(shift=1)), ("kv head h % Hkv", dict(heads="mod")),
                      ("one key short", "drop_last")):
        verdict = check_workload(r, mut)
        assert not verdict.ok, f"{name}: {what} passes (ratio {verdict.ratio:.3f}, LSE {verdict.lse_err:.2e})"


# ------------------------------------------------------------------ GPU: tile edges ------------------------------------

EDGES = [1, 63, 64, 65, 127, 128, 129, 191, 192, 193, 255, 256, 257]
PAIRS = [(sq, sk) for sq in EDGES for sk in EDGES]


def _check_rows(fails, label, out, lse, ref, kind, worst):
    v = compare(out, lse, ref, kind)
    worst[0], worst[1] = max(worst[0], v.ratio), max(worst[1], v.lse_err)
    if not v.ok:
        fails.append(f"{label}: {v.msg}")


@pytest.mark.gpu
@pytest.mark.parametrize("causal", [False, True])
@pytest.mark.parametrize("D", [64, 128])
def test_dense_tile_edges(tfa, D, causal):
    """Every (Sq, Sk) pair of tile edges, GQA group 2, the dtype alternating, 16-bit and fp32 output."""
    fails, worst = [], [0.0, 0.0]
    for idx, (Sq, Sk) in enumerate(PAIRS):
        kind = ("bf16", "fp16")[idx % 2]
        q, k, v = make_inputs(2, 4, 2, Sq, Sk, D, kind, seed=idx)
        ref = reference(q, k, v, causal, D ** -0.5)
        for f32 in (False, True):
            out, lse = tfa.attn_fwd(q, k, v, causal, D ** -0.5, num_splits=1, out_fp32=f32)
            _check_rows(fails, f"Sq {Sq} Sk {Sk} {kind} f32={f32}", out, lse, ref, kind, worst)
    print(f"\n[float64 reference] dense edges D {D} causal {causal}: max err/budget {worst[0]:.3f}, "
          f"max |dLSE| {worst[1]:.2e}")
    assert not fails, f"{len(fails)} failing: " + "; ".join(fails[:8])


@pytest.mark.gpu
@pytest.mark.parametrize("causal", [False, True])
def test_split_kv_tile_edges(tfa, causal):
    """Sk = 128 t +- 1 with 2, 3 and 5 splits, among them every split count whose last split holds one KV tile."""
    fails, worst, one_tile = [], [0.0, 0.0], set()
    D, kind = (128, "bf16") if causal else (64, "fp16")
    for t in range(2, 10):
        for Sk in (128 * t - 1, 128 * t + 1):
            for ns in (2, 3, 5):
                for Sq in (1, 129):
                    q, k, v = make_inputs(1, 4, 2, Sq, Sk, D, kind, seed=Sk * 7 + ns + Sq)
                    f32 = (t + ns) % 2 == 0
                    out, lse, n = tfa.attn_fwd(q, k, v, causal, D ** -0.5, num_splits=ns, out_fp32=f32,
                                               return_splits=True)
                    nkv = -(-Sk // 128)
                    assert 1 < n <= ns
                    tiles = -(-nkv // n)
                    if nkv - (n - 1) * tiles == 1:
                        one_tile.add(n)
                    ref = reference(q, k, v, causal, D ** -0.5)
                    _check_rows(fails, f"Sq {Sq} Sk {Sk} splits {n} f32={f32}", out, lse, ref, kind, worst)
    print(f"\n[float64 reference] split-KV edges causal {causal}: max err/budget {worst[0]:.3f}, "
          f"max |dLSE| {worst[1]:.2e}")
    assert {2, 3, 5} <= one_tile            # 4 too: 5 asked of 7 tiles runs 4 splits of 2, 2, 2, 1
    assert not fails, f"{len(fails)} failing: " + "; ".join(fails[:8])


@pytest.mark.gpu
@pytest.mark.parametrize("causal", [False, True])
def test_varlen_tile_edges(tfa, causal):
    """The 169 edge pairs as the sequences of one varlen call."""
    lq, lk = [p[0] for p in PAIRS], [p[1] for p in PAIRS]
    D, kind = (128, "bf16") if causal else (64, "fp16")
    q, k, v, cu_q, cu_k = make_batch(lq, lk, 4, 2, D, kind, seed=31)
    out, lse = tfa.attn_varlen_fwd(q, k, v, cu_q, cu_k, max(lq), causal, D ** -0.5, out_fp32=not causal)
    fails, worst = [], [0.0, 0.0]
    for (q0, q1), (k0, k1) in zip(offsets(lq), offsets(lk)):
        ref = reference(seq(q, q0, q1), seq(k, k0, k1), seq(v, k0, k1), causal, D ** -0.5)
        _check_rows(fails, f"Sq {q1 - q0} Sk {k1 - k0}", out[q0:q1].permute(1, 0, 2)[None], lse[:, q0:q1][None], ref,
                    kind, worst)
    print(f"\n[float64 reference] varlen edges causal {causal}: max err/budget {worst[0]:.3f}, "
          f"max |dLSE| {worst[1]:.2e}")
    assert not fails, f"{len(fails)} failing: " + "; ".join(fails[:8])


@pytest.mark.gpu
@pytest.mark.parametrize("causal,append", [(True, True), (False, False)])
def test_varlen_cache_tile_edges(tfa, causal, append):
    """The edge pairs as (query rows, cached length) of one varlen-cache call, page 128, so the cached lengths sit at
    page - 1, page, page + 1 and twice that; with the append each sequence then holds Sk + Sq keys."""
    sq, lens = [p[0] for p in PAIRS], [p[1] for p in PAIRS]
    kw = dict(sq=sq, lens=lens, Hq=4, Hkv=2, D=128 if causal else 64, kind="fp16" if causal else "bf16", page=128,
              causal=causal, append=append)
    r = run_workload(tfa, W("edges", "varlen_cache", 41, kw))
    verdict = check_workload(r)
    print(f"\n[float64 reference] varlen-cache edges causal {causal}: max err/budget {verdict.ratio:.3f}, "
          f"max |dLSE| {verdict.lse_err:.2e}")
    assert verdict.ok, verdict.msg


@pytest.mark.gpu
@pytest.mark.parametrize("Sq", [1, 63, 64, 65, 128, 129])
def test_cache_tile_edges(tfa, Sq):
    """One cache call per Sq, with the sequences' lengths at tile and page edges (key-less causal rows included)."""
    lens = [0, 1, 63, 64, 65, 127, 128, 129, 255, 256, 257]
    for causal in (False, True):
        kind, D = ("bf16", 128) if causal else ("fp16", 64)
        kw = dict(lens=lens, Sq=Sq, Hq=4, Hkv=2, D=D, kind=kind, page=128, causal=causal)
        r = run_workload(tfa, W("edges", "cache", 50 + Sq, kw))
        verdict = check_workload(r)
        print(f"\n[float64 reference] cache edges Sq {Sq} causal {causal}: max err/budget {verdict.ratio:.3f}, "
              f"max |dLSE| {verdict.lse_err:.2e}")
        assert verdict.ok, f"causal {causal}: {verdict.msg}"
