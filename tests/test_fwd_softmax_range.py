"""Every sm_90a forward mode on logits that move the running max, and at the edges of the accepted softmax scale.

The float64-reference suites draw q, k and v from N(0, 0.5^2): at D = 128 every row's softmax is then almost uniform
and the lazy rescale (fa_fwd_sm90.cuh, `(mx - m) * c > 8`) never fires.  Here the logits of each sequence are planted
as a function of the key index j counted from the sequence's first key, which is the index every mode tiles by.

Planting.  The last two dimensions of q and k carry the pattern (they sit above any rotary_dim used here, so rotary
leaves them alone); the others hold N(0, 0.5^2) noise.  A pattern gives every key a target logit u_j in log2 units
(exponent units of the kernel, c = fp32(scale * log2 e)); "peak" keys have no noise, so their score is exactly
k[D-2] + k[D-1] (two 16-bit values, the second the rounding rest of the first), which the kernel's fp32 S holds
exactly.  The planted q dimensions carry a per-head factor that alternates 1 and 2^-6, so a persistent CTA runs items
of very different magnitude one after another.  FP8 inputs are planted in float, quantized as a caller would, and the
reference is built from the codes.

Emulation (`emulate`).  The kernel's online softmax per row, tile by tile from the item's first key, with the split
boundaries of tfa_attn_num_splits: fp32 m and l, l in the kernel's own order (each thread of a row's quad sums its
16 pairs of a tile into a fresh partial, adds it into l with Kahan's compensated add, and the quad is summed by two
xor-shuffles at the end; mutation running_l is the earlier order, one fp32 add per pair into l), m set on tile 0 (-FLT_MAX / c while a row has no key), the rescale
decision `(mx - m) c > 8` with alpha = 2^((m - mx) c), P rounded to 16 bits or e4m3, every split through an fp32 LSE
and the combine's formula.  It shows that each GPU workload's pattern drives what it is named for (coverage), that the budget
covers it (soundness), and that the checker rejects a wrong rescale (six mutations).

Budget.  The float64 suite's budget (test_fwd_float64_reference.budget, test_fwd_fp8.budget) plus two terms that are
negligible there and not at wide logits:
  * S error.  S is an fp32 wgmma accumulation.  Every logit moves by at most eta_ij = scale EPS_S sum_d |q_id k_jd|,
    so every weight by a factor within e^(+-2 eta_i) and O by (e^(2 eta_i) - 1) A, and LSE by eta_i (the FP8 budget's
    own eta term, with its EPS_ACC).  EPS_S is twice S_MEASURED_BOUND, the bound test_wgmma_16bit_s_accumulation
    asserts over 16-bit S chains measured on the H100.
  * Split combine.  A split reaches the combine as LSE_s = fp32(fp32(m scale) + logf(l)): each rounding is within
    2^-24 |LSE_s| (the two together 2 2^-24 |LSE_s|); the combine rounds LSE_s - max (2^-24 |LSE_s - max| <= 2^-23
    max |LSE|), so each weight w_s is off by a factor e^(+-eps_s), eps_s <= 6 2^-24 max(|LSE_s|, |max|).  O =
    sum w_s O_s / sum w_s then moves by at most 2 max_s eps_s A.  A split with LSE_s = LSE - Delta has weight
    e^-Delta and |LSE_s| <= |LSE| + Delta, and e^-Delta Delta <= 1, so the term is 12 2^-24 (|LSE_ref| + 1) A.

The scale range.  Every call accepts scale (s' for FP8) >= 0 while fp32(scale log2 e) is finite; the CPU tests take,
for every entry point, the largest float accepted and the next one up.  Key-less rows give exactly 0 / +inf at every
accepted scale (a row without a key gets m = -FLT_MAX / max(c, 1), so -m c stays finite); the GPU boundary test runs
one call per mode at 1e9 and at the largest accepted scale, on integer inputs whose S is exact, so the float64 reference
stays meaningful."""
import ctypes
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

import test_fwd_fp8 as F8
from test_fwd_float64_reference import L_SUM, OUT_EMIN, OUT_P, U_P, guarded, lse_bound, reference
from test_kvcache_fp8 import FP8, bits, quantize
from test_kvcache_rotary import positions, rope, rope_tables
from test_varlen import offsets

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LOG2E = 1.4426950408889634
S_MEASURED_BOUND = 2.0 ** -19   # per 16-bit S chain, relative to sum |a b|: 1.79x the worst measured (1.07e-6, fp16,
                                # K = 128, H100 80GB HBM3 at 700 W), half the budget's EPS_S
EPS_S = 2 * S_MEASURED_BOUND
K_COMBINE = 12 * 2.0 ** -24
TINY = 2.0 ** -6                # the planted magnitude of every other head
BN = 128


def _m_none(c):
    """The kernel's running max of a row without a key (run_forward's p.m_none): fp32(-FLT_MAX / max(c, 1)), one ulp
    toward zero when -m_none * max(c, 1) would exceed FLT_MAX."""
    top, c = float(np.finfo(np.float32).max), float(np.float32(max(c, 1.0)))
    r = np.float32(np.float32(-top) / np.float32(c))
    return np.nextafter(r, np.float32(0)) if float(r) * c < -top else r


def c_of(scale):
    """The kernel's exponent scale c = fp32(scale * log2 e), floored at 1e-30 (scale 0)."""
    return max(float(np.float32(scale) * np.float32(LOG2E)), 1e-30)


# ------------------------------------------------------------------ patterns --------------------------------------------

PATTERNS = ["spread", "late_outlier", "staircase_up", "staircase_under", "at_threshold", "sink", "descending",
            "shifted_1e2", "shifted_1e3", "shifted_1e4", "uniform"]


def targets(pattern, Sk):
    """(u, peak): target logit of each key in log2 units and which keys carry no noise, for one sequence of Sk keys.
    The tile of key j is j // 128 (the sequence's own tiles)."""
    j = np.arange(Sk)
    T = j // BN
    u = np.zeros(Sk)
    peak = np.zeros(Sk, dtype=bool)
    first = j % BN == 0
    if pattern == "late_outlier":
        u[-1], peak[-1] = 40.0, True
    elif pattern in ("staircase_up", "staircase_under", "descending"):
        step = {"staircase_up": 12.0, "staircase_under": 7.5 + 2.0 ** -5, "descending": -10.0}[pattern]
        u = step * T - 4.0 * ~first
        peak = first
    elif pattern == "at_threshold":
        # tile 2i+1 rises 8 + 2^-6 above the running max (rescale); tile 2i+2 8 - 2^-6 above it (no rescale, P ~ 2^8)
        m, top = 0.0, [0.0]
        for t in range(1, T.max() + 1):
            if t % 2:
                m += 8.0 + 2.0 ** -6
                top.append(m)
            else:
                top.append(m + 8.0 - 2.0 ** -6)
        u = np.array(top)[T] - 4.0 * ~first
        peak = first
    elif pattern == "sink":
        u[0], peak[0] = 20.0 * LOG2E, True
    elif pattern.startswith("shifted"):
        u[:] = float(pattern.split("_")[1]) * LOG2E
    return u, peak


@dataclass
class Seq:
    q: torch.Tensor            # (Hq, Sq, D) float64, the values the kernel sees (rounded / dequantized)
    k: torch.Tensor            # (Hkv, Sk, D)
    v: torch.Tensor


def plant(pattern, Hq, Hkv, Sq, Sk, D, scale, kind, seed):
    """One sequence's q, k, v in float64, before any rounding to what the kernel reads."""
    g = torch.Generator().manual_seed(seed)
    rn = lambda *s: torch.empty(s, dtype=torch.float64).normal_(0.0, 0.5, generator=g)
    q, k, v = rn(Hq, Sq, D), rn(Hkv, Sk, D), rn(Hkv, Sk, D)
    mu = torch.tensor([1.0 if h % 2 == 0 else TINY for h in range(Hq)], dtype=torch.float64)
    if pattern == "spread":
        q = q * torch.where(mu == 1.0, 30.0, 1.0)[:, None, None]
    if pattern == "staircase_up":         # rows 8..15 of every 16 climb 24 per tile, rows 0..7 see a flat row:
        q = q * 0.01                      # the two row halves of a thread get alpha = 2^-24 and 1
        mu = mu[:, None] * (torch.where(torch.arange(Sq) % 16 >= 8, 2.0, 0.0)[None] if Sq >= 16 else 2.0)
    else:
        mu = mu[:, None].expand(Hq, Sq)
    u, peak = targets(pattern, Sk)
    c = c_of(scale)
    q[..., D - 2:] = 0.0
    k[..., D - 2:] = 0.0
    if pattern.startswith("shifted"):
        raw = torch.tensor(u / c / 2)                      # two halves: each stays inside fp16's range
        k[..., D - 2] = raw
        k[..., D - 1] = raw
        q[..., D - 2:] = mu[..., None]
    elif pattern not in ("spread", "uniform"):
        k[:, torch.from_numpy(peak), :D - 2] = 0.0
        raw = torch.tensor(u / c)
        hi = raw.to(_dt(kind)).double()
        k[..., D - 2] = hi
        k[..., D - 1] = raw - hi
        q[..., D - 2:] = mu[..., None]
    return q, k, v


def fp8_scale(xs):
    """A caller's per-tensor scale: the largest magnitude maps to 448."""
    return float(np.float32(max(float(x.abs().max()) for x in xs) / 448.0))


def to_fp8(x, s):
    return (x.float() / s).clamp(-448, 448).to(FP8)


# ------------------------------------------------------------------ emulation -------------------------------------------

def _round_p(p, rnd):
    if rnd == "fp16":
        return p.astype(np.float16).astype(np.float64)
    return torch.from_numpy(p.astype(np.float32)).to(torch.bfloat16 if rnd == "bf16" else FP8).double().numpy()


@dataclass
class Trace:
    rescales: np.ndarray = None      # per row: rescale events
    near: list = field(default_factory=lambda: [0, 0])   # decisions within 2^-5 of the threshold: [above, at/below]
    max_p: float = 0.0               # largest P (the stale max's P included)
    small_p: int = 0                 # P below 2^-14 (fp16 subnormal) / below 2^-10 (e4m3 flushed to 0)
    lse_spread: float = 0.0          # largest |LSE_s - LSE_s'| over a row's splits


@np.errstate(invalid="ignore", over="ignore", divide="ignore")     # -inf - -inf: a row without a key
def emulate(s, vis, v, scale, rnd, splits=None, mutation=None):
    """s (H, R, K) exact scores (float64; rounded to fp32 here), vis (R, K) visibility, v (H, K, D); splits: list of
    key ranges (the kernel's split boundaries, tiles counted from key 0).  Returns O (H, R, D), LSE (H, R), Trace."""
    H, R, K = s.shape
    c = np.float32(c_of(scale))
    none = _m_none(float(c))
    s = np.where(vis[None], s.astype(np.float32), np.float32(-np.inf))
    splits = splits or [(0, K)]
    tr = Trace(rescales=np.zeros((H, R), dtype=int))
    small = 2.0 ** -14 if rnd != "e4m3" else 2.0 ** -10
    parts = []
    for (k0, k1) in splits:
        m = np.zeros((H, R), np.float32)
        m_old = m.copy()
        l = np.zeros((H, R, 4), np.float32)      # per thread of the row's quad: l and its Kahan compensation
        lc = np.zeros((H, R, 4), np.float32)
        o = np.zeros((H, R, v.shape[2]))
        for t0 in range(k0, k1, BN):
            st = s[:, :, t0:min(t0 + BN, k1)]
            mx = st.max(-1)
            if t0 == k0:
                m = np.maximum(mx, none).astype(np.float32)                 # a row without a key so far: none
                m_old = m.copy()
            else:
                d = (mx - m) if mutation == "raw_threshold" else (mx - m) * c
                n = d.astype(np.float32) > 8
                dd = ((mx - m) * c).astype(np.float64)
                tr.near[0] += int(((dd > 8) & (dd < 8 + 2 ** -5)).sum())
                tr.near[1] += int(((dd <= 8) & (dd > 8 - 2 ** -5)).sum())
                alpha = np.where(n, np.exp2(((m - mx) * c).astype(np.float32)), 1.0).astype(np.float32)
                tr.rescales += n
                m_old = np.where(n, m, m_old)
                m = np.where(n, mx, m)
                if mutation != "no_l_rescale":
                    l = (l * alpha[..., None]).astype(np.float32)
                    lc = (lc * alpha[..., None]).astype(np.float32)
                if mutation == "swap_halves":        # alpha of row r applied to row r ^ 8
                    idx = np.arange(R)
                    idx[:R // 16 * 16] ^= 8
                    alpha = alpha[:, idx]
                if mutation != "no_o_rescale":
                    o = o * alpha[..., None]
            nm = (-m * c).astype(np.float32)
            p = np.exp2((st.astype(np.float64) * float(c) + nm[..., None]).astype(np.float32)).astype(np.float32)
            p = np.where(np.isnan(p), 0.0, p)
            tr.max_p = max(tr.max_p, float(p.max()) if p.size else 0.0)
            tr.small_p += int(((p > 0) & (p < small)).sum())
            # thread tq of a row's quad holds the tile's columns 8 i + 2 tq + e (i < 16, e < 2) and adds them in pairs
            pad = np.zeros((H, R, BN), np.float32)
            pad[..., :p.shape[-1]] = p
            pairs = pad.reshape(H, R, 16, 4, 2)
            pairs = (pairs[..., 0] + pairs[..., 1]).astype(np.float32)          # (H, R, i, tq)
            if mutation == "running_l":          # the pairs straight into l, one fp32 add per pair
                for i in range(16):
                    l = (l + pairs[..., i, :]).astype(np.float32)
            else:                                # a fresh tile partial, then Kahan's compensated add into l
                t = pairs[..., 0, :]
                for i in range(1, 16):
                    t = (t + pairs[..., i, :]).astype(np.float32)
                y = (t - lc).astype(np.float32)
                u = (l + y).astype(np.float32)
                lc = ((u - l).astype(np.float32) - y).astype(np.float32)
                l = u
            o = o + np.einsum("hrk,hkd->hrd", _round_p(p, rnd), v[:, t0:min(t0 + BN, k1)])
        l = (l - lc).astype(np.float32)
        l = (l + l[..., [1, 0, 3, 2]]).astype(np.float32)                      # the two xor-shuffles of the quad
        l = (l + l[..., [2, 3, 0, 1]]).astype(np.float32)[..., 0]
        if mutation == "no_reset":               # item h starts from item h - 1's l and O (a persistent CTA's)
            l, o = l.copy(), o.copy()
            l[1:] += l[:-1].copy()
            o[1:] += o[:-1].copy()
        with np.errstate(divide="ignore"):
            ms = m_old if mutation == "stale_lse" else m
            lse = np.where(l > 0, (ms * np.float32(scale)).astype(np.float32) + np.log(l).astype(np.float32),
                           -np.inf if len(splits) > 1 else np.inf).astype(np.float32)
        inv = np.where(l > 0, 1.0 / np.where(l > 0, l, 1.0), 0.0)
        parts.append(((o * inv[..., None]).astype(np.float32), lse))
    if len(parts) == 1:
        return parts[0][0].astype(np.float64), parts[0][1].astype(np.float64), tr
    lses = np.stack([p[1] for p in parts])
    fin = np.isfinite(lses)
    if fin.any():
        lo, hi = np.where(fin, lses, np.inf).min(0), np.where(fin, lses, -np.inf).max(0)
        both = fin.sum(0) > 1
        tr.lse_spread = float((hi - lo)[both].max()) if both.any() else 0.0
    mm = lses.max(0)
    with np.errstate(invalid="ignore"):
        w = np.where(np.isfinite(mm)[None], np.exp((lses - mm[None]).astype(np.float32)), 0.0).astype(np.float32)
    ws = w.sum(0).astype(np.float32)
    o = sum(w[i][..., None].astype(np.float64) * parts[i][0] for i in range(len(parts)))
    o = np.where(ws[..., None] > 0, o / np.where(ws > 0, ws, 1)[..., None], 0.0)
    with np.errstate(divide="ignore"):
        lse = np.where(ws > 0, mm + np.log(np.where(ws > 0, ws, 1)), np.inf)
    return o, lse.astype(np.float32).astype(np.float64), tr


# ------------------------------------------------------------------ reference and budget --------------------------------

def full_reference(sq, causal, scale, fp8, ks=1.0, vs=1.0):
    """(O, LSE, A, extra, eta) for one sequence: extra = the 16-bit fp16-subnormal term or the FP8 E_P + E_PV terms."""
    q, k, v = sq.q[None], sq.k[None], sq.v[None]
    if fp8:
        return F8.fp8_reference(q, k, v, causal, scale, 1.0, 1.0)
    o, lse, a, sub, pv16 = reference(q, k, v, causal, scale)
    Hq, Hkv = q.shape[1], k.shape[1]
    kk = k[:, torch.arange(Hq) // (Hq // Hkv)]
    Sq, Sk = q.shape[2], k.shape[2]
    vis = (torch.arange(Sk)[None] <= torch.arange(Sq)[:, None] + Sk - Sq) if causal else torch.ones(Sq, Sk).bool()
    eta = ((q.abs().cpu() @ kk.abs().cpu().transpose(-1, -2)) * (scale * EPS_S)).masked_fill(~vis, 0.0).amax(-1)
    return o, lse, a, sub, eta.to(q.device), pv16


def budget(ref, kind, out16, fp8, split):
    o_ref, l_ref, a, extra, eta = ref[:5]
    if fp8:
        b = extra + torch.expm1(2 * eta)[..., None] * a + 2.0 ** -14 * a + L_SUM * a + 1e-6
    else:
        b = U_P[kind] * a + 2.0 ** -14 * a + L_SUM * a + ref[5] + 1e-6 + torch.expm1(2 * eta)[..., None] * a
        if kind == "fp16":
            b = b + 2.0 ** -25 * extra
    if split:
        b = b + K_COMBINE * (l_ref.abs().masked_fill(torch.isinf(l_ref), 0.0) + 1.0)[..., None] * a
    if out16:
        x = o_ref.abs() + b
        _, e = torch.frexp(x)
        e = torch.where(x > 0, e.clamp(min=OUT_EMIN[kind]), torch.full_like(e, OUT_EMIN[kind]))
        b = b + 0.5 * torch.ldexp(torch.ones_like(x), e - OUT_P[kind])
    return b


def check(out, lse, ref, kind, fp8, split):
    """(ok, worst err / budget, worst |dLSE|, message) of out (1, Hq, S, D), lse (1, Hq, S)."""
    o_ref, l_ref = ref[0], ref[1]
    o, l = out.to(torch.float64).to(o_ref.device), lse.to(torch.float64).to(o_ref.device)
    keyless = torch.isinf(l_ref)
    if keyless.any() and not (bool((o[keyless] == 0).all()) and bool(torch.isposinf(l[keyless]).all())):
        return False, math.inf, math.inf, "a row without keys is not 0 / +inf"
    b = budget(ref, kind, out.dtype != torch.float32, fp8, split)
    ratio = torch.nan_to_num((o - o_ref).abs() / b, nan=math.inf).masked_fill(keyless[..., None], 0.0)
    lerr = torch.nan_to_num((l - l_ref).abs(), nan=math.inf).masked_fill(keyless, 0.0)
    lb = ref[4] + lse_bound(l_ref.masked_fill(keyless, 0.0))
    r, le = float(ratio.max()) if ratio.numel() else 0.0, float(lerr.max()) if lerr.numel() else 0.0
    if r > 1.0:
        at = np.unravel_index(int(ratio.argmax()), tuple(ratio.shape))
        return False, r, le, f"O over budget: ratio {r:.3f} at {tuple(int(x) for x in at)}"
    if bool((lerr > lb).any()):
        return False, r, le, f"LSE off by {le:.3e}"
    return True, r, le, ""


# ------------------------------------------------------------------ workloads -------------------------------------------

@dataclass
class W:
    name: str
    mode: str                # dense, varlen, cache, varlen_cache
    pattern: str
    kw: dict


def _lens_varlen(seed):
    rng = random.Random(seed)
    lq = [300] + [rng.choice([1, 64, 129, 200, 400]) for _ in range(5)]
    lk = [700] + [rng.choice([130, 300, 600, 900]) for _ in range(5)]
    return lq, lk


def _lens_cache(seed, B, page):
    rng = random.Random(seed)
    edges = [1, page - 1, page, page + 1, 2 * page + 1]
    return edges + [rng.randint(300, 1200) for _ in range(B - len(edges))]


def workloads():
    out = []
    for i, pat in enumerate(PATTERNS):
        big = pat == "staircase_up"                        # the >= 3 items per SM workload of each mode
        d128 = i % 2 == 0
        D = 128 if d128 else 64
        kind = "bf16" if i % 2 == 0 else "fp16"
        causal = i % 3 != 1
        ns = 1 if big else (1, 3, 5)[i % 3]    # staircase_up: every tile of a row in one split
        f32 = i % 4 == 3
        B, Hq = (4, 16) if big else (1, 4)
        out.append(W(f"dense_{pat}", "dense", pat, dict(B=B, Hq=Hq, Hkv=Hq // 2, Sq=1024 if big else 700,
                                                        Sk=1024 if big else 1100, D=D, kind=kind, causal=causal,
                                                        ns=ns, f32=f32)))
        lq, lk = _lens_varlen(200 + i)
        if big:
            lq, lk = lq * 8, lk * 8
        out.append(W(f"varlen_{pat}", "varlen", pat, dict(lq=lq, lk=lk, Hq=8 if big else 4, Hkv=2, D=D, kind=kind,
                                                          causal=causal, f32=f32)))
        if pat == "uniform":
            continue                                       # the cache calls take D^-0.5 here
        page = (128, 256)[i % 2]
        B = 48 if big else 8
        Sq, snew = ((1, 1), (4, 4), (200, 0))[i % 3]
        cns = 3 if Sq == 1 and not big else 1
        out.append(W(f"cache_{pat}", "cache", pat, dict(lens=_lens_cache(300 + i, B, page), Sq=Sq, snew=snew,
                                                        Hq=16, Hkv=4, D=D, kind=kind, page=page, causal=True,
                                                        ns=cns)))
        sq = ([300, 64, 1, 1, 129, 1] * (8 if big else 1))
        out.append(W(f"varlen_cache_{pat}", "varlen_cache", pat,
                     dict(sq=sq, lens=_lens_cache(400 + i, len(sq), 256)[:len(sq)], Hq=16 if big else 8, Hkv=4, D=D,
                          kind=kind, page=256, causal=True, append=True)))
        if not pat.startswith("shifted") or pat == "shifted_1e2":
            rd, il = ((64, False), (32, True))[i % 2]
            out.append(W(f"rotary_{pat}", "cache", pat, dict(lens=_lens_cache(500 + i, 48 if big else 8, 256),
                                                             Sq=1, snew=1, Hq=16, Hkv=4, D=D, kind=kind, page=256,
                                                             causal=True, ns=1, rotary=(rd, il))))
        if pat in ("at_threshold",) or pat.startswith("shifted"):
            continue                                       # e4m3 holds neither the 2^-6 steps nor 1e3-nat offsets
        fp8 = "auto"
        out.append(W(f"fp8_dense_{pat}", "dense", pat, dict(B=B if big else 1, Hq=Hq, Hkv=Hq // 2,
                                                            Sq=1024 if big else 500, Sk=1024 if big else 900, D=D,
                                                            kind=kind, causal=causal, ns=ns, f32=False, fp8=fp8)))
        lq, lk = _lens_varlen(600 + i)
        if big:
            lq, lk = lq * 8, lk * 8
        out.append(W(f"fp8_varlen_{pat}", "varlen", pat, dict(lq=lq, lk=lk, Hq=8 if big else 4, Hkv=2, D=D,
                                                              kind=kind, causal=causal, fp8=fp8)))
        out.append(W(f"fp8_cache_{pat}", "cache", pat, dict(lens=_lens_cache(700 + i, 48 if big else 8, 128),
                                                            Sq=1, snew=1, Hq=16, Hkv=4, D=D, kind=kind, page=128,
                                                            causal=True, ns=1 if big else 3, kvfp8="auto")))
        out.append(W(f"fp8_varlen_cache_{pat}", "varlen_cache", pat,
                     dict(sq=sq, lens=_lens_cache(800 + i, len(sq), 256)[:len(sq)], Hq=16 if big else 8, Hkv=4, D=D,
                          kind=kind, page=256, causal=True, append=True, kvfp8="auto")))
        # e4m3 queries against the FP8 cache: q, k and v quantized, both products on FP8 wgmma
        out.append(W(f"qkv8_cache_{pat}", "cache", pat, dict(lens=_lens_cache(900 + i, 48 if big else 8, 128),
                                                             Sq=1, snew=1, Hq=16, Hkv=4, D=D, kind=kind, page=128,
                                                             causal=True, ns=1 if big else 3, fp8=fp8, kvfp8=fp8)))
        out.append(W(f"qkv8_varlen_cache_{pat}", "varlen_cache", pat,
                     dict(sq=sq, lens=_lens_cache(1000 + i, len(sq), 256)[:len(sq)], Hq=16 if big else 8, Hkv=4,
                          D=D, kind=kind, page=256, causal=True, append=True, fp8=fp8, kvfp8=fp8)))
    return out


WORKLOADS = workloads()
BY_NAME = {w.name: w for w in WORKLOADS}


def _scale(w):
    """uniform: 0; staircase_up: 16, where c = 23 and a threshold in raw score units (8 c in log2 units) would let P
    overflow fp32."""
    return {"uniform": 0.0, "staircase_up": 16.0}.get(w.pattern, w.kw["D"] ** -0.5)


def sequences(w):
    """Per sequence: (Sq, Sk, seed) of workload w; cache modes count the appended keys in Sk."""
    kw = w.kw
    if w.mode == "dense":
        return [(kw["Sq"], kw["Sk"], 1000 * b + 7) for b in range(kw["B"])]
    if w.mode == "varlen":
        return [(a, b, 1000 * i + 11) for i, (a, b) in enumerate(zip(kw["lq"], kw["lk"]))]
    if w.mode == "cache":
        return [(kw["Sq"], L + kw["snew"], 1000 * b + 13) for b, L in enumerate(kw["lens"])]
    return [(n, L + (n if kw["append"] else 0), 1000 * b + 17) for b, (n, L) in enumerate(zip(kw["sq"], kw["lens"]))]


def planted(w):
    """The workload's sequences as the kernel reads them: a list of (Seq of float64 values, codes), and the FP8 scales
    (q, k, v).  FP8 attention: all three quantized, codes (q8, k8, v8); an FP8 cache: q 16-bit, codes (None, k8, v8);
    16-bit: codes None.  Scales "auto" map each tensor's largest magnitude over the workload to 448."""
    kw = w.kw
    raw = [plant(w.pattern, kw["Hq"], kw["Hkv"], Sq, Sk, kw["D"], _scale(w), kw["kind"], seed)
           for Sq, Sk, seed in sequences(w)]
    dt = _dt(kw["kind"])
    f8 = kw.get("fp8") or kw.get("kvfp8")
    if not f8:
        return [(Seq(*(x.to(dt).double() for x in t)), None) for t in raw], None
    sc = [fp8_scale([t[i] for t in raw]) for i in range(3)] if f8 == "auto" else list(f8)
    res = []
    for q, k, v in raw:
        k8, v8 = to_fp8(k, sc[1]), to_fp8(v, sc[2])
        kd, vd = k8.double() * sc[1], v8.double() * sc[2]
        if kw.get("fp8"):
            q8 = to_fp8(q, sc[0])
            res.append((Seq(q8.double() * sc[0], kd, vd), (q8, k8, v8)))
        else:
            res.append((Seq(q.to(dt).double(), kd, vd), (None, k8, v8)))
    return res, sc


def split_ranges(w, Sk):
    """The key ranges of the splits of one sequence (dense and cache split-KV: tiles of the whole capacity)."""
    ns = w.kw.get("ns", 1)
    if w.mode == "dense":
        nkv = -(-w.kw["Sk"] // BN)
    elif w.mode == "cache" and ns > 1:
        nkv = _mbps(w.kw["lens"], [w.kw["snew"]] * len(w.kw["lens"]), w.kw["page"]) * w.kw["page"] // BN
    else:
        return None
    n = min(ns, nkv)
    if n < 2:
        return None
    tiles = -(-nkv // n)
    r = [(BN * tiles * i, min(BN * tiles * (i + 1), Sk)) for i in range(n)]
    return [x for x in r if x[0] < x[1]] or None


def _mbps(lens, n_app, page):
    """Block-table width of a cache workload: one page more than its longest sequence needs."""
    return -(-max(L + a for L, a in zip(lens, n_app)) // page) + 1


def _table(B, mbps, seed, spare=3):
    g = torch.Generator().manual_seed(seed)
    nblk = B * mbps + spare
    return torch.randperm(nblk, generator=g)[:B * mbps].view(B, mbps).to(torch.int32), nblk


# ------------------------------------------------------------------ runners ---------------------------------------------

def _dt(kind):
    return torch.bfloat16 if kind == "bf16" else torch.float16


def run(tfa, w, scale=None):
    """Run workload w on the GPU.  Returns out, lse, q_rot (or None), the launch variant, the work items, and per
    sequence (out (1, Hq, Sq, D), lse (1, Hq, Sq), Seq the reference reads)."""
    kw = w.kw
    scale = _scale(w) if scale is None else scale
    seqs, sc = planted(w)
    D, kind, Hq, Hkv = kw["D"], kw["kind"], kw["Hq"], kw["Hkv"]
    dt = _dt(kind)
    fp8 = kw.get("fp8")
    qkw = dict(q_scale=sc[0], k_scale=sc[1], v_scale=sc[2], out_dtype=dt) if fp8 else {}
    q_rot = None
    if w.mode == "dense":
        if fp8:
            q, k, v = (torch.stack([c[i] for _, c in seqs]).cuda() for i in range(3))
        else:
            q, k, v = (torch.stack([getattr(s, x) for s, _ in seqs]).to(dt).cuda() for x in "qkv")
        f32 = kw.get("f32", False)
        ob, out = guarded(tuple(q.shape), torch.float32 if f32 else dt)
        lb, lse = guarded((len(seqs), Hq, q.shape[2]), torch.float32)
        _, _, n = tfa.attn_fwd(q, k, v, kw["causal"], scale, num_splits=kw["ns"], out_fp32=f32, out=out, lse=lse,
                               return_splits=True, **qkw)
        items = -(-q.shape[2] // BN) * len(seqs) * Hq * n
        per = [(out[b:b + 1], lse[b:b + 1]) for b in range(len(seqs))]
        guards = [(ob, out), (lb, lse)]
    elif w.mode == "varlen":
        if fp8:
            q, k, v = (torch.cat([c[i].permute(1, 0, 2) for _, c in seqs]).cuda() for i in range(3))
        else:
            q, k, v = (torch.cat([getattr(s, x).permute(1, 0, 2) for s, _ in seqs]).to(dt).cuda() for x in "qkv")
        lq, lk = kw["lq"], kw["lk"]
        cu_q = torch.tensor([0] + np.cumsum(lq).tolist(), dtype=torch.int32, device="cuda")
        cu_k = torch.tensor([0] + np.cumsum(lk).tolist(), dtype=torch.int32, device="cuda")
        f32 = kw.get("f32", False) and not fp8
        ob, out = guarded((sum(lq), Hq, D), torch.float32 if f32 else dt)
        lb, lse = guarded((Hq, sum(lq)), torch.float32)
        tfa.attn_varlen_fwd(q, k, v, cu_q, cu_k, max(lq), kw["causal"], scale, out_fp32=f32, out=out, lse=lse, **qkw)
        items = -(-max(lq) // BN) * len(lq) * Hq
        per = [(out[a:b].permute(1, 0, 2)[None], lse[:, a:b][None]) for a, b in offsets(lq)]
        guards = [(ob, out), (lb, lse)]
    else:
        out, lse, q_rot, items, per, guards, seqs = _run_cache(tfa, w, seqs, sc, scale)
    variant = tfa.lib().tfa_internal_last_variant()
    torch.cuda.synchronize()
    for buf, view in guards:
        assert not torch.isnan(view).any(), f"{w.name}: a row of out / lse was not written"
        assert torch.isnan(buf[:512]).all() and torch.isnan(buf[-512:]).all(), f"{w.name}: a guard element changed"
    return dict(out=out, lse=lse, q_rot=q_rot, variant=variant, items=items,
                seqs=[(o, l, s) for (o, l), (s, _) in zip(per, seqs)])


def _run_cache(tfa, w, seqs, sc, scale):
    """Both cache calls: the planted keys [0, L) sit in a paged pool (NaN / 0x7f elsewhere), keys [L, K) are
    appended; the reference reads the pool back after the call, and the appends must be exact."""
    kw = w.kw
    D, kind, Hq, Hkv, page = kw["D"], kw["kind"], kw["Hq"], kw["Hkv"], kw["page"]
    dt = _dt(kind)
    kvfp8 = kw.get("kvfp8")
    qkv8 = bool(kw.get("fp8"))      # e4m3 q codes against the FP8 cache, out in the workload's dtype
    qkw = dict(q_scale=sc[0], out_dtype=dt) if qkv8 else {}
    varlen = w.mode == "varlen_cache"
    B = len(seqs)
    n_app = [s.q.shape[1] if (varlen and kw["append"]) else (0 if varlen else kw["snew"]) for s, _ in seqs]
    lens = [s.k.shape[1] - a for (s, _), a in zip(seqs, n_app)]
    mbps = _mbps(lens, n_app, page)
    table, nblk = _table(B, mbps, 99 + B)
    pdt = FP8 if kvfp8 else dt
    fill = 0x7F if kvfp8 else None
    pools = []
    for x in ("k", "v"):
        pool = torch.empty((nblk, page, Hkv, D), dtype=pdt)
        if kvfp8:
            pool.view(torch.uint8).fill_(fill)
        else:
            pool.fill_(float("nan"))
        flat = pool.view(torch.uint8) if kvfp8 else pool
        for b, ((s, codes), L) in enumerate(zip(seqs, lens)):
            src = codes[1 if x == "k" else 2] if kvfp8 else getattr(s, x).to(dt)
            for j0 in range(0, L, page):
                j1 = min(L, j0 + page)
                blk = int(table[b, j0 // page])
                val = src[:, j0:j1].permute(1, 0, 2)
                flat[blk, :j1 - j0] = val.view(torch.uint8) if kvfp8 else val
        pools.append(pool.cuda())
    kp, vp = pools
    new = [(s.k[:, L:].permute(1, 0, 2), s.v[:, L:].permute(1, 0, 2)) for (s, _), L in zip(seqs, lens)]
    if kvfp8:    # the append quantizes the 16-bit new keys itself: hand it values whose quantization is the code
        new = [(kn.to(dt), vn.to(dt)) for kn, vn in new]
    else:
        new = [(kn.to(dt), vn.to(dt)) for kn, vn in new]
    ks, vs = (sc[1], sc[2]) if kvfp8 else (1.0, 1.0)
    k1, v1 = kp.clone(), vp.clone()
    sl = torch.tensor(lens, dtype=torch.int32, device="cuda")
    rotary = kw.get("rotary")
    q_rot = None
    if varlen:
        q = (torch.cat([c[0].permute(1, 0, 2) for _, c in seqs]) if qkv8 else
             torch.cat([s.q.permute(1, 0, 2) for s, _ in seqs]).to(dt)).cuda()
        cu = torch.tensor([0] + np.cumsum(kw["sq"]).tolist(), dtype=torch.int32, device="cuda")
        kn = torch.cat([x[0] for x in new]).cuda() if kw["append"] else None
        vn = torch.cat([x[1] for x in new]).cuda() if kw["append"] else None
        total = q.shape[0]
        ob, out = guarded((total, Hq, D), dt)
        lb, lse = guarded((Hq, total), torch.float32)
        tfa.attn_varlen_kvcache_fwd(q, k1, v1, cu, max(kw["sq"]), sl, table.cuda(), kn, vn, is_causal=kw["causal"],
                                    scale=scale, out=out, lse=lse, k_scale=ks, v_scale=vs, **qkw)
        items = -(-max(kw["sq"]) // BN) * B * Hq
        per = [(out[a:b].permute(1, 0, 2)[None], lse[:, a:b][None]) for a, b in offsets(kw["sq"])]
        qs = [s.q for s, _ in seqs]
    else:
        Sq, snew = kw["Sq"], kw["snew"]
        q = (torch.stack([c[0].permute(1, 0, 2) for _, c in seqs]) if qkv8 else
             torch.stack([s.q.permute(1, 0, 2) for s, _ in seqs]).to(dt)).cuda()
        kn = torch.stack([x[0] for x in new]).cuda() if snew else None
        vn = torch.stack([x[1] for x in new]).cuda() if snew else None
        rot = {}
        if rotary:
            rd, il = rotary
            seqlen_ro = mbps * page + 64
            cos, sin = rope_tables(seqlen_ro, rd, kind)
            q_rot = torch.full_like(q, float("nan"))
            rot = dict(rotary_cos=cos, rotary_sin=sin, rotary_interleaved=il, q_rot=q_rot)
        ob, out = guarded(tuple(q.shape), dt)
        lb, lse = guarded((B, Hq, Sq), torch.float32)
        _, _, n = tfa.attn_kvcache_fwd(q, k1, v1, sl, table.cuda(), kn, vn, is_causal=kw["causal"], scale=scale,
                                       num_splits=kw.get("ns", 1), out=out, lse=lse, return_splits=True, k_scale=ks,
                                       v_scale=vs, **rot, **qkw)
        items = -(-Sq // BN) * B * Hq * n
        per = [(out[b:b + 1].permute(0, 2, 1, 3), lse[b:b + 1]) for b in range(B)]
        qs = [s.q for s, _ in seqs]
        if rotary:
            cap = mbps * page
            qa = rope(q, positions(lens, cap, snew, Sq, True, True, seqlen_ro), cos, sin, rd, il)
            torch.cuda.synchronize()
            assert torch.equal(bits(q_rot), bits(qa)), f"{w.name}: q_rot differs from the eager fp32 rotation"
            kn = rope(kn, positions(lens, cap, snew, snew, True, False, seqlen_ro), cos, sin, rd, il)
            qs = [qa[b].permute(1, 0, 2).double().cpu() for b in range(B)]
        new = [(kn[b], vn[b]) for b in range(B)] if snew else new
    torch.cuda.synchronize()
    # the pools after the call: the planted rows and every appended row exact, nothing else touched
    for pool0, pool1, x, xs in ((kp, k1, 0, ks), (vp, v1, 1, vs)):
        want = pool0.clone()
        wv = want.view(torch.uint8) if kvfp8 else want
        for b, L in enumerate(lens):
            t = new[b][x]
            if t is None or t.shape[0] == 0:
                continue
            t = quantize(t, xs).view(torch.uint8).cuda() if kvfp8 else t.cuda()
            for i in range(t.shape[0]):
                j = L + i
                wv[int(table[b, j // page]), j % page] = t[i]
        assert torch.equal(bits(pool1), bits(want)), f"{w.name}: the appended cache rows"
    refs = []
    for b, L in enumerate(lens):
        K = L + n_app[b]
        kk, vv = [], []
        for pool, xs in ((k1, ks), (v1, vs)):
            rows = pool[table[b].long().cuda()].reshape(mbps * page, Hkv, D)[:K].permute(1, 0, 2)
            (kk if pool is k1 else vv).append((rows.float().double() * xs).cpu())
        refs.append((Seq(qs[b].double().cpu(), kk[0], vv[0]), None))
    guards = [(ob, out), (lb, lse)]
    return out, lse, q_rot, items, per, guards, refs


def portable(r):
    return {x: (r[x].cpu() if r[x] is not None else None) for x in ("out", "lse", "q_rot")} | {"variant": r["variant"]}


def check_run(w, r):
    kw = w.kw
    fp8 = bool(kw.get("fp8"))
    worst = [True, 0.0, 0.0, ""]
    for i, (out, lse, s) in enumerate(r["seqs"]):
        split = split_ranges(w, s.k.shape[1]) is not None
        ref = full_reference(Seq(s.q.cuda(), s.k.cuda(), s.v.cuda()), kw["causal"], _scale(w), fp8)
        ok, ra, le, msg = check(out, lse, ref, kw["kind"], fp8, split)
        worst[1], worst[2] = max(worst[1], ra), max(worst[2], le)
        if not ok and worst[0]:
            worst[0], worst[3] = False, f"sequence {i}: {msg}"
    return worst


# ------------------------------------------------------------------ CPU: coverage, soundness, sensitivity -------------

def _vis(Sq, Sk, causal):
    return (np.arange(Sk)[None] <= np.arange(Sq)[:, None] + Sk - Sq) if causal else np.ones((Sq, Sk), bool)


def _emulate_seq(w, s, mutation=None):
    kw = w.kw
    Hq, Hkv = kw["Hq"], kw["Hkv"]
    q, k, v = s.q.numpy(), s.k.numpy(), s.v.numpy()
    h = np.arange(Hq) // (Hq // Hkv)
    sc = np.einsum("hrd,hkd->hrk", q, k[h])
    rnd = "e4m3" if kw.get("fp8") else kw["kind"]
    return emulate(sc, _vis(q.shape[1], k.shape[1], kw["causal"]), v[h], _scale(w), rnd,
                   split_ranges(w, k.shape[1]), mutation)


def _emulated_check(w, mutation=None, limit=None):
    """The emulation of every sequence (or the first `limit`) against the float64 reference: (ok, ratio, traces)."""
    kw = w.kw
    fp8 = bool(kw.get("fp8"))
    ok, worst, traces = True, 0.0, []
    seqs = sorted(planted(w)[0], key=lambda x: -x[0].k.shape[1])      # the longest sequences first
    for s, _ in seqs[:limit]:
        o, lse, tr = _emulate_seq(w, s, mutation)
        traces.append(tr)
        ref = full_reference(s, kw["causal"], _scale(w), fp8)
        dt = torch.float32 if kw.get("f32") and not kw.get("fp8") else _dt(kw["kind"])
        good, r, _, _ = check(torch.from_numpy(o).to(dt)[None], torch.from_numpy(lse).float()[None], ref, kw["kind"],
                              fp8, split_ranges(w, s.k.shape[1]) is not None)
        ok, worst = ok and good, max(worst, r)
    return ok, worst, traces


def _cpu_workload(w):
    """A shorter copy of w for the CPU emulation: the same per-sequence shapes and pattern, fewer sequences."""
    kw = dict(w.kw)
    if w.mode == "dense":
        kw["B"] = 1
    elif w.mode == "varlen":
        kw["lq"], kw["lk"] = kw["lq"][:3], kw["lk"][:3]
    elif w.mode == "cache":
        kw["lens"] = kw["lens"][:6]
    else:
        kw["sq"], kw["lens"] = kw["sq"][:6], kw["lens"][:6]
    return W(w.name, w.mode, w.pattern, kw)


@pytest.mark.parametrize("name", [w.name for w in WORKLOADS])
def test_pattern_drives_its_branch_and_budget_covers_emulation(name):
    """Coverage at the GPU shapes: the emulation of each workload shows the branch its pattern is named for, and
    stays within budget."""
    w = _cpu_workload(BY_NAME[name])
    ok, ratio, traces = _emulated_check(w)
    assert ok, f"{name}: the emulation is over budget (ratio {ratio:.3f})"
    resc = max(int(t.rescales.max()) for t in traces)
    max_p = max(t.max_p for t in traces)
    small = sum(t.small_p for t in traces)
    near = [sum(t.near[0] for t in traces), sum(t.near[1] for t in traces)]
    spread = max(t.lse_spread for t in traces)
    pat = w.pattern
    if pat == "staircase_up":
        ntiles = max(-(-s.k.shape[1] // BN) for s, _ in planted(w)[0])
        nsplit = len(split_ranges(w, ntiles * BN) or [0])
        # every tile of a split rescales (under a causal mask the last climbing row may stop one tile short)
        assert resc >= -(-ntiles // nsplit) - 2 >= 1, (resc, ntiles)
    elif pat == "staircase_under":    # e4m3 rounds the planted steps: P still comes within 2^-1 of the bound
        assert max_p >= 2 ** (7.0 if w.kw.get("fp8") or w.kw.get("kvfp8") else 7.5), max_p
    elif pat == "at_threshold":
        assert max_p >= 2 ** 7.9 and near[0] > 0 and near[1] > 0, (max_p, near)
    elif pat == "late_outlier":
        assert resc >= 1
    elif pat == "sink":
        assert small > 0
    elif pat == "descending":
        assert resc == 0 and small > 0
    elif pat.startswith("shifted") and split_ranges(w, 10 ** 6):
        assert spread > 0
    elif pat == "uniform":
        assert resc == 0 and max_p == 1.0
    assert max_p <= 2.0 ** 8 * (1 + 2 ** -20), f"P above the lazy-rescale bound: {max_p}"


def test_budget_is_not_loose():
    """Over the staircase and threshold workloads the emulation uses a fair part of the budget: a budget orders of
    magnitude too wide would let a subtly wrong kernel through."""
    worst = 0.0
    for name in ("dense_staircase_under", "dense_at_threshold", "varlen_sink", "dense_shifted_1e4"):
        _, r, _ = _emulated_check(_cpu_workload(BY_NAME[name]), limit=1)
        worst = max(worst, r)
    assert worst > 0.05, worst


MUTATIONS = ["no_o_rescale", "no_l_rescale", "raw_threshold", "swap_halves", "stale_lse", "no_reset"]
SENSITIVE = [w.name for w in WORKLOADS if w.pattern == "staircase_up"]


@pytest.mark.parametrize("mutation", MUTATIONS)
@pytest.mark.parametrize("name", SENSITIVE)
def test_checker_rejects_wrong_rescale(name, mutation):
    """A rescale that is wrong in one way, emulated at a GPU shape, fails the checker."""
    w = _cpu_workload(BY_NAME[name])
    if mutation == "swap_halves" and max(s[0] for s in sequences(w)) < 16:
        pytest.skip("decode: a row's other half is a padding row")
    ok, ratio, _ = _emulated_check(w, mutation, limit=2)
    assert not ok, f"{name}: {mutation} passes (ratio {ratio:.3f})"


@pytest.mark.parametrize("Sk", [131072, 262144])
def test_row_sum_order_keeps_lse_bound_on_a_constant_tail(Sk):
    """One sink key and Sk - 1 keys at the same logit delta below it (repeated tokens, padding without rotary, FP8
    keys that share a code): summed as one fp32 add per key pair into a running l, l drifts with the tile count past
    the LSE bound 1e-4 + 2e-6 |LSE| (mutation running_l); the kernel's tile partials with a compensated add into l stay
    far inside it at every delta."""
    deltas = np.array([0.5, 1.0, 3.0, 6.0])
    scale = 1.0 / LOG2E
    s = np.zeros((1, len(deltas), Sk))
    s[0, :, 1:] = -deltas[:, None] / scale
    vis = np.ones((len(deltas), Sk), bool)
    v = np.ones((1, Sk, 1))
    lse_ref = np.log1p((Sk - 1) * np.exp(-deltas))
    bound = 1e-4 + 2e-6 * np.abs(lse_ref)
    err = {}
    for mut in (None, "running_l"):
        _, lse, _ = emulate(s, vis, v, scale, "bf16", mutation=mut)
        err[mut] = np.abs(lse[0] - lse_ref)
    print(f"\n[row sum] Sk {Sk}: |dLSE| per delta {deltas.tolist()}: tile partial + Kahan "
          f"{err[None].tolist()}, running l {err['running_l'].tolist()}, bound {bound.tolist()}")
    assert (err[None] <= bound / 16).all(), err[None]
    assert (err["running_l"] > bound).any(), err["running_l"]


# ------------------------------------------------------------------ CPU: the scale range --------------------------------

def largest_scale():
    """The largest float32 x with fp32(x * fp32(log2 e)) finite."""
    L = np.float32(LOG2E)
    lo, hi = np.float32(1e38).view(np.uint32), np.float32(np.finfo(np.float32).max).view(np.uint32)
    with np.errstate(over="ignore"):
        while lo + 1 < hi:
            mid = np.uint32((int(lo) + int(hi)) // 2)
            if np.isfinite(mid.view(np.float32) * L):
                lo = mid
            else:
                hi = mid
    return float(lo.view(np.float32)), float(hi.view(np.float32))


def test_largest_scale_is_where_log2_overflows():
    top, above = largest_scale()
    assert 2.3586e38 < top < 2.3588e38 and above == float(np.nextafter(np.float32(top), np.float32(np.inf)))


@pytest.fixture(scope="module")
def tfa(built):
    import tfa_ctypes
    tfa_ctypes.lib()
    return tfa_ctypes


def _has_gpu():
    return torch.cuda.is_available()


def test_every_entry_point_takes_the_largest_scale_and_rejects_the_next(tfa):
    """softmax_scale at the largest accepted float passes the scale check, the next float up is TFA_EINVAL_SCALE, in
    every call; for the FP8 calls the same for s', through k_scale and, for the e4m3-query calls, through q_scale.
    Accepted calls are stopped before any device work by a later argument error (split-KV without a workspace,
    max_seqlen_q = 0, more than 7 exchange peers), or by TFA_EARCH without an H100; the FP8 varlen calls' s' has no
    later check, so only a machine without an H100 takes the largest s' here."""
    top, above = largest_scale()
    L = tfa.lib()
    A = 0x100000
    gpu = _has_gpu()

    def attn(scale, ns=2):
        return tfa.AttnArgs(A, A, A, A, A, 1, 4, 2, 300, 500, 128, 4 * 300 * 128, 300 * 128, 128, 2 * 500 * 128,
                            500 * 128, 128, 0, 1, scale, 0, ns, None, 0, None)

    def quant(qs=1.0, ks=1.0):
        return tfa.QkvQuantArgs(2, qs, ks, 0.01)

    def varlen(scale, mq=0):
        return tfa.VarlenArgs(A, A, A, A, A, A, A, 2, 4, 2, 128, 600, 900, mq, 4 * 128, 128, 2 * 128, 128, 0, 1, scale,
                              0, None)

    def cache(scale, ns=2):
        return tfa.KvcacheArgs(A, A, A, A, A, A, A, A, A, 2, 4, 2, 1, 128, 8, 128, 4, 1, 4 * 128, 4 * 128, 128,
                               128 * 2 * 128, 2 * 128, 128, 4, 2 * 128, 2 * 128, 128, 0, 1, scale, 0, ns, None, 0, None)

    def vcache(scale, mq=0):
        return tfa.VarlenKvcacheArgs(A, A, A, A, A, A, A, A, A, A, 2, 4, 2, 128, 5, mq, 8, 128, 4, 4 * 128, 128,
                                     128 * 2 * 128, 2 * 128, 128, 4, 2 * 128, 128, 0, 1, scale, 0, None)

    rot = tfa.RotaryArgs(A, A, 1024, 64, 0, A)
    kvq = lambda ks=1.0: tfa.KvQuantArgs(2, ks, 0.01)
    by = ctypes.byref
    calls = {
        "tfa_attn_fwd": (lambda s: L.tfa_attn_fwd(by(attn(s))), (-11, -7)),
        "tfa_attn_fp8_fwd": (lambda s: L.tfa_attn_fp8_fwd(by(attn(s)), by(quant())), (-11, -7)),
        "tfa_attn_fp8_fwd s'": (lambda s: L.tfa_attn_fp8_fwd(by(attn(1.0)), by(quant(1.0, s))), (-11, -7)),
        "tfa_attn_varlen_fwd": (lambda s: L.tfa_attn_varlen_fwd(by(varlen(s))), (-12,)),
        "tfa_attn_varlen_fp8_fwd": (lambda s: L.tfa_attn_varlen_fp8_fwd(by(varlen(s)), by(quant())), (-12,)),
        "tfa_attn_kvcache_fwd": (lambda s: L.tfa_attn_kvcache_fwd(by(cache(s))), (-11, -7)),
        "tfa_attn_kvcache_rotary_fwd": (lambda s: L.tfa_attn_kvcache_rotary_fwd(by(cache(s)), by(rot)), (-11, -7)),
        "tfa_attn_kvcache_fp8_fwd": (lambda s: L.tfa_attn_kvcache_fp8_fwd(by(cache(s)), None, by(kvq())), (-11, -7)),
        "tfa_attn_kvcache_fp8_fwd s'": (lambda s: L.tfa_attn_kvcache_fp8_fwd(by(cache(1.0)), None, by(kvq(s))),
                                        (-11, -7)),
        "tfa_attn_varlen_kvcache_fwd": (lambda s: L.tfa_attn_varlen_kvcache_fwd(by(vcache(s))), (-12,)),
        "tfa_attn_varlen_kvcache_fp8_fwd": (lambda s: L.tfa_attn_varlen_kvcache_fp8_fwd(by(vcache(s)), by(kvq())),
                                            (-12,)),
        "tfa_attn_varlen_kvcache_rotary_fwd": (lambda s: L.tfa_attn_varlen_kvcache_rotary_fwd(by(vcache(s)), by(rot),
                                                                                             None), (-12,)),
        "tfa_attn_kvcache_qkv8_fwd": (lambda s: L.tfa_attn_kvcache_qkv8_fwd(by(cache(s)), by(quant())), (-11, -7)),
        "tfa_attn_kvcache_qkv8_fwd q_scale s'": (lambda s: L.tfa_attn_kvcache_qkv8_fwd(by(cache(1.0)), by(quant(s))),
                                                 (-11, -7)),
        "tfa_attn_kvcache_qkv8_fwd k_scale s'": (
            lambda s: L.tfa_attn_kvcache_qkv8_fwd(by(cache(1.0)), by(quant(1.0, s))), (-11, -7)),
        "tfa_attn_varlen_kvcache_qkv8_fwd": (lambda s: L.tfa_attn_varlen_kvcache_qkv8_fwd(by(vcache(s)), by(quant())),
                                             (-12,)),
        "tfa_fwd_multi": (lambda s: L.tfa_fwd_multi(by(tfa.FwdArgs(A, A, A, A, A, 1, 4, 256, 128, 4 * 256 * 128,
                                                                   256 * 128, 128, 0, 0, s, 0, None)),
                                                    (ctypes.c_void_p * 8)(*([A] * 8)), 8), (-3, -7)),
    }
    if not gpu:      # no later check: only a machine without an H100 stops these before device work
        calls["tfa_attn_varlen_fp8_fwd s'"] = (
            lambda s: L.tfa_attn_varlen_fp8_fwd(by(varlen(1.0, 300)), by(quant(1.0, s))), (-7,))
        calls["tfa_attn_varlen_kvcache_fp8_fwd s'"] = (
            lambda s: L.tfa_attn_varlen_kvcache_fp8_fwd(by(vcache(1.0, 1)), by(kvq(s))), (-7,))
        calls["tfa_attn_varlen_kvcache_qkv8_fwd q_scale s'"] = (
            lambda s: L.tfa_attn_varlen_kvcache_qkv8_fwd(by(vcache(1.0, 1)), by(quant(s))), (-7,))
        calls["tfa_attn_varlen_kvcache_qkv8_fwd k_scale s'"] = (
            lambda s: L.tfa_attn_varlen_kvcache_qkv8_fwd(by(vcache(1.0, 1)), by(quant(1.0, s))), (-7,))
    for name, (call, accepted) in calls.items():
        assert call(top) in accepted, (name, call(top))
        assert call(above) == -9, (name, call(above))
        if not name.endswith("'"):         # a non-finite k_scale is the quantization's own error
            assert call(math.inf) == -9 and call(math.nan) == -9, name
    # the two FP8 varlen calls reject s' above the bound before any device work on every machine
    assert L.tfa_attn_varlen_fp8_fwd(by(varlen(1.0, 300)), by(quant(1.0, above))) == -9
    assert L.tfa_attn_varlen_kvcache_fp8_fwd(by(vcache(1.0, 1)), by(kvq(above))) == -9
    assert L.tfa_attn_varlen_kvcache_qkv8_fwd(by(vcache(1.0, 1)), by(quant(above))) == -9
    assert L.tfa_attn_varlen_kvcache_qkv8_fwd(by(vcache(1.0, 1)), by(quant(1.0, above))) == -9
    # tfa_fwd and tfa_fwd_host: the next float up is rejected before any device work
    assert L.tfa_fwd(A, A, A, A, A, 1, 4, 256, 128, 0, 0, above, None) == -9
    h = np.zeros(64 * 64, dtype=np.uint16)
    o = np.zeros_like(h)
    lse = np.zeros(64, dtype=np.float32)
    p = lambda x: x.ctypes.data
    assert L.tfa_fwd_host(p(h), p(h), p(h), p(o), p(lse), 1, 1, 64, 64, 0, 0, above, 1) == -9
    got = L.tfa_fwd_host(p(h), p(h), p(h), p(o), p(lse), 1, 1, 64, 64, 0, 0, top, 1)
    assert (got == 0) if gpu else got not in (0, -9), got
    msg = L.tfa_error_string(-9).decode()
    assert "log2" in msg and "2.3587e38" in msg


# ------------------------------------------------------------------ GPU ---------------------------------------------------

def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.mark.gpu
def test_wgmma_16bit_s_accumulation(tfa):
    """S = Q K^T chains (K = 64 and 128, bf16 and fp16) on wide-range operands, from zero, against exact products:
    |C - exact| / sum |a b| stays within S_MEASURED_BOUND, half the budget's EPS_S."""
    L = tfa.lib()
    g = torch.Generator().manual_seed(11)
    worst = {}
    for dtype in ("bf16", "fp16"):
        dt = _dt(dtype)
        for K in (64, 128):
            for trial in range(6):
                a = torch.empty(128, K).normal_(0, 1, generator=g)
                b = torch.empty(128, K).normal_(0, 1, generator=g)
                if trial % 3 == 1:                       # one large term per row against many small ones
                    a[:, 0] *= 256.0
                    b[:, 0] *= 64.0
                if trial % 3 == 2:                       # the planted dimensions: a big sum and its rounding rest
                    a[:, -2:] = 1.0
                    b[:, -2] = torch.empty(128).uniform_(100, 60000, generator=g)
                a, b = a.to(dt), b.to(dt)
                ad, bd = a.cuda(), b.cuda()
                c = torch.full((128, 128), float("nan"), dtype=torch.float32, device="cuda")
                kn = (ctypes.c_int * 4)(0, 0, 0, 0)
                tfa.check(L.tfa_selftest_umma(ad.data_ptr(), bd.data_ptr(), c.data_ptr(), 128, K, 0,
                                              0 if dtype == "bf16" else 1, ctypes.byref(kn), None))
                torch.cuda.synchronize()
                exact = a.double() @ b.double().T
                mag = a.double().abs() @ b.double().abs().T
                err = (c.cpu().double() - exact).abs() / mag.clamp(min=1e-30)
                worst[(dtype, K)] = max(worst.get((dtype, K), 0.0), float(err.max()))
    print("\n[16-bit wgmma] S chains from zero, worst |C - exact| / sum|a b|: " +
          ", ".join(f"{k}: {v:.3e}" for k, v in worst.items()))
    assert max(worst.values()) <= S_MEASURED_BOUND, worst


@pytest.fixture(scope="module")
def auto_runs(tfa):
    res = {}
    for w in WORKLOADS:
        res[w.name] = run(tfa, w)
    return res


SCHEDULE_RUN = r'''
import os, sys, torch
sys.path.insert(0, os.path.join(os.environ["TFA_ROOT"], "tiny-flash-attention_b200"))
sys.path.insert(0, os.path.join(os.environ["TFA_ROOT"], "tests"))
import tfa_ctypes as tfa
from test_fwd_softmax_range import WORKLOADS, portable, run
res = {}
for w in WORKLOADS:
    res[w.name] = portable(run(tfa, w))
torch.save(res, os.environ["TFA_OUT"])
'''


@pytest.mark.gpu
def test_softmax_range_matrix(auto_runs):
    """Every workload within budget of the float64 reference, no pass fraction; the worst ratio per workload printed;
    per mode, the staircase workload runs at least 3 work items per SM."""
    sms = _sms()
    fails = []
    for w in WORKLOADS:
        r = auto_runs[w.name]
        if w.pattern == "staircase_up":
            assert r["items"] >= 3 * sms, f"{w.name}: {r['items']} work items for {sms} SMs"
        ok, ratio, dl, msg = check_run(w, r)
        print(f"[softmax range] {w.name}: {r['items']} items, schedule {r['variant']}, max err/budget {ratio:.3f}, "
              f"max |dLSE| {dl:.2e}")
        if not ok:
            fails.append(f"{w.name}: {msg}")
    assert not fails, "; ".join(fails)


@pytest.mark.gpu
def test_softmax_range_bitwise_equal_under_both_schedules(auto_runs):
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


# key-less rows inside keyed items, one call per mode, on inputs whose S is exact
BOUNDARY = [
    W("b_dense", "dense", "exact", dict(B=1, Hq=4, Hkv=2, Sq=300, Sk=200, D=128, kind="bf16", causal=True, ns=1)),
    W("b_dense_split", "dense", "exact", dict(B=1, Hq=4, Hkv=2, Sq=700, Sk=450, D=64, kind="fp16", causal=True,
                                              ns=3)),
    W("b_varlen", "varlen", "exact", dict(lq=[300, 129, 64], lk=[100, 129, 30], Hq=4, Hkv=2, D=128, kind="bf16",
                                          causal=True)),
    W("b_cache", "cache", "exact", dict(lens=[1, 5, 130, 300], Sq=200, snew=0, Hq=4, Hkv=2, D=64, kind="fp16",
                                        page=128, causal=True)),
    W("b_cache_split", "cache", "exact", dict(lens=[1, 5, 130, 900], Sq=4, snew=0, Hq=4, Hkv=2, D=128, kind="bf16",
                                              page=256, causal=True, ns=3)),
    W("b_varlen_cache", "varlen_cache", "exact", dict(sq=[200, 1, 64], lens=[10, 300, 1], Hq=4, Hkv=2, D=128,
                                                      kind="bf16", page=256, causal=True, append=False)),
    W("b_fp8_dense", "dense", "exact", dict(B=1, Hq=4, Hkv=2, Sq=300, Sk=200, D=128, kind="bf16", causal=True, ns=1,
                                            fp8=(1.0, 1.0, 1.0))),
    W("b_fp8_varlen", "varlen", "exact", dict(lq=[300, 129], lk=[100, 129], Hq=4, Hkv=2, D=64, kind="fp16",
                                              causal=True, fp8=(1.0, 1.0, 1.0))),
    W("b_fp8_cache", "cache", "exact", dict(lens=[1, 5, 130, 300], Sq=200, snew=0, Hq=4, Hkv=2, D=128, kind="bf16",
                                            page=128, causal=True, kvfp8=(1.0, 1.0, 1.0))),
    W("b_fp8_varlen_cache", "varlen_cache", "exact", dict(sq=[200, 1], lens=[10, 300], Hq=4, Hkv=2, D=64,
                                                          kind="fp16", page=256, causal=True, append=False,
                                                          kvfp8=(1.0, 1.0, 1.0))),
]


def _exact_plant(pattern, Hq, Hkv, Sq, Sk, D, scale, kind, seed):
    """Scores in {-1, 0, 1}: q and k hold 0 / +-1 in a few dimensions, so S is exact and |S| <= 1 keeps every
    exponent finite at the largest scale; each row's max is one key or a tie, which the float64 reference resolves
    exactly as the kernel."""
    g = torch.Generator().manual_seed(seed)
    q = torch.zeros(Hq, Sq, D, dtype=torch.float64)
    k = torch.zeros(Hkv, Sk, D, dtype=torch.float64)
    q[..., 0] = 1.0
    k[..., 0] = torch.randint(-1, 1, (Hkv, Sk), generator=g).double()      # -1 or 0
    hot = torch.randint(0, Sk, (Hkv,), generator=g)
    k[torch.arange(Hkv), hot, 0] = 1.0                                     # one key with S = 1
    v = torch.randint(-4, 5, (Hkv, Sk, D), generator=g).double() / 4
    return q, k, v


@pytest.mark.gpu
@pytest.mark.parametrize("scale", ["1e9", "largest"])
def test_keyless_rows_exact_at_large_scales(tfa, monkeypatch, scale):
    """One call per mode with key-less causal rows inside items that have keys: exactly out = 0 / lse = +inf on those
    rows, the others equal to the float64 reference within budget (S is exact: |S| <= 1 in small integers)."""
    s = 1e9 if scale == "1e9" else largest_scale()[0]
    monkeypatch.setattr(sys.modules[__name__], "plant", _exact_plant)
    fails = []
    for w in BOUNDARY:
        r = run(tfa, w, scale=s)
        keyless = 0
        for i, (out, lse, sq) in enumerate(r["seqs"]):
            fp8 = bool(w.kw.get("fp8"))
            o_ref, l_ref, a, sub, pv16 = reference(sq.q[None], sq.k[None], sq.v[None], True, s)
            kl = torch.isinf(l_ref)
            keyless += int(kl.sum())
            o, l = out.double().cpu(), lse.double().cpu()
            if not (bool((o[kl] == 0).all()) and bool(torch.isposinf(l[kl]).all())):
                fails.append(f"{w.name} seq {i}: a key-less row is not exactly 0 / +inf "
                             f"(nan {int(torch.isnan(o[kl]).sum())})")
                continue
            ref = (o_ref, l_ref, a, F8.fp8_reference(sq.q[None], sq.k[None], sq.v[None], True, s, 1.0, 1.0)[3]
                   if fp8 else sub, torch.zeros_like(l_ref), pv16)
            ok, ra, le, msg = check(out.cpu(), lse.cpu(), ref, w.kw["kind"], fp8,
                                    split_ranges(w, sq.k.shape[1]) is not None)
            if not ok:
                fails.append(f"{w.name} seq {i}: {msg}")
        assert keyless > 0, w.name
        print(f"[scale {s:.6g}] {w.name}: {keyless} key-less rows")
    assert not fails, "; ".join(fails[:6])
