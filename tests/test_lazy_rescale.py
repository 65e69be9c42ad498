"""GPU: the LAZY-RESCALE branch of the online softmax (O rescaled in registers, l *= alpha,
P carried against a stale max, values up to 2^8) against the CPU oracle.

The seeded N(0, 0.5^2) inputs of the other parity files never move the running row max by more than 2^8 between KV
tiles, so they never enter that branch (ADVICE r01).  Here the logits are made to: (a) spread widely (q x 30),
(b) jump late (a planted outlier key in the last KV tile), (c) grow monotonically tile after tile by a step just
above / just below the 2^8 threshold (below: P approaches 2^8 without a rescale -- the fp16 range case).

Reference arithmetic being matched: max on unscaled scores, p = exp(scale*s - scale*m), l summed in fp32 before P is
rounded to 16 bit (flash_attention_cutlass/csrc/flash_attention.cu:228-316,601; SURVEY.md A.1) == oracle.attn_exact.

Tolerances: LSE (= scale*m + ln l, no 16-bit rounding anywhere on its path) atol 2e-4 * max(1, |lse|) -- this is what
pins the carried (m_ref, l) pair.  O: the kernel rounds P = 2^((s-m_ref)c) with a STALE m_ref, the reference rounds
exp(scale(s-m)) with the true max.  Both round every p_i to 16 bit with a relative error <= 2^-9 (bf16) -- but they round
DIFFERENT numbers (the two scalings differ by a factor that is not a power of two), so for peaked rows, where the errors
do not average out, the two results differ by up to 2 * 2^-9 * sum_i p_i |v_i| / l.  That attention-weighted mean of |v|
is computed by the oracle itself (same scores, values |v|); budget = 1e-3 + 2^-8 * attn(|v|) (fp16 P: 2^-11, same test)."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

ATOL, RTOL = 1e-3, 2.0 ** -8


@pytest.fixture(scope="module")
def tfa(built):
    import tfa_ctypes
    tfa_ctypes.lib()
    return tfa_ctypes


def _oracle(q, k, v, causal, scale, kind):
    from oracle import oracle as orc
    mode = orc.ROUND_BF16 if kind == "bf16" else orc.ROUND_FP16
    return orc.attn_general(q.float().cpu().numpy(), k.float().cpu().numpy(), v.float().cpu().numpy(), causal, scale,
                            mode, False)


def _base(B, Hq, Hkv, Sq, Sk, D, seed):
    g = torch.Generator(device="cpu").manual_seed(seed)
    mk = lambda *s: torch.empty(s, dtype=torch.float32).normal_(0.0, 0.5, generator=g)
    return mk(B, Hq, Sq, D), mk(B, Hkv, Sk, D), mk(B, Hkv, Sk, D)


def make_case(pattern, B, Hq, Hkv, Sq, Sk, D, kind, seed=20):
    """Returns (q, k, v) 16-bit CUDA tensors whose raw scores exercise the rescale branch."""
    q, k, v = _base(B, Hq, Hkv, Sq, Sk, D, seed)
    scale = D ** -0.5
    log2e = 1.4426950408889634
    if pattern == "spread":
        q = q * 30.0                                   # score std ~ 7.5 nats: the row max moves by >> 2^8 all the time
    elif pattern == "late_outlier":
        k[:, :, Sk - 3, :] = 12.0 * torch.sign(q[:, :1, Sq - 1, :]).expand_as(k[:, :, Sk - 3, :])   # huge |q.k| at the very end
        k[:, :, Sk // 2 + 1, :] *= 25.0
    elif pattern in ("staircase_up", "staircase_under"):
        # s_ij = step_raw * (j // 128) + noise: the row max climbs by `step` (log2 units) per KV tile.
        step_log2 = 12.0 if pattern == "staircase_up" else 7.5     # 7.5 < 8: every other tile runs with P up to 2^7.5
        u = torch.zeros(D)
        u[0] = 1.0
        beta = 4.0
        step_raw = step_log2 / (scale * log2e)          # raw-score units
        alpha = step_raw / beta
        tile = (torch.arange(Sk) // 128).float()
        k = k * 0.25 + (alpha * tile)[None, None, :, None] * u
        q = q * 0.25
        q[..., 0] = beta
    else:
        raise ValueError(pattern)
    dt = torch.bfloat16 if kind == "bf16" else torch.float16
    return q.to(dt).cuda(), k.to(dt).cuda(), v.to(dt).cuda(), scale


def check(o32, lse, want32, want_lse, want_abs):
    o = o32.float().cpu().numpy()
    l = lse.cpu().numpy()
    assert np.all(np.isfinite(o)), "non-finite output"
    d = np.abs(o - want32)
    budget = ATOL + RTOL * want_abs                        # want_abs = attention-weighted mean of |v| (>= |O|)
    assert np.all(d <= budget), f"O: max excess {(d - budget).max():.3e} at {np.unravel_index((d - budget).argmax(), d.shape)}"
    fin = np.isfinite(want_lse)
    assert np.array_equal(np.isfinite(l), fin)
    dl = np.abs(l[fin] - want_lse[fin])
    assert np.all(dl <= 2e-4 * np.maximum(1.0, np.abs(want_lse[fin]))), f"LSE: max err {dl.max():.3e}"


CASES = [
    # pattern, B, H, S, D, causal, kind
    ("spread", 1, 2, 512, 128, False, "bf16"),
    ("spread", 1, 2, 640, 64, True, "bf16"),
    ("spread", 1, 1, 384, 128, True, "fp16"),
    ("late_outlier", 1, 2, 512, 128, False, "bf16"),
    ("late_outlier", 1, 2, 512, 64, True, "fp16"),
    ("staircase_up", 1, 2, 768, 128, False, "bf16"),
    ("staircase_up", 1, 2, 768, 64, True, "bf16"),
    ("staircase_up", 1, 1, 512, 128, True, "fp16"),
    ("staircase_under", 1, 2, 768, 128, False, "fp16"),     # P up to 2^7.5 in fp16 without a rescale
    ("staircase_under", 1, 2, 768, 64, False, "fp16"),
    ("staircase_under", 1, 1, 640, 128, True, "bf16"),
]


@pytest.mark.parametrize("pattern,B,H,S,D,causal,kind", CASES)
def test_rescale_branch_matches_oracle(tfa, pattern, B, H, S, D, causal, kind):
    q, k, v, scale = make_case(pattern, B, H, H, S, S, D, kind)
    want32, want_lse = _oracle(q, k, v, causal, scale, kind)
    want_abs, _ = _oracle(q, k, v.abs(), causal, scale, kind)
    o32, lse = tfa.fwd(q, k, v, causal, scale, out_fp32=True)
    torch.cuda.synchronize()
    check(o32, lse, want32, want_lse, want_abs)
    # the shipped 16-bit output is the rounding of the same arithmetic
    o16, lse2 = tfa.fwd(q, k, v, causal, scale)
    torch.cuda.synchronize()
    assert torch.equal(lse, lse2)
    ulp = 2.0 ** (np.floor(np.log2(np.maximum(np.abs(want32), 2.0 ** -14))) - (7 if kind == "bf16" else 10))
    d = np.abs(o16.float().cpu().numpy() - want32)
    assert np.all(d <= ATOL + RTOL * want_abs + 0.505 * ulp)


@pytest.mark.parametrize("pattern,kind,D,causal", [("spread", "bf16", 128, True), ("staircase_up", "bf16", 64, False),
                                                    ("staircase_under", "fp16", 128, False)])
def test_rescale_branch_gqa_and_split_kv(tfa, pattern, kind, D, causal):
    """Same stress through tfa_attn_fwd: grouped K/V heads, Sq != Sk, and split-KV partials (each split carries its own
    (m_ref, l) and its LSE feeds the combine kernel)."""
    B, Hq, Hkv, Sq, Sk = 1, 4, 2, 256, 1536
    q, k, v, scale = make_case(pattern, B, Hq, Hkv, Sq, Sk, D, kind)
    want32, want_lse = _oracle(q, k, v, causal, scale, kind)
    want_abs, _ = _oracle(q, k, v.abs(), causal, scale, kind)
    for ns in (1, 3):
        o32, lse = tfa.attn_fwd(q, k, v, causal, scale, num_splits=ns, out_fp32=True)
        torch.cuda.synchronize()
        check(o32, lse, want32, want_lse, want_abs)
