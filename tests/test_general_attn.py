"""GPU: the generalised problem of SURVEY.md 8f rows 2-3 through the C ABI (tfa_attn_fwd) --
grouped K/V heads, Sq != Sk with the bottom-right aligned causal mask, split-KV with the LSE merge --
against the generalised CPU oracle (pinned to the reference's C++ CPU path, tests/test_oracle.py) and the
committed golden vectors of that path.  Same tolerances as tests/test_fwd_parity.py."""
import ctypes

import numpy as np
import pytest
import torch

from helpers import bf16_ulp, fp16_ulp, golden

pytestmark = pytest.mark.gpu

RTOL = ATOL = 1e-3


@pytest.fixture(scope="module")
def tfa(built):
    import tfa_ctypes
    tfa_ctypes.lib()
    return tfa_ctypes


def make_inputs(B, Hq, Hkv, Sq, Sk, D, kind, seed=20):
    g = torch.Generator(device="cpu")
    g.manual_seed(seed)
    dt = torch.bfloat16 if kind == "bf16" else torch.float16
    mk = lambda *s: torch.empty(s, dtype=torch.float32).normal_(0.0, 0.5, generator=g).to(dt).cuda()
    return mk(B, Hq, Sq, D), mk(B, Hkv, Sk, D), mk(B, Hkv, Sk, D)


def oracle_general(q, k, v, causal, scale, kind, round_out):
    from oracle import oracle as orc
    mode = orc.ROUND_BF16 if kind == "bf16" else orc.ROUND_FP16
    return orc.attn_general(q.float().cpu().numpy(), k.float().cpu().numpy(), v.float().cpu().numpy(), causal, scale,
                            mode, round_out)


def check_out32(o32, want32, causal):
    """fp32-output build vs the oracle.  Non-causal: strict allclose(1e-3, 1e-3).  Causal: rows with a handful of
    visible keys have P ~ 0.5 per key, where ONE 16-bit rounding flip of P (ex2.approx vs expf, SURVEY.md A.3) moves
    O by ~1e-3: same criterion as tests/test_fwd_parity.py's causal golden check."""
    o = o32.float().cpu().numpy()
    diff = np.abs(o - want32)
    ok = diff <= ATOL + RTOL * np.abs(want32)
    msg = f"max_abs {diff.max():.3e} pass_frac {ok.mean():.6f} worst at {np.unravel_index(diff.argmax(), diff.shape)}"
    if causal:
        assert ok.mean() >= 0.9995 and diff.max() < 4e-3, msg
    else:
        assert ok.all(), msg


def check_lse(lse, want):
    lse = lse.cpu().numpy()
    inf = np.isinf(want)
    assert np.array_equal(np.isinf(lse), inf) and np.all(lse[inf] > 0)
    assert np.abs(lse[~inf] - want[~inf]).max() <= 2e-4


def check_out16(out, want32, kind):
    o = out.float().cpu().numpy()
    ulp = bf16_ulp(want32) if kind == "bf16" else fp16_ulp(want32)
    diff = np.abs(o - want32)
    budget = ATOL + RTOL * np.abs(want32) + 0.5 * ulp * 1.01
    bad = diff > budget
    assert bad.mean() <= 5e-4 and diff.max() < 1e-2, f"max excess {(diff - budget).max():.3e} frac {bad.mean():.2e}"


GENERAL = [
    # B, Hq, Hkv, Sq, Sk, D, causal, kind
    (2, 8, 2, 256, 256, 128, True, "bf16"),     # GQA, group 4
    (1, 4, 1, 300, 300, 64, False, "bf16"),     # MQA, ragged
    (1, 2, 2, 96, 224, 64, True, "bf16"),       # more keys than queries, offset 128
    (1, 4, 2, 128, 1000, 128, True, "bf16"),    # offset 872: the masked diagonal straddles two KV tiles
    (1, 2, 2, 130, 333, 64, True, "fp16"),      # everything ragged
    (2, 2, 2, 1, 777, 128, True, "bf16"),       # one query row (decode): causal == non-causal
    (2, 2, 1, 1, 777, 128, False, "fp16"),
    (1, 2, 1, 500, 200, 64, True, "bf16"),      # more queries than keys, causal: 300 rows see nothing
    (1, 2, 2, 400, 130, 128, False, "bf16"),    # more queries than keys, non-causal
    (1, 8, 2, 640, 384, 128, True, "fp16"),     # GQA + Sq > Sk + causal
]


@pytest.mark.parametrize("B,Hq,Hkv,Sq,Sk,D,causal,kind", GENERAL)
def test_general_matches_oracle(tfa, B, Hq, Hkv, Sq, Sk, D, causal, kind):
    q, k, v = make_inputs(B, Hq, Hkv, Sq, Sk, D, kind)
    scale = D ** -0.5
    want32, want_lse = oracle_general(q, k, v, causal, scale, kind, round_out=False)
    o32, lse = tfa.attn_fwd(q, k, v, causal, scale, num_splits=1, out_fp32=True)
    torch.cuda.synchronize()
    check_out32(o32, want32, causal)
    check_lse(lse, want_lse)
    o16, lse16 = tfa.attn_fwd(q, k, v, causal, scale, num_splits=1)
    torch.cuda.synchronize()
    check_out16(o16, want32, kind)
    check_lse(lse16, want_lse)
    if causal and Sk < Sq:                                  # rows without keys: exact zeros
        assert torch.count_nonzero(o16[:, :, : Sq - Sk]).item() == 0


def test_grouped_heads_equal_repeated_heads_bitwise(tfa):
    """kv head = h // group (archive_)/attn.cpp:61): the grouped call must equal the MHA call on repeated K/V."""
    q, k, v = make_inputs(2, 8, 2, 384, 384, 128, "bf16")
    a, la = tfa.attn_fwd(q, k, v, True, 0.1)
    kr, vr = k.repeat_interleave(4, dim=1).contiguous(), v.repeat_interleave(4, dim=1).contiguous()
    b, lb = tfa.fwd(q, kr, vr, True, 0.1)
    torch.cuda.synchronize()
    assert torch.equal(a, b) and torch.equal(la, lb)


def test_square_general_entry_equals_reference_entry_bitwise(tfa):
    q, k, v = make_inputs(1, 4, 4, 700, 700, 64, "fp16")
    a, la = tfa.attn_fwd(q, k, v, True, 0.125)
    b, lb = tfa.fwd(q, k, v, True, 0.125)
    torch.cuda.synchronize()
    assert torch.equal(a, b) and torch.equal(la, lb)


def test_golden_reference_cpp_sq_ne_sk(tfa):
    """Outputs of the reference's own C++ CPU module for Sq=96, Sk=224 (tests/golden/make_golden.py section 5)."""
    g = golden("ref_cpp_sq96_sk224.npz")
    q, k, v = (torch.from_numpy(g[n]).to(torch.bfloat16).cuda() for n in ("q", "k", "v"))
    scale = float(g["scale"])
    from oracle import oracle as orc
    for causal in (False, True):
        o32, _ = tfa.attn_fwd(q, k, v, causal, scale, out_fp32=True)
        torch.cuda.synchronize()
        # the fixture was computed from the fp32 inputs; bf16 quantisation of uniform[0,1) inputs moves the
        # output by < 4e-3, the reference's own bar is 1e-2 (flash_attention_c/test.py:82-83)
        assert np.abs(o32.cpu().numpy() - g[f"flash_causal{int(causal)}"]).max() < 1e-2
        # exact statement on the quantised inputs: the reference algorithm restated (pinned by test_oracle.py)
        want = orc.rowwise_general(q.float().cpu().numpy(), k.float().cpu().numpy(), v.float().cpu().numpy(), causal,
                                   scale)
        # (pure fp32 restatement, P not rounded: the kernel's 16-bit P adds up to 2^-9 relative per key)
        assert np.abs(o32.cpu().numpy() - want).max() < 4e-3


SPLIT = [
    # B, Hq, Hkv, Sq, Sk, D, causal, kind, num_splits
    (1, 2, 2, 256, 2048, 128, False, "bf16", 4),
    (1, 2, 2, 256, 2048, 128, True, "bf16", 4),       # offset 1792
    (1, 2, 1, 1024, 1024, 64, True, "bf16", 4),       # square causal: later splits lie above early tiles' diagonal
    (1, 2, 2, 1024, 1024, 128, True, "fp16", 3),      # uneven split (8 tiles -> 3,3,2)
    (2, 4, 2, 1, 4000, 128, False, "bf16", 8),        # decode, ragged keys
    (1, 1, 1, 300, 1500, 64, True, "bf16", 5),        # ragged everything; 12 tiles -> 3 per split -> 4 splits
    (1, 2, 2, 130, 640, 128, False, "fp16", 16),      # more splits asked than sensible: clamped to 5
    (1, 2, 1, 700, 400, 64, True, "bf16", 2),         # Sq > Sk causal + split
]


@pytest.mark.parametrize("B,Hq,Hkv,Sq,Sk,D,causal,kind,ns", SPLIT)
def test_split_kv_matches_oracle_and_single_pass(tfa, B, Hq, Hkv, Sq, Sk, D, causal, kind, ns):
    q, k, v = make_inputs(B, Hq, Hkv, Sq, Sk, D, kind, seed=7)
    scale = D ** -0.5
    want32, want_lse = oracle_general(q, k, v, causal, scale, kind, round_out=False)
    o32, lse, used = tfa.attn_fwd(q, k, v, causal, scale, num_splits=ns, out_fp32=True, return_splits=True)
    torch.cuda.synchronize()
    assert 2 <= used <= ns
    check_out32(o32, want32, causal)
    check_lse(lse, want_lse)
    o16, lse16 = tfa.attn_fwd(q, k, v, causal, scale, num_splits=ns)
    one, lse_one = tfa.attn_fwd(q, k, v, causal, scale, num_splits=1)
    torch.cuda.synchronize()
    check_out16(o16, want32, kind)
    check_lse(lse16, want_lse)
    # split and single pass agree to a 16-bit rounding step of each other
    ulp = bf16_ulp(want32) if kind == "bf16" else fp16_ulp(want32)
    assert np.all(np.abs(o16.float().cpu().numpy() - one.float().cpu().numpy()) <= 2e-3 + 1.01 * ulp)


@pytest.mark.parametrize("B,Hq,Hkv,Sq,Sk,D,kind,ns", [
    (1, 4, 2, 1024, 1024, 128, "bf16", 4),      # the first Q tiles' rows see keys of split 0 only
    (1, 2, 1, 700, 400, 64, "fp16", 2),         # and the first 300 rows see no key at all
])
def test_split_kv_result_does_not_depend_on_the_workspace(tfa, B, Hq, Hkv, Sq, Sk, D, kind, ns):
    """Causal split-KV: every split writes the LSE of every row, a split without keys too (-inf), and the combine
    reads them all.  A workspace full of NaN and a zeroed one give the same bits."""
    q, k, v = make_inputs(B, Hq, Hkv, Sq, Sk, D, kind, seed=11)
    L = tfa.lib()
    st = torch.cuda.current_stream().cuda_stream
    dtype = tfa.TFA_BF16 if kind == "bf16" else tfa.TFA_FP16
    for f32 in (0, 1):
        res = []
        for fill in (float("nan"), 0.0):
            out = torch.empty(q.shape, dtype=torch.float32 if f32 else q.dtype, device="cuda")
            lse = torch.empty((B, Hq, Sq), dtype=torch.float32, device="cuda")
            a = tfa.AttnArgs(q.data_ptr(), k.data_ptr(), v.data_ptr(), out.data_ptr(), lse.data_ptr(), B, Hq, Hkv, Sq,
                             Sk, D, Hq * Sq * D, Sq * D, D, Hkv * Sk * D, Sk * D, D, dtype, 1, D ** -0.5, f32, ns, None,
                             0, st)
            assert L.tfa_attn_num_splits(ctypes.byref(a)) == ns
            need = L.tfa_attn_workspace_bytes(ctypes.byref(a), ns)
            ws = torch.full((need // 4,), fill, dtype=torch.float32, device="cuda")
            a.workspace, a.workspace_bytes = ws.data_ptr(), need
            tfa.check(L.tfa_attn_fwd(ctypes.byref(a)))
            torch.cuda.synchronize()
            res.append((out, lse))
        (o_nan, l_nan), (o_zero, l_zero) = res
        assert torch.equal(o_nan, o_zero) and torch.equal(l_nan, l_zero), f32


def test_split_heuristic(tfa):
    """auto (num_splits=0): splits a long-key / few-row problem, leaves a grid that already fills the GPU alone."""
    q, k, v = make_inputs(1, 4, 4, 128, 16384, 128, "bf16")
    o, lse, used = tfa.attn_fwd(q, k, v, False, 128 ** -0.5, num_splits=0, return_splits=True)
    one, lse_one = tfa.attn_fwd(q, k, v, False, 128 ** -0.5, num_splits=1)
    torch.cuda.synchronize()
    assert used > 1
    assert np.abs(o.float().cpu().numpy() - one.float().cpu().numpy()).max() <= 4e-3
    assert np.abs(lse.cpu().numpy() - lse_one.cpu().numpy()).max() <= 2e-4
    q, k, v = make_inputs(4, 32, 32, 1024, 1024, 128, "bf16")
    _, _, used = tfa.attn_fwd(q, k, v, True, 0.1, num_splits=0, return_splits=True)
    assert used == 1


def test_scale_zero_is_a_prefix_mean(tfa):
    """softmax_scale = 0: every visible key gets the same weight (masked keys must stay masked, not 0 * -inf)."""
    q, k, v = make_inputs(1, 2, 2, 200, 200, 64, "bf16")
    o32, lse = tfa.attn_fwd(q, k, v, True, 0.0, out_fp32=True)
    torch.cuda.synchronize()
    vf = v.float()
    want = torch.cumsum(vf, dim=2) / torch.arange(1, 201, device="cuda").view(1, 1, -1, 1)
    assert torch.allclose(o32, want, rtol=2e-3, atol=2e-3)    # P = 1 exactly; V sums in fp32 on both sides
    assert torch.allclose(lse, torch.log(torch.arange(1, 201, device="cuda").float()).expand(1, 2, 200), atol=2e-4)


def test_scale_zero_causal_split_kv(tfa):
    """softmax_scale = 0 through causal split-KV: splits wholly above a row's diagonal must contribute weight 0
    (LSE_s = -inf), not a partial with l = 32 * 2^-126 and a finite LSE (ADVICE r01: ex2_poly2 clamps -inf)."""
    q, k, v = make_inputs(1, 2, 2, 256, 1024, 64, "bf16")
    for ns in (2, 4, 8):
        o32, lse = tfa.attn_fwd(q, k, v, True, 0.0, num_splits=ns, out_fp32=True)
        torch.cuda.synchronize()
        n_vis = torch.arange(1, 257, device="cuda") + (1024 - 256)               # bottom-right aligned mask
        csum = torch.cumsum(v.float(), dim=2)
        want = csum[:, :, n_vis - 1] / n_vis.view(1, 1, -1, 1)
        assert torch.allclose(o32, want, rtol=2e-3, atol=2e-3), ns
        assert torch.allclose(lse, torch.log(n_vis.float()).expand(1, 2, 256), atol=2e-4), ns


def test_extension_general_entry(built):
    import attention_cutlass as ac
    q, k, v = make_inputs(1, 4, 2, 200, 456, 128, "bf16")
    out, lse = ac.flash_attention_v2_general(q, k, v, True, 128 ** -0.5, 1)
    out2, lse2 = ac.flash_attention_v2_general(q, k, v, True, 128 ** -0.5, 2)
    torch.cuda.synchronize()
    want32, want_lse = oracle_general(q, k, v, True, 128 ** -0.5, "bf16", round_out=False)
    check_out16(out, want32, "bf16")
    check_out16(out2, want32, "bf16")
    check_lse(lse, want_lse)
    check_lse(lse2, want_lse)
    with pytest.raises(RuntimeError, match="multiple of K/V heads"):
        ac.flash_attention_v2_general(q, k[:, :1].repeat(1, 3, 1, 1).contiguous(), v[:, :1].repeat(1, 3, 1, 1).contiguous(),
                                      True, 0.1, 1)


def test_general_argument_errors(tfa):
    L = tfa.lib()
    q, k, v = make_inputs(1, 4, 3, 128, 128, 64, "bf16")
    out = torch.empty_like(q)
    a = tfa.AttnArgs(q.data_ptr(), k.data_ptr(), v.data_ptr(), out.data_ptr(), None, 1, 4, 3, 128, 128, 64,
                     4 * 128 * 64, 128 * 64, 64, 3 * 128 * 64, 128 * 64, 64, 0, 0, 0.1, 0, 1, None, 0, None)
    assert L.tfa_attn_fwd(ctypes.byref(a)) == -10            # TFA_EINVAL_HEADS
    a.Hkv = 2
    a.Sk = 1024                                               # (not dereferenced: rejected before any launch)
    a.num_splits = 4
    assert L.tfa_attn_fwd(ctypes.byref(a)) == -11            # TFA_EINVAL_WORKSPACE
    assert L.tfa_attn_num_splits(ctypes.byref(a)) == 4
    assert L.tfa_attn_workspace_bytes(ctypes.byref(a), 4) == 4 * 1 * 4 * 128 * 65 * 4
    torch.cuda.synchronize()
