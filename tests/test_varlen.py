"""The variable-length (packed, cu_seqlens) forward: tfa_attn_varlen_fwd / attention_cutlass.flash_attention_v2_varlen.

CPU: the entry point is declared and exported, every argument error comes back before any device work, and the barrier
protocol model accepts the consumers' "item without tiles" path.
GPU: each packed sequence equals the dense tfa_attn_fwd on that sequence bit for bit (where the dense path does the
same arithmetic) and the CPU oracle at tests/test_general_attn.py's tolerances; sequences do not leak into each other
or outside out / lse; both schedules agree; the call is one launch and replays from a CUDA graph with new lengths."""
import ctypes
import os
import random
import subprocess
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

TFA_EINVAL_SEQLENS = -12


def declared_functions():
    import re
    src = open(os.path.join(ROOT, "include", "tfa_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return set(re.findall(r"\b(tfa_[a-z0-9_]+)\s*\(", src))


# ------------------------------------------------------------------ CPU ------------------------------------------------

def test_header_declares_and_library_exports_varlen(built):
    import tfa_ctypes
    assert "tfa_attn_varlen_fwd" in declared_functions()
    assert "TFA_EINVAL_SEQLENS (-12)" in open(os.path.join(ROOT, "include", "tfa_b200.h")).read()
    L = ctypes.CDLL(tfa_ctypes.LIB_PATH)
    assert hasattr(L, "tfa_attn_varlen_fwd")


def test_varlen_error_string(built):
    import tfa_ctypes
    L = tfa_ctypes.lib()
    msg = L.tfa_error_string(TFA_EINVAL_SEQLENS)
    assert msg.startswith(b"tfa:") and b"cu_seqlens" in msg and b"max_seqlen_q" in msg


def test_varlen_argument_validation_without_device(built):
    """Host buffers only: every code must come back before anything touches a device (on a CPU-only box a call that
    got that far would fail with a CUDA error instead)."""
    import tfa_ctypes
    L = tfa_ctypes.lib()
    buf = ctypes.create_string_buffer(4096 + 16)
    base = (ctypes.addressof(buf) + 15) & ~15
    cu = base + 1024                                          # 16-byte aligned, so 4-byte aligned
    Hq, Hkv, D = 4, 2, 64

    def mk(**kw):
        return tfa_ctypes.VarlenArgs(
            kw.get("q", base), base, base, kw.get("out", base), None, kw.get("cu_q", cu), kw.get("cu_k", cu),
            kw.get("B", 2), kw.get("Hq", Hq), kw.get("Hkv", Hkv), kw.get("D", D), kw.get("total_q", 300),
            kw.get("total_k", 400), kw.get("max_q", 200), kw.get("qss", Hq * D), kw.get("qsh", D),
            kw.get("kss", Hkv * D), D, kw.get("dtype", 0), 1, kw.get("scale", 0.1), 0, None)

    call = lambda **kw: L.tfa_attn_varlen_fwd(ctypes.byref(mk(**kw)))
    assert L.tfa_attn_varlen_fwd(None) == -1                  # TFA_EINVAL_PTR
    assert call(q=None) == -1 and call(q=base + 2) == -1 and call(out=base + 8) == -1
    assert call(D=96) == -2                                   # TFA_EINVAL_DIM
    assert call(B=0) == -3 and call(total_q=0) == -3 and call(total_k=0) == -3 and call(Hq=0) == -3
    assert call(dtype=2) == -4                                # TFA_EINVAL_DTYPE
    assert call(qss=60) == -5 and call(qsh=12) == -5 and call(kss=30) == -5     # TFA_EINVAL_STRIDE
    assert call(scale=-1.0) == -9 and call(scale=float("nan")) == -9             # TFA_EINVAL_SCALE
    assert call(Hkv=3) == -10                                 # TFA_EINVAL_HEADS
    assert call(cu_q=None) == TFA_EINVAL_SEQLENS
    assert call(cu_k=None) == TFA_EINVAL_SEQLENS
    assert call(cu_q=cu + 2) == TFA_EINVAL_SEQLENS
    assert call(cu_k=cu + 1) == TFA_EINVAL_SEQLENS
    assert call(max_q=0) == TFA_EINVAL_SEQLENS
    assert call(max_q=301) == TFA_EINVAL_SEQLENS              # > total_q
    assert call(max_q=-5) == TFA_EINVAL_SEQLENS


def _protocol_model():
    sys.path.insert(0, os.path.join(ROOT, "scripts"))
    import protocol_model as pm
    return pm


def test_protocol_model_items_without_tiles():
    """Variable-length items whose rows see no key: the producer skips them, the softmax warpgroups write their rows
    without waiting on a barrier.  Mixed with skipped items and items with tiles, in both ring depths."""
    pm = _protocol_model()
    for trial in range(400):
        rng = random.Random(424242 + trial)
        items, empty = pm.random_varlen_items(rng)
        pm.Sim(items, rng.choice([4, 8]), rng, empty).run()
    rng = random.Random(5)
    pm.Sim([0, 3, 0, 0, 2], 4, rng, empty=[0, 2, 3]).run()   # empty items first, between and after loaded ones


def test_protocol_model_catches_a_wait_on_an_empty_item():
    """Mutation: the consumers wait for Q on an item the producer never loads -> deadlock (or a parity slip on the
    next item), which the model must report."""
    src = open(os.path.join(ROOT, "scripts", "protocol_model.py")).read()
    needle = "                if item in self.empty:                        # epilogue only: no barrier is touched\n" \
             "                    yield lambda: True\n"
    assert needle in src
    mutated = src.replace(needle, "                if item in self.empty:\n"
                                  "                    yield lambda p=qcnt & 1: self.q_full.done(p)\n")
    ns = {"__name__": "mutated_model"}
    exec(compile(mutated, "mutated_model", "exec"), ns)
    caught = 0
    for trial in range(40):
        rng = random.Random(7 + trial)
        items, empty = ns["random_varlen_items"](rng)
        if not empty:
            continue
        try:
            ns["Sim"](items, 4, rng, empty).run()
        except AssertionError:
            caught += 1
    assert caught > 5


# ------------------------------------------------------------------ GPU ------------------------------------------------

@pytest.fixture(scope="module")
def tfa(built):
    import tfa_ctypes
    tfa_ctypes.lib()
    return tfa_ctypes


def make_batch(lq, lk, Hq, Hkv, D, kind, seed=20):
    """Packed q (sum lq, Hq, D), k/v (sum lk, Hkv, D) ~ N(0, 0.5^2) and their int32 cu_seqlens on the GPU."""
    g = torch.Generator(device="cpu")
    g.manual_seed(seed)
    dt = torch.bfloat16 if kind == "bf16" else torch.float16
    mk = lambda *s: torch.empty(s, dtype=torch.float32).normal_(0.0, 0.5, generator=g).to(dt).cuda()
    q, k, v = mk(sum(lq), Hq, D), mk(sum(lk), Hkv, D), mk(sum(lk), Hkv, D)
    cu = lambda ls: torch.tensor(np.concatenate([[0], np.cumsum(ls)]), dtype=torch.int32, device="cuda")
    return q, k, v, cu(lq), cu(lk)


def seq(x, c0, c1):
    """Rows [c0, c1) of a packed (total, H, D) tensor as a contiguous (1, H, S, D) one."""
    return x[c0:c1].permute(1, 0, 2).unsqueeze(0).contiguous()


def offsets(ls):
    c = np.concatenate([[0], np.cumsum(ls)]).astype(int)
    return list(zip(c[:-1], c[1:]))


MIX = [1, 64, 127, 128, 129, 300, 1000, 2049]

BITWISE = [
    # causal, D, kind, Hq, Hkv, more_keys
    (True, 128, "bf16", 4, 4, False),
    (True, 64, "fp16", 8, 2, True),          # GQA group 4, Sk_b > Sq_b: bottom-right offset per sequence
    (False, 128, "fp16", 8, 2, False),
    (False, 64, "bf16", 2, 2, True),
    (True, 128, "bf16", 8, 2, True),
]


@pytest.mark.gpu
@pytest.mark.parametrize("causal,D,kind,Hq,Hkv,more_keys", BITWISE)
def test_varlen_equals_per_sequence_dense_bitwise(tfa, causal, D, kind, Hq, Hkv, more_keys):
    rng = random.Random(D + Hq + int(causal))
    lq = MIX[:]
    rng.shuffle(lq)
    lk = [s + rng.randint(1, 300) for s in lq] if more_keys else lq[:]
    q, k, v, cu_q, cu_k = make_batch(lq, lk, Hq, Hkv, D, kind)
    scale = D ** -0.5
    for f32 in (False, True):
        out, lse = tfa.attn_varlen_fwd(q, k, v, cu_q, cu_k, max(lq), causal, scale, out_fp32=f32)
        for (q0, q1), (k0, k1) in zip(offsets(lq), offsets(lk)):
            o_ref, l_ref = tfa.attn_fwd(seq(q, q0, q1), seq(k, k0, k1), seq(v, k0, k1), causal, scale, num_splits=1,
                                        out_fp32=f32)
            assert torch.equal(out[q0:q1], o_ref[0].permute(1, 0, 2)), (f32, q0, q1)
            assert torch.equal(lse[:, q0:q1], l_ref[0]), (f32, q0, q1)
    torch.cuda.synchronize()


ORACLE = [
    # lq, lk, causal, D, kind, Hq, Hkv
    ([300, 0, 200, 64, 129, 5], [100, 50, 0, 64, 500, 5], True, 128, "bf16", 4, 2),
    ([500, 77, 0, 1, 260], [200, 0, 10, 300, 260], True, 64, "fp16", 4, 1),
    ([300, 0, 200, 64, 129], [100, 50, 0, 64, 500], False, 64, "bf16", 2, 2),
]


@pytest.mark.gpu
@pytest.mark.parametrize("lq,lk,causal,D,kind,Hq,Hkv", ORACLE)
def test_varlen_matches_oracle(tfa, lq, lk, causal, D, kind, Hq, Hkv):
    """Causal Sq_b > Sk_b, Sk_b = 0 and Sq_b = 0 included: rows that see no key are exact zeros with LSE = +inf."""
    from test_general_attn import check_lse, check_out16, check_out32, oracle_general
    q, k, v, cu_q, cu_k = make_batch(lq, lk, Hq, Hkv, D, kind, seed=3)
    scale = D ** -0.5
    o32, lse32 = tfa.attn_varlen_fwd(q, k, v, cu_q, cu_k, max(lq), causal, scale, out_fp32=True)
    o16, lse16 = tfa.attn_varlen_fwd(q, k, v, cu_q, cu_k, max(lq), causal, scale)
    torch.cuda.synchronize()
    assert torch.equal(lse32, lse16)
    for (q0, q1), (k0, k1) in zip(offsets(lq), offsets(lk)):
        if q1 == q0:
            continue
        Sq, Sk = q1 - q0, k1 - k0
        n_empty = Sq if Sk == 0 else (max(0, Sq - Sk) if causal else 0)
        got32, got16 = o32[q0:q1].permute(1, 0, 2)[None], o16[q0:q1].permute(1, 0, 2)[None]
        got_lse = lse32[:, q0:q1][None]
        if n_empty:
            assert torch.count_nonzero(got32[:, :, :n_empty]).item() == 0
            assert torch.count_nonzero(got16[:, :, :n_empty]).item() == 0
            assert torch.all(torch.isposinf(got_lse[:, :, :n_empty]))
        if n_empty == Sq:
            continue
        want32, want_lse = oracle_general(seq(q, q0, q1), seq(k, k0, k1), seq(v, k0, k1), causal, scale, kind,
                                          round_out=False)
        check_out32(got32, want32, causal)
        check_out16(got16, want32, kind)
        check_lse(got_lse, want_lse)


@pytest.mark.gpu
@pytest.mark.parametrize("kind,causal", [("fp16", True), ("fp16", False), ("bf16", True)])
def test_varlen_sequences_are_isolated(tfa, kind, causal):
    """Other finite values (down to +-6e4 in fp16) in one sequence's q/k/v leave every other sequence's output
    bit-identical: the rows a TMA box pulls in from a neighbour are masked (keys) or never stored (queries)."""
    lq, lk = [129, 300, 1, 200, 64], [129, 500, 40, 64, 64]
    q, k, v, cu_q, cu_k = make_batch(lq, lk, 4, 2, 128, kind, seed=11)
    o1, l1 = tfa.attn_varlen_fwd(q, k, v, cu_q, cu_k, max(lq), causal, 0.1)
    big = 6.0e4                  # near the fp16 maximum; every score stays finite in fp32
    sq, sk = offsets(lq), offsets(lk)
    for victim in (1, 3):
        q2, k2, v2 = q.clone(), k.clone(), v.clone()
        (a, b), (c, d) = sq[victim], sk[victim]
        sign = torch.where(torch.rand(q2[a:b].shape, device="cuda") < 0.5, -1.0, 1.0)
        q2[a:b] = (sign * big).to(q.dtype)
        k2[c:d] = (-big if victim == 1 else big) * torch.ones_like(k2[c:d])
        v2[c:d] = torch.full_like(v2[c:d], -big)
        o2, l2 = tfa.attn_varlen_fwd(q2, k2, v2, cu_q, cu_k, max(lq), causal, 0.1)
        torch.cuda.synchronize()
        for i, (s0, s1) in enumerate(sq):
            if i != victim:
                assert torch.equal(o1[s0:s1], o2[s0:s1]) and torch.equal(l1[:, s0:s1], l2[:, s0:s1]), (victim, i)


@pytest.mark.gpu
@pytest.mark.parametrize("f32", [False, True])
def test_varlen_writes_every_row_and_nothing_else(tfa, f32):
    """NaN-filled out / lse with guard regions on both sides: every row of [0, total_q) is written, no guard byte
    changes (sequences with Sq_b = 0, Sk_b = 0 and causal Sq_b > Sk_b included)."""
    lq, lk = [200, 0, 129, 7, 300], [64, 90, 0, 7, 700]
    Hq, D, G = 4, 64, 64
    q, k, v, cu_q, cu_k = make_batch(lq, lk, Hq, 1, D, "bf16", seed=5)
    tq = sum(lq)
    dt = torch.float32 if f32 else q.dtype
    obuf = torch.full((G + tq + G, Hq, D), float("nan"), dtype=dt, device="cuda")
    lbuf = torch.full((G + Hq * tq + G,), float("nan"), dtype=torch.float32, device="cuda")
    out, lse = obuf[G:G + tq], lbuf[G:G + Hq * tq].view(Hq, tq)
    tfa.attn_varlen_fwd(q, k, v, cu_q, cu_k, max(lq), True, 0.125, out_fp32=f32, out=out, lse=lse)
    torch.cuda.synchronize()
    assert not torch.isnan(out).any() and not torch.isnan(lse).any()
    assert torch.isnan(obuf[:G]).all() and torch.isnan(obuf[G + tq:]).all()
    assert torch.isnan(lbuf[:G]).all() and torch.isnan(lbuf[G + Hq * tq:]).all()


@pytest.mark.gpu
def test_varlen_classic_and_persistent_agree_bitwise(tfa):
    code = r'''
import os, sys, torch
sys.path.insert(0, os.path.join(os.environ["TFA_ROOT"], "tiny-flash-attention_b200"))
sys.path.insert(0, os.path.join(os.environ["TFA_ROOT"], "tests"))
import tfa_ctypes as tfa
from test_varlen import make_batch
lq, lk = [1000, 0, 129, 2049, 64, 300], [1000, 30, 0, 2100, 20, 300]
res = []
for causal in (True, False):
    q, k, v, cu_q, cu_k = make_batch(lq, lk, 8, 2, 128, "bf16", seed=9)
    o, lse = tfa.attn_varlen_fwd(q, k, v, cu_q, cu_k, max(lq), causal, 128 ** -0.5)
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
def test_varlen_cuda_graph_reads_lengths_on_the_device(tfa):
    """Capture one call, rewrite cu_seqlens in place (same totals and max), replay: equals a fresh eager call."""
    lq1, lk1 = [100, 300, 50, 250], [400, 300, 50, 100]
    lq2, lk2 = [300, 100, 250, 50], [50, 100, 400, 300]
    q, k, v, cu_q, cu_k = make_batch(lq1, lk1, 4, 2, 128, "bf16", seed=13)
    out = torch.empty_like(q)
    lse = torch.empty((4, q.shape[0]), dtype=torch.float32, device="cuda")
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):                               # warm-up outside the capture
        tfa.attn_varlen_fwd(q, k, v, cu_q, cu_k, 300, True, 0.1, out=out, lse=lse)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        tfa.attn_varlen_fwd(q, k, v, cu_q, cu_k, 300, True, 0.1, out=out, lse=lse)
    g.replay()
    want1, wl1 = tfa.attn_varlen_fwd(q, k, v, cu_q.clone(), cu_k.clone(), 300, True, 0.1)
    torch.cuda.synchronize()
    assert torch.equal(out, want1) and torch.equal(lse, wl1)
    c2q, c2k = make_batch(lq2, lk2, 1, 1, 64, "bf16")[3:]
    cu_q.copy_(c2q)
    cu_k.copy_(c2k)
    g.replay()
    want2, wl2 = tfa.attn_varlen_fwd(q, k, v, c2q, c2k, 300, True, 0.1)
    torch.cuda.synchronize()
    assert not torch.equal(want1, want2)
    assert torch.equal(out, want2) and torch.equal(lse, wl2)


@pytest.mark.gpu
def test_varlen_is_one_launch(tfa):
    q, k, v, cu_q, cu_k = make_batch([500, 0, 64, 129], [200, 10, 0, 300], 4, 2, 64, "fp16", seed=1)
    for causal in (True, False):
        n0 = tfa.launch_count()
        tfa.attn_varlen_fwd(q, k, v, cu_q, cu_k, 500, causal, 0.1)
        tfa.attn_varlen_fwd(q, k, v, cu_q, cu_k, 500, causal, 0.1, out_fp32=True)
        assert tfa.launch_count() - n0 == 2
    torch.cuda.synchronize()


@pytest.mark.gpu
def test_extension_varlen_entry(built):
    import attention_cutlass as ac
    lq = [300, 1, 129, 640]
    H, D = 4, 128
    g = torch.Generator(device="cpu")
    g.manual_seed(17)
    qkv = torch.empty((sum(lq), 3, H, D), dtype=torch.float32).normal_(0, 0.5, generator=g).to(torch.bfloat16).cuda()
    cu = torch.tensor(np.concatenate([[0], np.cumsum(lq)]), dtype=torch.int32, device="cuda")
    q, k, v = qkv.unbind(1)
    out, lse = ac.flash_attention_v2_varlen(q, k, v, cu, cu, max(lq), True, D ** -0.5)
    out2, lse2 = ac.flash_attention_v2_varlen(q.contiguous(), k.contiguous(), v.contiguous(), cu, cu, max(lq), True,
                                              D ** -0.5)
    torch.cuda.synchronize()
    assert out.shape == (sum(lq), H, D) and out.dtype == torch.bfloat16 and lse.shape == (H, sum(lq))
    assert torch.equal(out, out2) and torch.equal(lse, lse2)
    with pytest.raises(RuntimeError, match="int32"):
        ac.flash_attention_v2_varlen(q, k, v, cu.long(), cu, max(lq), True, 0.1)
    with pytest.raises(RuntimeError, match="device"):
        ac.flash_attention_v2_varlen(q, k, v, cu.cpu(), cu.cpu(), max(lq), True, 0.1)
    with pytest.raises(RuntimeError, match="B \\+ 1"):
        ac.flash_attention_v2_varlen(q, k, v, cu, cu[:-1], max(lq), True, 0.1)
    with pytest.raises(RuntimeError, match="B \\+ 1"):
        ac.flash_attention_v2_varlen(q, k, v, cu[:1], cu[:1], max(lq), True, 0.1)
    with pytest.raises(RuntimeError, match="multiple of K/V heads"):
        ac.flash_attention_v2_varlen(q, k[:, :3], v[:, :3], cu, cu, max(lq), True, 0.1)
    with pytest.raises(RuntimeError, match="max_seqlen_q"):
        ac.flash_attention_v2_varlen(q, k, v, cu, cu, 0, True, 0.1)
