"""Every sm_90a forward mode on strided views inside poisoned buffers.

Each GPU case runs one call twice: once on clean contiguous tensors, once on the same values placed as strided views
inside buffers whose every other element is poison (+Inf, -Inf or NaN for 16-bit and fp32 elements, the e4m3 NaN codes
0x7f / 0xff for FP8 ones), with out, lse and q_rot written into poisoned buffers too.  The two runs must agree bit for
bit on out, lse, the appended cache rows and q_rot; no input byte and no output byte outside the output's own elements
may change; and the clean run must be within budget of the float64 reference (test_fwd_float64_reference, test_fwd_fp8).
A masked key's P = 0 does not cancel 0 * Inf or 0 * NaN, so a kernel that lets one byte it must not use into a product
turns a row into NaN here.

Layouts: dense q / k / v as a slice of a static (B, H, S + 200, D) cache, as BSHD, as views of one fused
(B, S, Hq + 2 Hkv, D) projection, as BSHD rows padded by 64 elements, and q and k / v on different layouts in one
call, out at q's strides (for FP8: q's element strides in a 16-bit or fp32 buffer); packed varlen tensors as views of
one fused (total, Hq + 2 Hkv, D) buffer or padded between heads; KV-cache pools as one layer of a stacked
(3, num_blocks, page, Hkv, D) buffer or as K and V interleaved in one (num_blocks, 2, page, Hkv, D) buffer, whose block
stride is then twice the pool's; unused slots, spare blocks and the block-table entries past each sequence's last page
(which point at a poisoned spare block) hold poison; q, k_new and v_new are views of head-padded buffers.

CPU: every layout's argument struct, on fake aligned addresses, passes every argument check and stops at the device or
workspace check; the poisoned-view builders put the clean values in the view and poison everywhere else."""
import ctypes
import math

import pytest
import torch

from test_fwd_float64_reference import compare, reference
from test_fwd_fp8 import compare as fp8_compare, deq, fp8_reference, make_fp8
from test_kvcache import gather, make_cache
from test_kvcache_fp8 import FP8, bits, make_fp8_cache
from test_kvcache_rotary import rope_tables
from test_varlen import offsets, seq

POISON16 = (math.inf, -math.inf, math.nan)
POISON8 = (0x7F, 0xFF)
GUARD = 256
TFA_EARCH, TFA_EINVAL_WORKSPACE = -7, -11


# ------------------------------------------------------------------ poisoned views --------------------------------------

def poison_full(shape, dtype, which, device):
    """A buffer every element of which is poison number `which`."""
    if dtype == FP8:
        return torch.full(shape, POISON8[which % 2], dtype=torch.uint8, device=device).view(FP8)
    return torch.full(shape, POISON16[which % 3], dtype=dtype, device=device)


class Poisoned:
    """A poison-filled buffer of `shape` and its view `fn(buf)`, which holds `clean` (or stays poison for an output)."""

    def __init__(self, shape, fn, dtype, which, device, clean=None):
        self.buf = poison_full(shape, dtype, which, device)
        self.fn = fn
        self.view = fn(self.buf)
        if clean is not None:
            assert self.view.shape == clean.shape
            bits(self.view).copy_(bits(clean))
        self.before = self.buf.clone()

    def outside(self):
        keep = torch.ones(self.buf.shape, dtype=torch.bool, device=self.buf.device)
        self.fn(keep).fill_(False)
        return keep

    def assert_kept(self, what, whole=False):
        """Inputs (`whole`): no byte changed.  Outputs: no byte outside the view changed."""
        if whole:
            assert torch.equal(bits(self.buf), bits(self.before)), f"{what}: an input byte changed"
        else:
            keep = self.outside()
            assert torch.equal(bits(self.buf)[keep], bits(self.before)[keep]), f"{what}: a byte outside it changed"


def guarded_layout(shape):
    """A contiguous tensor of `shape` between GUARD poison elements on both sides."""
    n = math.prod(shape)
    return (GUARD + n + GUARD,), lambda b: b[GUARD:GUARD + n].view(shape)


def dense_layout(name, B, H, S, D):
    """(buffer shape, view fn) of a logical (B, H, S, D) tensor."""
    if name == "static_cache":
        return (B, H, S + 200, D), lambda b: b[:, :, :S]
    if name == "bshd":
        return (B, S, H, D), lambda b: b.permute(0, 2, 1, 3)
    if name == "padded_rows":
        return (B, S, H * D + 64), lambda b: b[:, :, :H * D].unflatten(2, (H, D)).permute(0, 2, 1, 3)
    raise ValueError(name)


def fused_layout(B, S, Hq, Hkv, D):
    """q, k and v as views of one fused (B, S, Hq + 2 Hkv, D) projection: (buffer shape, [fn_q, fn_k, fn_v])."""
    cut = (0, Hq, Hq + Hkv, Hq + 2 * Hkv)
    return (B, S, Hq + 2 * Hkv, D), [lambda b, i=i: b[:, :, cut[i]:cut[i + 1]].permute(0, 2, 1, 3) for i in range(3)]


# q layout, k / v layout; "fused" puts all three in one buffer
DENSE_LAYOUTS = [("static_cache", "static_cache"), ("bshd", "bshd"), ("fused", "fused"),
                 ("padded_rows", "padded_rows"), ("bshd", "static_cache"), ("padded_rows", "bshd")]
DENSE_IDS = [f"q_{a}-kv_{b}" if a != b else a for a, b in DENSE_LAYOUTS]


def place_dense(layout, q, k, v, which, out_dtype):
    """The poisoned copies of q, k and v on `layout` and the poisoned out buffer at q's strides."""
    (B, Hq, Sq, D), Hkv, Sk = q.shape, k.shape[1], k.shape[2]
    lq, lkv = layout
    if lq == "fused":
        assert Sq == Sk
        shape, fns = fused_layout(B, Sq, Hq, Hkv, D)
        buf = Poisoned(shape, lambda b: b, q.dtype, which, q.device)
        for fn, t in zip(fns, (q, k, v)):
            bits(fn(buf.buf)).copy_(bits(t))
        buf.before = buf.buf.clone()
        ins = [buf]
        views = [fn(buf.buf) for fn in fns]
        oshape, ofn = shape, fns[0]
    else:
        qs, qfn = dense_layout(lq, B, Hq, Sq, D)
        ks, kfn = dense_layout(lkv, B, Hkv, Sk, D)
        ins = [Poisoned(qs, qfn, q.dtype, which, q.device, q), Poisoned(ks, kfn, k.dtype, which + 1, q.device, k),
               Poisoned(ks, kfn, v.dtype, which + 2, q.device, v)]
        views = [p.view for p in ins]
        oshape, ofn = qs, qfn
    out = Poisoned(oshape, ofn, out_dtype, which + 1, q.device)
    assert out.view.stride() == views[0].stride()
    return ins, views, out


# ------------------------------------------------------------------ calls -----------------------------------------------

def dense_call(tfa, q, k, v, out, lse, causal, scale, f32, ns, dt16, ws_fill=None, quant=None):
    """tfa_attn_fwd / tfa_attn_fp8_fwd on (B, H, S, D) views with unit head_dim stride, out at q's strides, through
    the argument struct itself.  dt16: the 16-bit type (q's, or an FP8 call's output type); `ws_fill`: the split-KV
    workspace's contents (None: uninitialised)."""
    assert k.stride() == v.stride() and q.stride(3) == 1 and k.stride(3) == 1 and out.stride() == q.stride()
    (B, Hq, Sq, D), Hkv, Sk = q.shape, k.shape[1], k.shape[2]
    dtype = tfa.TFA_BF16 if dt16 == torch.bfloat16 else tfa.TFA_FP16
    st = torch.cuda.current_stream().cuda_stream
    a = tfa.AttnArgs(q.data_ptr(), k.data_ptr(), v.data_ptr(), out.data_ptr(), lse.data_ptr(), B, Hq, Hkv, Sq, Sk, D,
                     *q.stride()[:3], *k.stride()[:3], dtype, int(causal), scale, int(f32), ns, None, 0, st)
    L = tfa.lib()
    n = int(L.tfa_attn_num_splits(ctypes.byref(a)))
    ws = None
    if n > 1:
        need = int(L.tfa_attn_workspace_bytes(ctypes.byref(a), n))
        ws = torch.empty((need + 3) // 4, dtype=torch.float32, device=q.device)
        if ws_fill is not None:
            ws.fill_(ws_fill)
        a.workspace, a.workspace_bytes = ws.data_ptr(), need
    if quant is not None:
        tfa.check(L.tfa_attn_fp8_fwd(ctypes.byref(a), ctypes.byref(tfa.QkvQuantArgs(2, *quant))))
    else:
        tfa.check(L.tfa_attn_fwd(ctypes.byref(a)))
    torch.cuda.synchronize()
    return n


def assert_same(what, clean, got):
    assert torch.equal(bits(clean), bits(got)), f"{what} differs from the clean run"


# ------------------------------------------------------------------ CPU -------------------------------------------------

@pytest.fixture(scope="module")
def tfa(built):
    import tfa_ctypes
    tfa_ctypes.lib()
    return tfa_ctypes


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16, torch.float32, FP8])
def test_poisoned_views_hold_clean_values_and_poison_elsewhere(dtype):
    """On CPU tensors: every builder's view equals the clean tensor bit for bit, every element outside it is poison."""
    g = torch.Generator().manual_seed(3)
    mk = lambda *s: (torch.empty(s).normal_(0, 0.5, generator=g) * 8).to(dtype)
    B, Hq, Hkv, S, D = 2, 4, 2, 33, 64
    q, k, v = mk(B, Hq, S, D), mk(B, Hkv, S, D), mk(B, Hkv, S, D)
    checked = []
    for which in range(3):
        for layout in DENSE_LAYOUTS:
            ins, views, out = place_dense(layout, q, k, v, which, dtype)
            for t, got in zip((q, k, v), views):
                assert torch.equal(bits(got), bits(t)), layout
            for j, p in enumerate(ins + [out]):   # the fused buffer has nothing outside its three views
                pv = poison_full((1,), dtype, which + (j if p is not out else 1), "cpu")
                if p is out:                      # an output's buffer: all poison before the call
                    assert torch.equal(bits(p.buf), bits(pv).expand(p.buf.shape))
                rest = bits(p.buf)[p.outside()]            # none for BSHD and the fused buffer
                assert torch.equal(rest, bits(pv).expand(rest.shape)), (layout, which)
                checked.append(rest.numel())
        for shape, fn, t in (guarded_layout((3, 5, 8)) + (mk(3, 5, 8),),
                             ((B * S, Hq, D + 64), lambda b: b[:, :, :D], mk(B * S, Hq, D))):
            p = Poisoned(shape, fn, dtype, which, "cpu", t)
            rest = bits(p.buf)[p.outside()]
            assert torch.equal(bits(p.view), bits(t)) and rest.numel() > 0
            assert torch.equal(rest, bits(poison_full((1,), dtype, which, "cpu")).expand(rest.shape))
    assert len(checked) == 3 * 4 * len(DENSE_LAYOUTS) - 3 * 2 and min(checked) == 0 < max(checked)


def _fake_dense(tfa, layout, B, Hq, Hkv, Sq, Sk, D, fp8):
    """AttnArgs of `layout` on fake, 16-byte aligned addresses, 2 splits without a workspace."""
    dt = FP8 if fp8 else torch.bfloat16
    meta = lambda s: torch.empty(s, dtype=dt, device="meta")
    q, k = meta((B, Hq, Sq, D)), meta((B, Hkv, Sk, D))
    if layout[0] == "fused":
        shape, fns = fused_layout(B, Sq, Hq, Hkv, D)
        qv, kv = fns[0](meta(shape)), fns[1](meta(shape))
    else:
        qs, qfn = dense_layout(layout[0], B, Hq, Sq, D)
        ks, kfn = dense_layout(layout[1], B, Hkv, Sk, D)
        qv, kv = qfn(meta(qs)), kfn(meta(ks))
    assert qv.shape == q.shape and kv.shape == k.shape
    return tfa.AttnArgs(0x10000, 0x20000, 0x30000, 0x40000, 0x50000, B, Hq, Hkv, Sq, Sk, D, *qv.stride()[:3],
                        *kv.stride()[:3], 0, 1, 0.1, 0, 2, None, 0, None)


def test_layout_arguments_pass_every_check(tfa):
    """Each dense and dense-FP8 layout, and each cache pool layout with a padded q and interleaved k_new / v_new, on
    fake aligned addresses: every argument check passes and the call stops at the workspace check (two splits of at
    least two KV tiles asked for without a workspace) or, without an H100, at the device check."""
    L = tfa.lib()
    for layout in DENSE_LAYOUTS:
        for B, Hq, Hkv, S, D in ((1, 4, 2, 300, 64), (2, 4, 1, 129, 128), (3, 2, 2, 257, 64)):
            for fp8 in (False, True):
                a = _fake_dense(tfa, layout, B, Hq, Hkv, S, S, D, fp8)
                rc = (L.tfa_attn_fp8_fwd(ctypes.byref(a), ctypes.byref(tfa.QkvQuantArgs(2, 0.02, 0.03, 0.01)))
                      if fp8 else L.tfa_attn_fwd(ctypes.byref(a)))
                assert rc in (TFA_EINVAL_WORKSPACE, TFA_EARCH), (layout, B, Hq, Hkv, S, D, fp8, rc)
    ints = ctypes.create_string_buffer(4096 + 16)
    ip = (ctypes.addressof(ints) + 15) & ~15           # cache_seqlens and block table: host ints, never read
    for pool in ("stacked", "interleaved"):
        for fp8 in (False, True):
            B, Sq, Hq, Hkv, D, page, nblk, mbps, snew = 3, 4, 8, 2, 128, 128, 16, 4, 4
            ps, pfns = cache_pool_layout(pool, nblk, page, Hkv, D)
            kp = pfns[0](torch.empty(ps, dtype=FP8 if fp8 else torch.float16, device="meta"))
            qs, qfn = head_padded((B, Sq, Hq, D))
            qv = qfn(torch.empty(qs, dtype=torch.float16, device="meta"))
            ns_, nfns = new_layout((B, snew, Hkv, D))
            kn = nfns[0](torch.empty(ns_, dtype=torch.float16, device="meta"))
            a = tfa.KvcacheArgs(0x10000, 0x20000, 0x30000, 0x60000, 0x70000, 0x40000, 0x50000, ip, ip, B, Hq, Hkv, Sq,
                                D, nblk, page, mbps, snew, qv.stride(0), qv.stride(1), qv.stride(2), *kp.stride()[:3],
                                mbps, *kn.stride()[:3], 1, 1, 0.1, 0, 2, None, 0, None)
            rc = (L.tfa_attn_kvcache_fp8_fwd(ctypes.byref(a), None, ctypes.byref(tfa.KvQuantArgs(2, 0.5, 0.25)))
                  if fp8 else L.tfa_attn_kvcache_fwd(ctypes.byref(a)))
            assert rc in (TFA_EINVAL_WORKSPACE, TFA_EARCH), (pool, fp8, rc)


@pytest.mark.skipif(torch.cuda.is_available(), reason="without split-KV the call gets past its checks to the device")
def test_packed_layout_arguments_pass_every_check_without_a_device(tfa):
    """The varlen, FP8 varlen and varlen-cache calls on the packed layouts, fake aligned addresses: TFA_EARCH, the
    device check, is the first error."""
    L = tfa.lib()
    ints = ctypes.create_string_buffer(4096 + 16)
    ip = (ctypes.addressof(ints) + 15) & ~15
    total, Hq, Hkv, D = 700, 4, 2, 128
    for name in ("fused", "head_padded"):
        for fp8 in (False, True):
            dt = FP8 if fp8 else torch.bfloat16
            if name == "fused":
                shape, fns = packed_fused(total, Hq, Hkv, D)
                qv, kv = fns[0](torch.empty(shape, dtype=dt, device="meta")), fns[1](torch.empty(shape, dtype=dt,
                                                                                                 device="meta"))
            else:
                qs, qfn = head_padded((total, Hq, D))
                ks, kfn = head_padded((total, Hkv, D))
                qv, kv = qfn(torch.empty(qs, dtype=dt, device="meta")), kfn(torch.empty(ks, dtype=dt, device="meta"))
            a = tfa.VarlenArgs(0x10000, 0x20000, 0x30000, 0x40000, 0x50000, ip, ip, 3, Hq, Hkv, D, total, total, 300,
                               qv.stride(0), qv.stride(1), kv.stride(0), kv.stride(1), 0, 1, 0.1, 0, None)
            rc = (L.tfa_attn_varlen_fp8_fwd(ctypes.byref(a), ctypes.byref(tfa.QkvQuantArgs(2, 0.02, 0.03, 0.01)))
                  if fp8 else L.tfa_attn_varlen_fwd(ctypes.byref(a)))
            assert rc == TFA_EARCH, (name, fp8, rc)
    for pool in ("stacked", "interleaved"):
        for fp8 in (False, True):
            nblk, page, mbps = 16, 128, 4
            ps, pfns = cache_pool_layout(pool, nblk, page, Hkv, D)
            kp = pfns[0](torch.empty(ps, dtype=FP8 if fp8 else torch.float16, device="meta"))
            qs, qfn = head_padded((total, Hq, D))
            qv = qfn(torch.empty(qs, dtype=torch.float16, device="meta"))
            ns_, nfns = new_layout((total, Hkv, D))
            kn = nfns[0](torch.empty(ns_, dtype=torch.float16, device="meta"))
            a = tfa.VarlenKvcacheArgs(0x10000, 0x20000, 0x30000, 0x60000, 0x70000, 0x40000, 0x50000, ip, ip, ip, 3, Hq,
                                      Hkv, D, total, 300, nblk, page, mbps, qv.stride(0), qv.stride(1),
                                      *kp.stride()[:3], mbps, kn.stride(0), kn.stride(1), 1, 1, 0.1, 0, None)
            rc = (L.tfa_attn_varlen_kvcache_fp8_fwd(ctypes.byref(a), ctypes.byref(tfa.KvQuantArgs(2, 0.5, 0.25)))
                  if fp8 else L.tfa_attn_varlen_kvcache_fwd(ctypes.byref(a)))
            assert rc == TFA_EARCH, (pool, fp8, rc)


# ------------------------------------------------------------------ GPU: dense ------------------------------------------

# B, Hq, Hkv, Sq, Sk: tile edges, B = 1 and Hkv = 1 (make_tmap's size-1 strides), causal Sq > Sk (key-less rows)
DENSE_SHAPES = [(1, 4, 2, 127, 300), (2, 2, 1, 129, 129), (2, 4, 4, 300, 127), (1, 2, 1, 1, 300), (3, 2, 2, 300, 1),
                (2, 4, 1, 129, 300)]


def _dense_cases(D):
    i = 0
    for causal in (False, True):
        for kind in ("bf16", "fp16"):
            for f32 in (False, True):
                for ns in (1, 3):
                    yield i, causal, kind, f32, ns, DENSE_SHAPES[(i + D // 64) % len(DENSE_SHAPES)]
                    i += 1


def _dense_pair(tfa, layout, q, k, v, causal, scale, f32, ns, which, odt, quant=None):
    """The clean and the poisoned run of one dense call; returns the clean (out, lse) after checking the other."""
    (B, Hq, Sq, D) = q.shape
    out_dt = torch.float32 if f32 else odt
    out = torch.empty(q.shape, dtype=out_dt, device="cuda")
    lse = torch.empty((B, Hq, Sq), dtype=torch.float32, device="cuda")
    n0 = dense_call(tfa, q, k, v, out, lse, causal, scale, f32, ns, odt, quant=quant)
    ins, (qv, kv, vv), pout = place_dense(layout, q, k, v, which, out_dt)
    plse = Poisoned(*guarded_layout((B, Hq, Sq)), torch.float32, which, "cuda")
    n1 = dense_call(tfa, qv, kv, vv, pout.view, plse.view, causal, scale, f32, ns, odt, ws_fill=math.nan, quant=quant)
    assert n0 == n1
    for p in ins:
        p.assert_kept("q / k / v", whole=True)
    pout.assert_kept("out")
    plse.assert_kept("lse")
    assert_same("out", out, pout.view)
    assert_same("lse", lse, plse.view)
    return out, lse, n0


@pytest.mark.gpu
@pytest.mark.parametrize("D", [64, 128])
@pytest.mark.parametrize("layout", DENSE_LAYOUTS, ids=DENSE_IDS)
def test_dense_poisoned_layouts(tfa, layout, D):
    """tfa_attn_fwd: causal and not, bf16 and fp16, 16-bit and fp32 out, one pass and 3 splits (the combine writes
    into the strided out), against the float64 reference."""
    fails, splits = [], set()
    for i, causal, kind, f32, ns, (B, Hq, Hkv, Sq, Sk) in _dense_cases(D):
        if layout[0] == "fused":
            Sk = Sq
        g = torch.Generator().manual_seed(1000 * D + i)
        dt = torch.bfloat16 if kind == "bf16" else torch.float16
        mk = lambda *s: torch.empty(s).normal_(0.0, 0.5, generator=g).to(dt).cuda()
        q, k, v = mk(B, Hq, Sq, D), mk(B, Hkv, Sk, D), mk(B, Hkv, Sk, D)
        out, lse, n = _dense_pair(tfa, layout, q, k, v, causal, D ** -0.5, f32, ns, i, dt)
        splits.add(n)
        verdict = compare(out, lse, reference(q, k, v, causal, D ** -0.5), kind)
        if not verdict.ok:
            fails.append(f"B{B} Hq{Hq} Hkv{Hkv} Sq{Sq} Sk{Sk} {kind} causal={causal} f32={f32} ns={n}: {verdict.msg}")
    assert splits >= {1, 3} or layout[0] == "fused", splits
    assert not fails, "; ".join(fails[:6])


@pytest.mark.gpu
@pytest.mark.parametrize("D", [64, 128])
@pytest.mark.parametrize("layout", DENSE_LAYOUTS, ids=DENSE_IDS)
def test_dense_fp8_poisoned_layouts(tfa, layout, D):
    """tfa_attn_fp8_fwd on e4m3 views whose strides are multiples of 16, out at q's element strides inside a 16-bit or
    fp32 poison buffer, against the float64 reference of the dequantized problem."""
    scales = (0.0213, 0.0171, 0.0119)
    fails = []
    for i, causal, kind, f32, ns, (B, Hq, Hkv, Sq, Sk) in _dense_cases(D):
        if layout[0] == "fused":
            Sk = Sq
        q8, k8, v8 = make_fp8(B, Hq, Hkv, Sq, Sk, D, seed=2000 * D + i, scales=scales, device="cuda")
        dt = torch.bfloat16 if kind == "bf16" else torch.float16
        out, lse, n = _dense_pair(tfa, layout, q8, k8, v8, causal, D ** -0.5, f32, ns, i, dt, quant=scales)
        ref = fp8_reference(deq(q8, scales[0]), k8, v8, causal, D ** -0.5, scales[1], scales[2])
        ok, r, _, msg = fp8_compare(out, lse, ref, kind)
        if not ok:
            fails.append(f"B{B} Hq{Hq} Hkv{Hkv} Sq{Sq} Sk{Sk} {kind} causal={causal} f32={f32} ns={n}: {msg}")
    assert not fails, "; ".join(fails[:6])


# ------------------------------------------------------------------ GPU: varlen -----------------------------------------

def packed_fused(total, Hq, Hkv, D):
    """q, k and v of a packed batch as views of one fused (total, Hq + 2 Hkv, D) buffer."""
    cut = (0, Hq, Hq + Hkv, Hq + 2 * Hkv)
    return (total, Hq + 2 * Hkv, D), [lambda b, i=i: b[:, cut[i]:cut[i + 1]] for i in range(3)]


def head_padded(shape):
    """(..., H, D) with 64 poison elements after every head's D."""
    *lead, D = shape
    return (*lead, D + 64), lambda b: b[..., :D]


VARLEN = {
    # name: (lq, lk); "fused" shares cu_seqlens between q and k / v
    "fused": ([127, 1, 0, 300, 129, 64, 200], None),
    "head_padded": ([127, 1, 0, 300, 129, 64, 5], [300, 129, 5, 0, 1, 64, 257]),
}


@pytest.mark.gpu
@pytest.mark.parametrize("fp8", [False, True])
@pytest.mark.parametrize("name", list(VARLEN))
def test_varlen_poisoned_layouts(tfa, name, fp8):
    """tfa_attn_varlen_fwd / tfa_attn_varlen_fp8_fwd on packed views, out and lse contiguous between poison guards."""
    import numpy as np
    lq, lk = VARLEN[name]
    lk = lk or lq
    Hq, Hkv = 4, 2
    scales = (0.0213, 0.0171, 0.0119)
    cu = lambda ls: torch.tensor(np.concatenate([[0], np.cumsum(ls)]), dtype=torch.int32, device="cuda")
    cu_q, cu_k = cu(lq), cu(lk)
    tq, tk = sum(lq), sum(lk)
    fails = []
    for i, (causal, kind, f32, D) in enumerate([(True, "bf16", False, 128), (False, "fp16", True, 64),
                                                 (True, "fp16", True, 64), (False, "bf16", False, 128)]):
        dt = torch.bfloat16 if kind == "bf16" else torch.float16
        if fp8:
            q, k, v = (t[0].permute(1, 0, 2).contiguous() for t in make_fp8(1, Hq, Hkv, tq, tk, D, seed=50 + i,
                                                                               scales=scales, device="cuda"))
            kw = dict(q_scale=scales[0], k_scale=scales[1], v_scale=scales[2], out_dtype=dt)
        else:
            g = torch.Generator().manual_seed(50 + i)
            mk = lambda *s: torch.empty(s).normal_(0.0, 0.5, generator=g).to(dt).cuda()
            q, k, v = mk(tq, Hq, D), mk(tk, Hkv, D), mk(tk, Hkv, D)
            kw = {}
        out_dt = torch.float32 if f32 else dt
        scale = D ** -0.5
        out, lse = tfa.attn_varlen_fwd(q, k, v, cu_q, cu_k, max(lq), causal, scale, out_fp32=f32, **kw)
        if name == "fused":
            shape, fns = packed_fused(tq, Hq, Hkv, D)
            buf = Poisoned(shape, lambda b: b, q.dtype, i, "cuda")
            for fn, t in zip(fns, (q, k, v)):
                bits(fn(buf.buf)).copy_(bits(t))
            buf.before = buf.buf.clone()
            ins, (qv, kv, vv) = [buf], [fn(buf.buf) for fn in fns]
        else:
            ins = [Poisoned(*head_padded(t.shape), t.dtype, i + j, "cuda", t) for j, t in enumerate((q, k, v))]
            qv, kv, vv = (p.view for p in ins)
        pout = Poisoned(*guarded_layout(tuple(out.shape)), out_dt, i + 1, "cuda")
        plse = Poisoned(*guarded_layout(tuple(lse.shape)), torch.float32, i + 2, "cuda")
        tfa.attn_varlen_fwd(qv, kv, vv, cu_q, cu_k, max(lq), causal, scale, out_fp32=f32, out=pout.view, lse=plse.view,
                            **kw)
        torch.cuda.synchronize()
        for p in ins:
            p.assert_kept("q / k / v", whole=True)
        pout.assert_kept("out")
        plse.assert_kept("lse")
        assert_same("out", out, pout.view)
        assert_same("lse", lse, plse.view)
        for (q0, q1), (k0, k1) in zip(offsets(lq), offsets(lk)):
            if q1 == q0:
                continue
            o_b, l_b = out[q0:q1].permute(1, 0, 2)[None], lse[:, q0:q1][None]
            if fp8 and k1 > k0:
                ref = fp8_reference(deq(seq(q, q0, q1), scales[0]), seq(k, k0, k1), seq(v, k0, k1), causal, scale,
                                    scales[1], scales[2])
                ok, _, _, msg = fp8_compare(o_b, l_b, ref, kind)
            elif fp8:                             # no key: every row exactly 0 / +inf
                verdict = compare(o_b, l_b, reference(deq(seq(q, q0, q1), scales[0]), seq(k, k0, k1), seq(v, k0, k1),
                                                      causal, scale), kind)
                ok, msg = verdict.ok, verdict.msg
            else:
                verdict = compare(o_b, l_b, reference(seq(q, q0, q1), seq(k, k0, k1), seq(v, k0, k1), causal, scale),
                                  kind)
                ok, msg = verdict.ok, verdict.msg
            if not ok:
                fails.append(f"case {i} sequence Sq {q1 - q0} Sk {k1 - k0}: {msg}")
    assert not fails, "; ".join(fails[:6])


# ------------------------------------------------------------------ GPU: KV cache ---------------------------------------

def cache_pool_layout(name, nblk, page, Hkv, D):
    """K and V pools (num_blocks, page, Hkv, D): layer 1 of stacked (3, ...) buffers (one per pool), or K and V
    interleaved in one (num_blocks, 2, page, Hkv, D) buffer.  Returns (buffer shape, [fn_k, fn_v])."""
    if name == "stacked":
        return (3, nblk, page, Hkv, D), [lambda b: b[1], lambda b: b[1]]
    if name == "interleaved":
        return (nblk, 2, page, Hkv, D), [lambda b: b[:, 0], lambda b: b[:, 1]]
    raise ValueError(name)


def new_layout(shape):
    """k_new / v_new as slots 0 and 1 of one buffer, heads padded by 64 poison elements: (shape, [fn_k, fn_v])."""
    *lead, Hkv, D = shape
    return (*lead, 2, Hkv, D + 64), [lambda b: b[..., 0, :, :D], lambda b: b[..., 1, :, :D]]


def valid_slots(table, Ks, nblk, page):
    """(num_blocks, page) mask of the slots that hold key < K_b of some sequence b."""
    m = torch.zeros((nblk, page), dtype=torch.bool)
    tab = table.cpu().tolist()
    for b, K in enumerate(Ks):
        for key in range(K):
            m[tab[b][key // page], key % page] = True
    return m.cuda()


def retable(table, pool_k, pool_v, Ks_after, page):
    """Point every table entry past sequence b's last page (of its K_b keys after the append) at a spare block, which
    holds no sequence's keys; returns the new table."""
    nblk = pool_k.shape[0]
    used = set(table.flatten().tolist())
    spare = next(b for b in range(nblk) if b not in used)
    t = table.clone()
    for b, K in enumerate(Ks_after):
        t[b, -(-K // page):] = spare
    return t


class CachePools:
    """The clean pools (unused slots 0) and their poisoned copies on `layout`: the valid keys of each sequence (before
    the append) in the view, every other slot, the spare blocks and every other byte of the buffer poison."""

    def __init__(self, layout, kp, vp, table, lens_now, which):
        nblk, page, Hkv, D = kp.shape
        shape, fns = cache_pool_layout(layout, nblk, page, Hkv, D)
        valid = valid_slots(table, lens_now, nblk, page)
        self.bufs = []
        if layout == "interleaved":
            buf = poison_full(shape, kp.dtype, which, "cuda")
            self.bufs = [buf]
            views = [fn(buf) for fn in fns]
        else:
            self.bufs = [poison_full(shape, kp.dtype, which + j, "cuda") for j in range(2)]
            views = [fn(b) for fn, b in zip(fns, self.bufs)]
        for view, clean in zip(views, (kp, vp)):
            bits(view)[valid] = bits(clean)[valid]
        self.fns, self.views, self.before = fns, views, [b.clone() for b in self.bufs]

    def assert_after(self, clean_k, clean_v, table, Ks_after):
        """After the call: the slots of keys < K_b hold the clean run's (appended rows included), every other byte of
        the buffers is what it was."""
        nblk, page = clean_k.shape[:2]
        valid = valid_slots(table, Ks_after, nblk, page)
        want = [b.clone() for b in self.before]
        wviews = [fn(w) for fn, w in zip(self.fns, want if len(want) == 2 else want * 2)]
        for wv, clean in zip(wviews, (clean_k, clean_v)):
            bits(wv)[valid] = bits(clean)[valid]
        for got, w in zip(self.bufs, want):
            assert torch.equal(bits(got), bits(w)), "a cache byte other than the appended rows changed, or an " \
                                                     "appended row differs from the clean run"


def _gather(pool, table, b, K):
    if pool.dtype == FP8:
        return gather(pool.view(torch.uint8), table, b, K).view(FP8)
    return gather(pool, table, b, K)


def quantize_q(q, fp8):
    """q for the call: 16-bit as given, or with fp8 = (q_scale, k_scale, v_scale) e4m3 codes as a caller quantizes."""
    return (q.float() / fp8[0]).clamp(-448, 448).to(FP8) if fp8 is not None and len(fp8) == 3 else q


def check_seq(q, k, v, out, lse, causal, scale, fp8, kind):
    """(ok, message) of one sequence against the float64 reference: the FP8 budget for e4m3 q (fp8 of length 3),
    the 16-bit one otherwise (and for a sequence without keys, whose rows must be exactly 0 / +inf)."""
    ks, vs = fp8[-2:] if fp8 else (1.0, 1.0)
    if fp8 is not None and len(fp8) == 3:
        qd = deq(q, fp8[0])
        if k.shape[2]:
            ok, _, _, msg = fp8_compare(out, lse, fp8_reference(qd, k, v, causal, scale, ks, vs), kind)
            return ok, msg
        q = qd
    verdict = compare(out, lse, reference(q, k, v, causal, scale, ks, vs), kind)
    return verdict.ok, verdict.msg


# name, pool layout, FP8 scales or None, Sq, snew, num_splits, rotary (rotary_dim, interleaved) or None.  FP8 scales
# (k_scale, v_scale): an FP8 cache with a 16-bit q; (q_scale, k_scale, v_scale): e4m3 q codes too (kCacheQkv8)
CACHE = [
    ("stacked", "stacked", None, 1, 1, 1, None),
    ("stacked_splits", "stacked", None, 4, 4, 3, None),
    ("interleaved", "interleaved", None, 4, 0, 1, None),
    ("interleaved_splits", "interleaved", None, 1, 1, 3, None),
    ("fp8_stacked", "stacked", (0.0213, 0.0117), 1, 1, 3, None),
    ("fp8_interleaved", "interleaved", (0.0311, 0.0089), 4, 4, 1, None),
    ("rotary_decode", "interleaved", None, 1, 1, 3, (64, False)),
    ("fp8_rotary_decode", "stacked", (0.0213, 0.0117), 1, 1, 1, (128, True)),
    ("qkv8_stacked", "stacked", (0.0213, 0.0171, 0.0117), 1, 1, 3, None),
    ("qkv8_interleaved", "interleaved", (0.0213, 0.0311, 0.0089), 4, 4, 1, None),
]


@pytest.mark.gpu
@pytest.mark.parametrize("name,pool,fp8,Sq,snew,ns,rotary", CACHE, ids=[c[0] for c in CACHE])
def test_cache_poisoned_layouts(tfa, name, pool, fp8, Sq, snew, ns, rotary):
    """tfa_attn_kvcache_fwd (16-bit and FP8 pools, rotary, e4m3 q): q a view of a head-padded buffer (for e4m3 q its
    strides are multiples of 16 bytes), out at q's element strides inside poison, k_new / v_new interleaved views, the
    pools as above."""
    lens = [0, 1, 127, 128, 129, 300, 255, 511]
    Hq, Hkv, page = 8, 2, 128
    D = 64 if (fp8 is None) == (ns == 1) else 128
    kind = "bf16" if ns == 1 else "fp16"
    dt = torch.bfloat16 if kind == "bf16" else torch.float16
    causal = Sq > 1 or rotary is not None
    B = len(lens)
    if fp8:
        q, kp, vp, table, sl = make_fp8_cache(lens, Sq, Hq, Hkv, D, kind, page, seed=70, fill=0, snew=snew)
    else:
        q, kp, vp, table, sl = make_cache(lens, Sq, Hq, Hkv, D, kind, page, seed=70, fill=0.0, snew=snew)
    cap = table.shape[1] * page
    Ks = [min(max(L, 0), cap - snew) + snew for L in lens]
    table = retable(table, kp, vp, Ks, page)
    g = torch.Generator().manual_seed(71)
    kn, vn = ((torch.empty(B, snew, Hkv, D).normal_(0, 0.5, generator=g).to(dt).cuda() for _ in range(2)) if snew
              else (None, None))
    q = quantize_q(q, fp8)
    ks, vs = fp8[-2:] if fp8 else (1.0, 1.0)
    qkw = dict(q_scale=fp8[0], out_dtype=dt) if len(fp8 or ()) == 3 else {}
    scale = D ** -0.5
    rot, rot_p = {}, {}
    if rotary:
        rd, il = rotary
        cos, sin = rope_tables(cap + 64, rd, kind)
        rot = dict(rotary_cos=cos, rotary_sin=sin, rotary_interleaved=il, q_rot=torch.empty_like(q))
    k1, v1 = kp.clone(), vp.clone()
    out, lse = tfa.attn_kvcache_fwd(q, k1, v1, sl, table, kn, vn, is_causal=causal, scale=scale, num_splits=ns,
                                    k_scale=ks, v_scale=vs, **rot, **qkw)
    torch.cuda.synchronize()
    # the poisoned run
    which = len(name)
    pools = CachePools(pool, kp, vp, table, [min(max(L, 0), cap - snew) for L in lens], which)
    pq = Poisoned(*head_padded(tuple(q.shape)), q.dtype, which, "cuda", q)
    pout = Poisoned(*head_padded(tuple(q.shape)), dt, which + 1, "cuda")
    plse = Poisoned(*guarded_layout((B, Hq, Sq)), torch.float32, which + 2, "cuda")
    pn = None
    if snew:
        shape, fns = new_layout(tuple(kn.shape))
        pn = Poisoned(shape, lambda b: b, dt, which, "cuda")
        bits(fns[0](pn.buf)).copy_(bits(kn))
        bits(fns[1](pn.buf)).copy_(bits(vn))
        pn.before = pn.buf.clone()
        kn2, vn2 = fns[0](pn.buf), fns[1](pn.buf)
    else:
        kn2 = vn2 = None
    if rotary:
        pr = Poisoned(*guarded_layout(tuple(q.shape)), dt, which, "cuda")
        rot_p = dict(rot, q_rot=pr.view)
    assert pout.view.stride() == pq.view.stride()
    tfa.attn_kvcache_fwd(pq.view, pools.views[0], pools.views[1], sl, table, kn2, vn2, is_causal=causal, scale=scale,
                         num_splits=ns, out=pout.view, lse=plse.view, k_scale=ks, v_scale=vs, **rot_p, **qkw)
    torch.cuda.synchronize()
    pq.assert_kept("q", whole=True)
    if pn is not None:
        pn.assert_kept("k_new / v_new", whole=True)
    pout.assert_kept("out")
    plse.assert_kept("lse")
    assert_same("out", out, pout.view)
    assert_same("lse", lse, plse.view)
    pools.assert_after(k1, v1, table, Ks)
    qa = q
    if rotary:
        pr.assert_kept("q_rot")
        assert_same("q_rot", rot["q_rot"], pr.view)
        qa = rot["q_rot"]
    fails = []
    for b, K in enumerate(Ks):
        ok, msg = check_seq(qa[b:b + 1].permute(0, 2, 1, 3), _gather(k1, table, b, K), _gather(v1, table, b, K),
                            out[b:b + 1].permute(0, 2, 1, 3), lse[b:b + 1], causal, scale, fp8, kind)
        if not ok:
            fails.append(f"sequence {b} (K {K}): {msg}")
    assert not fails, "; ".join(fails)


@pytest.mark.gpu
@pytest.mark.parametrize("pool", ["stacked", "interleaved"])
@pytest.mark.parametrize("fp8", [None, (0.0371, 0.0093), (0.0213, 0.0371, 0.0093)])
def test_varlen_cache_poisoned_layouts(tfa, pool, fp8):
    """tfa_attn_varlen_kvcache_fwd (16-bit and FP8 pools, e4m3 q): one mixed batch of prefill chunks and one-token
    decodes with an append, packed q a view of a head-padded buffer, k_new / v_new interleaved views, out and lse
    between poison guards."""
    import numpy as np
    sq = [129, 1, 1, 300, 0, 1, 64, 1]
    lens = [0, 1, 127, 128, 300, 255, 513, 383]
    Hq, Hkv, page = 8, 2, 128
    D, kind = (128, "bf16") if fp8 is None else (64, "fp16")
    dt = torch.bfloat16 if kind == "bf16" else torch.float16
    B, total = len(sq), sum(sq)
    if fp8:
        _, kp, vp, table, sl = make_fp8_cache(lens, 1, Hq, Hkv, D, kind, page, seed=80, fill=0, snew=max(sq))
    else:
        _, kp, vp, table, sl = make_cache(lens, 1, Hq, Hkv, D, kind, page, seed=80, fill=0.0, snew=max(sq))
    cap = table.shape[1] * page
    Ls = [min(max(L, 0), cap - n) for L, n in zip(lens, sq)]
    Ks = [L + n for L, n in zip(Ls, sq)]
    table = retable(table, kp, vp, Ks, page)
    g = torch.Generator().manual_seed(81)
    mk = lambda *s: torch.empty(s).normal_(0.0, 0.5, generator=g).to(dt).cuda()
    q, kn, vn = mk(total, Hq, D), mk(total, Hkv, D), mk(total, Hkv, D)
    q = quantize_q(q, fp8)
    cu = torch.tensor(np.concatenate([[0], np.cumsum(sq)]), dtype=torch.int32, device="cuda")
    ks, vs = fp8[-2:] if fp8 else (1.0, 1.0)
    qkw = dict(q_scale=fp8[0], out_dtype=dt) if len(fp8 or ()) == 3 else {}
    scale = D ** -0.5
    k1, v1 = kp.clone(), vp.clone()
    out, lse = tfa.attn_varlen_kvcache_fwd(q, k1, v1, cu, max(sq), sl, table, kn, vn, is_causal=True, scale=scale,
                                           k_scale=ks, v_scale=vs, **qkw)
    torch.cuda.synchronize()
    which = 2 if fp8 is None else len(fp8) - 1
    pools = CachePools(pool, kp, vp, table, Ls, which)
    pq = Poisoned(*head_padded(tuple(q.shape)), q.dtype, which, "cuda", q)
    shape, fns = new_layout(tuple(kn.shape))
    pn = Poisoned(shape, lambda b: b, dt, which + 1, "cuda")
    bits(fns[0](pn.buf)).copy_(bits(kn))
    bits(fns[1](pn.buf)).copy_(bits(vn))
    pn.before = pn.buf.clone()
    pout = Poisoned(*guarded_layout(tuple(out.shape)), dt, which, "cuda")
    plse = Poisoned(*guarded_layout(tuple(lse.shape)), torch.float32, which + 1, "cuda")
    tfa.attn_varlen_kvcache_fwd(pq.view, pools.views[0], pools.views[1], cu, max(sq), sl, table, fns[0](pn.buf),
                                fns[1](pn.buf), is_causal=True, scale=scale, out=pout.view, lse=plse.view, k_scale=ks,
                                v_scale=vs, **qkw)
    torch.cuda.synchronize()
    pq.assert_kept("q", whole=True)
    pn.assert_kept("k_new / v_new", whole=True)
    pout.assert_kept("out")
    plse.assert_kept("lse")
    assert_same("out", out, pout.view)
    assert_same("lse", lse, plse.view)
    pools.assert_after(k1, v1, table, Ks)
    fails = []
    for b, ((r0, r1), K) in enumerate(zip(offsets(sq), Ks)):
        if r1 == r0:
            continue
        ok, msg = check_seq(q[r0:r1].permute(1, 0, 2)[None], _gather(k1, table, b, K), _gather(v1, table, b, K),
                            out[r0:r1].permute(1, 0, 2)[None], lse[:, r0:r1][None], True, scale, fp8, kind)
        if not ok:
            fails.append(f"sequence {b} (Sq {r1 - r0}, K {K}): {msg}")
    assert not fails, "; ".join(fails)
