"""Rotary position embedding in the KV-cache forward: tfa_attn_kvcache_rotary_fwd /
attention_cutlass.flash_attention_v2_kvcache_rotary / tfa_ctypes.attn_kvcache_fwd(rotary_cos=...).

CPU: the entry point is declared and exported, its error code and string exist, every argument error comes back before
any device work, the host-callable position rule matches its definition exhaustively (clamp included), and the
existing KV-cache binding keeps its signature and docstring.
GPU: out, lse and the whole K/V pool equal, bit for bit, rotating q / k_new in eager torch fp32 and calling the
unrotated forward; a float64 reference agrees within the KV-cache tolerances; the call writes exactly the appended
tokens (rotated K, verbatim tail dimensions, unrotated V, dropped tokens), leaves its inputs and every guard byte alone,
never reads a cos/sin row past seqlen_ro - 1, replays from a CUDA graph with new lengths and tables, and is 2 / 3
launches."""
import ctypes
import os

import pytest
import torch

from test_kvcache import _dt, bits, check_keyless, declared_functions, make_cache, scatter_append

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

TFA_EINVAL_PTR = -1
TFA_EINVAL_ROTARY = -14


# ------------------------------------------------------------------ CPU ------------------------------------------------

def test_header_declares_and_library_exports_kvcache_rotary(built):
    import tfa_ctypes
    assert "tfa_attn_kvcache_rotary_fwd" in declared_functions()
    header = open(os.path.join(ROOT, "include", "tfa_b200.h")).read()
    assert "TFA_EINVAL_ROTARY (-14)" in header and "typedef struct tfa_rotary_args" in header
    assert "#define TFA_ABI_VERSION 2" in header
    L = ctypes.CDLL(tfa_ctypes.LIB_PATH)
    assert hasattr(L, "tfa_attn_kvcache_rotary_fwd")


def test_rotary_error_string(built):
    import tfa_ctypes
    msg = tfa_ctypes.lib().tfa_error_string(TFA_EINVAL_ROTARY)
    assert msg.startswith(b"tfa:") and b"rotary_dim" in msg and b"seqlen_ro" in msg and b"k_new" in msg


def test_rotary_argument_validation_without_device(built):
    """Host buffers only: every code must come back before anything touches a device (a call that got that far would
    fail with a CUDA error on a CPU-only box, and must never happen with host pointers on a GPU box)."""
    import tfa_ctypes
    L = tfa_ctypes.lib()
    buf = ctypes.create_string_buffer(8192 + 16)
    base = (ctypes.addressof(buf) + 15) & ~15
    ints = base + 1024
    tabs = base + 2048                                        # 16-byte aligned cos / sin / q_rot stand-ins
    Hq, Hkv, D, page, mbps = 4, 2, 64, 256, 4
    cap = page * mbps

    def kv(**kw):
        return tfa_ctypes.KvcacheArgs(
            base, base, base, kw.get("k_new", base), kw.get("v_new", base), base, None, ints, ints, 2, Hq, Hkv, 1,
            kw.get("D", D), 8, page, mbps, 1, Hq * D, Hq * D, D, page * Hkv * D, Hkv * D, D, mbps, Hkv * D, Hkv * D,
            D, 0, kw.get("causal", 1), 0.1, 0, 1, None, 0, None)

    def ro(**kw):
        return tfa_ctypes.RotaryArgs(kw.get("cos", tabs), kw.get("sin", tabs + 512), kw.get("seqlen_ro", cap),
                                     kw.get("rd", D), kw.get("il", 0), kw.get("q_rot", tabs + 1024))

    def call(kva=None, **kw):
        return L.tfa_attn_kvcache_rotary_fwd(ctypes.byref(kva or kv()), ctypes.byref(ro(**kw)))

    E = TFA_EINVAL_ROTARY
    assert L.tfa_attn_kvcache_rotary_fwd(None, ctypes.byref(ro())) == TFA_EINVAL_PTR
    assert L.tfa_attn_kvcache_rotary_fwd(ctypes.byref(kv()), None) == TFA_EINVAL_PTR
    for rd in (15, 17, 24, 40, 0, -16, D + 16, 2 * D, 8):     # odd, not a multiple of 16, 0, negative, > D
        assert call(rd=rd) == E, rd
    for name in ("cos", "sin", "q_rot"):
        assert call(**{name: None}) == E, name
        for off in (2, 8):
            assert call(**{name: tabs + 2048 + off}) == E, (name, off)
    assert call(seqlen_ro=cap - 1) == E and call(seqlen_ro=0) == E and call(seqlen_ro=-5) == E
    assert call(kv(k_new=None, v_new=None)) == E              # rotary rotates the appended keys: they are required
    assert call(kv(k_new=None, v_new=None), il=1) == E
    # the cache / shape checks keep their own codes and come first
    assert call(kv(k_new=base, v_new=None)) == -13
    assert call(kv(D=96)) == -2 and call(kv(D=96), rd=8) == -2


def _rotary_pos_lib():
    import tfa_ctypes
    L = tfa_ctypes.lib()
    L.tfa_internal_rotary_pos.argtypes = [ctypes.c_int] * 5
    L.tfa_internal_rotary_pos.restype = ctypes.c_int
    return L


def test_rotary_pos_exhaustively(built):
    """Keys at L + i; queries at L + i (causal) or L (not); clamped to seqlen_ro - 1, for every clamped cache length of
    small capacities and every row a call can have."""
    L = _rotary_pos_lib()
    for cap in (1, 7, 128, 200):
        for seqlen_ro in sorted({cap, cap + 1, cap + 33}):
            for Ln in range(0, cap + 1):
                for i in range(0, min(cap, 40) + 8):
                    for causal in (0, 1):
                        for is_q in (0, 1):
                            pos = Ln if (is_q and not causal) else Ln + i
                            want = min(pos, seqlen_ro - 1)
                            assert L.tfa_internal_rotary_pos(Ln, i, causal, is_q, seqlen_ro) == want, \
                                (cap, seqlen_ro, Ln, i, causal, is_q)


KVCACHE_DOC = (
    "flash_attention_v2_kvcache(arg0: torch.Tensor, arg1: torch.Tensor, arg2: torch.Tensor, arg3: torch.Tensor, "
    "arg4: torch.Tensor | None, arg5: torch.Tensor | None, arg6: torch.Tensor | None, arg7: bool, "
    "arg8: typing.SupportsFloat, arg9: typing.SupportsInt) -> list[torch.Tensor]\n\n"
    "attention against a (paged) KV cache with an optional in-place append: (q, k_cache, v_cache, cache_seqlens, "
    "block_table, k_new, v_new, is_causal, scale, num_splits)\n")


def test_kvcache_binding_unchanged_and_rotary_binding_present(built):
    import attention_cutlass as ac
    assert ac.flash_attention_v2_kvcache.__doc__ == KVCACHE_DOC
    doc = ac.flash_attention_v2_kvcache_rotary.__doc__
    assert doc.startswith("flash_attention_v2_kvcache_rotary(arg0: torch.Tensor")
    assert "arg12: typing.SupportsInt) -> list[torch.Tensor]" in doc and "rotary_cos, rotary_sin" in doc


# ------------------------------------------------------------------ GPU ------------------------------------------------

@pytest.fixture(scope="module")
def tfa(built):
    import tfa_ctypes
    tfa_ctypes.lib()
    return tfa_ctypes


def rope_tables(seqlen_ro, rd, kind, base=10000.0, guard=0):
    """flash-attn's cos / sin tables (seqlen_ro, rd / 2) in the 16-bit dtype, computed in float64; with `guard` > 0
    they are views of buffers followed by `guard` NaN rows."""
    inv = 1.0 / base ** (torch.arange(0, rd, 2, dtype=torch.float64) / rd)
    ang = torch.outer(torch.arange(seqlen_ro, dtype=torch.float64), inv)
    out = []
    for t in (torch.cos(ang), torch.sin(ang)):
        full = torch.full((seqlen_ro + guard, rd // 2), float("nan"), dtype=_dt(kind))
        full[:seqlen_ro] = t.to(_dt(kind))
        out.append(full.cuda()[:seqlen_ro])
    return out


def rope(x, pos, cos, sin, rd, interleaved, ftype=torch.float32):
    """x (B, S, H, D) rotated at positions pos (B, S): each pair in `ftype` as x0 c - x1 s, x0 s + x1 c, rounded once
    to x's dtype; dimensions >= rd copied."""
    c = cos[pos].to(ftype).unsqueeze(2)
    s = sin[pos].to(ftype).unsqueeze(2)
    if interleaved:
        i0, i1 = slice(0, rd, 2), slice(1, rd, 2)
    else:
        i0, i1 = slice(0, rd // 2), slice(rd // 2, rd)
    x0, x1 = x[..., i0].to(ftype), x[..., i1].to(ftype)
    y = x.clone()
    y[..., i0] = (x0 * c - x1 * s).to(x.dtype)
    y[..., i1] = (x0 * s + x1 * c).to(x.dtype)
    return y


def positions(raw_lens, cap, snew, S, causal, is_query, seqlen_ro):
    """(B, S) table rows of the rule in include/tfa_b200.h, on the GPU."""
    rows = []
    for raw in raw_lens:
        Lb = min(max(raw, 0), cap - snew)
        rows.append([min(Lb if (is_query and not causal) else Lb + i, seqlen_ro - 1) for i in range(S)])
    return torch.tensor(rows, dtype=torch.long, device="cuda")


def new_tokens(B, snew, Hkv, D, kind, seed):
    g = torch.Generator(device="cpu")
    g.manual_seed(seed)
    mk = lambda: torch.empty((B, snew, Hkv, D)).normal_(0, 0.5, generator=g).to(_dt(kind)).cuda()
    return mk(), mk()


class Case:
    """A cache (paged, or its contiguous gather), new tokens and rotary tables for one parameter set."""

    def __init__(self, D, kind, rd, Sq, snew, paged, lens, Hq=8, Hkv=2, page=256, cap=1024, seed=30, extra_ro=64,
                 ro_guard=0, fill=0.0):
        self.D, self.kind, self.rd, self.Sq, self.snew, self.paged = D, kind, rd, Sq, snew, paged
        self.raw = lens
        self.cap, self.page = cap, page
        mbps = cap // page
        data_lens = [min(max(L, 0), cap - snew) for L in lens]
        q, kp, vp, table, _ = make_cache(data_lens, Sq, Hq, Hkv, D, kind, page, seed=seed, fill=fill, mbps=mbps)
        self.q, self.table = q, table
        if paged:
            self.k0, self.v0 = kp, vp
        else:                          # the same keys, gathered into a contiguous (B, capacity, Hkv, D) cache
            B = len(lens)
            self.k0 = kp[table.long()].reshape(B, cap, Hkv, D).contiguous()
            self.v0 = vp[table.long()].reshape(B, cap, Hkv, D).contiguous()
        self.sl = torch.tensor(lens, dtype=torch.int32, device="cuda")
        self.kn, self.vn = new_tokens(len(lens), snew, Hkv, D, kind, seed + 1)
        self.seqlen_ro = cap + extra_ro
        self.cos, self.sin = rope_tables(self.seqlen_ro, rd, kind, guard=ro_guard)

    @property
    def tab(self):
        return self.table if self.paged else None

    def pos(self, causal, is_query, S):
        return positions(self.raw, self.cap, self.snew, S, causal, is_query, self.seqlen_ro)

    def fused(self, tfa, causal, il, ns, **kw):
        kc, vc = self.k0.clone(), self.v0.clone()
        out, lse = tfa.attn_kvcache_fwd(self.q, kc, vc, self.sl, self.tab, self.kn, self.vn, is_causal=causal,
                                        num_splits=ns, rotary_cos=self.cos, rotary_sin=self.sin, rotary_interleaved=il,
                                        **kw)
        return out, lse, kc, vc

    def unfused(self, tfa, causal, il, ns, ftype=torch.float32):
        qr = rope(self.q, self.pos(causal, True, self.Sq), self.cos, self.sin, self.rd, il, ftype)
        kr = rope(self.kn, self.pos(causal, False, self.snew), self.cos, self.sin, self.rd, il, ftype)
        kc, vc = self.k0.clone(), self.v0.clone()
        out, lse = tfa.attn_kvcache_fwd(qr, kc, vc, self.sl, self.tab, kr, self.vn, is_causal=causal, num_splits=ns)
        return out, lse, kc, vc, qr, kr


BITWISE = [
    # D, kind, rotary_dim, interleaved, causal, Sq, Snew, paged, num_splits
    (128, "bf16", 128, False, True, 1, 1, True, 1),
    (128, "fp16", 64, True, False, 4, 4, True, 3),
    (64, "bf16", 16, False, False, 1, 1, False, 1),
    (64, "fp16", 32, True, True, 4, 4, False, 4),
    (128, "bf16", 16, True, True, 4, 4, True, 1),
    (64, "bf16", 64, True, False, 1, 1, True, 2),
    (128, "fp16", 128, False, True, 6, 2, True, 1),        # Sq > Snew, causal
    (64, "fp16", 32, False, False, 3, 5, False, 1),        # Sq < Snew, non-causal
    (128, "bf16", 64, False, True, 4, 4, False, 3),
]
LENS = [300, 0, 129, 1000, 77, 5000, -3]                   # the last two clamp to capacity - Snew and 0


@pytest.mark.gpu
@pytest.mark.parametrize("D,kind,rd,il,causal,Sq,snew,paged,ns", BITWISE)
def test_rotary_equals_unfused_torch_rotation_bitwise(tfa, D, kind, rd, il, causal, Sq, snew, paged, ns):
    """out, lse, q_rot and the whole K/V pool after the call equal rotating q / k_new in eager torch fp32 and calling
    the unrotated forward on the same starting cache."""
    c = Case(D, kind, rd, Sq, snew, paged, LENS, page=256 if paged and D == 128 else 128, seed=40 + D + Sq)
    q_in, kn_in = c.q.clone(), c.kn.clone()
    q_rot = torch.empty_like(c.q)
    o1, l1, k1, v1 = c.fused(tfa, causal, il, ns, q_rot=q_rot)
    o2, l2, k2, v2, qr, _ = c.unfused(tfa, causal, il, ns)
    torch.cuda.synchronize()
    assert torch.equal(bits(q_rot), bits(qr))
    assert torch.equal(o1, o2) and torch.equal(l1, l2)
    assert torch.equal(bits(k1), bits(k2)) and torch.equal(bits(v1), bits(v2))
    assert torch.equal(bits(c.q), bits(q_in)) and torch.equal(bits(c.kn), bits(kn_in))
    assert torch.isfinite(o1).all()


@pytest.mark.gpu
@pytest.mark.parametrize("D,kind,rd,il,causal,Sq,snew", [(128, "bf16", 64, False, True, 4, 4),
                                                         (64, "fp16", 64, True, False, 1, 1),
                                                         (128, "fp16", 128, True, True, 6, 2)])
def test_rotary_matches_float64_oracle(tfa, D, kind, rd, il, causal, Sq, snew):
    """Rotate in float64 (rounded once to 16 bits), append, attend with the float64 oracle: the fused call agrees within
    the KV-cache tolerances (a float64 rotation may round a few elements one unit apart from the fp32 one)."""
    from test_kvcache import check_vs_oracle
    lens = [300, 0, 129, 1000]
    c = Case(D, kind, rd, Sq, snew, True, lens, page=128, seed=70)
    scale = D ** -0.5
    out, lse, kc, vc = c.fused(tfa, causal, il, 1, scale=scale)
    torch.cuda.synchronize()
    qr = rope(c.q, c.pos(causal, True, Sq), c.cos, c.sin, rd, il, torch.float64)
    kr = rope(c.kn, c.pos(causal, False, snew), c.cos, c.sin, rd, il, torch.float64)
    nblk = c.k0.shape[0]
    kw = scatter_append(c.k0, c.table, lens, kr, c.page, nblk)
    vw = scatter_append(c.v0, c.table, lens, c.vn, c.page, nblk)
    for b, raw in enumerate(lens):
        K = min(max(raw, 0), c.cap - snew) + snew
        rows = max(0, Sq - K) if causal else 0
        if rows:
            check_keyless(out, lse, b, rows)
        check_vs_oracle(out, lse, qr, kw, vw, c.table, b, K, causal, scale, kind)


@pytest.mark.gpu
@pytest.mark.parametrize("il", [False, True])
def test_rotary_append_writes_its_tokens_and_nothing_else(tfa, il):
    """NaN in every unused cache slot, a sequence whose append crosses into a page with an out-of-range table entry:
    the pool after the call is the torch scatter of rot(k_new) / v_new (V unrotated, K's dimensions >= rotary_dim
    verbatim), every other byte unchanged; out / lse / q_rot sit between NaN guard regions that stay NaN."""
    D, kind, rd, Sq, snew, G = 128, "bf16", 64, 4, 4, 64
    lens = [300, 0, 254, 1000, 77]
    c = Case(D, kind, rd, Sq, snew, True, lens, page=128, seed=90, fill=float("nan"))
    nblk = c.k0.shape[0]
    c.table[2, 2] = nblk + 5            # sequence 2 appends keys 254..257: the last two fall into logical page 2
    B, Hq = len(lens), c.q.shape[2]
    n = B * Sq * Hq * D
    obuf = torch.full((G + n + G,), float("nan"), dtype=c.q.dtype, device="cuda")
    qbuf = torch.full((G + n + G,), float("nan"), dtype=c.q.dtype, device="cuda")
    lbuf = torch.full((G + B * Hq * Sq + G,), float("nan"), dtype=torch.float32, device="cuda")
    out, q_rot = obuf[G:G + n].view(c.q.shape), qbuf[G:G + n].view(c.q.shape)
    lse = lbuf[G:G + B * Hq * Sq].view(B, Hq, Sq)
    q_in, kn_in, vn_in = c.q.clone(), c.kn.clone(), c.vn.clone()
    _, _, kc, vc = c.fused(tfa, True, il, 1, out=out, lse=lse, q_rot=q_rot)
    torch.cuda.synchronize()
    kr = rope(c.kn, c.pos(True, False, snew), c.cos, c.sin, rd, il)
    want_k = scatter_append(c.k0, c.table, lens, kr, c.page, nblk)
    want_v = scatter_append(c.v0, c.table, lens, c.vn, c.page, nblk)
    assert torch.equal(bits(kc), bits(want_k)) and torch.equal(bits(vc), bits(want_v))
    assert torch.equal(bits(kr[..., rd:]), bits(c.kn[..., rd:]))        # the tail dimensions pass through
    assert not torch.equal(bits(kr[..., :rd]), bits(c.kn[..., :rd]))
    for t, t0 in ((c.q, q_in), (c.kn, kn_in), (c.vn, vn_in)):
        assert torch.equal(bits(t), bits(t0))
    assert not torch.isnan(out).any() and not torch.isnan(lse).any() and not torch.isnan(q_rot).any()
    for buf, m in ((obuf, n), (qbuf, n), (lbuf, B * Hq * Sq)):
        assert torch.isnan(buf[:G]).all() and torch.isnan(buf[G + m:]).all()


@pytest.mark.gpu
@pytest.mark.parametrize("il", [False, True])
def test_rotary_query_positions_clamp_to_the_table(tfa, il):
    """A sequence at L_b = capacity - Snew with Sq > Snew, causal: its last query rows ask for positions past the
    table, which holds exactly `capacity` rows followed by NaN.  They are clamped to its last row: every output is
    finite and equals the unfused call with clamped positions."""
    D, kind, rd, Sq, snew = 64, "fp16", 64, 6, 2
    lens = [5000, 1024 - 2, 10, 0]                  # the first two sit at the capacity
    c = Case(D, kind, rd, Sq, snew, True, lens, page=128, seed=11, extra_ro=0, ro_guard=16)
    assert c.seqlen_ro == c.cap and int(c.pos(True, True, Sq).max()) == c.cap - 1
    q_rot = torch.empty_like(c.q)
    o1, l1, k1, v1 = c.fused(tfa, True, il, 1, q_rot=q_rot)
    o2, l2, k2, v2, qr, _ = c.unfused(tfa, True, il, 1)
    torch.cuda.synchronize()
    assert torch.isfinite(o1).all() and not torch.isnan(l1).any() and torch.isfinite(q_rot).all()
    assert torch.equal(bits(q_rot), bits(qr)) and torch.equal(o1, o2) and torch.equal(l1, l2)
    assert torch.equal(bits(k1), bits(k2))


@pytest.mark.gpu
def test_rotary_cuda_graph_replays_with_new_lengths_and_table(tfa):
    """Capture one rotary decode step (rotary append + attention + split-KV combine), rewrite cache_seqlens and the
    block table in place and replay: positions follow the new lengths, and every replay equals an eager call."""
    D, kind, rd = 128, "bf16", 128
    c = Case(D, kind, rd, 1, 1, True, [300, 5, 1000, 129], page=256, seed=13)
    B, mbps = 4, c.cap // c.page
    kp, vp = c.k0.clone(), c.v0.clone()
    out = torch.empty_like(c.q)
    lse = torch.empty((B, c.q.shape[2], 1), dtype=torch.float32, device="cuda")
    q_rot = torch.empty_like(c.q)
    step = lambda: tfa.attn_kvcache_fwd(c.q, kp, vp, c.sl, c.table, c.kn, c.vn, is_causal=True, num_splits=3, out=out,
                                        lse=lse, rotary_cos=c.cos, rotary_sin=c.sin, q_rot=q_rot)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        step()
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        step()
    results = []
    for lens, perm_seed in (([300, 5, 1000, 129], None), ([1000, 700, 0, 256], 3)):
        if perm_seed is not None:
            gp = torch.Generator(device="cpu")
            gp.manual_seed(perm_seed)
            c.sl.copy_(torch.tensor(lens, dtype=torch.int32))
            c.table.copy_(torch.randperm(kp.shape[0], generator=gp)[:B * mbps].to(torch.int32).view(B, mbps))
            c.raw = lens
        kp.copy_(c.k0)
        vp.copy_(c.v0)
        graph.replay()
        want_o, want_l, want_k, want_v = c.fused(tfa, True, False, 3)
        ref_o, _, ref_k, _, qr, _ = c.unfused(tfa, True, False, 3)
        torch.cuda.synchronize()
        assert torch.equal(out, want_o) and torch.equal(lse, want_l)
        assert torch.equal(bits(kp), bits(want_k)) and torch.equal(bits(vp), bits(want_v))
        assert torch.equal(bits(q_rot), bits(qr)) and torch.equal(out, ref_o) and torch.equal(bits(kp), bits(ref_k))
        results.append(q_rot.clone())
    assert not torch.equal(results[0], results[1])          # new lengths, new query positions


@pytest.mark.gpu
def test_rotary_launch_counts(tfa):
    c = Case(64, "fp16", 32, 1, 1, True, [500, 0, 64, 129], page=128, seed=1)
    for ns, want in ((1, 2), (3, 3)):
        n0 = tfa.launch_count()
        c.fused(tfa, True, False, ns)
        assert tfa.launch_count() - n0 == want, ns
    torch.cuda.synchronize()


@pytest.mark.gpu
def test_extension_kvcache_rotary_entry(built, tfa):
    import attention_cutlass as ac
    c = Case(128, "bf16", 64, 4, 4, True, [300, 1, 0, 640], page=256, seed=17)
    scale = 128 ** -0.5
    for il in (False, True):
        k1, v1 = c.k0.clone(), c.v0.clone()
        out, lse = ac.flash_attention_v2_kvcache_rotary(c.q, k1, v1, c.sl, c.table, c.kn, c.vn, c.cos, c.sin, il, True,
                                                        scale, 1)
        want, wl, wk, wv = c.fused(tfa, True, il, 1, scale=scale)
        torch.cuda.synchronize()
        assert out.shape == c.q.shape and lse.shape == (4, 8, 4)
        assert torch.equal(out, want) and torch.equal(lse, wl) and torch.equal(bits(k1), bits(wk))
    # contiguous cache and automatic splits
    kc = c.k0[c.table.long()].reshape(4, c.cap, 2, 128).contiguous()
    o3, l3 = ac.flash_attention_v2_kvcache_rotary(c.q, kc, kc.clone(), c.sl, None, c.kn, c.vn, c.cos, c.sin, False,
                                                  False, scale, 0)
    torch.cuda.synchronize()
    assert torch.isfinite(o3).all()
    call = lambda **kw: ac.flash_attention_v2_kvcache_rotary(
        c.q, c.k0.clone(), c.v0.clone(), c.sl, c.table, kw.get("kn", c.kn), kw.get("vn", c.vn),
        kw.get("cos", c.cos), kw.get("sin", c.sin), False, True, scale, 1)
    with pytest.raises(RuntimeError, match="k_new"):
        call(kn=None, vn=None)
    with pytest.raises(RuntimeError, match="dtype"):
        call(cos=c.cos.float(), sin=c.sin.float())
    with pytest.raises(RuntimeError, match="device"):
        call(cos=c.cos.cpu(), sin=c.sin.cpu())
    with pytest.raises(RuntimeError, match="seqlen_ro"):
        call(cos=c.cos[:c.cap - 1], sin=c.sin[:c.cap - 1])
    with pytest.raises(RuntimeError, match="rotary_dim"):
        call(cos=c.cos[:, :4].contiguous(), sin=c.sin[:, :4].contiguous())
    with pytest.raises(RuntimeError, match="contiguous"):
        call(cos=c.cos[:, ::2], sin=c.sin[:, ::2])
    with pytest.raises(RuntimeError, match="seqlen_ro, rotary_dim"):
        call(cos=c.cos, sin=c.sin[:, :16].contiguous())
