"""CPU: the C-ABI library loads, exports every symbol include/tfa_b200.h declares, and rejects bad
arguments with the documented codes before touching any device (no compute calls without a GPU)."""
import ctypes
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def declared_functions():
    src = open(os.path.join(ROOT, "include", "tfa_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(tfa_[a-z0-9_]+)\s*\(", src)))


def test_header_declares_expected_entry_points():
    names = declared_functions()
    for n in ("tfa_fwd", "tfa_fwd_ex", "tfa_fwd_host", "tfa_error_string", "tfa_abi_version", "tfa_fwd_multi",
              "tfa_attn_fwd", "tfa_attn_num_splits", "tfa_attn_workspace_bytes",
              "tfa_launch_count", "tfa_debug_record", "tfa_selftest_tma", "tfa_selftest_umma"):
        assert n in names


def test_library_exports_every_declared_symbol(built):
    import tfa_ctypes
    L = ctypes.CDLL(tfa_ctypes.LIB_PATH)
    for n in declared_functions():
        assert hasattr(L, n), f"{n} declared in include/tfa_b200.h but not exported"


def test_abi_version_and_error_strings(built):
    import tfa_ctypes
    L = tfa_ctypes.lib()
    assert L.tfa_abi_version() == 2
    assert L.tfa_error_string(0) == b"success"
    for code in range(-11, 0):
        assert L.tfa_error_string(code).startswith(b"tfa:")


def test_argument_validation_without_device(built):
    import tfa_ctypes
    L = tfa_ctypes.lib()
    buf = ctypes.create_string_buffer(4096 + 16)
    base = (ctypes.addressof(buf) + 15) & ~15
    ok = ctypes.c_void_p(base)
    bad_align = ctypes.c_void_p(base + 2)
    f = lambda **kw: L.tfa_fwd(kw.get("q", ok), ok, ok, ok, None, kw.get("B", 1), kw.get("H", 1), kw.get("S", 128),
                               kw.get("D", 64), kw.get("dtype", 0), 0, 1.0, None)
    assert f(q=None) == -1            # TFA_EINVAL_PTR
    assert f(q=bad_align) == -1
    assert f(D=96) == -2              # TFA_EINVAL_DIM
    assert f(D=256) == -2
    assert f(B=0) == -3               # TFA_EINVAL_SHAPE
    assert f(S=0) == -3
    assert f(dtype=2) == -4           # TFA_EINVAL_DTYPE
    g = lambda sc: L.tfa_fwd(ok, ok, ok, ok, None, 1, 1, 128, 64, 0, 0, sc, None)
    assert g(-1.0) == -9 and g(float("nan")) == -9 and g(float("inf")) == -9    # TFA_EINVAL_SCALE
    # host path validates the same way
    assert L.tfa_fwd_host(None, ok, ok, ok, None, 1, 1, 128, 64, 0, 0, 1.0, 1) == -1
    assert L.tfa_fwd_host(ok, ok, ok, ok, None, 1, 1, 128, 80, 0, 0, 1.0, 1) == -2
    assert L.tfa_fwd_ex(None) == -1
    # generalised entry: same checks plus head grouping, before any device work
    A = tfa_ctypes.AttnArgs
    mk = lambda **kw: A(kw.get("q", base), base, base, base, None, 1, kw.get("Hq", 4), kw.get("Hkv", 2),
                        kw.get("Sq", 128), kw.get("Sk", 256), kw.get("D", 64), 4 * 128 * 64, 128 * 64, 64,
                        2 * 256 * 64, 256 * 64, kw.get("kss", 64), 0, 1, kw.get("scale", 0.1), 0,
                        kw.get("ns", 1), None, 0, None)
    call = lambda **kw: L.tfa_attn_fwd(ctypes.byref(mk(**kw)))
    assert L.tfa_attn_fwd(None) == -1
    assert call(q=None) == -1
    assert call(D=32) == -2
    assert call(Sk=0) == -3 and call(ns=-1) == -3
    assert call(Hkv=3) == -10         # TFA_EINVAL_HEADS
    assert call(kss=60) == -5         # TFA_EINVAL_STRIDE
    assert call(scale=-0.5) == -9
    # split bookkeeping is pure host arithmetic
    a = mk(Sq=1, Sk=128 * 64, ns=8)
    assert L.tfa_attn_num_splits(ctypes.byref(a)) == 8
    assert L.tfa_attn_workspace_bytes(ctypes.byref(a), 8) == 8 * 1 * 4 * 1 * 65 * 4
    assert L.tfa_attn_workspace_bytes(ctypes.byref(a), 1) == 0
    a = mk(Sq=1, Sk=300, ns=8)        # 3 KV tiles: at most 3 non-empty splits
    assert L.tfa_attn_num_splits(ctypes.byref(a)) == 3


def test_no_fallback_on_cpu_only_box(built):
    """Without a CUDA device a well-formed call must FAIL (arch/driver error), never compute on the CPU."""
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    import tfa_ctypes
    L = tfa_ctypes.lib()
    buf = ctypes.create_string_buffer(1 << 16)
    base = ctypes.c_void_p((ctypes.addressof(buf) + 15) & ~15)
    rc = L.tfa_fwd(base, base, base, base, None, 1, 1, 128, 64, 0, 0, 1.0, None)
    assert rc != 0


def test_product_path_never_imports_oracle():
    """The shipped package must not reference oracle/ in any way."""
    pkg = os.path.join(ROOT, "tiny-flash-attention_b200")
    for dirpath, _, files in os.walk(pkg):
        for fn in files:
            if fn.endswith((".py", ".cu", ".cuh", ".cpp", ".h")):
                txt = open(os.path.join(dirpath, fn), errors="ignore").read()
                assert "import oracle" not in txt and "from oracle" not in txt and "attn_oracle" not in txt, fn


def test_split_bookkeeping_invariants(built):
    """tfa_attn_num_splits: never an empty split, never more splits than asked, workspace grows linearly."""
    import tfa_ctypes
    L = tfa_ctypes.lib()
    buf = ctypes.create_string_buffer(64)
    base = (ctypes.addressof(buf) + 15) & ~15
    A = tfa_ctypes.AttnArgs
    for Sk in (1, 127, 128, 129, 1000, 4096, 65536, 100000):
        nkv = (Sk + 127) // 128
        for ns in (0, 1, 2, 3, 5, 8, 19, 64, 1000):
            a = A(base, base, base, base, None, 1, 8, 8, 128, Sk, 128, 8 * 128 * 128, 128 * 128, 128, 8 * Sk * 128,
                  Sk * 128, 128, 0, 0, 0.1, 0, ns, None, 0, None)
            n = L.tfa_attn_num_splits(ctypes.byref(a))
            assert 1 <= n <= max(1, nkv)
            if ns >= 1:
                assert n <= ns
            if n > 1:
                tiles = -(-nkv // n)
                assert (n - 1) * tiles < nkv <= n * tiles          # the last split is not empty, all keys covered
                assert L.tfa_attn_workspace_bytes(ctypes.byref(a), n) == n * 8 * 128 * 129 * 4
            else:
                assert L.tfa_attn_workspace_bytes(ctypes.byref(a), n) == 0


def test_launch_order_mapping_is_a_bijection(built):
    """decode_work (csrc/fa_fwd_sm90.cuh) -- the SAME function the kernel runs, called on the host: every CTA index maps
    to a distinct, in-range (batch*head, split, pair); inside a chunk of heads the order is heaviest pair first."""
    import tfa_ctypes
    L = tfa_ctypes.lib()
    f = L.tfa_internal_decode_work
    f.argtypes = [ctypes.c_int] * 5 + [ctypes.POINTER(ctypes.c_int * 3)]
    f.restype = ctypes.c_int
    out = (ctypes.c_int * 3)()
    for BH in (1, 2, 7, 8, 9, 15, 16, 17, 33, 128, 131):
        for npairs in (1, 2, 3, 16):
            for nsplit in (1, 2, 5):
                hc = min(8, BH)
                n = BH * npairs * nsplit
                seen = set()
                prev = None
                for blk in range(n):
                    f(blk, npairs, nsplit, hc, BH, ctypes.byref(out))
                    bh, split, pr = out[0], out[1], out[2]
                    assert 0 <= bh < BH and 0 <= split < nsplit and 0 <= pr < npairs, (BH, npairs, nsplit, blk)
                    assert (bh, split, pr) not in seen
                    seen.add((bh, split, pr))
                    chunk = bh // hc
                    if prev is not None and prev[0] == chunk:
                        # same chunk: (split, pair) index never decreases, pair goes heavy -> light inside a split
                        assert (split, -pr) >= (prev[1], -prev[2])
                    if prev is not None:
                        assert chunk >= prev[0]                      # chunks are taken in order
                    prev = (chunk, split, pr)
                assert len(seen) == n


def test_kernel_selection_rule_on_the_host(built):
    """choose_kernel (csrc/tfa_api.cu) through its host-callable twin, on an H100's 132 SMs: the shapes of the H100 A/B
    (profiles/h100_kernel_choice.txt).  0 = one CTA per work item, 4 = persistent.  (TFA_KERNEL forces one kernel and is
    read once per process.)"""
    if os.environ.get("TFA_KERNEL"):
        pytest.skip("TFA_KERNEL forces a kernel in this process")
    import tfa_ctypes
    f = tfa_ctypes.lib().tfa_internal_choose_kernel
    f.argtypes = [ctypes.c_int] * 9
    f.restype = ctypes.c_int
    CLASSIC, PERSIST = 0, 4

    def pick(B, H, S, D, causal, nsplit=1, sms=132, n_extra=0, Sk=None):
        return f(D, int(causal), S, S if Sk is None else Sk, B, H, nsplit, sms, n_extra)

    assert pick(4, 32, 4096, 128, True) == CLASSIC          # cfg3
    assert pick(64, 32, 4096, 128, True) == CLASSIC         # cfg5
    assert pick(1, 32, 16384, 128, True) == CLASSIC         # cfg4: few, very long causal items
    assert pick(2, 32, 8192, 128, True) == CLASSIC
    assert pick(16, 32, 1024, 128, True) == PERSIST         # short causal items
    assert pick(4, 32, 4096, 128, False) == PERSIST
    assert pick(2, 32, 8192, 128, False) == PERSIST
    assert pick(1, 32, 16384, 128, False) == PERSIST        # 128 KV tiles per item, 31 items per SM
    assert pick(1, 32, 16384, 128, False, nsplit=2) == PERSIST
    assert pick(4, 16, 2048, 64, False) == PERSIST          # cfg2
    assert pick(1, 32, 16384, 64, False) == PERSIST
    assert pick(4, 32, 4096, 64, True) == CLASSIC           # D=64 causal
    assert pick(32, 32, 512, 64, True) == PERSIST           # ... except short items
    assert pick(1, 32, 16384, 128, True, n_extra=1) == PERSIST   # the fused exchange keeps the persistent schedule
    # causal Sq > Sk: chosen for the Sk rows that see a key
    assert pick(4, 32, 8192, 128, True, Sk=128) == PERSIST
    assert pick(4, 32, 8192, 128, True, Sk=4096) == CLASSIC
    assert pick(4, 32, 8192, 128, False, Sk=128) == PERSIST
