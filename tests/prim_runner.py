"""Runs ONE bring-up case of the sm_90a primitives in its own process and prints a JSON verdict.

Used by tests/test_umma_primitives.py (each case in a subprocess: a device trap poisons the CUDA context
of the process that hit it, so cases must not share one) and directly:
    python tests/prim_runner.py tma
    python tests/prim_runner.py umma '{"N":128,"K":128,"mode":2,"dtype":"bf16"}'
"""
import ctypes
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tiny-flash-attention_b200"))
import tfa_ctypes  # noqa: E402


def tma_case(D=128, S=300, BH=3, x0=64, y0=256, z0=2):
    """Expected smem image of a SWIZZLE_128B (64 x 128) box: row r at byte r*128, its eight 16-byte
    chunks permuted by chunk ^= (r % 8); rows beyond S are zero filled."""
    L = tfa_ctypes.lib()
    n = BH * S * D
    src = (torch.arange(n, dtype=torch.int32) % 30000).to(torch.int16).view(BH, S, D).cuda()   # bit patterns
    dump = torch.zeros(16384 // 2, dtype=torch.int16, device="cuda")
    tfa_ctypes.check(L.tfa_selftest_tma(src.data_ptr(), D, S, BH, x0, y0, z0, dump.data_ptr(), None))
    torch.cuda.synchronize()
    got = dump.cpu().numpy().reshape(128, 8, 8)          # row, physical chunk, 8 elements
    want = np.zeros((128, 8, 8), dtype=np.int16)
    s = src.cpu().numpy()
    for r in range(128):
        if y0 + r < S:
            row = s[z0, y0 + r, x0:x0 + 64].reshape(8, 8)
            for c in range(8):
                want[r, c ^ (r % 8)] = row[c]
    bad = int((got != want).sum())
    return {"case": "tma", "mismatches": bad, "ok": bad == 0}


def make_operands(N, K, mode, dtype, seed=0):
    g = torch.Generator().manual_seed(seed)
    dt = torch.bfloat16 if dtype == "bf16" else torch.float16
    # small integers / 4: every product and partial sum is exact in fp32 -> expect bit equality
    a = (torch.randint(-4, 5, (128, K), generator=g).float() / 4).to(dt)
    if mode == 0:
        b = (torch.randint(-4, 5, (N, K), generator=g).float() / 4).to(dt)      # (N x K)
        c = a.float() @ b.float().t()
    else:
        b = (torch.randint(-4, 5, (K, N), generator=g).float() / 4).to(dt)      # (K x N)
        c = a.float() @ b.float()
    return a, b, c


def umma_case(N=128, K=128, mode=0, dtype="bf16", knobs=None, seed=0):
    L = tfa_ctypes.lib()
    a, b, want = make_operands(N, K, mode, dtype, seed)
    a, b = a.cuda(), b.cuda()
    c = torch.full((128, N), float("nan"), dtype=torch.float32, device="cuda")
    kn = (ctypes.c_int * 4)(*(knobs or [0, 0, 0, 0]))
    tfa_ctypes.check(L.tfa_selftest_umma(a.data_ptr(), b.data_ptr(), c.data_ptr(), N, K, mode,
                                         0 if dtype == "bf16" else 1, ctypes.byref(kn), None))
    torch.cuda.synchronize()
    got = c.cpu()
    err = (got - want).abs()
    nan = int(torch.isnan(got).sum())
    maxerr = float(torch.nan_to_num(err, nan=1e9).max())
    return {"case": "umma", "N": N, "K": K, "mode": mode, "dtype": dtype, "knobs": list(knobs or []),
            "max_abs_err": maxerr, "nan": nan, "ok": maxerr == 0.0 and nan == 0}


if __name__ == "__main__":
    kind = sys.argv[1]
    kw = json.loads(sys.argv[2]) if len(sys.argv) > 2 else {}
    try:
        res = {"tma": tma_case, "umma": umma_case}[kind](**kw)
    except Exception as e:  # noqa: BLE001
        res = {"case": kind, "ok": False, "error": repr(e), "debug": tfa_ctypes.debug_record()}
    print("PRIM_RESULT " + json.dumps(res))
