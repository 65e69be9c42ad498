"""GPU: bring-up tests of the Hopper primitives the forward kernel is made of (TMA SWIZZLE_128B
loads, SS-form wgmma with K-major and MN-major B, RS-form wgmma with A in registers).
Each case runs in its own process (tests/prim_runner.py)."""
import json
import os
import subprocess
import sys

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
pytestmark = pytest.mark.gpu


def run_case(kind, **kw):
    p = subprocess.run([sys.executable, os.path.join(HERE, "prim_runner.py"), kind, json.dumps(kw)],
                       capture_output=True, text=True, timeout=600)
    for line in p.stdout.splitlines():
        if line.startswith("PRIM_RESULT "):
            return json.loads(line[len("PRIM_RESULT "):])
    raise AssertionError(f"no result from prim_runner: rc={p.returncode}\n{p.stdout[-2000:]}\n{p.stderr[-2000:]}")


def test_tma_swizzle128_box_and_oob_fill(built):
    r = run_case("tma")
    assert r["ok"], r


@pytest.mark.parametrize("dtype", ["bf16", "fp16"])
@pytest.mark.parametrize("N,K", [(128, 64), (128, 128), (64, 128)])
def test_umma_ss_kmajor(built, N, K, dtype):
    """S = Q K^T shape: both operands K-major, 128-byte swizzle, K/16 chained MMAs."""
    r = run_case("umma", N=N, K=K, mode=0, dtype=dtype)
    assert r["ok"], r


@pytest.mark.parametrize("N,K", [(128, 128), (64, 128), (128, 64)])
def test_umma_ss_mnmajor_b(built, N, K):
    """B = V tile consumed in place as an MN-major operand (no transpose)."""
    r = run_case("umma", N=N, K=K, mode=1, dtype="bf16")
    assert r["ok"], r


@pytest.mark.parametrize("dtype", ["bf16", "fp16"])
@pytest.mark.parametrize("N,K", [(128, 128), (64, 128)])
def test_umma_ts_a_in_tmem(built, N, K, dtype):
    """O += P V shape (the name is from the Blackwell build, where A sat in tensor memory): RS-form wgmma, A (=P)
    packed two 16-bit values per register, B (=V) MN-major."""
    r = run_case("umma", N=N, K=K, mode=2, dtype=dtype)
    assert r["ok"], r
