"""The dense causal bf16 D=128 forward (the benchmark's kernel, both schedules) runs its softmax's exponentials while
its PV wgmma is in flight, in the compiled code.

In the KV loop a softmax warpgroup issues S_j = Q K_j^T and PV_{j-1} = P_{j-1} V_{j-1}, waits for S_j alone
(WARPGROUP.DEPBAR.LE gsb0, 0x1), runs the softmax of tile j and only then waits for PV_{j-1}
(WARPGROUP.DEPBAR.LE gsb0, 0x0).  ptxas is free to move that second wait up, and does so whenever the softmax writes a
register it ties to the in-flight wgmma; it serializes every wgmma (one DEPBAR after each HGMMA) whenever a non-wgmma
instruction defines a wgmma's input registers inside the pipeline or in a branch it takes for divergent.  Neither
shows in the results, only in the time, so this reads the SASS of the built library: CPU only, no GPU needed.
"""
import os
import re
import subprocess

import build as tfa_build  # tiny-flash-attention_b200/build.py

D = 128
KSTEPS = 8                 # HGMMAs per chain: S = D/16 k-steps of Q K^T, PV = 128 keys / 16
EXP_PER_TILE = 64          # exponentials per thread per 128-key tile (2 rows x 32 keys)
KERNELS = {
    # fa_fwd_sm90_kernel<D=128, CAUSAL, IS_BF16, OUT_F32=false, PERSIST, kDense>
    "classic": f"_ZN3tfa18fa_fwd_sm90_kernelILi{D}ELb1ELb1ELb0ELb0ELi0EEEv14CUtensorMap_stS1_S1_NS_9FwdParamsE",
    "persistent": f"_ZN3tfa18fa_fwd_sm90_kernelILi{D}ELb1ELb1ELb0ELb1ELi0EEEv14CUtensorMap_stS1_S1_NS_9FwdParamsE",
}
_INSN = re.compile(r"/\*([0-9a-f]{4,})\*/\s+(.*?)\s*;")


def _sass(lib, fun):
    cuobjdump = os.path.join(os.path.dirname(tfa_build.NVCC), "cuobjdump")
    assert os.path.exists(cuobjdump), (
        f"cuobjdump not found next to nvcc ({tfa_build.NVCC}): the SASS order check needs the CUDA toolkit's cuobjdump")
    out = subprocess.run([cuobjdump, "-sass", "-fun", fun, lib], stdout=subprocess.PIPE, stderr=subprocess.DEVNULL,
                         text=True, check=True).stdout
    insns = [m.group(2) for m in map(_INSN.search, out.splitlines()) if m]
    assert insns, f"{fun} not found in {lib}"
    return insns


def _chains(insns):
    """(first index, last index, is_pv) of every HGMMA chain: HGMMAs up to the one that carries gsb0."""
    chains, start, pv = [], None, False
    for i, s in enumerate(insns):
        if not s.startswith("HGMMA") and " HGMMA" not in s:
            continue
        if start is None:
            start, pv = i, "tnspB" in s      # PV reads V from shared memory as an MN-major (transposed) operand
        if "gsb0" in s:
            chains.append((start, i, pv))
            start = None
    return chains


def _hgmma_count(insns, a, b):
    return sum(1 for s in insns[a:b + 1] if "HGMMA" in s)


def _check(name, insns):
    chains = _chains(insns)
    assert chains, f"{name}: no HGMMA in the kernel"
    broken = [(a, b) for a, b, _ in chains if _hgmma_count(insns, a, b) != KSTEPS]
    assert not broken, (
        f"{name}: {len(broken)} of {len(chains)} wgmma chains are not {KSTEPS} HGMMAs under one commit: ptxas "
        f"serialized them (a WARPGROUP.DEPBAR after each HGMMA; look for C7513 / C7520 in the -Xptxas -v log)")
    steps = 0
    for a, b, pv in chains:
        if not pv:
            continue
        # the first wait after PV_{j-1}: 0x1 (S_j only) in a loop step, 0x0 after the last tile's PV
        waits = [i for i in range(b + 1, len(insns)) if insns[i].startswith("WARPGROUP.DEPBAR")]
        if not waits or not insns[waits[0]].endswith("0x1"):
            continue
        w1 = waits[0]
        w0 = next((i for i in waits if insns[i].endswith("0x0")), None)
        assert w0 is not None, f"{name}: no wait for PV after the chain at instruction {b}"
        exps = sum(1 for s in insns[w1:w0] if s.startswith("MUFU.EX2"))   # unpredicated: the softmax, not alpha
        assert exps >= EXP_PER_TILE, (
            f"{name}: only {exps} MUFU.EX2 between the S_j wait (DEPBAR.LE gsb0, 0x1) and the PV_(j-1) wait "
            f"(DEPBAR.LE gsb0, 0x0) of a KV-loop step; the softmax's {EXP_PER_TILE} exponentials run after PV is done")
        steps += 1
    assert steps >= 1, f"{name}: found no KV-loop step (PV chain followed by DEPBAR.LE gsb0, 0x1)"


def test_softmax_exponentials_run_under_pv_wgmma(built):
    lib = os.path.join(built, tfa_build.LIB_NAME)
    for name, fun in KERNELS.items():
        _check(name, _sass(lib, fun))
