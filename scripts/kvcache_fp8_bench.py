#!/usr/bin/env python
"""Attention against an FP8 (e4m3) KV cache (tfa_attn_kvcache_fp8_fwd) on one GPU, against the 16-bit cache call.

Workloads K1-K4 of scripts/kvcache_bench.py (bf16 q, Hq 32 / Hkv 8, D 128, page 256), each with an append of one key
per sequence (Sq keys for K4), and M1 of scripts/varlen_kvcache_bench.py (4 prefill chunks of 512 + 60 decodes,
causal, appending its step's keys) through the variable-length calls.  Arms:

  fp8          the FP8 call: quantizing append + attention reading the e4m3 pool (+ the split-KV combine)
  bf16         the 16-bit call on a bf16 pool of the same lengths
  dequant_bf16 what a caller with an FP8 cache does without the FP8 call: dequantize the pool in torch, then the
               16-bit call

Ring depths: the fp8 arm of K1 and K3 under the shipped library (16-bit ring 4 + raw ring 2 at D 128) and under the
variant libraries libtfa_b200_fp8r3w4.so (3 + 4) and libtfa_b200_fp8r2w6.so (2 + 6), built beforehand with
`python tiny-flash-attention_b200/build.py --variant fp8r3w4 -DTFA_FP8_RING128=3 -DTFA_FP8_RAW128=4` (and 2 / 6), each
in its own subprocess (TFA_LIB), alternated.

Before timing, the FP8 call's out / lse must equal the 16-bit call on the widened pool (softmax scale s' =
scale * k_scale, v_scale = 1) bit for bit.  One call per sample after a 256 MB write that flushes the L2, CUDA events,
arms alternated; ROUNDS rounds of REPS samples, the medians of each round recorded with the overall median.  A schedule
A/B (TFA_KERNEL=classic|persist, read once per process) of the fp8 arm runs in alternating subprocesses.  The card's
name, power limit and the median SM clock sampled during the timed sections are recorded with the numbers.

Run from the repository root after build():   python scripts/kvcache_fp8_bench.py OUT.json
"""
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tiny-flash-attention_b200"))
sys.path.insert(0, os.path.join(ROOT, "scripts"))
import tfa_ctypes as tfa  # noqa: E402
from kvcache_bench import HQ, HKV, D, PAGE, SCALE, workloads  # noqa: E402
from varlen_kvcache_bench import workloads as varlen_workloads  # noqa: E402
from varlen_bench import ClockSampler, gpu_identity  # noqa: E402

ROUNDS, REPS = 5, 10
K_SCALE, V_SCALE = 0.02, 1.0


class Workload:
    def __init__(self, lens, Sq, causal, seed):
        self.lens, self.Sq, self.causal = lens, Sq, causal
        B = len(lens)
        g = torch.Generator(device="cuda").manual_seed(seed)
        mbps = -(-(max(lens) + Sq) // PAGE)
        nblk = B * mbps + 8
        self.q = torch.empty((B, Sq, HQ, D), dtype=torch.bfloat16, device="cuda").normal_(0, 0.5, generator=g)
        self.kn = torch.empty((B, Sq, HKV, D), dtype=torch.bfloat16, device="cuda").normal_(0, 0.5, generator=g)
        self.vn = torch.empty_like(self.kn).normal_(0, 0.5, generator=g)
        # e4m3 codes of N(0, 0.5^2) / k_scale: the pool a quantizing serving engine would hold
        mk = lambda: (torch.empty((nblk, PAGE, HKV, D), device="cuda").normal_(0, 0.5, generator=g) / K_SCALE).clamp(
            -448, 448).to(torch.float8_e4m3fn)
        self.k8, self.v8 = mk(), mk()
        self.k16, self.v16 = self.k8.to(torch.bfloat16), self.v8.to(torch.bfloat16)
        perm = torch.randperm(nblk, generator=torch.Generator().manual_seed(seed))[:B * mbps]
        self.table = perm.to(torch.int32).view(B, mbps).cuda()
        self.sl = torch.tensor(lens, dtype=torch.int32, device="cuda")
        self.out = torch.empty_like(self.q)
        self.lse = torch.empty((B, HQ, Sq), dtype=torch.float32, device="cuda")

    def fp8(self):
        return tfa.attn_kvcache_fwd(self.q, self.k8, self.v8, self.sl, self.table, self.kn, self.vn,
                                    is_causal=self.causal, scale=SCALE, num_splits=0, out=self.out, lse=self.lse,
                                    k_scale=K_SCALE, v_scale=V_SCALE)

    def bf16(self):
        return tfa.attn_kvcache_fwd(self.q, self.k16, self.v16, self.sl, self.table, self.kn, self.vn,
                                    is_causal=self.causal, scale=SCALE, num_splits=0, out=self.out, lse=self.lse)

    def dequant_bf16(self):
        kd = (self.k8.to(torch.bfloat16) * K_SCALE)
        vd = (self.v8.to(torch.bfloat16) * V_SCALE)
        return tfa.attn_kvcache_fwd(self.q, kd, vd, self.sl, self.table, self.kn, self.vn, is_causal=self.causal,
                                    scale=SCALE, num_splits=0, out=self.out, lse=self.lse)

    def check(self):
        """The FP8 call (no append) against the 16-bit call on the widened pool with s', bit for bit."""
        s_eff = float(torch.tensor(SCALE, dtype=torch.float32) * torch.tensor(K_SCALE, dtype=torch.float32))
        o1, l1 = tfa.attn_kvcache_fwd(self.q, self.k8, self.v8, self.sl, self.table, is_causal=self.causal,
                                      scale=SCALE, num_splits=0, k_scale=K_SCALE, v_scale=V_SCALE)
        o2, l2 = tfa.attn_kvcache_fwd(self.q, self.k16, self.v16, self.sl, self.table, is_causal=self.causal,
                                      scale=s_eff, num_splits=0)
        torch.cuda.synchronize()
        return bool(torch.equal(o1, o2) and torch.equal(l1, l2))


class VarlenWorkload:
    """M1 through tfa_attn_varlen_kvcache(_fp8)_fwd: packed q / k_new / v_new, causal, with the append."""

    def __init__(self, sq, lens, seed):
        self.sq, self.lens = sq, lens
        B, tq = len(sq), sum(sq)
        g = torch.Generator(device="cuda").manual_seed(seed)
        mk = lambda *s: torch.empty(s, dtype=torch.bfloat16, device="cuda").normal_(0, 0.5, generator=g)
        self.q, self.kn, self.vn = mk(tq, HQ, D), mk(tq, HKV, D), mk(tq, HKV, D)
        mbps = -(-(max(lens) + max(sq)) // PAGE)
        nblk = B * mbps + 8
        e4 = lambda: (torch.empty((nblk, PAGE, HKV, D), device="cuda").normal_(0, 0.5, generator=g) / K_SCALE).clamp(
            -448, 448).to(torch.float8_e4m3fn)
        self.k8, self.v8 = e4(), e4()
        self.k16, self.v16 = self.k8.to(torch.bfloat16), self.v8.to(torch.bfloat16)
        perm = torch.randperm(nblk, generator=torch.Generator().manual_seed(seed))[:B * mbps]
        self.table = perm.to(torch.int32).view(B, mbps).cuda()
        self.sl = torch.tensor(lens, dtype=torch.int32, device="cuda")
        self.cu = torch.tensor([0] + list(torch.tensor(sq).cumsum(0)), dtype=torch.int32, device="cuda")
        self.out = torch.empty_like(self.q)
        self.lse = torch.empty((HQ, tq), dtype=torch.float32, device="cuda")

    def _call(self, kp, vp, kn=True, **kw):
        return tfa.attn_varlen_kvcache_fwd(self.q, kp, vp, self.cu, max(self.sq), self.sl, self.table,
                                           self.kn if kn else None, self.vn if kn else None, is_causal=True,
                                           scale=kw.pop("scale", SCALE), out=self.out, lse=self.lse, **kw)

    def fp8(self):
        return self._call(self.k8, self.v8, k_scale=K_SCALE, v_scale=V_SCALE)

    def bf16(self):
        return self._call(self.k16, self.v16)

    def dequant_bf16(self):
        return self._call((self.k8.to(torch.bfloat16) * K_SCALE), (self.v8.to(torch.bfloat16) * V_SCALE))

    def check(self):
        s_eff = float(torch.tensor(SCALE, dtype=torch.float32) * torch.tensor(K_SCALE, dtype=torch.float32))
        o1, l1 = (t.clone() for t in self._call(self.k8, self.v8, kn=False, k_scale=K_SCALE, v_scale=V_SCALE))
        o2, l2 = self._call(self.k16, self.v16, kn=False, scale=s_eff)
        torch.cuda.synchronize()
        return bool(torch.equal(o1, o2) and torch.equal(l1, l2))


_FLUSH = None


def time_arms(arms, rounds=ROUNDS, reps=REPS):
    """arms: name -> fn.  One call per sample after an L2 flush, arms alternated.  Returns name -> [[ms] per round]."""
    global _FLUSH
    if _FLUSH is None:
        _FLUSH = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    for fn in arms.values():
        for _ in range(3):
            fn()
    torch.cuda.synchronize()
    res = {name: [[] for _ in range(rounds)] for name in arms}
    for r in range(rounds):
        for _ in range(reps):
            for name, fn in arms.items():
                _FLUSH.fill_(1)
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                fn()
                e1.record()
                torch.cuda.synchronize()
                res[name][r].append(e0.elapsed_time(e1))
    return res


def summary(rounds):
    flat = [x for r in rounds for x in r]
    return {"us_median": round(statistics.median(flat) * 1e3, 2),
            "us_round_medians": [round(statistics.median(r) * 1e3, 2) for r in rounds],
            "us_min": round(min(flat) * 1e3, 2), "us_max": round(max(flat) * 1e3, 2)}


def child(names):
    """One subprocess of the schedule or ring-depth A/B: the fp8 arm of `names` under this process's TFA_KERNEL /
    TFA_LIB."""
    res = {}
    for i, (name, w) in enumerate(workloads().items()):
        if name not in names:
            continue
        wl = Workload(w["lens"], w["Sq"], w["causal"], seed=10 + i)
        res[name] = [x for r in time_arms({"fp8": wl.fp8}, rounds=1, reps=20)["fp8"] for x in r]
        del wl
        torch.cuda.empty_cache()
    print("RES " + json.dumps({"res": res, "variant": tfa.lib().tfa_internal_last_variant()}))


def run_children(envs, names, passes=2):
    """envs: label -> extra environment.  Alternates one child per label, `passes` times; returns label -> workload ->
    summary over the passes (each pass is one round)."""
    out = {label: {} for label in envs}
    for _ in range(passes):
        for label, extra in envs.items():
            p = subprocess.run([sys.executable, os.path.abspath(__file__), "--child", ",".join(names)],
                               env=dict(os.environ, **extra), capture_output=True, text=True)
            if p.returncode != 0:
                raise SystemExit(p.stderr[-3000:])
            r = json.loads([l for l in p.stdout.splitlines() if l.startswith("RES ")][0][4:])
            if "TFA_KERNEL" in extra:
                assert r["variant"] == (0 if extra["TFA_KERNEL"] == "classic" else 4), r
            for w, ms in r["res"].items():
                out[label].setdefault(w, []).append(ms)
    return {label: {w: summary(ms) for w, ms in d.items()} for label, d in out.items()}


def main(out_path):
    assert torch.cuda.is_available(), "kvcache_fp8_bench needs a GPU"
    tfa.lib()
    gpu_id, name, power = gpu_identity()
    report = {"gpu": name, "power_limit_w": power, "dtype": "bf16 q, e4m3 cache", "Hq": HQ, "Hkv": HKV, "D": D,
              "page": PAGE, "k_scale": K_SCALE, "v_scale": V_SCALE,
              "timing": f"one call per sample after a 256 MB L2 flush, CUDA events, {ROUNDS} rounds x {REPS}, arms "
                        "alternated"}
    samples = []
    for i, (wname, w) in enumerate(workloads().items()):
        wl = Workload(w["lens"], w["Sq"], w["causal"], seed=10 + i)
        ok = wl.check()
        if not ok:
            raise SystemExit(f"{wname}: the FP8 call differs from the 16-bit call on the widened cache")
        with ClockSampler(gpu_id) as clk:
            r = time_arms({"fp8": wl.fp8, "bf16": wl.bf16, "dequant_bf16": wl.dequant_bf16})
        samples += clk.samples
        entry = {"B": len(wl.lens), "Sq": wl.Sq, "causal": wl.causal, "keys_total": sum(wl.lens),
                 "append_per_seq": wl.Sq, "fp8_bitwise_equal_widened_bf16": ok,
                 **{k: summary(v) for k, v in r.items()}}
        entry["bf16_over_fp8"] = round(entry["bf16"]["us_median"] / entry["fp8"]["us_median"], 3)
        entry["dequant_over_fp8"] = round(entry["dequant_bf16"]["us_median"] / entry["fp8"]["us_median"], 3)
        entry["bf16_over_fp8_per_round"] = [round(b / f, 3) for b, f in zip(entry["bf16"]["us_round_medians"],
                                                                            entry["fp8"]["us_round_medians"])]
        report[wname] = entry
        print(wname, json.dumps(entry), flush=True)
        del wl
        torch.cuda.empty_cache()
    sq, lens = varlen_workloads()["M1"]
    wl = VarlenWorkload(sq, lens, seed=30)
    if not wl.check():
        raise SystemExit("M1: the FP8 varlen call differs from the 16-bit call on the widened cache")
    with ClockSampler(gpu_id) as clk:
        r = time_arms({"fp8": wl.fp8, "bf16": wl.bf16, "dequant_bf16": wl.dequant_bf16})
    samples += clk.samples
    entry = {"B": len(sq), "rows": sum(sq), "causal": True, "keys_total": sum(lens), "append": "each sequence's rows",
             "fp8_bitwise_equal_widened_bf16": True, **{k: summary(v) for k, v in r.items()}}
    entry["bf16_over_fp8"] = round(entry["bf16"]["us_median"] / entry["fp8"]["us_median"], 3)
    entry["dequant_over_fp8"] = round(entry["dequant_bf16"]["us_median"] / entry["fp8"]["us_median"], 3)
    entry["bf16_over_fp8_per_round"] = [round(b / f, 3) for b, f in zip(entry["bf16"]["us_round_medians"],
                                                                        entry["fp8"]["us_round_medians"])]
    report["M1_varlen"] = entry
    print("M1", json.dumps(entry), flush=True)
    del wl
    torch.cuda.empty_cache()
    report["sm_clock_mhz_median"] = statistics.median(samples) if samples else None
    report["sm_clock_samples"] = len(samples)

    report["schedules_fp8"] = run_children({"classic": {"TFA_KERNEL": "classic"}, "persist": {"TFA_KERNEL": "persist"}},
                                           list(workloads()))
    here = os.path.join(ROOT, "tiny-flash-attention_b200")
    depths = {"ring4_raw2": {}}
    for label, name in (("ring3_raw4", "fp8r3w4"), ("ring2_raw6", "fp8r2w6")):
        path = os.path.join(here, f"libtfa_b200_{name}.so")
        if os.path.exists(path):
            depths[label] = {"TFA_LIB": path}
    if len(depths) > 1:
        report["ring_depths_d128_fp8"] = run_children(depths, ["K1", "K3"], passes=3)
    os.makedirs(os.path.dirname(os.path.abspath(out_path)), exist_ok=True)
    with open(out_path, "w") as f:
        json.dump(report, f, indent=1)
    print(json.dumps(report))


if __name__ == "__main__":
    if "--child" in sys.argv:
        child(sys.argv[sys.argv.index("--child") + 1].split(","))
    else:
        main(sys.argv[1] if len(sys.argv) > 1 else "kvcache_fp8_bench.json")
