#!/usr/bin/env python
"""The FP8 variable-length forward (tfa_attn_varlen_fp8_fwd: packed e4m3 Q/K/V, e4m3 wgmma) against the ways an FP8
caller could run the same packed batch without it, and a classic / persistent A/B of the new call.

  W1   equal lengths: 4 x 4096 packed, H32 D128 causal (scripts/varlen_bench.py's W1).
  W2   mixed lengths: the 64 lengths of scripts/varlen_bench.py's W2 in [256, 8192], H32 D128 causal.
  GQA  mixed lengths: 32 lengths drawn with a fixed seed from [128, 4096], Hq32 Hkv8 D128 causal.

Arms: the FP8 varlen call; tfa_attn_varlen_fwd in bf16 on the dequantized values; tfa_attn_fp8_fwd on the batch padded
to the longest sequence; one tfa_attn_fp8_fwd call per sequence.  Before any timing the FP8 varlen outputs must equal
the per-sequence FP8 calls' bit for bit.  Method: CUDA events around each call (the per-sequence arm: around all its
calls), the arms alternated over ROUNDS rounds of REPS calls, the median per arm over all samples and per round.
Useful work is F = 4 Hq D sum_b Sq_b (Sq_b + 1) / 2 (causal, Sq_b = Sk_b), so padding counts as overhead.  The card's
name and power limit are read before and after, and the SM clock is sampled during the timed rounds; nothing is set.

Usage: python scripts/varlen_fp8_bench.py [--out PATH] [--rounds N] [--reps N]"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import threading

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tiny-flash-attention_b200"))
import tfa_ctypes as tfa  # noqa: E402

D = 128
SCALES = (0.0213, 0.0171, 0.0119)
FP8 = torch.float8_e4m3fn


def workloads():
    return {
        "W1": ([4096] * 4, 32, 32),
        "W2": ([int(x) for x in np.random.default_rng(2024).integers(256, 8193, size=64)], 32, 32),
        "GQA": ([int(x) for x in np.random.default_rng(7).integers(128, 4097, size=32)], 32, 8),
    }


def useful_flops(lens, Hq):
    return sum(4 * Hq * D * (s * (s + 1) // 2) for s in lens)


def card():
    return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                           "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()


class ClockSampler:
    """Reads the SM clock every 0.5 s while running (read only)."""
    def __init__(self):
        self.samples, self.stop = [], threading.Event()
        self.t = threading.Thread(target=self.run, daemon=True)

    def run(self):
        while not self.stop.wait(0.5):
            r = subprocess.run(["nvidia-smi", "--query-gpu=clocks.sm", "--format=csv,noheader,nounits"],
                               capture_output=True, text=True).stdout.strip()
            if r.isdigit():
                self.samples.append(int(r))

    def __enter__(self):
        self.t.start()
        return self

    def __exit__(self, *a):
        self.stop.set()
        self.t.join()


def per_seq(x, c):
    return [x[c[i]:c[i + 1]].permute(1, 0, 2).unsqueeze(0).contiguous() for i in range(len(c) - 1)]


def padded(x, lens, c):
    out = torch.zeros((len(lens), x.shape[1], max(lens), D), dtype=x.dtype, device=x.device)
    for i, s in enumerate(lens):
        out[i, :, :s] = x[c[i]:c[i + 1]].permute(1, 0, 2)
    return out


class Workload:
    def __init__(self, lens, Hq, Hkv, seed=1):
        self.lens, self.Hq = lens, Hq
        g = torch.Generator(device="cuda").manual_seed(seed)
        mk = lambda s, H: (torch.randn((sum(lens), H, D), device="cuda", generator=g) * 0.5 / s).clamp(-448, 448).to(FP8)
        self.q8, self.k8, self.v8 = mk(SCALES[0], Hq), mk(SCALES[1], Hkv), mk(SCALES[2], Hkv)
        self.q16, self.k16, self.v16 = ((x.float() * s).bfloat16() for x, s in zip((self.q8, self.k8, self.v8), SCALES))
        c = np.concatenate([[0], np.cumsum(lens)]).astype(int)
        self.c = c
        self.cu = torch.tensor(c, dtype=torch.int32, device="cuda")
        self.out = torch.empty(self.q16.shape, dtype=torch.bfloat16, device="cuda")
        self.lse = torch.empty((Hq, sum(lens)), dtype=torch.float32, device="cuda")
        self.out16, self.lse16 = torch.empty_like(self.out), torch.empty_like(self.lse)
        self.seqs = list(zip(per_seq(self.q8, c), per_seq(self.k8, c), per_seq(self.v8, c)))
        self.pad = [padded(x, lens, c) for x in (self.q8, self.k8, self.v8)]
        self.kw = dict(q_scale=SCALES[0], k_scale=SCALES[1], v_scale=SCALES[2], out_dtype=torch.bfloat16)

    def fp8_varlen(self):
        tfa.attn_varlen_fwd(self.q8, self.k8, self.v8, self.cu, self.cu, max(self.lens), True, D ** -0.5, out=self.out,
                            lse=self.lse, **self.kw)

    def bf16_varlen(self):
        tfa.attn_varlen_fwd(self.q16, self.k16, self.v16, self.cu, self.cu, max(self.lens), True, D ** -0.5,
                            out=self.out16, lse=self.lse16)

    def fp8_padded(self):
        return tfa.attn_fwd(*self.pad, True, D ** -0.5, num_splits=1, **self.kw)

    def fp8_per_sequence(self):
        return [tfa.attn_fwd(q, k, v, True, D ** -0.5, num_splits=1, **self.kw) for q, k, v in self.seqs]

    def check_bitwise(self):
        self.fp8_varlen()
        for i, (o, l) in enumerate(self.fp8_per_sequence()):
            a, b = self.c[i], self.c[i + 1]
            assert torch.equal(self.out[a:b].view(torch.int16), o[0].permute(1, 0, 2).view(torch.int16)), i
            assert torch.equal(self.lse[:, a:b].view(torch.int32), l[0].view(torch.int32)), i
        torch.cuda.synchronize()


def time_ms(fn, reps):
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    return ts


ARMS = ["fp8_varlen", "bf16_varlen", "fp8_padded", "fp8_per_sequence"]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_varlen_fp8.json"))
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--ab", action="store_true", help="(internal) the FP8 varlen call's timings as JSON on stdout")
    args = ap.parse_args()
    if args.ab:
        res = {}
        for name, (lens, Hq, Hkv) in workloads().items():
            w = Workload(lens, Hq, Hkv)
            time_ms(w.fp8_varlen, 3)
            res[name] = dict(median_ms=statistics.median(time_ms(w.fp8_varlen, args.rounds * args.reps)),
                             variant=tfa.lib().tfa_internal_last_variant())
            del w
            torch.cuda.empty_cache()
        print(json.dumps(res))
        return
    result = {"card_before": card(), "method": __doc__.split("\n\n")[2], "workloads": {}}
    with ClockSampler() as clk:
        for name, (lens, Hq, Hkv) in workloads().items():
            w = Workload(lens, Hq, Hkv)
            w.check_bitwise()
            fns = {a: getattr(w, a) for a in ARMS}
            for f in fns.values():
                time_ms(f, 2)
            t = {a: [] for a in ARMS}
            rounds = {a: [] for a in ARMS}
            for _ in range(args.rounds):
                for a in ARMS:
                    ts = time_ms(fns[a], args.reps)
                    t[a] += ts
                    rounds[a].append(statistics.median(ts))
            med = {a: statistics.median(t[a]) for a in ARMS}
            f = useful_flops(lens, Hq)
            result["workloads"][name] = dict(
                B=len(lens), Hq=Hq, Hkv=Hkv, D=D, causal=True, total_tokens=sum(lens), max_len=max(lens),
                median_ms=med, per_round_median_ms=rounds, spread_ms={a: [min(t[a]), max(t[a])] for a in ARMS},
                useful_tflops={a: f / med[a] / 1e9 for a in ARMS},
                fp8_varlen_speedup_over={a: med[a] / med["fp8_varlen"] for a in ARMS[1:]},
                per_round_speedup_range={a: [min(x / y for x, y in zip(rounds[a], rounds["fp8_varlen"])),
                                             max(x / y for x, y in zip(rounds[a], rounds["fp8_varlen"]))]
                                         for a in ARMS[1:]},
                bitwise_equal_to_per_sequence_fp8=True)
            print(name, json.dumps(result["workloads"][name]), flush=True)
            del w, fns
            torch.cuda.empty_cache()
    result["sm_clock_mhz_during_rounds"] = dict(median=statistics.median(clk.samples) if clk.samples else None,
                                                min=min(clk.samples, default=None), max=max(clk.samples, default=None),
                                                n=len(clk.samples))
    sched = {}
    for variant in ("classic", "persist", "classic", "persist"):
        env = dict(os.environ, TFA_KERNEL=variant)
        p = subprocess.run([sys.executable, os.path.abspath(__file__), "--ab", "--rounds", str(args.rounds), "--reps",
                            str(args.reps)], env=env, capture_output=True, text=True)
        sched.setdefault(variant, []).append(json.loads(p.stdout.strip().splitlines()[-1]) if p.returncode == 0
                                             else p.stderr[-2000:])
    result["fp8_varlen_schedule_ab"] = sched
    result["card_after"] = card()
    os.makedirs(os.path.dirname(args.out), exist_ok=True)
    with open(args.out, "w") as fh:
        json.dump(result, fh, indent=1)
    print(json.dumps(result, indent=1))


if __name__ == "__main__":
    main()
