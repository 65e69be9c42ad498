"""The FP8 attention call (tfa_attn_fp8_fwd: e4m3 Q/K/V, e4m3 wgmma) against tfa_attn_fwd in bf16 on the same
dequantized values, and a classic / persistent A/B of the FP8 call.

Workloads: bench.py's cfg5 (B64 H32 S4096 D128 causal), cfg3, cfg4, cfg2 (D64 non-causal), its GQA row and its
split-KV row.  Method: CUDA events around each launch, the arms alternated over ROUNDS rounds, the median per arm;
FLOPs as bench.py counts them (4 B H Sq Sk D, halved for causal Sq = Sk).  The card's name, power limit and SM clock
are read in the same run.  Writes profiles/h100_fp8_fwd.json (or --out).

Usage: python scripts/fp8_fwd_bench.py [--out PATH] [--rounds N]"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tiny-flash-attention_b200"))

# name, B, Hq, Hkv, Sq, Sk, D, causal, num_splits
WORKLOADS = [
    ("cfg5", 64, 32, 32, 4096, 4096, 128, True, 1),
    ("cfg3", 4, 32, 32, 4096, 4096, 128, True, 1),
    ("cfg4", 1, 32, 32, 16384, 16384, 128, True, 1),
    ("cfg2", 4, 16, 16, 2048, 2048, 64, False, 1),
    ("gqa", 4, 32, 8, 4096, 4096, 128, True, 1),
    ("splitkv", 1, 8, 8, 128, 65536, 128, False, 0),
]
SCALES = (0.0213, 0.0171, 0.0119)


def flops(B, Hq, Sq, Sk, D, causal):
    f = 4.0 * B * Hq * Sq * Sk * D
    return f / 2 if causal and Sq == Sk else f


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


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    return q


def arms(B, Hq, Hkv, Sq, Sk, D, causal, ns):
    import tfa_ctypes as tfa
    g = torch.Generator(device="cuda").manual_seed(1)
    mk = lambda s, *shape: (torch.randn(shape, device="cuda", generator=g) * 0.5 / s).clamp(-448, 448).to(
        torch.float8_e4m3fn)
    q8, k8, v8 = mk(SCALES[0], B, Hq, Sq, D), mk(SCALES[1], B, Hkv, Sk, D), mk(SCALES[2], B, Hkv, Sk, D)
    q16, k16, v16 = ((x.float() * s).bfloat16() for x, s in zip((q8, k8, v8), SCALES))
    scale = D ** -0.5
    out8, lse8 = torch.empty_like(q16), torch.empty((B, Hq, Sq), device="cuda")
    out16, lse16 = torch.empty_like(q16), torch.empty((B, Hq, Sq), device="cuda")
    fp8 = lambda: tfa.attn_fwd(q8, k8, v8, causal, scale, num_splits=ns, out=out8, lse=lse8, q_scale=SCALES[0],
                               k_scale=SCALES[1], v_scale=SCALES[2], out_dtype=torch.bfloat16)
    bf16 = lambda: tfa.attn_fwd(q16, k16, v16, causal, scale, num_splits=ns, out=out16, lse=lse16)
    return fp8, bf16, (out8, out16)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_fp8_fwd.json"))
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--ab", action="store_true", help="(internal) one schedule's FP8 timings as JSON on stdout")
    args = ap.parse_args()
    if args.ab:
        res = {}
        for name, B, Hq, Hkv, Sq, Sk, D, causal, ns in WORKLOADS:
            fp8, _, _ = arms(B, Hq, Hkv, Sq, Sk, D, causal, ns)
            time_ms(fp8, 3)
            res[name] = statistics.median(time_ms(fp8, args.reps * args.rounds))
        print(json.dumps(res))
        return
    result = {"card_before": card(), "method": __doc__.split("\n\n")[1], "workloads": {}}
    for name, B, Hq, Hkv, Sq, Sk, D, causal, ns in WORKLOADS:
        fp8, bf16, (o8, o16) = arms(B, Hq, Hkv, Sq, Sk, D, causal, ns)
        time_ms(fp8, 3)
        time_ms(bf16, 3)
        t8, t16 = [], []
        for _ in range(args.rounds):
            t8 += time_ms(fp8, args.reps)
            t16 += time_ms(bf16, args.reps)
        m8, m16 = statistics.median(t8), statistics.median(t16)
        f = flops(B, Hq, Sq, Sk, D, causal)
        result["workloads"][name] = dict(
            shape=dict(B=B, Hq=Hq, Hkv=Hkv, Sq=Sq, Sk=Sk, D=D, causal=causal, num_splits=ns),
            fp8_ms=m8, bf16_ms=m16, fp8_tflops=f / m8 / 1e9, bf16_tflops=f / m16 / 1e9, speedup=m16 / m8,
            fp8_ms_spread=[min(t8), max(t8)], bf16_ms_spread=[min(t16), max(t16)],
            max_abs_diff_fp8_vs_bf16=float((o8.float() - o16.float()).abs().max()))
        print(name, result["workloads"][name], flush=True)
        del fp8, bf16, o8, o16
        torch.cuda.empty_cache()
    sched = {}
    for variant in ("classic", "persist"):
        env = dict(os.environ, TFA_KERNEL=variant)
        p = subprocess.run([sys.executable, os.path.abspath(__file__), "--ab", "--rounds", str(args.rounds), "--reps",
                            str(args.reps)], env=env, capture_output=True, text=True)
        sched[variant] = json.loads(p.stdout.strip().splitlines()[-1]) if p.returncode == 0 else p.stderr[-2000:]
    result["fp8_schedule_ab_ms"] = sched
    result["card_after"] = card()
    os.makedirs(os.path.dirname(args.out), exist_ok=True)
    with open(args.out, "w") as fh:
        json.dump(result, fh, indent=1)
    print(json.dumps(result, indent=1))


if __name__ == "__main__":
    main()
