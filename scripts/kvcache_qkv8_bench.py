#!/usr/bin/env python
"""e4m3 queries against an FP8 (e4m3) KV cache (tfa_attn_kvcache_qkv8_fwd / tfa_attn_varlen_kvcache_qkv8_fwd) on one
GPU, against the widening FP8-cache call and the 16-bit cache call.

Workloads K1-K4 of scripts/kvcache_bench.py (Hq 32 / Hkv 8, D 128, page 256), each with an append of one key per sequence
(Sq keys for K4), and M1 of scripts/varlen_kvcache_bench.py (4 prefill chunks of 512 + 60 decodes, causal, appending
its step's keys) through the variable-length calls, exactly as scripts/kvcache_fp8_bench.py runs them.  Arms:

  qkv8        the new call: e4m3 q, quantizing append of bf16 k_new / v_new, attention on e4m3 wgmma (+ the split-KV
              combine), bf16 output
  fp8         tfa_attn_kvcache_fp8_fwd (tfa_attn_varlen_kvcache_fp8_fwd for M1) with bf16 q on the same e4m3 pool: the
              call that widens every cache tile to 16 bits
  bf16        the 16-bit cache call on a bf16 pool of the same lengths
  quantize_q  torch's (q / q_scale).clamp(-448, 448).to(float8_e4m3fn) of the step's bf16 q, timed alone: what a caller
              of the new call pays to make its input

Before timing, every sequence of every workload is checked: the new call's out and lse (after its append, on a copy of
the pool) must equal tfa_attn_fp8_fwd (num_splits = 1) on that sequence alone, with its first K_b keys gathered, bit for
bit.  The timed calls use num_splits = 0 (the library's choice) as the other cache benchmarks do.  One call per sample
after a 256 MB write that flushes the L2, CUDA events, arms alternated; ROUNDS rounds of REPS samples, the medians of each
round recorded with the overall median.  A schedule A/B (TFA_KERNEL=classic|persist, read once per process) of the qkv8
arm runs in alternating subprocesses.  The card's name, power limit and the median SM clock sampled during the timed
sections are recorded with the numbers.

Run from the repository root after build():   python scripts/kvcache_qkv8_bench.py OUT.json
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
from kvcache_fp8_bench import summary, time_arms  # noqa: E402
from varlen_kvcache_bench import workloads as varlen_workloads  # noqa: E402
from varlen_bench import ClockSampler, gpu_identity  # noqa: E402

ROUNDS, REPS = 5, 10
Q_SCALE, K_SCALE, V_SCALE = 0.01, 0.02, 0.02
FP8 = torch.float8_e4m3fn


def quantize(x, s):
    return (x.float() / s).clamp(-448, 448).to(FP8)


def gather(pool, table, b, K):
    idx = torch.arange(K, device=pool.device)
    rows = pool[table[b].long()[idx // PAGE], idx % PAGE]
    return rows.permute(1, 0, 2)[None].contiguous()


def same_as_fp8_forward(out, lse, q8, k8, v8, table, b, K, causal):
    """Sequence b's rows of the new call (out (Sq, Hq, D), lse (Hq, Sq)) against tfa_attn_fp8_fwd on it alone."""
    if K == 0:
        return bool((out == 0).all() and torch.isposinf(lse).all())
    o, l = tfa.attn_fwd(q8.permute(1, 0, 2)[None].contiguous(), gather(k8, table, b, K), gather(v8, table, b, K),
                        causal, SCALE, num_splits=1, q_scale=Q_SCALE, k_scale=K_SCALE, v_scale=V_SCALE,
                        out_dtype=torch.bfloat16)
    return bool(torch.equal(out.contiguous().view(torch.int16), o[0].permute(1, 0, 2).contiguous().view(torch.int16))
                and torch.equal(lse.contiguous().view(torch.int32), l[0].view(torch.int32)))


class Workload:
    def __init__(self, lens, Sq, causal, seed):
        self.lens, self.Sq, self.causal = lens, Sq, causal
        B = len(lens)
        g = torch.Generator(device="cuda").manual_seed(seed)
        mbps = -(-(max(lens) + Sq) // PAGE)
        nblk = B * mbps + 8
        self.cap = mbps * PAGE
        self.q = torch.empty((B, Sq, HQ, D), dtype=torch.bfloat16, device="cuda").normal_(0, 0.5, generator=g)
        self.q8 = quantize(self.q, Q_SCALE)
        self.kn = torch.empty((B, Sq, HKV, D), dtype=torch.bfloat16, device="cuda").normal_(0, 0.5, generator=g)
        self.vn = torch.empty_like(self.kn).normal_(0, 0.5, generator=g)
        mk = lambda s: quantize(torch.empty((nblk, PAGE, HKV, D), device="cuda").normal_(0, 0.5, generator=g), s)
        self.k8, self.v8 = mk(K_SCALE), mk(V_SCALE)
        self.k16, self.v16 = self.k8.to(torch.bfloat16), self.v8.to(torch.bfloat16)
        perm = torch.randperm(nblk, generator=torch.Generator().manual_seed(seed))[:B * mbps]
        self.table = perm.to(torch.int32).view(B, mbps).cuda()
        self.sl = torch.tensor(lens, dtype=torch.int32, device="cuda")
        self.out = torch.empty_like(self.q)
        self.lse = torch.empty((B, HQ, Sq), dtype=torch.float32, device="cuda")

    def qkv8(self, k8=None, v8=None, **kw):
        return tfa.attn_kvcache_fwd(self.q8, self.k8 if k8 is None else k8, self.v8 if v8 is None else v8, self.sl,
                                    self.table, self.kn, self.vn, is_causal=self.causal, scale=SCALE,
                                    num_splits=kw.pop("num_splits", 0), out=kw.pop("out", self.out),
                                    lse=kw.pop("lse", self.lse), q_scale=Q_SCALE, k_scale=K_SCALE, v_scale=V_SCALE,
                                    out_dtype=torch.bfloat16)

    def fp8(self):
        return tfa.attn_kvcache_fwd(self.q, self.k8, self.v8, self.sl, self.table, self.kn, self.vn,
                                    is_causal=self.causal, scale=SCALE, num_splits=0, out=self.out, lse=self.lse,
                                    k_scale=K_SCALE, v_scale=V_SCALE)

    def bf16(self):
        return tfa.attn_kvcache_fwd(self.q, self.k16, self.v16, self.sl, self.table, self.kn, self.vn,
                                    is_causal=self.causal, scale=SCALE, num_splits=0, out=self.out, lse=self.lse)

    def quantize_q(self):
        return quantize(self.q, Q_SCALE)

    def check(self):
        """The new call with its append on a copy of the pool, every sequence against tfa_attn_fp8_fwd."""
        k8, v8 = self.k8.clone(), self.v8.clone()
        out, lse = self.qkv8(k8, v8, num_splits=1, out=None, lse=None)
        for b, raw in enumerate(self.lens):
            K = min(max(raw, 0), self.cap - self.Sq) + self.Sq
            if not same_as_fp8_forward(out[b], lse[b], self.q8[b], k8, v8, self.table, b, K, self.causal):
                return False
        torch.cuda.synchronize()
        return True


class VarlenWorkload:
    """M1 through tfa_attn_varlen_kvcache_(qkv8|fp8)_fwd: packed q / k_new / v_new, causal, with the append."""

    def __init__(self, sq, lens, seed):
        self.sq, self.lens = sq, lens
        B, tq = len(sq), sum(sq)
        g = torch.Generator(device="cuda").manual_seed(seed)
        mk = lambda *s: torch.empty(s, dtype=torch.bfloat16, device="cuda").normal_(0, 0.5, generator=g)
        self.q, self.kn, self.vn = mk(tq, HQ, D), mk(tq, HKV, D), mk(tq, HKV, D)
        self.q8 = quantize(self.q, Q_SCALE)
        mbps = -(-(max(lens) + max(sq)) // PAGE)
        nblk = B * mbps + 8
        self.cap = mbps * PAGE
        e4 = lambda s: quantize(torch.empty((nblk, PAGE, HKV, D), device="cuda").normal_(0, 0.5, generator=g), s)
        self.k8, self.v8 = e4(K_SCALE), e4(V_SCALE)
        self.k16, self.v16 = self.k8.to(torch.bfloat16), self.v8.to(torch.bfloat16)
        perm = torch.randperm(nblk, generator=torch.Generator().manual_seed(seed))[:B * mbps]
        self.table = perm.to(torch.int32).view(B, mbps).cuda()
        self.sl = torch.tensor(lens, dtype=torch.int32, device="cuda")
        self.starts = [0] + torch.tensor(sq).cumsum(0).tolist()
        self.cu = torch.tensor(self.starts, dtype=torch.int32, device="cuda")
        self.out = torch.empty_like(self.q)
        self.lse = torch.empty((HQ, tq), dtype=torch.float32, device="cuda")

    def _call(self, q, kp, vp, out=None, lse=None, **kw):
        return tfa.attn_varlen_kvcache_fwd(q, kp, vp, self.cu, max(self.sq), self.sl, self.table, self.kn, self.vn,
                                           is_causal=True, scale=SCALE, out=self.out if out is None else out,
                                           lse=self.lse if lse is None else lse, **kw)

    def qkv8(self, k8=None, v8=None, **kw):
        return self._call(self.q8, self.k8 if k8 is None else k8, self.v8 if v8 is None else v8, q_scale=Q_SCALE,
                          k_scale=K_SCALE, v_scale=V_SCALE, out_dtype=torch.bfloat16, **kw)

    def fp8(self):
        return self._call(self.q, self.k8, self.v8, k_scale=K_SCALE, v_scale=V_SCALE)

    def bf16(self):
        return self._call(self.q, self.k16, self.v16)

    def quantize_q(self):
        return quantize(self.q, Q_SCALE)

    def check(self):
        k8, v8 = self.k8.clone(), self.v8.clone()
        out, lse = self.qkv8(k8, v8, out=torch.empty_like(self.out), lse=torch.empty_like(self.lse))
        for b, n in enumerate(self.sq):
            r0 = self.starts[b]
            K = min(max(self.lens[b], 0), max(self.cap - n, 0)) + min(n, self.cap)
            if not same_as_fp8_forward(out[r0:r0 + n], lse[:, r0:r0 + n], self.q8[r0:r0 + n], k8, v8, self.table, b,
                                       K, True):
                return False
        torch.cuda.synchronize()
        return True


def ratios(entry):
    for arm in ("fp8", "bf16"):
        entry[f"{arm}_over_qkv8"] = round(entry[arm]["us_median"] / entry["qkv8"]["us_median"], 3)
        entry[f"{arm}_over_qkv8_per_round"] = [round(a / b, 3) for a, b in zip(entry[arm]["us_round_medians"],
                                                                               entry["qkv8"]["us_round_medians"])]
    entry["qkv8_plus_quantize_q_us"] = round(entry["qkv8"]["us_median"] + entry["quantize_q"]["us_median"], 2)
    return entry


def child(names):
    """One subprocess of the schedule A/B: the qkv8 arm of `names` under this process's TFA_KERNEL."""
    res = {}
    for i, (name, w) in enumerate(workloads().items()):
        if name not in names:
            continue
        wl = Workload(w["lens"], w["Sq"], w["causal"], seed=10 + i)
        res[name] = [x for r in time_arms({"qkv8": wl.qkv8}, rounds=1, reps=20)["qkv8"] for x in r]
        del wl
        torch.cuda.empty_cache()
    print("RES " + json.dumps({"res": res, "variant": tfa.lib().tfa_internal_last_variant()}))


def run_children(envs, names, passes=2):
    out = {label: {} for label in envs}
    for _ in range(passes):
        for label, extra in envs.items():
            p = subprocess.run([sys.executable, os.path.abspath(__file__), "--child", ",".join(names)],
                               env=dict(os.environ, **extra), capture_output=True, text=True)
            if p.returncode != 0:
                raise SystemExit(p.stderr[-3000:])
            r = json.loads([l for l in p.stdout.splitlines() if l.startswith("RES ")][0][4:])
            assert r["variant"] == (0 if extra["TFA_KERNEL"] == "classic" else 4), r
            for w, ms in r["res"].items():
                out[label].setdefault(w, []).append(ms)
    return {label: {w: summary(ms) for w, ms in d.items()} for label, d in out.items()}


def main(out_path):
    assert torch.cuda.is_available(), "kvcache_qkv8_bench needs a GPU"
    tfa.lib()
    gpu_id, name, power = gpu_identity()
    report = {"gpu": name, "power_limit_w": power, "dtype": "e4m3 q (qkv8) or bf16 q, e4m3 / bf16 cache, bf16 out",
              "Hq": HQ, "Hkv": HKV, "D": D, "page": PAGE, "q_scale": Q_SCALE, "k_scale": K_SCALE, "v_scale": V_SCALE,
              "timing": f"one call per sample after a 256 MB L2 flush, CUDA events, {ROUNDS} rounds x {REPS}, arms "
                        "alternated"}
    samples = []
    names = list(workloads()) + ["M1_varlen"]
    for i, wname in enumerate(names):
        if wname == "M1_varlen":
            sq, lens = varlen_workloads()["M1"]
            wl = VarlenWorkload(sq, lens, seed=30)
            shape = {"B": len(sq), "rows": sum(sq), "causal": True, "keys_total": sum(lens),
                     "append": "each sequence's rows"}
        else:
            w = workloads()[wname]
            wl = Workload(w["lens"], w["Sq"], w["causal"], seed=10 + i)
            shape = {"B": len(wl.lens), "Sq": wl.Sq, "causal": wl.causal, "keys_total": sum(wl.lens),
                     "append_per_seq": wl.Sq}
        if not wl.check():
            raise SystemExit(f"{wname}: the qkv8 call differs from tfa_attn_fp8_fwd on a sequence")
        with ClockSampler(gpu_id) as clk:
            r = time_arms({"qkv8": wl.qkv8, "fp8": wl.fp8, "bf16": wl.bf16, "quantize_q": wl.quantize_q})
        samples += clk.samples
        entry = ratios({**shape, "qkv8_bitwise_equal_fp8_forward_per_sequence": True,
                        **{k: summary(v) for k, v in r.items()}})
        report[wname] = entry
        print(wname, json.dumps(entry), flush=True)
        del wl
        torch.cuda.empty_cache()
    report["sm_clock_mhz_median"] = statistics.median(samples) if samples else None
    report["sm_clock_samples"] = len(samples)
    report["schedules_qkv8"] = run_children({"classic": {"TFA_KERNEL": "classic"},
                                             "persist": {"TFA_KERNEL": "persist"}}, list(workloads()))
    os.makedirs(os.path.dirname(os.path.abspath(out_path)), exist_ok=True)
    with open(out_path, "w") as f:
        json.dump(report, f, indent=1)
    print(json.dumps(report))


if __name__ == "__main__":
    if "--child" in sys.argv:
        child(sys.argv[sys.argv.index("--child") + 1].split(","))
    else:
        main(sys.argv[1] if len(sys.argv) > 1 else "kvcache_qkv8_bench.json")
