#!/usr/bin/env python
"""Attention against a paged KV cache (tfa_attn_kvcache_fwd) on one GPU: what paging costs, and which schedule wins.

  K1  B16, Hq32 Hkv8 D128 bf16, Sq = 1, 8192 cached keys each, page 256
  K2  B1, the same heads, 131072 cached keys (split-KV)
  K3  B64, lengths drawn with a fixed seed from [256, 16384]
  K4  B16, Sq = 4 causal, 4096 cached keys

Each workload runs paged (a random permuted block table over a pool with spare blocks) and contiguous (block_table
NULL, capacity = the longest sequence); K1 also runs tfa_attn_fwd on a pre-gathered (B, Hkv, S, D) cache.  Split-KV is
left to the library (num_splits = 0) in every arm.  One call is timed at a time with CUDA events, after a 256 MB write
that flushes the L2, over REPS repetitions with the arms alternated; the time covers every kernel of the call (the
split-KV combine included).  Decode is HBM-bound, so the figure of merit is bytes over time: the algorithmic bytes are
the valid K/V read once plus Q, O and LSE, against the H100 SXM data sheet's 3.35 TB/s (a data-sheet figure, not a
measured peak).  Before any timing the paged output must equal the contiguous one bit for bit.  Both schedules
(TFA_KERNEL=classic|persist, read once per process) are timed on the paged arms in alternating subprocesses.  The
card's name, power limit and the median SM clock sampled during the timed sections are recorded with the numbers.

Run from the repository root after build():   python scripts/kvcache_bench.py OUT.json
"""
import json
import os
import statistics
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tiny-flash-attention_b200"))
sys.path.insert(0, os.path.join(ROOT, "scripts"))
import tfa_ctypes as tfa  # noqa: E402
from varlen_bench import ClockSampler, gpu_identity  # noqa: E402

HQ, HKV, D, PAGE = 32, 8, 128, 256
SCALE = D ** -0.5
REPS = 30
HBM_DATASHEET_BPS = 3.35e12


def workloads():
    k3 = [int(x) for x in np.random.default_rng(2024).integers(256, 16385, size=64)]
    return {"K1": dict(lens=[8192] * 16, Sq=1, causal=False),
            "K2": dict(lens=[131072], Sq=1, causal=False),
            "K3": dict(lens=k3, Sq=1, causal=False),
            "K4": dict(lens=[4096] * 16, Sq=4, causal=True)}


def algo_bytes(lens, Sq):
    B = len(lens)
    return sum(lens) * HKV * D * 2 * 2 + 2 * B * Sq * HQ * D * 2 + B * HQ * Sq * 4


class Workload:
    def __init__(self, lens, Sq, causal, seed):
        self.lens, self.Sq, self.causal = lens, Sq, causal
        B = len(lens)
        g = torch.Generator(device="cuda").manual_seed(seed)
        cap = max(lens)
        mbps = -(-cap // PAGE)
        self.q = torch.empty((B, Sq, HQ, D), dtype=torch.bfloat16, device="cuda").normal_(0, 0.5, generator=g)
        self.kc = torch.empty((B, mbps * PAGE, HKV, D), dtype=torch.bfloat16, device="cuda").normal_(0, 0.5,
                                                                                                      generator=g)
        self.vc = torch.empty_like(self.kc).normal_(0, 0.5, generator=g)
        nblk = B * mbps + 8
        perm = torch.randperm(nblk, generator=torch.Generator().manual_seed(seed))[:B * mbps]
        self.table = perm.to(torch.int32).view(B, mbps).cuda()
        self.kp = torch.empty((nblk, PAGE, HKV, D), dtype=torch.bfloat16, device="cuda")
        self.vp = torch.empty_like(self.kp)
        self.kp[perm.cuda()] = self.kc.view(B * mbps, PAGE, HKV, D)
        self.vp[perm.cuda()] = self.vc.view(B * mbps, PAGE, HKV, D)
        self.sl = torch.tensor(lens, dtype=torch.int32, device="cuda")
        self.out = torch.empty_like(self.q)
        self.lse = torch.empty((B, HQ, Sq), dtype=torch.float32, device="cuda")

    def paged(self):
        return tfa.attn_kvcache_fwd(self.q, self.kp, self.vp, self.sl, self.table, is_causal=self.causal, scale=SCALE,
                                    num_splits=0, out=self.out, lse=self.lse)

    def contiguous(self):
        return tfa.attn_kvcache_fwd(self.q, self.kc, self.vc, self.sl, None, is_causal=self.causal, scale=SCALE,
                                    num_splits=0, out=self.out, lse=self.lse)

    def add_gathered(self):
        """(B, Hkv, S, D) copies for tfa_attn_fwd (all lengths equal)."""
        S = self.lens[0]
        self.dq = self.q.permute(0, 2, 1, 3).contiguous()
        self.dk = self.kc[:, :S].permute(0, 2, 1, 3).contiguous()
        self.dv = self.vc[:, :S].permute(0, 2, 1, 3).contiguous()

    def dense(self):
        return tfa.attn_fwd(self.dq, self.dk, self.dv, self.causal, SCALE, num_splits=0)

    def check(self):
        o1, l1 = (t.clone() for t in self.paged())
        o2, l2 = self.contiguous()
        torch.cuda.synchronize()
        return bool(torch.equal(o1, o2) and torch.equal(l1, l2))


_FLUSH = None


def time_arms(arms):
    """arms: name -> fn.  One call per sample after an L2 flush; arms alternated.  Returns name -> [ms]."""
    global _FLUSH
    if _FLUSH is None:
        _FLUSH = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    for fn in arms.values():
        for _ in range(3):
            fn()
    torch.cuda.synchronize()
    res = {name: [] for name in arms}
    for _ in range(REPS):
        for name, fn in arms.items():
            _FLUSH.fill_(1)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            fn()
            e1.record()
            torch.cuda.synchronize()
            res[name].append(e0.elapsed_time(e1))
    return res


def summary(ms, nbytes):
    med = statistics.median(ms)
    bps = nbytes / (med * 1e-3)
    return {"us_median": round(med * 1e3, 2), "us_min": round(min(ms) * 1e3, 2), "us_max": round(max(ms) * 1e3, 2),
            "GBps": round(bps / 1e9, 1), "of_datasheet_3p35TBps": round(bps / HBM_DATASHEET_BPS, 3)}


def schedule_child():
    """One subprocess of the schedule A/B: the paged arm of every workload under this process's TFA_KERNEL."""
    res = {}
    for i, (name, w) in enumerate(workloads().items()):
        wl = Workload(w["lens"], w["Sq"], w["causal"], seed=10 + i)
        res[name] = time_arms({"paged": wl.paged})["paged"]
        del wl
        torch.cuda.empty_cache()
    print("RES " + json.dumps({"res": res, "variant": tfa.lib().tfa_internal_last_variant()}))


def main(out_path):
    assert torch.cuda.is_available(), "kvcache_bench needs a GPU"
    tfa.lib()
    gpu_id, name, power = gpu_identity()
    report = {"gpu": name, "power_limit_w": power, "dtype": "bf16", "Hq": HQ, "Hkv": HKV, "D": D, "page": PAGE,
              "timing": "one call per sample after a 256 MB L2 flush, CUDA events, median of %d" % REPS,
              "hbm_datasheet_TBps": 3.35}
    samples = []
    for i, (wname, w) in enumerate(workloads().items()):
        wl = Workload(w["lens"], w["Sq"], w["causal"], seed=10 + i)
        ok = wl.check()
        n_split = tfa.attn_kvcache_fwd(wl.q, wl.kp, wl.vp, wl.sl, wl.table, is_causal=wl.causal, num_splits=0,
                                       return_splits=True)[2]
        arms = {"paged": wl.paged, "contiguous": wl.contiguous}
        if wname == "K1":
            wl.add_gathered()
            arms["dense_pregathered"] = wl.dense
        with ClockSampler(gpu_id) as clk:
            r = time_arms(arms)
        samples += clk.samples
        nb = algo_bytes(wl.lens, wl.Sq)
        entry = {"B": len(wl.lens), "Sq": wl.Sq, "causal": wl.causal, "keys_total": sum(wl.lens),
                 "keys_min": min(wl.lens), "keys_max": max(wl.lens), "num_splits": n_split,
                 "paged_bitwise_equal_contiguous": ok, "algorithmic_bytes": nb,
                 **{k: summary(v, nb) for k, v in r.items()}}
        entry["paged_over_contiguous"] = round(entry["paged"]["us_median"] / entry["contiguous"]["us_median"], 4)
        if "dense_pregathered" in entry:
            entry["paged_over_dense"] = round(entry["paged"]["us_median"] / entry["dense_pregathered"]["us_median"], 4)
        report[wname] = entry
        if not ok:
            raise SystemExit("paged output differs from the contiguous one: " + json.dumps(report))
        del wl
        torch.cuda.empty_cache()
    report["sm_clock_mhz_median"] = statistics.median(samples) if samples else None
    report["sm_clock_samples"] = len(samples)

    sched = {"classic": {}, "persist": {}}
    for _ in range(2):
        for var in ("classic", "persist"):
            env = dict(os.environ, TFA_KERNEL=var)
            p = subprocess.run([sys.executable, os.path.abspath(__file__), "--schedule-child"], env=env,
                               capture_output=True, text=True)
            if p.returncode != 0:
                raise SystemExit(p.stderr[-3000:])
            r = json.loads([l for l in p.stdout.splitlines() if l.startswith("RES ")][0][4:])
            assert r["variant"] == (0 if var == "classic" else 4), r
            for w, ms in r["res"].items():
                sched[var].setdefault(w, []).extend(ms)
    wls = workloads()
    report["schedules_paged"] = {var: {w: summary(ms, algo_bytes(wls[w]["lens"], wls[w]["Sq"]))
                                       for w, ms in sched[var].items()} for var in sched}
    os.makedirs(os.path.dirname(os.path.abspath(out_path)), exist_ok=True)
    with open(out_path, "w") as f:
        json.dump(report, f, indent=1)
    print(json.dumps(report))


if __name__ == "__main__":
    if "--schedule-child" in sys.argv:
        schedule_child()
    else:
        main(sys.argv[1] if len(sys.argv) > 1 else "kvcache_bench.json")
