#!/usr/bin/env python
"""A variable-length batch of queries against a paged KV cache (tfa_attn_varlen_kvcache_fwd) on one GPU, against what a
caller had to do before it existed.

Common: Hq32 Hkv8 D128 bf16, page 256, causal, every call appends its queries' keys (k_new / v_new).
  M1  mixed step: 4 prefill chunks of 512 tokens on cached lengths drawn from [0, 4096] + 60 decodes on cached lengths
      drawn from [256, 8192].  Against tfa_attn_kvcache_fwd(B = 60, Sq = 1) + tfa_attn_kvcache_fwd(B = 4, Sq = 512),
      and against one cache call with every sequence padded to 512 query rows.
  M2  ragged chunked prefill: 16 chunks of lengths drawn from [1, 1024] on cached lengths drawn from [0, 8192].
      Against one cache call per sequence, and against one call padded to the longest chunk.
  M3  pure decode: B64, Sq_b = 1, cached lengths drawn from [256, 8192].  Against tfa_attn_kvcache_fwd(Sq = 1,
      num_splits = 1): what the varlen grid and its per-item decode cost.
The cache calls leave the split count to the library (num_splits = 0) except in M3.  Padded arms put each sequence's
real rows first and zeros after, and append all of them.  Before timing, the new call's out, lse and pools must equal
the equivalent arm's (M1: the two calls, M2: the per-sequence calls, M3: the one call) bit for bit, with that arm run
in one pass (num_splits = 1: a split-KV result is merged in fp32 and rounds differently).  One call (or the
arm's sequence of calls) is timed at a time with CUDA events after a 256 MB write that flushes the L2, over REPS
repetitions with the arms alternated, in ROUNDS rounds; each arm's median over all samples is reported, with the
per-round medians and the range of the per-round ratios to the new call, which is the run-to-run spread that a
difference between arms has to exceed to mean anything.  Both schedules (TFA_KERNEL=classic|persist, read once per
process) are timed on the new call in alternating subprocesses, and the work items launched but empty (past their
sequence's rows) are counted.  The card's name, power limit and the median SM clock sampled during the timed sections
are recorded with the numbers.

Run from the repository root after build():   python scripts/varlen_kvcache_bench.py OUT.json
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
ROUNDS = 5          # timed rounds per workload (REPS samples of every arm each), to show the run-to-run spread


def workloads():
    r = np.random.default_rng(77)
    m1_sq = [512] * 4 + [1] * 60
    m1_lens = [int(x) for x in r.integers(0, 4097, size=4)] + [int(x) for x in r.integers(256, 8193, size=60)]
    m2_sq = [int(x) for x in r.integers(1, 1025, size=16)]
    m2_lens = [int(x) for x in r.integers(0, 8193, size=16)]
    m3_lens = [int(x) for x in r.integers(256, 8193, size=64)]
    return {"M1": (m1_sq, m1_lens), "M2": (m2_sq, m2_lens), "M3": ([1] * 64, m3_lens)}


def bits(t):
    return t.view(torch.int16)


class Workload:
    """Packed q / k_new / v_new of the step, a pool behind a random permuted block table whose capacity also holds the
    padded arm's appends, and the padded tensors."""

    def __init__(self, sq, lens, seed):
        self.sq, self.lens = sq, lens
        B, tq, pad = len(sq), sum(sq), max(sq)
        g = torch.Generator(device="cuda").manual_seed(seed)
        mk = lambda *s: torch.empty(s, dtype=torch.bfloat16, device="cuda").normal_(0, 0.5, generator=g)
        self.q, self.kn, self.vn = mk(tq, HQ, D), mk(tq, HKV, D), mk(tq, HKV, D)
        mbps = -(-(max(lens) + pad) // PAGE)
        nblk = B * mbps + 8
        perm = torch.randperm(nblk, generator=torch.Generator().manual_seed(seed))[:B * mbps]
        self.table = perm.to(torch.int32).view(B, mbps).cuda()
        self.k0, self.v0 = mk(nblk, PAGE, HKV, D), mk(nblk, PAGE, HKV, D)
        self.kp, self.vp = self.k0.clone(), self.v0.clone()
        self.sl = torch.tensor(lens, dtype=torch.int32, device="cuda")
        c = np.concatenate([[0], np.cumsum(sq)]).astype(int)
        self.off = list(zip(c[:-1].tolist(), c[1:].tolist()))
        self.cu = torch.tensor(c, dtype=torch.int32, device="cuda")
        self.out = torch.empty_like(self.q)
        self.lse = torch.empty((HQ, tq), dtype=torch.float32, device="cuda")
        # padded (B, pad, H, D): real rows first, zeros after
        self.pq = torch.zeros((B, pad, HQ, D), dtype=torch.bfloat16, device="cuda")
        self.pk = torch.zeros((B, pad, HKV, D), dtype=torch.bfloat16, device="cuda")
        self.pv = torch.zeros_like(self.pk)
        for b, (q0, q1) in enumerate(self.off):
            self.pq[b, :q1 - q0] = self.q[q0:q1]
            self.pk[b, :q1 - q0] = self.kn[q0:q1]
            self.pv[b, :q1 - q0] = self.vn[q0:q1]
        self.pout = torch.empty_like(self.pq)
        self.plse = torch.empty((B, HQ, pad), dtype=torch.float32, device="cuda")

    def varlen_cache(self, kp=None, vp=None):
        return tfa.attn_varlen_kvcache_fwd(self.q, self.kp if kp is None else kp, self.vp if vp is None else vp, self.cu,
                                           max(self.sq), self.sl, self.table, self.kn, self.vn, is_causal=True,
                                           scale=SCALE, out=self.out, lse=self.lse)

    def groups(self, num_splits=0, kp=None, vp=None):
        """One cache call per run of sequences with the same query length (M1: decodes, prefills; M2: per sequence
        when all lengths differ).  Returns [(sequence indices, out, lse)]."""
        kp, vp = (self.kp, self.vp) if kp is None else (kp, vp)
        by = {}
        for b, s in enumerate(self.sq):
            by.setdefault(s, []).append(b)
        res = []
        for s, bs in by.items():
            idx = torch.tensor(bs, device="cuda")
            rows = torch.cat([torch.arange(self.off[b][0], self.off[b][1], device="cuda") for b in bs])
            q = self.q[rows].view(len(bs), s, HQ, D)
            kn, vn = self.kn[rows].view(len(bs), s, HKV, D), self.vn[rows].view(len(bs), s, HKV, D)
            o, l = tfa.attn_kvcache_fwd(q, kp, vp, self.sl[idx], self.table[idx], kn, vn, is_causal=True, scale=SCALE,
                                        num_splits=num_splits)
            res.append((bs, o, l))
        return res

    def prepare_groups(self, num_splits=0):
        """The grouped arm with its inputs gathered once, outside the timed region (as a caller that keeps its batch
        grouped would)."""
        by = {}
        for b, s in enumerate(self.sq):
            by.setdefault(s, []).append(b)
        self.calls = []
        for s, bs in by.items():
            idx = torch.tensor(bs, device="cuda")
            rows = torch.cat([torch.arange(self.off[b][0], self.off[b][1], device="cuda") for b in bs])
            self.calls.append(dict(q=self.q[rows].view(len(bs), s, HQ, D).contiguous(),
                                   kn=self.kn[rows].view(len(bs), s, HKV, D).contiguous(),
                                   vn=self.vn[rows].view(len(bs), s, HKV, D).contiguous(),
                                   sl=self.sl[idx].contiguous(), tab=self.table[idx].contiguous()))
        self.ns = num_splits

    def grouped(self):
        for c in self.calls:
            tfa.attn_kvcache_fwd(c["q"], self.kp, self.vp, c["sl"], c["tab"], c["kn"], c["vn"], is_causal=True,
                                 scale=SCALE, num_splits=self.ns)

    def padded(self):
        return tfa.attn_kvcache_fwd(self.pq, self.kp, self.vp, self.sl, self.table, self.pk, self.pv, is_causal=True,
                                    scale=SCALE, num_splits=0, out=self.pout, lse=self.plse)

    def check(self):
        """New call against the grouped calls in one pass, on fresh pool copies: out, lse and pools bit for bit."""
        k1, v1, k2, v2 = self.k0.clone(), self.v0.clone(), self.k0.clone(), self.v0.clone()
        o, l = (t.clone() for t in self.varlen_cache(k1, v1))
        ok = True
        for bs, og, lg in self.groups(1, k2, v2):
            for j, b in enumerate(bs):
                q0, q1 = self.off[b]
                ok &= torch.equal(o[q0:q1], og[j]) and torch.equal(l[:, q0:q1], lg[j])
        torch.cuda.synchronize()
        return bool(ok and torch.equal(bits(k1), bits(k2)) and torch.equal(bits(v1), bits(v2)))

    def items(self):
        pairs = -(-max(self.sq) // 128)
        busy = sum(-(-s // 128) for s in self.sq) * HQ
        return {"launched": len(self.sq) * HQ * pairs, "with_rows": busy, "empty": len(self.sq) * HQ * pairs - busy}


_FLUSH = None


def time_arms(arms):
    """arms: name -> fn.  One call (sequence) per sample after an L2 flush; arms alternated.  Returns name -> [ms]."""
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


def summary(ms):
    return {"us_median": round(statistics.median(ms) * 1e3, 2), "us_min": round(min(ms) * 1e3, 2),
            "us_max": round(max(ms) * 1e3, 2)}


def schedule_child():
    res = {}
    for i, (name, (sq, lens)) in enumerate(workloads().items()):
        wl = Workload(sq, lens, seed=30 + i)
        res[name] = time_arms({"varlen_kvcache": wl.varlen_cache})["varlen_kvcache"]
        del wl
        torch.cuda.empty_cache()
    print("RES " + json.dumps({"res": res, "variant": tfa.lib().tfa_internal_last_variant()}))


def main(out_path):
    assert torch.cuda.is_available(), "varlen_kvcache_bench needs a GPU"
    tfa.lib()
    gpu_id, name, power = gpu_identity()
    report = {"gpu": name, "power_limit_w": power, "dtype": "bf16", "Hq": HQ, "Hkv": HKV, "D": D, "page": PAGE,
              "causal": True, "append": True,
              "timing": "one call (or the arm's calls) per sample after a 256 MB L2 flush, CUDA events, median of %d"
                        % REPS}
    samples = []
    for i, (wname, (sq, lens)) in enumerate(workloads().items()):
        wl = Workload(sq, lens, seed=30 + i)
        ns = 1 if wname == "M3" else 0
        ok = wl.check()
        if not ok:
            raise SystemExit(f"{wname}: the new call differs from the equivalent calls")
        wl.prepare_groups(ns)
        arms = {"varlen_kvcache": wl.varlen_cache}
        arms[{"M1": "two_cache_calls", "M2": "cache_call_per_sequence", "M3": "cache_call_splits1"}[wname]] = wl.grouped
        if wname != "M3":
            arms["one_cache_call_padded"] = wl.padded
        rounds = []
        with ClockSampler(gpu_id) as clk:
            for _ in range(ROUNDS):
                rounds.append(time_arms(arms))
        samples += clk.samples
        r = {k: [x for rd in rounds for x in rd[k]] for k in arms}
        med = lambda ms: statistics.median(ms)
        entry = {"B": len(sq), "query_rows": sum(sq), "max_seqlen_q": max(sq), "cached_min": min(lens),
                 "cached_max": max(lens), "cache_calls_in_grouped_arm": len(wl.calls),
                 "bitwise_equal_to_equivalent_arm": ok, "items": wl.items(),
                 **{k: dict(summary(v), round_medians_us=[round(med(rd[k]) * 1e3, 1) for rd in rounds])
                    for k, v in r.items()}}
        base = entry["varlen_kvcache"]["us_median"]
        entry["speedup_over"] = {k: round(entry[k]["us_median"] / base, 3) for k in r if k != "varlen_kvcache"}
        entry["speedup_over_per_round_range"] = {
            k: [round(min(med(rd[k]) / med(rd["varlen_kvcache"]) for rd in rounds), 3),
                round(max(med(rd[k]) / med(rd["varlen_kvcache"]) for rd in rounds), 3)]
            for k in r if k != "varlen_kvcache"}
        report[wname] = entry
        del wl
        torch.cuda.empty_cache()
    report["sm_clock_mhz_median"] = statistics.median(samples) if samples else None
    report["sm_clock_samples"] = len(samples)

    sched = {"classic": {}, "persist": {}}
    sched_rounds = {"classic": {}, "persist": {}}
    for _ in range(3):
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
                sched_rounds[var].setdefault(w, []).append(round(statistics.median(ms) * 1e3, 1))
    report["schedules_varlen_kvcache"] = {var: {w: dict(summary(ms), round_medians_us=sched_rounds[var][w])
                                                for w, ms in sched[var].items()} for var in sched}
    report["schedule_auto"] = "persist (causal, ceil(max_seqlen_q / 128) <= 8)"
    os.makedirs(os.path.dirname(os.path.abspath(out_path)), exist_ok=True)
    with open(out_path, "w") as f:
        json.dump(report, f, indent=1)
    print(json.dumps(report))


if __name__ == "__main__":
    if "--schedule-child" in sys.argv:
        schedule_child()
    else:
        main(sys.argv[1] if len(sys.argv) > 1 else "varlen_kvcache_bench.json")
