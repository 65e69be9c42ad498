#!/usr/bin/env python
"""Split-KV in the variable-length KV-cache call (tfa_attn_varlen_kvcache_split_fwd) on one GPU: the long decodes of a
mixed step spread over the SMs, against the same call in one pass and against what a caller had to do before.

Common: D128 bf16, page 256, causal, every call appends its queries' keys (k_new / v_new).
  L1  2 decodes at 131072 cached keys, Hq32 Hkv8.  Also against tfa_attn_kvcache_fwd(B = 2, Sq = 1) at the same
      num_splits, which it should tie.
  L2  one 1024-token prefill chunk on 8192 cached keys + 3 decodes on 65536-131072 cached keys, Hq32 Hkv8.  Also
      against the two-call alternative: tfa_attn_kvcache_fwd for the decodes at 16 splits + the unsplit varlen call
      for the chunk.
  L3  the heads one GPU holds under tensor parallelism: Hq8 Hkv1, 8 decodes at 32768 cached keys.
  M1, M3  the mixed and pure-decode steps of scripts/varlen_kvcache_bench.py (Hq32 Hkv8): num_splits = 1 against the
      call without split (what one pass costs through the new entry point), and what auto picks.
Arms: the split call at num_splits 2, 4, 8, 16 and 0 (auto), and the unsplit varlen call.  Before timing, every arm's
out, lse and pools are checked: num_splits = 1 bit for bit against the call without split, each split count per
sequence bit for bit against tfa_attn_kvcache_fwd at that count (L1; on L2 the two-call arm's decodes at 16).  One call (or the arm's calls) is timed at a time with CUDA events after a 256 MB
write that flushes the L2, REPS repetitions with the arms alternated, in ROUNDS rounds; medians over all samples, the
per-round medians, and the range of the per-round ratios to the unsplit call.  The combine kernel's own time comes
from a torch.profiler pass of its own.  The card's name, power limit and the median SM clock sampled during the timed
sections are recorded with the numbers.

Run from the repository root after build():   python scripts/varlen_kvcache_split_bench.py OUT.json
"""
import ctypes
import json
import os
import statistics
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tiny-flash-attention_b200"))
sys.path.insert(0, os.path.join(ROOT, "scripts"))
import tfa_ctypes as tfa  # noqa: E402
from varlen_bench import ClockSampler, gpu_identity  # noqa: E402
from varlen_kvcache_bench import workloads as base_workloads  # noqa: E402

D, PAGE = 128, 256
SCALE = D ** -0.5
REPS = 20
ROUNDS = 5
SPLITS = (2, 4, 8, 16, 0)


def workloads():
    r = np.random.default_rng(91)
    base = base_workloads()
    l2_lens = [8192] + [int(x) for x in r.integers(65536, 131073, size=3)]
    return {"L1": ([1, 1], [131072, 131072], 32, 8),
            "L2": ([1024, 1, 1, 1], l2_lens, 32, 8),
            "L3": ([1] * 8, [32768] * 8, 8, 1),
            "M1": (*base["M1"], 32, 8),
            "M3": (*base["M3"], 32, 8)}


def bits(t):
    return t.view(torch.int16)


class Workload:
    def __init__(self, sq, lens, hq, hkv, seed):
        self.sq, self.lens, self.hq, self.hkv = sq, lens, hq, hkv
        B, tq = len(sq), sum(sq)
        g = torch.Generator(device="cuda").manual_seed(seed)
        mk = lambda *s: torch.empty(s, dtype=torch.bfloat16, device="cuda").normal_(0, 0.5, generator=g)
        self.q, self.kn, self.vn = mk(tq, hq, D), mk(tq, hkv, D), mk(tq, hkv, D)
        self.mbps = -(-(max(l + s for l, s in zip(lens, sq))) // PAGE)
        nblk = B * self.mbps + 8
        perm = torch.randperm(nblk, generator=torch.Generator().manual_seed(seed))[:B * self.mbps]
        self.table = perm.to(torch.int32).view(B, self.mbps).cuda()
        self.k0, self.v0 = mk(nblk, PAGE, hkv, D), mk(nblk, PAGE, hkv, D)
        self.kp, self.vp = self.k0.clone(), self.v0.clone()
        self.sl = torch.tensor(lens, dtype=torch.int32, device="cuda")
        c = np.concatenate([[0], np.cumsum(sq)]).astype(int)
        self.off = list(zip(c[:-1].tolist(), c[1:].tolist()))
        self.cu = torch.tensor(c, dtype=torch.int32, device="cuda")
        self.out = torch.empty_like(self.q)
        self.lse = torch.empty((hq, tq), dtype=torch.float32, device="cuda")
        self.ws = {}

    def call(self, ns, kp=None, vp=None, out=None, lse=None):
        """The varlen call at num_splits ns (1: the call without split), with a workspace allocated once per count."""
        if ns != 1 and ns not in self.ws:
            a = ctypes.byref(tfa.VarlenKvcacheArgs(B=len(self.sq), Hq=self.hq, D=D, total_q=sum(self.sq),
                                                   max_seqlen_q=max(self.sq), page_block_size=PAGE,
                                                   max_blocks_per_seq=self.mbps, is_causal=1))
            n = tfa.lib().tfa_attn_varlen_kvcache_num_splits(a, ns)
            need = tfa.lib().tfa_attn_varlen_kvcache_workspace_bytes(a, n)
            self.ws[ns] = torch.empty(max(need // 4, 1), dtype=torch.float32, device="cuda")
        return tfa.attn_varlen_kvcache_fwd(self.q, self.kp if kp is None else kp, self.vp if vp is None else vp,
                                           self.cu, max(self.sq), self.sl, self.table, self.kn, self.vn,
                                           is_causal=True, scale=SCALE, out=self.out if out is None else out,
                                           lse=self.lse if lse is None else lse, num_splits=ns,
                                           workspace=self.ws.get(ns), return_splits=True)

    def split_count(self, ns):
        return self.call(ns, self.k0.clone(), self.v0.clone(), torch.empty_like(self.out),
                         torch.empty_like(self.lse))[2]

    def dense_decodes(self, ns, idx, kp=None, vp=None):
        """tfa_attn_kvcache_fwd over the decodes `idx` (Sq = 1) at num_splits ns, on inputs gathered beforehand
        (prepare_dense), as a caller that keeps its decodes apart would hold them."""
        d = self.dense[tuple(idx)]
        return tfa.attn_kvcache_fwd(d["q"], self.kp if kp is None else kp, self.vp if vp is None else vp, d["sl"],
                                    d["tab"], d["kn"], d["vn"], is_causal=True, scale=SCALE, num_splits=ns), d["rows"]

    def prepare_dense(self, idx):
        rows = [self.off[b][0] for b in idx]
        r, it = torch.tensor(rows, device="cuda"), torch.tensor(idx, device="cuda")
        self.dense = getattr(self, "dense", {})
        self.dense[tuple(idx)] = dict(q=self.q[r][:, None].contiguous(), kn=self.kn[r][:, None].contiguous(),
                                      vn=self.vn[r][:, None].contiguous(), sl=self.sl[it].contiguous(),
                                      tab=self.table[it].contiguous(), rows=rows)

    def chunk_call(self):
        """The unsplit varlen call over the prefill chunk (sequence 0) alone."""
        q0, q1 = self.off[0]
        if not hasattr(self, "chunk"):
            self.chunk = dict(cu=torch.tensor([0, q1 - q0], dtype=torch.int32, device="cuda"),
                              sl=self.sl[:1].clone(), tab=self.table[:1].contiguous(), q=self.q[q0:q1],
                              kn=self.kn[q0:q1], vn=self.vn[q0:q1])
        c = self.chunk
        return tfa.attn_varlen_kvcache_fwd(c["q"], self.kp, self.vp, c["cu"], q1 - q0, c["sl"], c["tab"], c["kn"],
                                           c["vn"], is_causal=True, scale=SCALE)


_FLUSH = None


def time_arms(arms):
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


def combine_us(fn):
    """Median device time of the combine kernel over 10 calls of fn, from torch.profiler."""
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(10):
            fn()
        torch.cuda.synchronize()
    ts = [e.device_time for e in prof.events() if "splitkv_combine" in e.name]
    return round(statistics.median(ts), 2) if ts else None


def check(wl, name):
    """num_splits = 1 equals the call without split bit for bit; on L1 every split count, and on L2 the two-call arm's
    decodes at 16, equal tfa_attn_kvcache_fwd at that count per sequence bit for bit."""
    res = {}
    k1, v1, k2, v2 = (wl.k0.clone() for _ in range(4))
    o_ref, l_ref, _ = wl.call(1, k1, v1, torch.empty_like(wl.out), torch.empty_like(wl.lse))
    o_ref, l_ref = o_ref.clone(), l_ref.clone()
    o1, l1 = torch.empty_like(wl.out), torch.empty_like(wl.lse)
    tfa.attn_varlen_kvcache_fwd(wl.q, k2, v2, wl.cu, max(wl.sq), wl.sl, wl.table, wl.kn, wl.vn, is_causal=True,
                                scale=SCALE, out=o1, lse=l1, num_splits=1, workspace=_EMPTY)
    torch.cuda.synchronize()
    res["splits1_bitwise_equal_to_unsplit"] = bool(torch.equal(bits(o1), bits(o_ref)) and torch.equal(l1, l_ref) and
                                                   torch.equal(bits(k1), bits(k2)) and torch.equal(bits(v1), bits(v2)))
    if name == "L1":
        idx = list(range(len(wl.sq)))
        wl.prepare_dense(idx)
        ok = True
        for ns in (2, 4, 8, 16):
            ka, va, kb, vb = (wl.k0.clone() for _ in range(4))
            o, l, _ = wl.call(ns, ka, va, torch.empty_like(wl.out), torch.empty_like(wl.lse))
            (od, ld), rows = wl.dense_decodes(ns, idx, kb, vb)
            torch.cuda.synchronize()
            ok &= bool(torch.equal(bits(o[rows]), bits(od[:, 0])) and torch.equal(l[:, rows], ld[:, :, 0].T) and
                       torch.equal(bits(ka), bits(kb)))
        res["splits_bitwise_equal_to_kvcache_call"] = ok
    if name == "L2":
        idx = list(range(1, len(wl.sq)))
        wl.prepare_dense(idx)
        ka, va, kb, vb = (wl.k0.clone() for _ in range(4))
        o, l, _ = wl.call(16, ka, va, torch.empty_like(wl.out), torch.empty_like(wl.lse))
        (od, ld), rows = wl.dense_decodes(16, idx, kb, vb)
        torch.cuda.synchronize()
        res["two_call_decodes_bitwise_equal_at_16_splits"] = bool(
            torch.equal(bits(o[rows]), bits(od[:, 0])) and torch.equal(l[:, rows], ld[:, :, 0].T))
    return res


def main(out_path):
    assert torch.cuda.is_available(), "varlen_kvcache_split_bench needs a GPU"
    tfa.lib()
    gpu_id, gname, power = gpu_identity()
    report = {"gpu": gname, "power_limit_w": power, "dtype": "bf16", "D": D, "page": PAGE, "causal": True,
              "append": True, "sms": torch.cuda.get_device_properties(0).multi_processor_count,
              "timing": "one call (or the arm's calls) per sample after a 256 MB L2 flush, CUDA events, %d rounds of "
                        "%d" % (ROUNDS, REPS)}
    samples = []
    for i, (wname, (sq, lens, hq, hkv)) in enumerate(workloads().items()):
        wl = Workload(sq, lens, hq, hkv, seed=50 + i)
        entry = {"B": len(sq), "Hq": hq, "Hkv": hkv, "query_rows": sum(sq), "max_seqlen_q": max(sq),
                 "cached": lens if len(lens) <= 8 else [min(lens), max(lens)], "capacity": wl.mbps * PAGE}
        entry.update(check(wl, wname))
        arms = {"unsplit": lambda: wl.call(1)}
        if wname in ("M1", "M3"):
            arms["splits_1"] = lambda: tfa.attn_varlen_kvcache_fwd(
                wl.q, wl.kp, wl.vp, wl.cu, max(wl.sq), wl.sl, wl.table, wl.kn, wl.vn, is_causal=True, scale=SCALE,
                out=wl.out, lse=wl.lse, num_splits=1, workspace=_EMPTY)
            arms["auto"] = lambda: wl.call(0)
        else:
            for ns in SPLITS:
                arms["auto" if ns == 0 else f"splits_{ns}"] = (lambda n: (lambda: wl.call(n)))(ns)
        if wname == "L1":
            idx = list(range(len(sq)))
            for ns in (2, 4, 8, 16):
                arms[f"kvcache_splits_{ns}"] = (lambda n: (lambda: wl.dense_decodes(n, idx)))(ns)
        if wname == "L2":
            idx = list(range(1, len(sq)))
            arms["two_calls_splits_16"] = lambda: (wl.dense_decodes(16, idx), wl.chunk_call())
        entry["split_counts"] = {k: wl.split_count(0 if k == "auto" else int(k.split("_")[1]))
                                 for k in arms if k == "auto" or (k.startswith("splits_") and k != "splits_1")}
        rounds = []
        with ClockSampler(gpu_id) as clk:
            for _ in range(ROUNDS):
                rounds.append(time_arms(arms))
        samples += clk.samples
        med = lambda ms: statistics.median(ms)
        r = {k: [x for rd in rounds for x in rd[k]] for k in arms}
        for k, v in r.items():
            entry[k] = dict(summary(v), round_medians_us=[round(med(rd[k]) * 1e3, 1) for rd in rounds])
        base = entry["unsplit"]["us_median"]
        entry["speedup_over_unsplit"] = {k: round(base / entry[k]["us_median"], 3) for k in r if k != "unsplit"}
        entry["speedup_over_unsplit_per_round_range"] = {
            k: [round(min(med(rd["unsplit"]) / med(rd[k]) for rd in rounds), 3),
                round(max(med(rd["unsplit"]) / med(rd[k]) for rd in rounds), 3)] for k in r if k != "unsplit"}
        best = max((k for k in r if k.startswith("splits_") or k == "auto"), key=lambda k: -entry[k]["us_median"],
                   default=None)
        if best and best != "splits_1":
            n = 0 if best == "auto" else int(best.split("_")[1])
            entry["combine_us_at_" + best] = combine_us(lambda: wl.call(n))
        report[wname] = entry
        print(wname, json.dumps(entry), flush=True)
        del wl, arms
        torch.cuda.empty_cache()
    report["sm_clock_mhz_median"] = statistics.median(samples) if samples else None
    report["sm_clock_samples"] = len(samples)
    os.makedirs(os.path.dirname(os.path.abspath(out_path)), exist_ok=True)
    with open(out_path, "w") as f:
        json.dump(report, f, indent=1)
    print(json.dumps(report))


_EMPTY = None

if __name__ == "__main__":
    if torch.cuda.is_available():
        _EMPTY = torch.empty(0, device="cuda")
    main(sys.argv[1] if len(sys.argv) > 1 else "varlen_kvcache_split_bench.json")
