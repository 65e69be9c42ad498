#!/usr/bin/env python
"""The KV-cache forward with rotary position embedding (tfa_attn_kvcache_rotary_fwd) against the unfused path.

  K1  B16, Hq32 Hkv8 D128 bf16, Sq = Snew = 1, 8192 keys after the append, page 256
  K4  B16, Sq = Snew = 4 causal, 4096 keys after the append
  P   B4, Sq = Snew = 512 causal (a chunked-prefill step), 4096 keys cached before it

Arms, one call each on the same paged cache (kvcache_bench.py's workload set-up, split-KV left to the library):
  fused    tfa_attn_kvcache_rotary_fwd: one launch rotates q into a scratch buffer and appends rot(k_new) / v_new, then
           the forward (and the split-KV combine)
  unfused  what a caller does without it: gather cos / sin at the device-side positions cache_seqlens[b] + i, rotate q
           and k_new in eager torch fp32, cast back, then tfa_attn_kvcache_fwd with the plain append
  plain    tfa_attn_kvcache_fwd with the plain append and no rotation: the forward's own cost, which fused - plain
           separates from the rotation's (the q_rot write and re-read matter only on P)
rotary_dim = D (GPT-NeoX pairs).  Before any timing the fused out, lse and K/V pool must equal the unfused ones bit for
bit.  Timing, L2 flush, card, power limit and the median SM clock: as kvcache_bench.py.

Run from the repository root after build():   python scripts/kvcache_rotary_bench.py OUT.json
"""
import json
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tiny-flash-attention_b200"))
sys.path.insert(0, os.path.join(ROOT, "scripts"))
import tfa_ctypes as tfa  # noqa: E402
from kvcache_bench import D, HKV, HQ, PAGE, SCALE, Workload, summary, time_arms  # noqa: E402
from varlen_bench import ClockSampler, gpu_identity  # noqa: E402

ROTARY_DIM = D


def workloads():
    return {"K1": dict(B=16, S=1, keys=8192, causal=False),
            "K4": dict(B=16, S=4, keys=4096, causal=True),
            "P": dict(B=4, S=512, keys=4096 + 512, causal=True)}


def rope_tables(n, rd):
    inv = 1.0 / 10000.0 ** (torch.arange(0, rd, 2, dtype=torch.float64) / rd)
    ang = torch.outer(torch.arange(n, dtype=torch.float64), inv)
    return torch.cos(ang).to(torch.bfloat16).cuda(), torch.sin(ang).to(torch.bfloat16).cuda()


def rope(x, pos, cos, sin, rd):
    """GPT-NeoX rotation of x (B, S, H, D) at positions pos (B, S) in fp32, rounded once: the unfused arm."""
    c, s = cos[pos].float().unsqueeze(2), sin[pos].float().unsqueeze(2)
    x0, x1 = x[..., :rd // 2].float(), x[..., rd // 2:rd].float()
    return torch.cat([(x0 * c - x1 * s).to(x.dtype), (x0 * s + x1 * c).to(x.dtype), x[..., rd:]], dim=-1)


class RotaryWorkload(Workload):
    def __init__(self, B, S, keys, causal, seed):
        # the cache holds keys - S tokens per sequence, capacity `keys`: the append fills it
        super().__init__([keys] * B, S, causal, seed)
        self.sl.fill_(keys - S)
        self.cap = self.table.shape[1] * PAGE
        g = torch.Generator(device="cuda").manual_seed(seed + 1)
        self.kn = torch.empty((B, S, HKV, D), dtype=torch.bfloat16, device="cuda").normal_(0, 0.5, generator=g)
        self.vn = torch.empty_like(self.kn).normal_(0, 0.5, generator=g)
        self.cos, self.sin = rope_tables(self.cap, ROTARY_DIM)
        self.q_rot = torch.empty_like(self.q)
        self.ar = torch.arange(S, device="cuda")

    def fused(self):
        return tfa.attn_kvcache_fwd(self.q, self.kp, self.vp, self.sl, self.table, self.kn, self.vn,
                                    is_causal=self.causal, scale=SCALE, num_splits=0, out=self.out, lse=self.lse,
                                    rotary_cos=self.cos, rotary_sin=self.sin, q_rot=self.q_rot)

    def unfused(self):
        L = self.sl.clamp(0, self.cap - self.Sq).long().unsqueeze(1)
        pk = L + self.ar                                    # Sq == Snew: queries and keys share positions
        pq = pk if self.causal else L.expand_as(pk)
        qr = rope(self.q, pq, self.cos, self.sin, ROTARY_DIM)
        kr = rope(self.kn, pk, self.cos, self.sin, ROTARY_DIM)
        return tfa.attn_kvcache_fwd(qr, self.kp, self.vp, self.sl, self.table, kr, self.vn, is_causal=self.causal,
                                    scale=SCALE, num_splits=0, out=self.out, lse=self.lse)

    def plain(self):
        return tfa.attn_kvcache_fwd(self.q, self.kp, self.vp, self.sl, self.table, self.kn, self.vn,
                                    is_causal=self.causal, scale=SCALE, num_splits=0, out=self.out, lse=self.lse)

    def check(self):
        k0, v0 = self.kp.clone(), self.vp.clone()
        o1, l1 = (t.clone() for t in self.fused())
        k1, v1 = self.kp.clone(), self.vp.clone()
        self.kp.copy_(k0)
        self.vp.copy_(v0)
        o2, l2 = self.unfused()
        torch.cuda.synchronize()
        return bool(torch.equal(o1, o2) and torch.equal(l1, l2) and torch.equal(k1.view(torch.int16),
                    self.kp.view(torch.int16)) and torch.equal(v1.view(torch.int16), self.vp.view(torch.int16)))


def main(out_path):
    assert torch.cuda.is_available(), "kvcache_rotary_bench needs a GPU"
    tfa.lib()
    gpu_id, name, power = gpu_identity()
    report = {"gpu": name, "power_limit_w": power, "dtype": "bf16", "Hq": HQ, "Hkv": HKV, "D": D, "page": PAGE,
              "rotary_dim": ROTARY_DIM, "rotary_interleaved": False,
              "timing": "one call per sample after a 256 MB L2 flush, CUDA events, arms alternated (kvcache_bench.py)"}
    samples = []
    for i, (wname, w) in enumerate(workloads().items()):
        wl = RotaryWorkload(w["B"], w["S"], w["keys"], w["causal"], seed=30 + i)
        ok = wl.check()
        if not ok:
            raise SystemExit(f"{wname}: the fused output or cache differs from the unfused one")
        n0 = tfa.launch_count()
        wl.fused()
        launches = tfa.launch_count() - n0
        with ClockSampler(gpu_id) as clk:
            r = time_arms({"fused": wl.fused, "unfused": wl.unfused, "plain": wl.plain})
        samples += clk.samples
        B, S = w["B"], w["S"]
        # the rotation's own traffic: q in and q_rot out, k_new in and rot(k_new) out, the cos / sin rows it reads
        q_bytes = 2 * B * S * HQ * D * 2
        entry = {"B": B, "Sq": S, "Snew": S, "causal": w["causal"], "keys_after_append": w["keys"],
                 "fused_launches": launches, "fused_bitwise_equal_unfused": ok, "q_rot_bytes": q_bytes,
                 **{k: summary(v, 1) for k, v in r.items()}}
        for k in ("fused", "unfused", "plain"):
            entry[k] = {m: entry[k][m] for m in ("us_median", "us_min", "us_max")}
        f, u, p = (entry[k]["us_median"] for k in ("fused", "unfused", "plain"))
        entry["fused_over_unfused"] = round(f / u, 4)
        entry["fused_minus_plain_us"] = round(f - p, 2)
        report[wname] = entry
        del wl
        torch.cuda.empty_cache()
    report["sm_clock_mhz_median"] = statistics.median(samples) if samples else None
    report["sm_clock_samples"] = len(samples)
    os.makedirs(os.path.dirname(os.path.abspath(out_path)), exist_ok=True)
    with open(out_path, "w") as f:
        json.dump(report, f, indent=1)
    print(json.dumps(report))


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else "kvcache_rotary_bench.json")
