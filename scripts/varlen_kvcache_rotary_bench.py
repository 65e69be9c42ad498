#!/usr/bin/env python
"""The variable-length KV-cache call with rotary position embedding (tfa_attn_varlen_kvcache_rotary_fwd) against the
unfused path, on a 16-bit and an FP8 (e4m3) cache.

Workloads M1, M2 and M3 of varlen_kvcache_bench.py (Hq32 Hkv8 D128 bf16, page 256, causal, every call appends its
queries' keys), with rotary_dim = D and GPT-NeoX pairs.  Arms, one call (or the arm's calls) each on the same pools:
  fused    tfa_attn_varlen_kvcache_rotary_fwd (FP8: with the cache's tfa_kv_quant_args): one launch rotates q into a
           scratch buffer and appends rot(k_new) / v_new, then the forward
  unfused  what a caller does without it: with the per-token positions L_b + i of the step given (a scheduler knows
           them on the host), gather cos / sin, rotate q and k_new in eager torch fp32, cast back, then the plain
           variable-length cache call
  plain    the variable-length cache call without rotation: the forward's and the append's own cost, which
           fused - plain separates from the rotation's
Before any timing the fused out, lse and pools must equal the unfused ones bit for bit.  Timing, the L2 flush, the
alternated arms and the ROUNDS rounds are those of varlen_kvcache_bench.py; the card's name, power limit and the median
SM clock sampled during the timed sections are recorded with the numbers.

Run from the repository root after build():   python scripts/varlen_kvcache_rotary_bench.py OUT.json
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
from varlen_bench import ClockSampler, gpu_identity  # noqa: E402
from varlen_kvcache_bench import D, HKV, HQ, PAGE, REPS, ROUNDS, SCALE, Workload, summary, time_arms, workloads  # noqa

ROTARY_DIM = D
FP8_SCALES = (0.5, 0.25)          # k_scale, v_scale of the FP8 cache


def rope_tables(n, rd):
    inv = 1.0 / 10000.0 ** (torch.arange(0, rd, 2, dtype=torch.float64) / rd)
    ang = torch.outer(torch.arange(n, dtype=torch.float64), inv)
    return torch.cos(ang).to(torch.bfloat16).cuda(), torch.sin(ang).to(torch.bfloat16).cuda()


def rope(x, pos, cos, sin, rd):
    """GPT-NeoX rotation of packed x (total, H, D) at positions pos (total,) in fp32, rounded once: the unfused arm."""
    c, s = cos[pos].float().unsqueeze(1), sin[pos].float().unsqueeze(1)
    x0, x1 = x[..., :rd // 2].float(), x[..., rd // 2:rd].float()
    return torch.cat([(x0 * c - x1 * s).to(x.dtype), (x0 * s + x1 * c).to(x.dtype), x[..., rd:]], dim=-1)


class RotaryWorkload(Workload):
    def __init__(self, sq, lens, seed, fp8):
        super().__init__(sq, lens, seed)
        self.cap = self.table.shape[1] * PAGE
        if fp8:
            self.k0, self.v0 = (t.float().clamp(-448, 448).to(torch.float8_e4m3fn) for t in (self.k0, self.v0))
            self.kp, self.vp = self.k0.clone(), self.v0.clone()
        self.qkw = dict(k_scale=FP8_SCALES[0], v_scale=FP8_SCALES[1]) if fp8 else {}
        self.cos, self.sin = rope_tables(self.cap, ROTARY_DIM)
        self.q_rot = torch.empty_like(self.q)
        # the step's per-token positions (causal: queries and keys both at L_b + i), as a scheduler has them
        pos = []
        for (q0, q1), L in zip(self.off, lens):
            Lb = min(max(L, 0), self.cap - (q1 - q0))
            pos += range(Lb, Lb + q1 - q0)
        self.pos = torch.tensor(pos, dtype=torch.long, device="cuda")

    def call(self, q, kn, kp=None, vp=None, **kw):
        return tfa.attn_varlen_kvcache_fwd(q, self.kp if kp is None else kp, self.vp if vp is None else vp, self.cu,
                                           max(self.sq), self.sl, self.table, kn, self.vn, is_causal=True, scale=SCALE,
                                           out=self.out, lse=self.lse, **self.qkw, **kw)

    def fused(self, kp=None, vp=None):
        return self.call(self.q, self.kn, kp, vp, rotary_cos=self.cos, rotary_sin=self.sin, q_rot=self.q_rot)

    def unfused(self, kp=None, vp=None):
        qr = rope(self.q, self.pos, self.cos, self.sin, ROTARY_DIM)
        kr = rope(self.kn, self.pos, self.cos, self.sin, ROTARY_DIM)
        return self.call(qr, kr, kp, vp)

    def plain(self):
        return self.call(self.q, self.kn)

    def check(self):
        """fused against unfused on fresh pool copies: out, lse and pools bit for bit."""
        k1, v1, k2, v2 = self.k0.clone(), self.v0.clone(), self.k0.clone(), self.v0.clone()
        o1, l1 = (t.clone() for t in self.fused(k1, v1))
        o2, l2 = (t.clone() for t in self.unfused(k2, v2))
        torch.cuda.synchronize()
        u8 = lambda t: t.view(torch.uint8)
        return bool(torch.equal(o1, o2) and torch.equal(l1, l2) and torch.equal(u8(k1), u8(k2)) and
                    torch.equal(u8(v1), u8(v2)))


def main(out_path):
    assert torch.cuda.is_available(), "varlen_kvcache_rotary_bench needs a GPU"
    tfa.lib()
    gpu_id, name, power = gpu_identity()
    report = {"gpu": name, "power_limit_w": power, "dtype": "bf16", "Hq": HQ, "Hkv": HKV, "D": D, "page": PAGE,
              "causal": True, "append": True, "rotary_dim": ROTARY_DIM, "rotary_interleaved": False,
              "fp8_cache_scales": FP8_SCALES,
              "timing": "one call (or the arm's calls) per sample after a 256 MB L2 flush, CUDA events, arms alternated, "
                        "%d rounds of %d samples per arm (varlen_kvcache_bench.py)" % (ROUNDS, REPS)}
    samples = []
    med = statistics.median
    for cache in ("bf16", "fp8"):
        for i, (wname, (sq, lens)) in enumerate(workloads().items()):
            wl = RotaryWorkload(sq, lens, 30 + i, cache == "fp8")
            ok = wl.check()
            if not ok:
                raise SystemExit(f"{cache} {wname}: the fused output or cache differs from the unfused one")
            n0 = tfa.launch_count()
            wl.fused()
            launches = tfa.launch_count() - n0
            arms = {"fused": wl.fused, "unfused": wl.unfused, "plain": wl.plain}
            rounds = []
            with ClockSampler(gpu_id) as clk:
                for _ in range(ROUNDS):
                    rounds.append(time_arms(arms))
            samples += clk.samples
            r = {k: [x for rd in rounds for x in rd[k]] for k in arms}
            entry = {"B": len(sq), "query_rows": sum(sq), "max_seqlen_q": max(sq), "fused_launches": launches,
                     "fused_bitwise_equal_unfused": ok,
                     **{k: dict(summary(v), round_medians_us=[round(med(rd[k]) * 1e3, 1) for rd in rounds])
                        for k, v in r.items()}}
            f, u, p = (entry[k]["us_median"] for k in ("fused", "unfused", "plain"))
            entry["fused_over_unfused"] = round(f / u, 4)
            entry["fused_over_plain"] = round(f / p, 4)
            entry["fused_minus_plain_us"] = round(f - p, 2)
            entry["per_round_range"] = {
                k: [round(min(med(rd["fused"]) / med(rd[k]) for rd in rounds), 4),
                    round(max(med(rd["fused"]) / med(rd[k]) for rd in rounds), 4)] for k in ("unfused", "plain")}
            report.setdefault(cache + "_cache", {})[wname] = entry
            del wl
            torch.cuda.empty_cache()
    report["sm_clock_mhz_median"] = statistics.median(samples) if samples else None
    report["sm_clock_samples"] = len(samples)
    os.makedirs(os.path.dirname(os.path.abspath(out_path)), exist_ok=True)
    with open(out_path, "w") as f:
        json.dump(report, f, indent=1)
    print(json.dumps(report))


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else "varlen_kvcache_rotary_bench.json")
