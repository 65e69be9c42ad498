#!/usr/bin/env python
"""The e4m3-query cache calls fed from a bf16 q (tfa_attn_kvcache_qkv8_q16_fwd / tfa_attn_varlen_kvcache_qkv8_q16_fwd)
on one GPU: q rotated (RoPE) and quantized in the append's launch, against the paths a caller has without them.

Workloads K1-K4 and M1 of scripts/kvcache_qkv8_bench.py (Hq 32 / Hkv 8, D 128, page 256, e4m3 pools, bf16 q / k_new /
v_new, with the append).  Two variants: `rope` (rotary_dim = D, GPT-NeoX pairs) and `quantize_only` (no rotary).  Arms:

  fused    the new call: one launch rotates and quantizes q into an e4m3 scratch and appends rot(k_new) / v_new
           quantized, then the attention on e4m3 wgmma (+ the split-KV combine)
  unfused  what a caller does without it: eager torch rotates q and k_new in fp32 at the step's positions (a scheduler
           has them on the host) as scripts/varlen_kvcache_rotary_bench.py does, quantizes q with
           (q / q_scale).clamp(-448, 448).to(float8_e4m3fn), then the e4m3-query call with the rotated k_new
  fp8      the widening FP8-cache call (tfa_attn_kvcache_fp8_fwd / tfa_attn_varlen_kvcache_rotary_fwd) with rotary
  bf16     the 16-bit cache call with rotary on a bf16 pool of the same values
(quantize_only: the same arms without any rotation.)

Before timing, the fused call's out, lse, appended pools and q8 must equal the unfused path's bit for bit, on fresh
pool copies.  One call (or the arm's calls) per sample after a 256 MB write that flushes the L2, CUDA events, arms
alternated; ROUNDS rounds of REPS samples, each round's median recorded with the overall median.  The timed calls use
num_splits = 0 (the library's choice).  The card's name, power limit and the median SM clock sampled during the timed
sections are recorded with the numbers.

Run from the repository root after build():   python scripts/kvcache_qkv8_q16_bench.py OUT.json
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
from kvcache_bench import D, PAGE, SCALE, workloads  # noqa: E402
from kvcache_fp8_bench import summary, time_arms  # noqa: E402
from kvcache_qkv8_bench import K_SCALE, Q_SCALE, V_SCALE, VarlenWorkload, Workload, quantize  # noqa: E402
from varlen_bench import ClockSampler, gpu_identity  # noqa: E402
from varlen_kvcache_bench import workloads as varlen_workloads  # noqa: E402

ROUNDS, REPS = 5, 10
ROTARY_DIM = D
FP8 = torch.float8_e4m3fn


def rope_tables(n, rd):
    inv = 1.0 / 10000.0 ** (torch.arange(0, rd, 2, dtype=torch.float64) / rd)
    ang = torch.outer(torch.arange(n, dtype=torch.float64), inv)
    return torch.cos(ang).to(torch.bfloat16).cuda(), torch.sin(ang).to(torch.bfloat16).cuda()


def rope(x, pos, cos, sin, rd=ROTARY_DIM):
    """GPT-NeoX rotation of x (..., H, D) at positions pos (x.shape[:-2]) in fp32, rounded once: the unfused arm."""
    c, s = cos[pos].float().unsqueeze(-2), sin[pos].float().unsqueeze(-2)
    x0, x1 = x[..., :rd // 2].float(), x[..., rd // 2:rd].float()
    return torch.cat([(x0 * c - x1 * s).to(x.dtype), (x0 * s + x1 * c).to(x.dtype), x[..., rd:]], dim=-1)


class Q16:
    """The four arms over a kvcache_qkv8_bench workload `w` (its bf16 q, k_new, v_new, e4m3 and bf16 pools), with q's
    and k_new's positions qpos / kpos and `call(q, k_new, kp, vp, out, lse, **kw)` the workload's cache call."""

    def __init__(self, w, rotary, qpos, kpos, call):
        self.w, self.call = w, call
        self.rotary = rotary
        self.cos, self.sin = rope_tables(w.cap, ROTARY_DIM)
        self.rot = dict(rotary_cos=self.cos, rotary_sin=self.sin) if rotary else {}
        self.qpos, self.kpos = qpos, kpos
        self.q8 = torch.empty(w.q.shape, dtype=FP8, device="cuda")
        self.q_rot = torch.empty_like(w.q)
        self.quant = dict(k_scale=K_SCALE, v_scale=V_SCALE)

    def fused(self, kp=None, vp=None, out=None, lse=None):
        w = self.w
        return self.call(w.q, w.kn, kp if kp is not None else w.k8, vp if vp is not None else w.v8, out, lse,
                         q8_scale=Q_SCALE, q8=self.q8, **self.quant, **self.rot)

    def unfused(self, kp=None, vp=None, out=None, lse=None):
        w = self.w
        qr, kr = w.q, w.kn
        if self.rotary:
            qr, kr = rope(w.q, self.qpos, self.cos, self.sin), rope(w.kn, self.kpos, self.cos, self.sin)
        q8 = quantize(qr, Q_SCALE)
        o, l = self.call(q8, kr, kp if kp is not None else w.k8, vp if vp is not None else w.v8, out, lse,
                         q_scale=Q_SCALE, out_dtype=torch.bfloat16, **self.quant)
        return o, l, q8

    def fp8(self):
        w = self.w
        return self.call(w.q, w.kn, w.k8, w.v8, None, None, q_rot=self.q_rot, **self.quant, **self.rot)

    def bf16(self):
        w = self.w
        return self.call(w.q, w.kn, w.k16, w.v16, None, None, q_rot=self.q_rot, **self.rot)

    def check(self):
        """fused against unfused on fresh pool copies: out, lse, pools and q8 bit for bit."""
        w = self.w
        k1, v1, k2, v2 = w.k8.clone(), w.v8.clone(), w.k8.clone(), w.v8.clone()
        o1, l1 = (t.clone() for t in self.fused(k1, v1, torch.empty_like(w.out), torch.empty_like(w.lse)))
        o2, l2, q8 = self.unfused(k2, v2, torch.empty_like(w.out), torch.empty_like(w.lse))
        torch.cuda.synchronize()
        u8 = lambda t: t.view(torch.uint8)
        return bool(torch.equal(o1.view(torch.int16), o2.view(torch.int16)) and
                    torch.equal(l1.view(torch.int32), l2.view(torch.int32)) and
                    torch.equal(u8(k1), u8(k2)) and torch.equal(u8(v1), u8(v2)) and torch.equal(u8(self.q8), u8(q8)))


def dense(wname, i, rotary):
    spec = workloads()[wname]
    w = Workload(spec["lens"], spec["Sq"], spec["causal"], seed=10 + i)
    B, Sq = len(w.lens), w.Sq
    Lb = torch.tensor([min(max(x, 0), w.cap - Sq) for x in w.lens], device="cuda")[:, None]
    ii = torch.arange(Sq, device="cuda")[None]
    kpos = Lb + ii
    qpos = kpos if w.causal else Lb.expand(B, Sq)

    def call(q, kn, kp, vp, out, lse, **kw):
        return tfa.attn_kvcache_fwd(q, kp, vp, w.sl, w.table, kn, w.vn, is_causal=w.causal, scale=SCALE, num_splits=0,
                                    out=w.out if out is None else out, lse=w.lse if lse is None else lse, **kw)
    shape = {"B": B, "Sq": Sq, "causal": w.causal, "keys_total": sum(w.lens), "append_per_seq": Sq}
    return Q16(w, rotary, qpos, kpos, call), shape


def varlen(rotary):
    sq, lens = varlen_workloads()["M1"]
    w = VarlenWorkload(sq, lens, seed=30)
    pos = []
    for n, L in zip(sq, lens):
        Lb = min(max(L, 0), max(w.cap - n, 0))
        pos += range(Lb, Lb + n)
    pos = torch.tensor(pos, dtype=torch.long, device="cuda")

    def call(q, kn, kp, vp, out, lse, **kw):
        return tfa.attn_varlen_kvcache_fwd(q, kp, vp, w.cu, max(w.sq), w.sl, w.table, kn, w.vn, is_causal=True,
                                           scale=SCALE, out=w.out if out is None else out,
                                           lse=w.lse if lse is None else lse, **kw)
    shape = {"B": len(sq), "rows": sum(sq), "causal": True, "keys_total": sum(lens), "append": "each sequence's rows"}
    return Q16(w, rotary, pos, pos, call), shape


def main(out_path):
    assert torch.cuda.is_available(), "kvcache_qkv8_q16_bench needs a GPU"
    tfa.lib()
    gpu_id, name, power = gpu_identity()
    report = {"gpu": name, "power_limit_w": power, "dtype": "bf16 q / k_new / v_new, e4m3 (or bf16) cache, bf16 out",
              "Hq": 32, "Hkv": 8, "D": D, "page": PAGE, "q_scale": Q_SCALE, "k_scale": K_SCALE, "v_scale": V_SCALE,
              "rotary_dim": ROTARY_DIM, "rotary_interleaved": False,
              "timing": f"one call (or the arm's calls) per sample after a 256 MB L2 flush, CUDA events, {ROUNDS} rounds "
                        f"x {REPS}, arms alternated, num_splits = 0"}
    samples = []
    for variant in ("rope", "quantize_only"):
        for i, wname in enumerate(list(workloads()) + ["M1_varlen"]):
            arms, shape = varlen(variant == "rope") if wname == "M1_varlen" else dense(wname, i, variant == "rope")
            if not arms.check():
                raise SystemExit(f"{variant} {wname}: the fused call differs from the unfused path")
            n0 = tfa.launch_count()
            arms.fused()
            launches = tfa.launch_count() - n0
            with ClockSampler(gpu_id) as clk:
                r = time_arms({"fused": arms.fused, "unfused": arms.unfused, "fp8": arms.fp8, "bf16": arms.bf16},
                              rounds=ROUNDS, reps=REPS)
            samples += clk.samples
            entry = {**shape, "fused_launches": launches, "fused_bitwise_equal_unfused": True,
                     **{k: summary(v) for k, v in r.items()}}
            for arm in ("unfused", "fp8", "bf16"):
                entry[f"{arm}_over_fused"] = round(entry[arm]["us_median"] / entry["fused"]["us_median"], 3)
                entry[f"{arm}_over_fused_per_round"] = [
                    round(a / b, 3) for a, b in zip(entry[arm]["us_round_medians"], entry["fused"]["us_round_medians"])]
            report.setdefault(variant, {})[wname] = entry
            print(variant, wname, json.dumps(entry), flush=True)
            del arms
            torch.cuda.empty_cache()
    report["sm_clock_mhz_median"] = statistics.median(samples) if samples else None
    report["sm_clock_samples"] = len(samples)
    os.makedirs(os.path.dirname(os.path.abspath(out_path)), exist_ok=True)
    with open(out_path, "w") as f:
        json.dump(report, f, indent=1)
    print(json.dumps(report))


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else "kvcache_qkv8_q16_bench.json")
