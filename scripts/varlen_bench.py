#!/usr/bin/env python
"""Variable-length forward (tfa_attn_varlen_fwd) against the dense forward on the same work, on one GPU.

  W1  equal lengths: 4 x 4096 packed, H32 D128 bf16 causal, against dense B4 S4096 (bench.py's cfg3).
  W2  mixed lengths: 64 lengths drawn with a fixed seed from [256, 8192], H32 D128 bf16 causal, against
      (a) dense with every sequence padded to the longest one and (b) one dense call per sequence.

Useful work is F = 4 * Hq * D * sum_b visible_pairs_b (for a square causal sequence 2 * H * S^2 * D up to the
diagonal's half, bench.py's count), so padding counts as overhead, not as throughput.  Every arm is warmed up,
timed with CUDA events over back-to-back calls, and the arms are alternated in one process; the medians over the
repetitions are reported with their spread.  Before any timing, the varlen outputs (O and LSE) must equal the
per-sequence dense outputs bit for bit.  Both schedules of the kernel (TFA_KERNEL=classic|persist, read once per
process) are timed on W1 and W2 in alternating subprocesses.  The card's name, power limit and the median SM clock
sampled during the timed sections are recorded with the numbers.

Run from the repository root after build():   python scripts/varlen_bench.py OUT.json
"""
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

H, D = 32, 128
SCALE = D ** -0.5
REPS = 7


def w1_lengths():
    return [4096] * 4


def w2_lengths():
    return [int(x) for x in np.random.default_rng(2024).integers(256, 8193, size=64)]


def useful_flops(lens):
    return sum(4 * H * D * (s * (s + 1) // 2) for s in lens)      # causal, Sq_b == Sk_b


def packed(lens, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    mk = lambda: torch.empty((sum(lens), H, D), dtype=torch.bfloat16, device="cuda").normal_(0, 0.5, generator=g)
    cu = torch.tensor(np.concatenate([[0], np.cumsum(lens)]), dtype=torch.int32, device="cuda")
    return mk(), mk(), mk(), cu


def per_seq(x, lens):
    """(total, H, D) -> list of contiguous (1, H, S, D), one per sequence."""
    c = np.concatenate([[0], np.cumsum(lens)])
    return [x[c[i]:c[i + 1]].permute(1, 0, 2).unsqueeze(0).contiguous() for i in range(len(lens))]


def padded(x, lens):
    """(total, H, D) -> (B, H, max, D) with zeros after each sequence."""
    S = max(lens)
    out = torch.zeros((len(lens), H, S, D), dtype=x.dtype, device=x.device)
    c = np.concatenate([[0], np.cumsum(lens)])
    for i, s in enumerate(lens):
        out[i, :, :s] = x[c[i]:c[i + 1]].permute(1, 0, 2)
    return out


class Workload:
    def __init__(self, lens, seed):
        self.lens = lens
        self.q, self.k, self.v, self.cu = packed(lens, seed)
        self.out = torch.empty_like(self.q)
        self.lse = torch.empty((H, sum(lens)), dtype=torch.float32, device="cuda")

    def varlen(self):
        tfa.attn_varlen_fwd(self.q, self.k, self.v, self.cu, self.cu, max(self.lens), True, SCALE, out=self.out,
                            lse=self.lse)

    def add_loop(self):
        self.sq, self.sk, self.sv = (per_seq(t, self.lens) for t in (self.q, self.k, self.v))
        self.so = [torch.empty_like(t) for t in self.sq]
        self.sl = [torch.empty((1, H, t.shape[2]), dtype=torch.float32, device="cuda") for t in self.sq]

    def loop(self):
        for q, k, v, o, l in zip(self.sq, self.sk, self.sv, self.so, self.sl):
            tfa.fwd(q, k, v, True, SCALE, out=o, lse=l)

    def add_padded(self):
        self.pq, self.pk, self.pv = (padded(t, self.lens) for t in (self.q, self.k, self.v))
        self.po = torch.empty_like(self.pq)
        self.pl = torch.empty((len(self.lens), H, max(self.lens)), dtype=torch.float32, device="cuda")

    def padded_dense(self):
        tfa.fwd(self.pq, self.pk, self.pv, True, SCALE, out=self.po, lse=self.pl)

    def check_bitwise(self):
        """varlen O / LSE == the per-sequence dense calls', bit for bit."""
        self.varlen()
        self.variant = {0: "classic", 4: "persist"}[tfa.lib().tfa_internal_last_variant()]
        self.loop()
        torch.cuda.synchronize()
        c = np.concatenate([[0], np.cumsum(self.lens)])
        for i in range(len(self.lens)):
            if not (torch.equal(self.out[c[i]:c[i + 1]], self.so[i][0].permute(1, 0, 2)) and
                    torch.equal(self.lse[:, c[i]:c[i + 1]], self.sl[i][0])):
                return False
        return True


def time_arms(arms, calls):
    """arms: name -> fn.  Returns name -> list of ms per call, one entry per repetition, arms alternated."""
    for fn in arms.values():            # warm-up of every shape
        for _ in range(2):
            fn()
    torch.cuda.synchronize()
    res = {name: [] for name in arms}
    for _ in range(REPS):
        for name, fn in arms.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(calls[name]):
                fn()
            e1.record()
            torch.cuda.synchronize()
            res[name].append(e0.elapsed_time(e1) / calls[name])
    return res


def summary(ms, flops):
    med = statistics.median(ms)
    return {"ms_median": round(med, 4), "ms_min": round(min(ms), 4), "ms_max": round(max(ms), 4),
            "useful_tflops": round(flops / (med * 1e-3) / 1e12, 1)}


class ClockSampler:
    """SM clock of this GPU from nvidia-smi (read-only query) every 0.25 s while the timed sections run."""

    def __init__(self, gpu_id):
        self.gpu_id, self.samples, self.stop = gpu_id, [], threading.Event()
        self.t = threading.Thread(target=self.run, daemon=True)

    def run(self):
        while not self.stop.is_set():
            try:
                r = subprocess.run(["nvidia-smi", "-i", self.gpu_id, "--query-gpu=clocks.sm",
                                    "--format=csv,noheader,nounits"], capture_output=True, text=True, timeout=10)
                self.samples.append(float(r.stdout.strip().splitlines()[0]))
            except Exception:
                pass
            self.stop.wait(0.25)

    def __enter__(self):
        self.t.start()
        return self

    def __exit__(self, *exc):
        self.stop.set()
        self.t.join()


def gpu_identity():
    props = torch.cuda.get_device_properties(0)
    gpu_id = "GPU-" + str(props.uuid) if hasattr(props, "uuid") else "0"
    r = subprocess.run(["nvidia-smi", "-i", gpu_id, "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"],
                       capture_output=True, text=True)
    if r.returncode != 0:
        gpu_id = "0"
        r = subprocess.run(["nvidia-smi", "-i", gpu_id, "--query-gpu=name,power.limit",
                            "--format=csv,noheader,nounits"], capture_output=True, text=True)
    name, power = [x.strip() for x in r.stdout.strip().splitlines()[0].split(",")]
    return gpu_id, name, float(power)


def schedule_child():
    """One subprocess of the schedule A/B: varlen W1 and W2 under the TFA_KERNEL of this process."""
    w1, w2 = Workload(w1_lengths(), 1), Workload(w2_lengths(), 2)
    res = time_arms({"w1": w1.varlen, "w2": w2.varlen}, {"w1": 10, "w2": 5})
    print("RES " + json.dumps({"res": res, "variant": tfa.lib().tfa_internal_last_variant()}))


def main(out_path):
    assert torch.cuda.is_available(), "varlen_bench needs a GPU"
    tfa.lib()
    gpu_id, name, power = gpu_identity()
    report = {"gpu": name, "power_limit_w": power, "dtype": "bf16", "H": H, "D": D, "causal": True}

    w1 = Workload(w1_lengths(), 1)
    w1.add_loop()
    w2 = Workload(w2_lengths(), 2)
    w2.add_loop()
    ok1, ok2 = w1.check_bitwise(), w2.check_bitwise()
    report["bitwise_equal_to_per_sequence_calls"] = {"W1": ok1, "W2": ok2}
    report["auto_schedule"] = {"W1": w1.variant, "W2": w2.variant}
    if not (ok1 and ok2):
        raise SystemExit("varlen output differs from the per-sequence dense calls: " + json.dumps(report))
    w2.add_padded()
    # W1's dense arm is the B4 S4096 problem itself: the four sequences laid out as (B, H, S, D)
    dq, dk, dv = (torch.cat(t) for t in (w1.sq, w1.sk, w1.sv))
    do, dl = torch.empty_like(dq), torch.empty((4, H, 4096), dtype=torch.float32, device="cuda")
    dense_cfg3 = lambda: tfa.fwd(dq, dk, dv, True, SCALE, out=do, lse=dl)

    with ClockSampler(gpu_id) as clk:
        r1 = time_arms({"varlen": w1.varlen, "dense_B4_S4096": dense_cfg3}, {"varlen": 20, "dense_B4_S4096": 20})
        r2 = time_arms({"varlen": w2.varlen, "dense_padded": w2.padded_dense, "per_sequence_loop": w2.loop},
                       {"varlen": 5, "dense_padded": 3, "per_sequence_loop": 5})
    f1, f2 = useful_flops(w1.lens), useful_flops(w2.lens)
    report["W1"] = {"lengths": w1.lens, "useful_flop": f1, **{k: summary(v, f1) for k, v in r1.items()}}
    report["W1"]["varlen_over_dense"] = round(report["W1"]["varlen"]["ms_median"] /
                                              report["W1"]["dense_B4_S4096"]["ms_median"], 4)
    report["W2"] = {"lengths": w2.lens, "useful_flop": f2, **{k: summary(v, f2) for k, v in r2.items()}}
    for arm in ("dense_padded", "per_sequence_loop"):
        report["W2"]["speedup_vs_" + arm] = round(report["W2"][arm]["ms_median"] / report["W2"]["varlen"]["ms_median"],
                                                  3)
    report["sm_clock_mhz_median"] = statistics.median(clk.samples) if clk.samples else None
    report["sm_clock_samples"] = len(clk.samples)
    del w1, w2, dq, dk, dv, do, dl
    torch.cuda.empty_cache()

    # schedule A/B: both kernels, alternating subprocesses
    sched = {"classic": {"w1": [], "w2": []}, "persist": {"w1": [], "w2": []}}
    for _ in range(2):
        for var in ("classic", "persist"):
            env = dict(os.environ, TFA_KERNEL=var)
            p = subprocess.run([sys.executable, os.path.abspath(__file__), "--schedule-child"], env=env,
                               capture_output=True, text=True)
            if p.returncode != 0:
                raise SystemExit(p.stderr[-3000:])
            r = json.loads([l for l in p.stdout.splitlines() if l.startswith("RES ")][0][4:])
            assert r["variant"] == (0 if var == "classic" else 4), r
            for w in ("w1", "w2"):
                sched[var][w] += r["res"][w]
    report["schedules"] = {var: {w.upper(): summary(sched[var][w], f1 if w == "w1" else f2) for w in ("w1", "w2")}
                           for var in sched}
    os.makedirs(os.path.dirname(os.path.abspath(out_path)), exist_ok=True)
    with open(out_path, "w") as f:
        json.dump(report, f, indent=1)
    print(json.dumps(report))


if __name__ == "__main__":
    if "--schedule-child" in sys.argv:
        schedule_child()
    else:
        main(sys.argv[1] if len(sys.argv) > 1 else "varlen_bench.json")
