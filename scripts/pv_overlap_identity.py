#!/usr/bin/env python
"""Bit-for-bit comparison of two builds of the library on seeded inputs: out and lse of every call must be
torch.equal.  The softmax's schedule inside the KV loop (its exponentials under the in-flight PV wgmma, P in two
register sets) moves instructions, not arithmetic, so any difference is a bug.

Build the other library first (python tiny-flash-attention_b200/build.py --variant <name>, from the sources to
compare against), then run from the repository root on the GPU:

    python scripts/pv_overlap_identity.py --a <lib A> --b <lib B> --out <json>

Each library runs in a subprocess of its own (TFA_LIB selects it) and saves its results; this process compares them.
Calls: the benchmark's workload (B64 H32 S4096 D128 bf16 causal; its first and last 8 (batch, head) compared
element-wise, the whole out / lse by SHA-256), cfg2-cfg4, an fp16 D=64 causal call with an odd tile count, a split-KV
fp32-output call, a varlen batch, a paged bf16 cache, a paged FP8 cache, e4m3 (Q, K, V) dense and varlen calls, and
cache calls that append k_new (their caches compared too): dense-query with rotary, with an e4m3 q, and with a 16-bit q
quantized after rotary; variable-length with split-KV, with an FP8 cache, with an e4m3 q, and with a 16-bit q
quantized after rotary.  Together they reach every forward mode and both cache calls' appends: 16-bit, rotary, FP8,
and FP8 with the quantized q."""
import argparse
import hashlib
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def run_cases(path):
    import torch
    sys.path.insert(0, os.path.join(ROOT, "tiny-flash-attention_b200"))
    import tfa_ctypes as tfa
    dev = "cuda"
    res = {}

    def gen(seed):
        return torch.Generator(device=dev).manual_seed(seed)

    def rnd(g, *shape, dtype=torch.bfloat16):
        return torch.empty(*shape, dtype=dtype, device=dev).normal_(0.0, 0.5, generator=g)

    def digest(t):
        return hashlib.sha256(t.contiguous().view(torch.uint8).cpu().numpy().tobytes()).hexdigest()

    # the benchmark's workload, through the same call (tfa_fwd_ex)
    B, H, S, D = 64, 32, 4096, 128
    g = gen(20)
    q, k, v = (rnd(g, B, H, S, D) for _ in range(3))
    out, lse = tfa.fwd(q, k, v, True, D ** -0.5)
    o2, l2 = out.view(B * H, S, D), lse.view(B * H, S)
    res["bench B64 H32 S4096 D128 bf16 causal"] = {
        "out_first8": o2[:8].cpu(), "out_last8": o2[-8:].cpu(), "lse_first8": l2[:8].cpu(), "lse_last8": l2[-8:].cpu(),
        "out_sha256": digest(out), "lse_sha256": digest(lse)}
    del q, k, v, out, lse, o2, l2
    torch.cuda.empty_cache()

    dense = {"cfg2 B4 H16 S2048 D64 bf16 non-causal": (4, 16, 2048, 64, False, torch.bfloat16),
             "cfg3 B4 H32 S4096 D128 bf16 causal": (4, 32, 4096, 128, True, torch.bfloat16),
             "cfg4 B1 H32 S16384 D128 bf16 causal": (1, 32, 16384, 128, True, torch.bfloat16),
             "B2 H8 S640 D64 fp16 causal (5 KV tiles)": (2, 8, 640, 64, True, torch.float16)}
    for name, (B, H, S, D, causal, dt) in dense.items():
        g = gen(21)
        q, k, v = (rnd(g, B, H, S, D, dtype=dt) for _ in range(3))
        out, lse = tfa.fwd(q, k, v, causal, D ** -0.5)
        res[name] = {"out": out.cpu(), "lse": lse.cpu()}

    g = gen(22)
    q, k, v = rnd(g, 1, 8, 256, 128), rnd(g, 1, 8, 8192, 128), rnd(g, 1, 8, 8192, 128)
    out, lse = tfa.attn_fwd(q, k, v, False, 128 ** -0.5, num_splits=4, out_fp32=True)
    res["split-KV x4 fp32 out B1 H8 Sq256 Sk8192 D128 bf16"] = {"out": out.cpu(), "lse": lse.cpu()}

    g = gen(23)
    lens = [1000, 77, 2048, 513]
    cu = torch.tensor([0] + list(torch.tensor(lens).cumsum(0)), dtype=torch.int32, device=dev)
    q, k, v = (rnd(g, sum(lens), 16, 128) for _ in range(3))
    out, lse = tfa.attn_varlen_fwd(q, k, v, cu, cu, max(lens), True, 128 ** -0.5)
    res["varlen 4 seqs H16 D128 bf16 causal"] = {"out": out.cpu(), "lse": lse.cpu()}

    # paged caches: 4 sequences of up to 3000 keys in 256-row pages, 64 causal query rows each
    g = gen(24)
    Bc, Hq, Hkv, Dc, page, Sq = 4, 16, 4, 128, 256, 64
    nper = 12
    table = torch.randperm(Bc * nper, generator=torch.Generator().manual_seed(24)).view(Bc, nper).int().to(dev)
    sl = torch.tensor([3000, 129, 1800, 2560], dtype=torch.int32, device=dev)
    qc = rnd(g, Bc, Sq, Hq, Dc)
    kc, vc = rnd(g, Bc * nper, page, Hkv, Dc), rnd(g, Bc * nper, page, Hkv, Dc)
    out, lse = tfa.attn_kvcache_fwd(qc, kc, vc, sl, table, is_causal=True)
    res["paged bf16 cache B4 Hq16 Hkv4 D128 page256 Sq64 causal"] = {"out": out.cpu(), "lse": lse.cpu()}
    k8, v8 = (x.float().div(0.25).clamp(-448, 448).to(torch.float8_e4m3fn) for x in (kc, vc))
    out, lse = tfa.attn_kvcache_fwd(qc, k8, v8, sl, table, is_causal=True, k_scale=0.25, v_scale=0.25)
    res["paged FP8 cache B4 Hq16 Hkv4 D128 page256 Sq64 causal"] = {"out": out.cpu(), "lse": lse.cpu()}

    g = gen(25)
    q, k, v = (rnd(g, 2, 16, 2048, 128).float().div(0.25).to(torch.float8_e4m3fn) for _ in range(3))
    out, lse = tfa.attn_fwd(q, k, v, True, 128 ** -0.5, q_scale=0.25, k_scale=0.25, v_scale=0.25,
                            out_dtype=torch.bfloat16)
    res["e4m3 Q/K/V B2 H16 S2048 D128 causal, bf16 out"] = {"out": out.cpu(), "lse": lse.cpu()}

    g = gen(26)
    lens = [1000, 77, 2048, 513]
    cu = torch.tensor([0] + list(torch.tensor(lens).cumsum(0)), dtype=torch.int32, device=dev)
    q, k, v = (rnd(g, sum(lens), 16, 128).float().div(0.25).to(torch.float8_e4m3fn) for _ in range(3))
    out, lse = tfa.attn_varlen_fwd(q, k, v, cu, cu, max(lens), True, 128 ** -0.5, q_scale=0.25, k_scale=0.25,
                                   v_scale=0.25, out_dtype=torch.bfloat16)
    res["e4m3 varlen 4 seqs H16 D128 causal, bf16 out"] = {"out": out.cpu(), "lse": lse.cpu()}

    # calls that append k_new to the paged caches above (a fresh copy each), the cache after the call compared too:
    # the dense-query calls append 64 rows per sequence, the variable-length ones each sequence's query rows
    g = gen(27)
    e4m3 = lambda x: x.float().div(0.25).clamp(-448, 448).to(torch.float8_e4m3fn)    # noqa: E731
    cos, sin = (rnd(g, nper * page, 32) for _ in range(2))                            # rotary_dim 64
    kn, vn = rnd(g, Bc, Sq, Hkv, Dc), rnd(g, Bc, Sq, Hkv, Dc)
    qlens = [64, 1, 37, 100]
    cuq = torch.tensor([0] + list(torch.tensor(qlens).cumsum(0)), dtype=torch.int32, device=dev)
    qv, knv, vnv = rnd(g, sum(qlens), Hq, Dc), rnd(g, sum(qlens), Hkv, Dc), rnd(g, sum(qlens), Hkv, Dc)
    fp8 = dict(k_scale=0.25, v_scale=0.25)
    appends = {
        "paged bf16 cache + rotary append B4 Sq64 causal": (qc, kc, vc, dict(rotary_cos=cos, rotary_sin=sin)),
        "paged e4m3 q + FP8 cache append B4 Sq64 causal": (e4m3(qc), k8, v8, dict(q_scale=0.25,
                                                                                 out_dtype=torch.bfloat16, **fp8)),
        "paged 16-bit q quantized + rotary, FP8 cache append B4 Sq64 causal": (
            qc, k8, v8, dict(q8_scale=0.25, rotary_cos=cos, rotary_sin=sin, **fp8)),
        "varlen paged bf16 cache append, split-KV x4": (qv, kc, vc, dict(num_splits=4)),
        "varlen paged FP8 cache append": (qv, k8, v8, fp8),
        "varlen paged e4m3 q + FP8 cache append": (e4m3(qv), k8, v8, dict(q_scale=0.25, out_dtype=torch.bfloat16,
                                                                          **fp8)),
        "varlen paged 16-bit q quantized + rotary, FP8 cache append": (
            qv, k8, v8, dict(q8_scale=0.25, rotary_cos=cos, rotary_sin=sin, **fp8)),
    }
    for name, (qa, kca, vca, kw) in appends.items():
        kca, vca = kca.clone(), vca.clone()
        if qa.dim() == 4:
            out, lse = tfa.attn_kvcache_fwd(qa, kca, vca, sl, table, k_new=kn, v_new=vn, is_causal=True, **kw)
        else:
            out, lse = tfa.attn_varlen_kvcache_fwd(qa, kca, vca, cuq, max(qlens), sl, table, k_new=knv, v_new=vnv,
                                                   is_causal=True, **kw)
        res[name] = {"out": out.cpu(), "lse": lse.cpu(), "k_cache": kca.view(torch.uint8).cpu(),
                     "v_cache": vca.view(torch.uint8).cpu()}
    torch.cuda.synchronize()
    torch.save(res, path)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--a", help="library A (e.g. the parent commit's, built with build.py --variant)")
    ap.add_argument("--b", help="library B")
    ap.add_argument("--out", help="JSON result")
    ap.add_argument("--save", help=argparse.SUPPRESS)       # the child: run the cases on $TFA_LIB, save to this path
    args = ap.parse_args()
    if args.save:
        run_cases(args.save)
        return
    import torch
    with tempfile.TemporaryDirectory() as tmp:
        got = {}
        for tag, lib in (("a", args.a), ("b", args.b)):
            path = os.path.join(tmp, tag + ".pt")
            subprocess.run([sys.executable, os.path.abspath(__file__), "--save", path], check=True,
                           env=dict(os.environ, TFA_LIB=os.path.abspath(lib)))
            got[tag] = torch.load(path)
    calls = {}
    for name, ta in got["a"].items():
        tb = got["b"][name]
        calls[name] = {key: (ta[key] == tb[key]) if isinstance(ta[key], str) else bool(torch.equal(ta[key], tb[key]))
                       for key in ta}
    line = {"what": "torch.equal of out and lse (SHA-256 where marked) between two builds on seeded inputs",
            "a": os.path.basename(args.a), "b": os.path.basename(args.b),
            "gpu": torch.cuda.get_device_name(0),
            "all_equal": all(all(c.values()) for c in calls.values()), "calls": calls}
    print(json.dumps(line, indent=1))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(line, f, indent=1)
    sys.exit(0 if line["all_equal"] else 1)


if __name__ == "__main__":
    main()
