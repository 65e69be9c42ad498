#!/usr/bin/env python
"""A/B of the two schedules of the forward kernel (TFA_KERNEL=classic|persist, read once per process, so each arm runs in
a subprocess): median of 15 CUDA-event-timed launches per shape after 3 warm-ups, both arms twice, min of the two
medians reported.  Run from the repository root on the GPU after build(); the result behind choose_kernel
(csrc/tfa_api.cu) is profiles/h100_kernel_choice.txt."""
import json, os, subprocess, sys
CASES = [(4,32,4096,128,True),(1,32,16384,128,True),(16,32,1024,128,True),(1,32,16384,128,False),(2,32,8192,128,False),
         (4,16,2048,64,False),(4,32,4096,64,True),(32,32,512,64,True),(2,32,8192,128,True),(64,32,4096,128,True),(1,32,16384,64,False)]
CODE = r'''
import json, os, sys, torch
sys.path.insert(0, "tiny-flash-attention_b200")
import tfa_ctypes as tfa
res = []
for (B, H, S, D, causal) in json.loads(os.environ["CASES"]):
    g = torch.Generator(device="cuda").manual_seed(20)
    q, k, v = (torch.empty(B, H, S, D, dtype=torch.bfloat16, device="cuda").normal_(0, 0.5, generator=g) for _ in range(3))
    out = torch.empty_like(q); lse = torch.empty(B, H, S, device="cuda")
    for _ in range(3): tfa.fwd(q, k, v, causal, D ** -0.5, out=out, lse=lse)
    torch.cuda.synchronize(); ts = []
    for _ in range(15):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(); tfa.fwd(q, k, v, causal, D ** -0.5, out=out, lse=lse); e1.record(); torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    ts.sort(); res.append(ts[len(ts)//2])
    del q, k, v, out, lse; torch.cuda.empty_cache()
print("RES", json.dumps(res))
'''
out = {}
for rep in range(2):
    for var in ("classic", "persist"):
        env = dict(os.environ, TFA_KERNEL=var, CASES=json.dumps(CASES))
        p = subprocess.run([sys.executable, "-c", CODE], env=env, capture_output=True, text=True)
        r = json.loads([l for l in p.stdout.splitlines() if l.startswith("RES")][0][4:]) if p.returncode == 0 else p.stderr[-500:]
        out.setdefault(var, []).append(r)
for i, c in enumerate(CASES):
    a = min(x[i] for x in out["classic"]); b = min(x[i] for x in out["persist"])
    print(c, "classic %.4f persist %.4f ms  -> %s" % (a, b, "classic" if a < b else "persist"), "spread c", [round(x[i],4) for x in out["classic"]], "p", [round(x[i],4) for x in out["persist"]])
