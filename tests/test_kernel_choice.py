"""GPU: which kernel the library picks on its own (`choose_kernel`, csrc/tfa_api.cu) for the shapes the rule was measured on
(an A/B of both schedules on one H100, profiles/h100_kernel_choice.txt).  The rule is host logic, but the only observable is
the variant of the last launch, so the shapes are launched for real -- in a subprocess, because TFA_KERNEL (which forces one
kernel) is read once per process."""
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu

CLASSIC, PERSIST = 0, 4
CASES = [
    # B, H, S, D, causal, expected, why (H100 A/B, median ms one-CTA-per-item / persistent)
    (4, 32, 4096, 128, True, CLASSIC, "cfg3: 0.913 / 1.002"),
    (1, 32, 16384, 128, True, CLASSIC, "cfg4, few very long causal items: 3.16 / 3.66"),
    (16, 32, 1024, 128, True, PERSIST, "short causal items: 0.423 / 0.378"),
    (1, 32, 16384, 128, False, PERSIST, "non-causal, 128 KV tiles per item, 31 items per SM: 7.22 / 6.75"),
    (2, 32, 8192, 128, False, PERSIST, "non-causal, 64 KV tiles per item: 3.36 / 3.26"),
    (4, 16, 2048, 64, False, PERSIST, "cfg2: 0.235 / 0.225"),
    (4, 32, 4096, 64, True, CLASSIC, "D=64 causal: 0.817 / 0.893"),
    (32, 32, 512, 64, True, PERSIST, "D=64 causal, S <= 512: 0.227 / 0.189"),
]

CODE = r'''
import json, os, sys, torch
sys.path.insert(0, os.path.join(os.environ["TFA_ROOT"], "tiny-flash-attention_b200"))
import tfa_ctypes as tfa
out = []
for (B, H, S, D, causal) in json.loads(os.environ["TFA_CASES"]):
    q = torch.randn(B, H, S, D, device="cuda", dtype=torch.bfloat16)
    o, lse = tfa.fwd(q, q, q, bool(causal), D ** -0.5)
    torch.cuda.synchronize()
    assert bool(torch.isfinite(lse).all())
    out.append(int(tfa.lib().tfa_internal_last_variant()))
print("VARIANTS", json.dumps(out))
'''


def test_auto_kernel_choice_follows_the_measured_rule(built):
    import json
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    env = {k: v for k, v in os.environ.items() if k != "TFA_KERNEL"}
    env.update(TFA_ROOT=root, TFA_CASES=json.dumps([c[:5] for c in CASES]))
    p = subprocess.run([sys.executable, "-c", CODE], env=env, capture_output=True, text=True, timeout=600)
    assert p.returncode == 0, p.stderr[-2000:]
    line = [ln for ln in p.stdout.splitlines() if ln.startswith("VARIANTS")][-1]
    got = json.loads(line.split(" ", 1)[1])
    for c, g in zip(CASES, got):
        assert g == c[5], f"{c[:5]} ({c[6]}): launched variant {g}, rule says {c[5]}"
