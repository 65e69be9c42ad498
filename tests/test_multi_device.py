"""GPU, >= 2 devices in ONE process (skipped on the 1-GPU box): per-device host state (ADVICE r01).  The dynamic shared
memory opt-in, the SM count and the host-buffer workspace all belong to a device;
a process that runs the forward on cuda:0 and then on cuda:1 must get the oracle's result on both."""
import numpy as np
import pytest
import torch

from helpers import ref_inputs

pytestmark = pytest.mark.gpu


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs >= 2 GPUs in one process")
def test_second_device_in_the_same_process(built):
    import tfa_ctypes as tfa
    from oracle import oracle as orc
    tfa.lib()
    q0, k0, v0 = ref_inputs(1, 2, 512, 128, torch.bfloat16, seed=20, device="cpu")
    want, want_lse = orc.attn_exact(q0.float().numpy(), k0.float().numpy(), v0.float().numpy(), True, 128 ** -0.5,
                                    orc.ROUND_BF16, False)
    for dev in (0, 1, 0):
        with torch.cuda.device(dev):
            q, k, v = (t.to(f"cuda:{dev}") for t in (q0, k0, v0))
            o32, lse = tfa.fwd(q, k, v, True, 128 ** -0.5, out_fp32=True)
            torch.cuda.synchronize(dev)
            np.testing.assert_allclose(o32.cpu().numpy(), want, rtol=1e-3, atol=1e-3)
            np.testing.assert_allclose(lse.cpu().numpy(), want_lse, rtol=0, atol=2e-4)
            # host-buffer path: its workspace and streams are per device too
            hq, hk, hv = (t.pin_memory() for t in (q0, k0, v0))
            ho = torch.empty_like(q0).pin_memory()
            hl = torch.empty(1, 2, 512, dtype=torch.float32).pin_memory()
            tfa.fwd_host(hq, hk, hv, ho, hl, True, 128 ** -0.5, n_chunks=2)
            assert np.abs(ho.float().numpy() - want).max() <= 1e-2
            np.testing.assert_allclose(hl.numpy(), want_lse, rtol=0, atol=2e-4)
