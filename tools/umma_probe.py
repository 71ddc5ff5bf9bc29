"""Diagnostic: run the wgmma self-test kernel over M / major-ness variants and report the error of the product
against an f64 matmul."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
from tianshou_b200 import _cabi
from tianshou_b200._cabi import call, ptr, stream_ptr
_cabi.use_diagnostics_library()      # ts_umma_selftest lives in the diagnostics build (python -m tianshou_b200.csrc.build --diag)

dev = "cuda:0"
rng = np.random.default_rng(0)

for M in (128, 64):
    for a_mn, b_mn in ((0, 0), (1, 0), (0, 1), (1, 1)):
        for N, K in ((64, 64), (16, 128), (8, 32), (128, 48)):
            a = rng.standard_normal((M, K)).astype(np.float32); b = rng.standard_normal((N, K)).astype(np.float32)
            ref = a.astype(np.float64) @ b.astype(np.float64).T
            d = torch.full((M, N), float("nan"), dtype=torch.float32, device=dev)
            ta, tb = torch.from_numpy(a).to(dev), torch.from_numpy(b).to(dev)
            try:
                call("ts_umma_selftest", ptr(ta), ptr(tb), ptr(d), M, N, K, 1, a_mn, b_mn, 0, stream_ptr())
                torch.cuda.synchronize()
                err = float(np.abs(d.cpu().numpy() - ref).max() / np.abs(ref).max())
            except Exception as e:  # noqa: BLE001
                err = f"ERR {e}"
            print(f"bf16x3 M={M} a_mn={a_mn} b_mn={b_mn} N={N} K={K}: {err}", flush=True)
