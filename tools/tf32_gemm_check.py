"""Validates the wgmma GEMM + row-norm kernel (limbo_b200/csrc/tf32_query.cu, tf32 and fp16 operands) against torch.
usage: python tools/tf32_gemm_check.py [M N K]"""
import ctypes as C
import os
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from limbo_b200 import _lib  # noqa: E402

M, N, K = (int(x) for x in sys.argv[1:4]) if len(sys.argv) > 3 else (256, 512, 512)
lib = _lib.load()
lib.lb_debug_tf32_gemm.argtypes = [C.c_void_p, C.c_void_p, C.c_longlong, C.c_longlong, C.c_longlong, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_int]
sms = torch.cuda.get_device_properties(0).multi_processor_count
torch.manual_seed(0)
A = torch.randn(M, K, device="cuda", dtype=torch.float32)
B = torch.randn(N, K, device="cuda", dtype=torch.float32)
for f16 in (0, 1):
    for tri in (0, 1):
        Bt = torch.tril(B) if tri else B
        Ah, Bh = (A.half(), Bt.half()) if f16 else (A, Bt)
        D = torch.zeros(M, N, device="cuda", dtype=torch.float32)
        nrm = torch.zeros(M, device="cuda", dtype=torch.float32)
        torch.cuda.synchronize()
        t0 = time.time()
        rc = lib.lb_debug_tf32_gemm(Ah.data_ptr(), Bh.data_ptr(), M, N, K, tri, nrm.data_ptr(), D.data_ptr(), sms, f16)
        dt = time.time() - t0
        ref = (Ah.double() @ Bh.double().T)
        err = (D.double() - ref).abs().max().item()
        scale = ref.abs().max().item()
        nerr = ((nrm.double() - (ref ** 2).sum(1)).abs() / (ref ** 2).sum(1)).max().item()
        print(f"f16={f16} tri={tri} rc={rc} max|D-ref|={err:.3e} (scale {scale:.2f}, rel {err / scale:.2e}) norm rel err {nerr:.2e} "
              f"time {dt * 1e3:.1f} ms", flush=True)
        assert rc == 0 and err / scale < 5e-3 and nerr < 5e-3
print("TF32 GEMM OK")
