"""time (CUDA events) and check the four encoder GEMM shapes of one layer through bg_op_gemm_f16, M = B x 4000 tokens.
"""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from brepgen_b200 import _ffi

torch.backends.cuda.matmul.allow_tf32 = False
B = int(os.environ.get("B", 64))
M = B * 4000
g = torch.Generator(device="cuda").manual_seed(3)
# name, N, K, out_f16, relu, residual
SHAPES = [("qkv (q|k rows)", 1536, 768, 1, 0, False), ("v rows, hi|lo", 768, 1536, 1, 0, False), ("out-proj, hi|lo", 768, 1536, 0, 0, True),
          ("ffn1", 1024, 768, 1, 1, False), ("ffn2", 768, 1024, 0, 0, True)]
for name, N, K, f16, relu, res in SHAPES:
    A = torch.randn(M, K, generator=g, device="cuda").half()
    W = (torch.randn(N, K, generator=g, device="cuda") / K ** 0.5).half()
    bias = torch.randn(N, generator=g, device="cuda")
    X = torch.randn(M, N, generator=g, device="cuda") if res else None
    out = X.clone() if res else torch.empty(M, N, device="cuda", dtype=torch.float16 if f16 else torch.float32)
    call = lambda: _ffi.check(_ffi.lib().bg_op_gemm_f16(A.data_ptr(), K, W.data_ptr(), K, M, N, K, out.data_ptr(), N, f16, relu, bias.data_ptr(),
                                                      out.data_ptr() if res else None, N, None, 1, N, _ffi.current_stream()), "gemm")
    call()
    torch.cuda.synchronize()
    rows = slice(0, 4096)                                  # parity on the first rows (the reference GEMM is the slow part)
    ref = A[rows].float() @ W.float().t() + bias
    if res:
        ref = ref + X[rows]
    if relu:
        ref = ref.relu()
    err = float((out[rows].double() - ref.double()).norm() / ref.double().norm())
    if os.environ.get("ONCE"):          # one launch per shape (for profiler captures)
        print(f"{name:16s} M={M} N={N} K={K}: rel_l2={err:.2e}", flush=True)
        continue
    for _ in range(2):
        call()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(10):
        call()
    e1.record()
    torch.cuda.synchronize()
    us = e0.elapsed_time(e1) * 100
    nbytes = M * K * 2 + N * K * 2 + M * N * (2 if f16 else 4) * (2 if res else 1)
    print(f"{name:16s} M={M} N={N} K={K}: {us:7.1f} us  {2 * M * N * K / us / 1e6:6.0f} TF/s  {nbytes / us / 1e3:6.0f} GB/s  rel_l2={err:.2e}", flush=True)
