#!/usr/bin/env python
"""Steady-state timing (CUDA events, back-to-back launches) of the hot dense-contraction shapes and epilogues, with the
bytes each launch has to move, to see how far each is from the HBM roofline."""
import os
import sys

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
import torch  # noqa: E402

from cmgan_b200 import ops  # noqa: E402
from cmgan_b200.ops import call, gemm  # noqa: E402

ops.set_precision(os.environ.get("CMGAN_PRECISION", "tf32"))
dev = "cuda"
M = 129684
torch.manual_seed(0)


def timeit(fn, reps=20):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps * 1e3


def report(name, us, nbytes):
    print(f"{name:38s} {us:8.1f} us   {nbytes / 1e6:7.1f} MB   {nbytes / us / 1e3:7.1f} GB/s")


x64, x128, x256 = torch.randn(M, 64, device=dev), torch.randn(M, 128, device=dev), torch.randn(M, 256, device=dev)
o64, o128, o256, o256b = torch.empty(M, 64, device=dev), torch.empty(M, 128, device=dev), torch.empty(M, 256, device=dev), torch.empty(M, 256, device=dev)
r64 = torch.randn(M, 64, device=dev)
W = {(n, k): torch.randn(n, k, device=dev) * 0.1 for n in (64, 128, 192, 256) for k in (64, 128, 256)}
b = {n: torch.randn(n, device=dev) for n in (64, 128, 192, 256)}
st = torch.empty(M, 2, device=dev)
call("cmgan_ln_stats", x64, 64, M, st)
g64, be64 = torch.randn(64, device=dev), torch.randn(64, device=dev)
F4 = 4

# copy baseline
big = torch.empty(M, 320, device=dev)
report("torch copy (M,256) r+w", timeit(lambda: o256.copy_(x256)), 2 * M * 256 * F4)
report("torch copy (M,64) r+w", timeit(lambda: o64.copy_(x64)), 2 * M * 64 * F4)

for (N, K, xin, out) in ((256, 64, x64, o256), (128, 64, x64, o128), (64, 64, x64, o64), (64, 256, x256, o64), (64, 128, x128, o64), (192, 64, x64, None)):
    if out is None:
        out = torch.empty(M, N, device=dev)
    report(f"rows N={N} K={K} plain+bias", timeit(lambda: gemm(A=xin, lda=K, W=W[(N, K)], sb_k=1, sb_n=K, bias=b[N], C=out, ldc=N, M=M, N=N, Cin=K)),
           M * (N + K) * F4)
report("rows N=256 K=64 SWISH_DUAL", timeit(lambda: gemm(A=x64, lda=64, W=W[(256, 64)], sb_k=1, sb_n=64, bias=b[256], C=o256, ldc=256, M=M, N=256, Cin=64,
                                                      epi=ops.EPI_SWISH_DUAL, C2=o256b, ldc2=256, seed=5, drop_p=0.2)), M * (64 + 512) * F4)
report("rows N=256 K=64 DSWISH_DROP", timeit(lambda: gemm(A=x64, lda=64, W=W[(64, 256)], sb_k=256, sb_n=1, C=o256, ldc=256, M=M, N=256, Cin=64,
                                                       epi=ops.EPI_DSWISH_DROP, aux=x256, ldaux=256, seed=5, drop_p=0.2)), M * (64 + 512) * F4)
report("rows N=64 K=256 DROP_RES", timeit(lambda: gemm(A=x256, lda=256, W=W[(64, 256)], sb_k=1, sb_n=256, bias=b[64], C=o64, ldc=64, M=M, N=64, Cin=256,
                                                    epi=ops.EPI_DROP_RES, alpha=0.5, R=r64, ldr=64, seed=2, drop_p=0.2)), M * (256 + 128) * F4)
report("rows N=64 K=64 DROP_RES", timeit(lambda: gemm(A=x64, lda=64, W=W[(64, 64)], sb_k=1, sb_n=64, bias=b[64], C=o64, ldc=64, M=M, N=64, Cin=64,
                                                   epi=ops.EPI_DROP_RES, alpha=1.0, R=r64, ldr=64, seed=2, drop_p=0.2)), M * (64 + 128) * F4)
report("rows N=256 K=64 PRO_LN", timeit(lambda: gemm(A=x64, lda=64, W=W[(256, 64)], sb_k=1, sb_n=64, bias=b[256], C=o256, ldc=256, M=M, N=256, Cin=64,
                                                  pro=ops.PRO_LN, p0=st, p1=g64, p2=be64)), M * (64 + 256) * F4)
# wgrads
dw = torch.zeros(256, 64, device=dev)
db = torch.zeros(256, device=dev)
report("wgrad N=256 K=64 (+dbias)", timeit(lambda: gemm(wgrad=True, W=None, C=dw, ldc=0, dbias=db, A=x64, lda=64, Cin=64, D=x256, ldd=256, N=256, sb_k=1,
                                                      sb_n=64, M=M)), M * (64 + 256) * F4)
report("wgrad N=256 K=64 (no dbias)", timeit(lambda: gemm(wgrad=True, W=None, C=dw, ldc=0, A=x64, lda=64, Cin=64, D=x256, ldd=256, N=256, sb_k=1,
                                                       sb_n=64, M=M)), M * (64 + 256) * F4)
dw2 = torch.zeros(64, 256, device=dev)
db2 = torch.zeros(64, device=dev)
report("wgrad N=64 K=256 (+dbias)", timeit(lambda: gemm(wgrad=True, W=None, C=dw2, ldc=0, dbias=db2, A=x256, lda=256, Cin=256, D=x64, ldd=64, N=64, sb_k=1,
                                                      sb_n=256, M=M)), M * (64 + 256) * F4)
dw3 = torch.zeros(64, 64, device=dev)
report("wgrad N=64 K=64 (+dbias)", timeit(lambda: gemm(wgrad=True, W=None, C=dw3, ldc=0, dbias=db2, A=x64, lda=64, Cin=64, D=r64, ldd=64, N=64, sb_k=1,
                                                     sb_n=64, M=M)), M * (64 + 64) * F4)
