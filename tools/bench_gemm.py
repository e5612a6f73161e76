"""Microbenchmark of the MLP GEMM variants on the PPO shapes (diagnostic, not bench values): phc_gemm_tc5 (pre-split operands),
phc_gemm (mma.sync), phc_gemm_tc5s with 128 x 128 x 32 (s128) and 128 x 256 x 16 (w256) tiles.
usage: python tools/bench_gemm.py [iters]   -- prints per shape/variant: us, TFLOP/s of tensor work (3 MMAs per product)."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from phc_b200 import _lib

lib = _lib.load()
dev = "cuda:0"
iters = int(sys.argv[1]) if len(sys.argv) > 1 else 20
only = sys.argv[2] if len(sys.argv) > 2 else None


def r4(x):
    return (x + 3) & ~3


def split(x):
    hi, lo = torch.zeros_like(x), torch.zeros_like(x)
    _lib.check(lib.phc_split_tf32(x.data_ptr(), x.stride(0), x.shape[0], x.shape[1], hi.data_ptr(), lo.data_ptr(), x.stride(0), None))
    return hi, lo


def run(name, M, N, K, a_k, b_k, splits=1, mask=False, split_out=False):
    # operand storage: k-major operand is [rows, K]; mn-major is [K, rows]
    A = torch.randn((M, r4(K)) if a_k else (K, r4(M)), device=dev)
    B = torch.randn((N, r4(K)) if b_k else (K, r4(N)), device=dev)
    C = torch.zeros(M, r4(N), device=dev)
    Ch, Cl = (torch.zeros_like(C), torch.zeros_like(C)) if split_out else (None, None)
    Mk = torch.randn(M, r4(N), device=dev) if mask else None
    Ah, Al = split(A)
    Bh, Bl = split(B)
    acc = 1 if splits > 1 else 0
    variants = [("presplit", "tc5"), ("mma.sync", None), ("s128", 128), ("w256", 256)]
    out = []
    for vname, env in variants:
        if only and vname not in only.split(","):
            continue
        if isinstance(env, int):
            lib.phc_gemm_tc5s_set_tile(env)

        def call():
            if isinstance(env, int):      # split in shared memory (gemm_wgmma.cu): raw operands
                return lib.phc_gemm_tc5s(A.data_ptr(), A.stride(0), int(a_k), B.data_ptr(), B.stride(0), int(b_k), C.data_ptr(), C.stride(0),
                                         M, N, K, 1.0, None, 0, None if Mk is None else Mk.data_ptr(), 0 if Mk is None else Mk.stride(0), acc, splits, None)
            if env is None:
                return lib.phc_gemm(A.data_ptr(), A.stride(0), int(a_k), B.data_ptr(), B.stride(0), int(b_k), C.data_ptr(), C.stride(0),
                                    M, N, K, 1.0, None, 0, None if Mk is None else Mk.data_ptr(), 0 if Mk is None else Mk.stride(0), acc, splits, None)
            return lib.phc_gemm_tc5(Ah.data_ptr(), Al.data_ptr(), A.stride(0), int(a_k), Bh.data_ptr(), Bl.data_ptr(), B.stride(0), int(b_k),
                                    C.data_ptr(), None if Ch is None else Ch.data_ptr(), None if Cl is None else Cl.data_ptr(), C.stride(0),
                                    M, N, K, 1.0, None, 0, None if Mk is None else Mk.data_ptr(), 0 if Mk is None else Mk.stride(0), acc, splits, None)
        for _ in range(3):
            _lib.check(call())
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(iters):
            call()
        e1.record()
        torch.cuda.synchronize()
        us = e0.elapsed_time(e1) * 1e3 / iters
        out.append(f"{vname}: {us:8.1f} us {3 * 2.0 * M * N * K / us * 1e-6:7.1f} TF/s")
    print(f"{name:34s} M={M:6d} N={N:5d} K={K:6d} s={splits:2d} | " + " | ".join(out), flush=True)


run("fwd  obs->1024 (B=16384)", 16384, 1024, 934, True, True, split_out=True)
run("fwd  1024->512 (B=16384)", 16384, 512, 1024, True, True, split_out=True)
run("fwd  amp->1024 (B=12288)", 12288, 1024, 1960, True, True, split_out=True)
run("dX   512->1024 (B=16384) +mask", 16384, 1024, 512, True, False, mask=True, split_out=True)
run("dW   1024x934  (K=16384) s=5", 1024, 934, 16384, False, False, splits=5)
run("dW   1024x934  (K=16384) s=9", 1024, 934, 16384, False, False, splits=9)
run("dW   512x1024  (K=16384) s=10", 512, 1024, 16384, False, False, splits=10)
run("dW   512x1024  (K=16384) s=18", 512, 1024, 16384, False, False, splits=18)
run("fwd  rollout obs->1024 (B=4096)", 4096, 1024, 934, True, True, split_out=True)
run("fwd  big square 8192^3/8", 8192, 8192, 1024, True, True)
