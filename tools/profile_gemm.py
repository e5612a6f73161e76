"""ncu driver for the MLP GEMMs: one warm launch and one profiled launch of three PPO shapes for ONE kernel variant.
usage: python tools/profile_gemm.py {presplit|s|w}     (capture with: ncu -k regex:gemm_wgmma -s 3 -c 3 ...)
presplit: phc_gemm_tc5 (operands pre-split in global memory); s: 128 x 128 x 32 tiles; w: 128 x 256 x 16 tiles."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from phc_b200 import _lib

lib = _lib.load()
dev = "cuda:0"
variant = sys.argv[1] if len(sys.argv) > 1 else "s"
r4 = lambda x: (x + 3) & ~3
lib.phc_gemm_tc5s_set_tile(256 if variant == "w" else 128)


def split(x):
    hi, lo = torch.zeros_like(x), torch.zeros_like(x)
    _lib.check(lib.phc_split_tf32(x.data_ptr(), x.stride(0), x.shape[0], x.shape[1], hi.data_ptr(), lo.data_ptr(), x.stride(0), None))
    return hi, lo


def make(M, N, K, a_k, b_k, splits=1, mask=False, bias=False, relu=False):
    A = torch.randn((M, r4(K)) if a_k else (K, r4(M)), device=dev)
    B = torch.randn((N, r4(K)) if b_k else (K, r4(N)), device=dev)
    C = torch.zeros(M, r4(N), device=dev)
    Mk = torch.randn(M, r4(N), device=dev) if mask else None
    bs = torch.randn(N, device=dev) if bias else None
    acc = 1 if splits > 1 else 0
    if variant in ("s", "w"):
        return lambda: lib.phc_gemm_tc5s(A.data_ptr(), A.stride(0), int(a_k), B.data_ptr(), B.stride(0), int(b_k), C.data_ptr(), C.stride(0), M, N, K,
                                         1.0, None if bs is None else bs.data_ptr(), int(relu), None if Mk is None else Mk.data_ptr(),
                                         0 if Mk is None else Mk.stride(0), acc, splits, None), (A, B, C, Mk, bs)
    Ah, Al = split(A)
    Bh, Bl = split(B)
    Ch, Cl = (torch.zeros_like(C), torch.zeros_like(C)) if not acc else (None, None)
    return lambda: lib.phc_gemm_tc5(Ah.data_ptr(), Al.data_ptr(), A.stride(0), int(a_k), Bh.data_ptr(), Bl.data_ptr(), B.stride(0), int(b_k),
                                    C.data_ptr(), None if Ch is None else Ch.data_ptr(), None if Cl is None else Cl.data_ptr(), C.stride(0), M, N, K,
                                    1.0, None if bs is None else bs.data_ptr(), int(relu), None if Mk is None else Mk.data_ptr(),
                                    0 if Mk is None else Mk.stride(0), acc, splits, None), (Ah, Al, Bh, Bl, C, Ch, Cl, Mk, bs)


calls = [make(16384, 1024, 934, True, True, bias=True, relu=True),       # forward obs -> 1024
         make(16384, 1024, 512, True, False, mask=True),                 # dX 512 -> 1024 with the ReLU mask
         make(1024, 934, 16384, False, False, splits=9)]                 # dW 1024 x 934 over the batch
for _ in range(2):
    for fn, _keep in calls:
        _lib.check(fn())
    torch.cuda.synchronize()
print("done", variant)
