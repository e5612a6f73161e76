"""GPU parity of the grouped wgmma GEMM with the 3xTF32 split done in shared memory (phc_gemm_tc5s / phc_gemm_group,
gemm_wgmma.cu) in its three layer forms and both tile shapes (128 x 128 x 32, 128 x 256 x 16), against an
fp64 product with the fp32-equivalence criterion |err| <= tol * |A||B|^T."""
import ctypes as C
import math

import pytest
import torch

from phc_b200 import _lib
from phc_b200.learning.networks import round4
from tests.test_gpu_learner import gemm_close, padded

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


@pytest.fixture(params=[(1, 256), (1, 128), (2, 128)], ids=["wide128x256x16", "cta128x128x32", "pair256x128x32"], autouse=True)
def ctas(request):
    """The tile configurations phc_gemm_group accepts: 128 x 256 x 16 and 128 x 128 x 32 tiles; a request for two CTAs per tile is
    accepted and runs the one-CTA 128 x 128 tiles."""
    lib = _lib.load()
    n, tile = request.param
    _lib.check(lib.phc_gemm_tc5s_set_ctas(n))
    _lib.check(lib.phc_gemm_tc5s_set_tile(tile))
    yield n
    lib.phc_gemm_tc5s_set_ctas(0)
    lib.phc_gemm_tc5s_set_tile(0)


def tc5s(A, a_k, B, b_k, Cm, M, N, K, alpha=1.0, bias=None, act=0, aux=None, accumulate=False, k_splits=1):
    lib = _lib.load()
    rc = lib.phc_gemm_tc5s(A.data_ptr(), A.stride(0), int(a_k), B.data_ptr(), B.stride(0), int(b_k), Cm.data_ptr(), Cm.stride(0), M, N, K,
                           alpha, None if bias is None else bias.data_ptr(), int(act), None if aux is None else aux.data_ptr(),
                           0 if aux is None else aux.stride(0), int(accumulate), k_splits, None)
    _lib.check(rc, "phc_gemm_tc5s")
    torch.cuda.synchronize()


@pytest.mark.parametrize("M,N,K", [(128, 128, 32), (128, 128, 256), (300, 70, 934), (4096, 1024, 936), (130, 1, 512), (257, 69, 512),
                                   (260, 200, 100), (256, 256, 32), (1000, 520, 2048), (5, 3, 7)])
def test_forward_form(M, N, K):
    g = torch.Generator().manual_seed(M + N + K)
    A, B, bias = torch.randn(M, K, generator=g), torch.randn(N, K, generator=g) / math.sqrt(K), torch.randn(N, generator=g)
    Cm = torch.zeros(M, round4(N), device=DEV)
    tc5s(padded(A), True, padded(B), True, Cm, M, N, K, bias=bias.to(DEV), act=_lib.PHC_ACT_RELU)
    gemm_close(Cm[:, :N], A, B, "tc5s fwd", extra=lambda e, b: (torch.relu(e + bias.double()), b + bias.double().abs()))
    assert float(Cm[:, N:].abs().sum()) == 0.0


@pytest.mark.parametrize("M,N,K", [(256, 936, 1024), (100, 72, 69), (64, 1960, 40)])
def test_input_grad_form(M, N, K):
    g = torch.Generator().manual_seed(1)
    dY, W, H = torch.randn(M, K, generator=g), torch.randn(K, N, generator=g) / math.sqrt(K), torch.randn(M, N, generator=g)
    Cm = torch.zeros(M, round4(N), device=DEV)
    tc5s(padded(dY), True, padded(W), False, Cm, M, N, K, aux=padded(H))
    gemm_close(Cm[:, :N], dY, W.T.contiguous(), "tc5s dX", extra=lambda e, b: (e * (H > 0), b))


@pytest.mark.parametrize("M,N,K,splits", [(1024, 934, 4096, 4), (69, 512, 2048, 16), (1, 512, 1000, 1), (33, 17, 515, 2), (512, 1024, 16384, 9)])
def test_weight_grad_form(M, N, K, splits):
    g = torch.Generator().manual_seed(2)
    dY, X = torch.randn(K, M, generator=g), torch.randn(K, N, generator=g)
    Cm = torch.ones(M, round4(N), device=DEV)
    tc5s(padded(dY), False, padded(X), False, Cm, M, N, K, alpha=0.5, accumulate=True, k_splits=splits)
    gemm_close(Cm[:, :N], dY.T.contiguous(), X.T.contiguous(), "tc5s dW", extra=lambda e, b: (1.0 + 0.5 * e, 1.0 + 0.5 * b))
    assert float((Cm[:, N:] - 1.0).abs().sum()) == 0.0


def test_silu_forward_writes_preactivation_and_backward_uses_it():
    g = torch.Generator().manual_seed(5)
    M, N, K = 300, 200, 260
    A, B, bias = torch.randn(M, K, generator=g), torch.randn(N, K, generator=g) / math.sqrt(K), torch.randn(N, generator=g)
    Cm, Z = torch.zeros(M, round4(N), device=DEV), torch.zeros(M, round4(N), device=DEV)
    tc5s(padded(A), True, padded(B), True, Cm, M, N, K, bias=bias.to(DEV), act=_lib.PHC_ACT_SILU, aux=Z)
    z = A.double() @ B.double().T + bias.double()
    assert torch.allclose(Z[:, :N].double().cpu(), z, rtol=2e-5, atol=2e-5)
    assert torch.allclose(Cm[:, :N].double().cpu(), z * torch.sigmoid(z), rtol=2e-5, atol=2e-5)
    dY, W = torch.randn(M, K, generator=g), torch.randn(K, N, generator=g) / math.sqrt(K)
    D = torch.zeros(M, round4(N), device=DEV)
    tc5s(padded(dY), True, padded(W), False, D, M, N, K, act=_lib.PHC_ACT_SILU_BWD, aux=Z)
    zz = Z[:, :N].double().cpu()
    sg = torch.sigmoid(zz)
    exp = (dY.double() @ W.double()) * (sg * (1 + zz * (1 - sg)))
    assert torch.allclose(D[:, :N].double().cpu(), exp, rtol=3e-5, atol=3e-5)


def test_group_of_heterogeneous_problems_equals_single_launches():
    """One launch over three forward problems (different M, N, K), one dX and one split-K dW: the same results as five launches."""
    lib = _lib.load()
    g = torch.Generator().manual_seed(11)
    probs, keep, singles = [], [], []

    def add(A, a_k, B, b_k, M, N, K, bias=None, act=0, aux=None, acc=False, ks=1, init=0.0):
        Cg = torch.full((M, round4(N)), init, device=DEV)
        Cs = torch.full((M, round4(N)), init, device=DEV)
        keep.extend([A, B, bias, aux, Cg, Cs])
        d = _lib.PhcGemmDesc(A.data_ptr(), A.stride(0), int(a_k), B.data_ptr(), B.stride(0), int(b_k), Cg.data_ptr(), Cg.stride(0), M, N, K, 1.0,
                             None if bias is None else bias.data_ptr(), act, None if aux is None else aux.data_ptr(),
                             0 if aux is None else aux.stride(0), int(acc), ks)
        probs.append(d)
        singles.append((A, a_k, B, b_k, Cs, M, N, K, bias, act, aux, acc, ks, Cg))

    r = lambda *s: torch.randn(*s, generator=g)
    add(padded(r(700, 934)), True, padded(r(1024, 934) / 30), True, 700, 1024, 934, bias=r(1024).to(DEV), act=_lib.PHC_ACT_RELU)
    add(padded(r(700, 934)), True, padded(r(512, 934) / 30), True, 700, 512, 934, bias=r(512).to(DEV), act=_lib.PHC_ACT_RELU)
    add(padded(r(384, 1960)), True, padded(r(1024, 1960) / 44), True, 384, 1024, 1960, bias=r(1024).to(DEV))
    add(padded(r(700, 512)), True, padded(r(512, 1024) / 22), False, 700, 1024, 512, aux=padded(r(700, 1024)))
    add(padded(r(2048, 69)), False, padded(r(2048, 512)), False, 69, 512, 2048, acc=True, ks=4, init=1.0)
    arr = (_lib.PhcGemmDesc * len(probs))(*probs)
    _lib.check(lib.phc_gemm_group(arr, len(probs), None), "phc_gemm_group")
    torch.cuda.synchronize()
    for (A, a_k, B, b_k, Cs, M, N, K, bias, act, aux, acc, ks, Cg) in singles:
        tc5s(A, a_k, B, b_k, Cs, M, N, K, bias=bias, act=act, aux=aux, accumulate=acc, k_splits=ks)
        if acc:      # split-K partial sums arrive in a different order: equal up to fp32 re-association
            assert torch.allclose(Cg, Cs, rtol=1e-5, atol=1e-4)
        else:
            assert torch.equal(Cg, Cs)


def test_ppo_shapes_against_fp64_on_device():
    """The bench shapes (batch 16384): forward obs -> 1024 with bias + ReLU, and the weight gradient 1024 x 934 over the batch."""
    g = torch.Generator(device=DEV).manual_seed(3)
    M, N, K = 16384, 1024, 934
    A = torch.zeros(M, round4(K), device=DEV)
    A[:, :K] = torch.randn(M, K, device=DEV, generator=g)
    B = torch.zeros(N, round4(K), device=DEV)
    B[:, :K] = torch.randn(N, K, device=DEV, generator=g) / math.sqrt(K)
    bias = torch.randn(N, device=DEV, generator=g)
    Cm = torch.zeros(M, N, device=DEV)
    tc5s(A, True, B, True, Cm, M, N, K, bias=bias, act=_lib.PHC_ACT_RELU)
    exp = torch.relu(A[:, :K].double() @ B[:, :K].double().T + bias.double())
    bound = A[:, :K].double().abs() @ B[:, :K].double().abs().T + bias.double().abs()
    ratio = float(((Cm.double() - exp).abs() / bound).max())
    assert ratio < 4e-6, ratio
    dY = torch.randn(M, N, device=DEV, generator=g)
    G = torch.zeros(N, round4(K), device=DEV)
    tc5s(dY, False, A, False, G, N, K, M, accumulate=True, k_splits=9)
    exp = dY.double().T @ A[:, :K].double()
    bound = dY.double().abs().T @ A[:, :K].double().abs()
    ratio = float(((G[:, :K].double() - exp).abs() / bound).max())
    assert ratio < 4e-6, ratio


def test_relu_sign_bits_forward_and_masked_backward():
    """PHC_ACT_RELU_BITS writes one bit per element (x > 0); PHC_ACT_MASK_BITS applies it: the same results as the fp32-mask path."""
    g = torch.Generator().manual_seed(7)
    M, N, K = 333, 200, 96
    A, B, bias = torch.randn(M, K, generator=g), torch.randn(N, K, generator=g) / math.sqrt(K), torch.randn(N, generator=g)
    W = (N + 31) // 32
    H, Hb = torch.zeros(M, round4(N), device=DEV), torch.zeros(M, round4(N), device=DEV)
    bits = torch.zeros(M, W + 1, dtype=torch.int32, device=DEV)           # one spare word per row: ldaux > ceil(N / 32)
    tc5s(padded(A), True, padded(B), True, H, M, N, K, bias=bias.to(DEV), act=_lib.PHC_ACT_RELU)
    tc5s(padded(A), True, padded(B), True, Hb, M, N, K, bias=bias.to(DEV), act=_lib.PHC_ACT_RELU_BITS, aux=bits)
    assert torch.equal(H, Hb)
    cols = torch.arange(N, device=DEV)
    got = (bits[:, cols // 32] >> (cols % 32)) & 1
    assert torch.equal(got.bool(), H[:, :N] > 0)
    assert int(bits[:, W].abs().sum()) == 0
    if N % 32:      # bits beyond column N stay clear
        assert int(((bits[:, W - 1].long() & 0xFFFFFFFF) >> (N % 32)).sum()) == 0
    dY, Wt = torch.randn(M, K, generator=g), torch.randn(K, N, generator=g) / math.sqrt(K)
    D1, D2 = torch.zeros(M, round4(N), device=DEV), torch.zeros(M, round4(N), device=DEV)
    tc5s(padded(dY), True, padded(Wt), False, D1, M, N, K, aux=H)                                  # fp32 mask (aux > 0)
    tc5s(padded(dY), True, padded(Wt), False, D2, M, N, K, act=_lib.PHC_ACT_MASK_BITS, aux=bits)   # bit mask
    assert torch.equal(D1, D2)


def test_single_pass_tf32_mode_has_its_own_tolerance_and_switches_back():
    """PHC_GEMM_TF32_SINGLE_PASS (opt-in, BASELINE configs[3]): one tensor-core product per fp32 product -- operands truncated to tf32,
    fp32 accumulation: |err| <= 2.5e-3 |A||B|^T (two truncations of 2^-10 each), all three layer forms; switching back restores the
    fp32-equivalent results bit for bit."""
    lib = _lib.load()
    g = torch.Generator().manual_seed(13)
    M, N, K = 700, 300, 934
    A, B, bias = torch.randn(M, K, generator=g), torch.randn(N, K, generator=g) / math.sqrt(K), torch.randn(N, generator=g)
    C3, C1, C3b = (torch.zeros(M, round4(N), device=DEV) for _ in range(3))
    tc5s(padded(A), True, padded(B), True, C3, M, N, K, bias=bias.to(DEV))
    _lib.check(lib.phc_gemm_set_precision(_lib.PHC_GEMM_TF32_SINGLE_PASS))
    try:
        tc5s(padded(A), True, padded(B), True, C1, M, N, K, bias=bias.to(DEV))
        r_fwd = gemm_close(C1[:, :N], A, B, "tf32 single pass fwd", extra=lambda e, b: (e + bias.double(), b + bias.double().abs()), tol=2.5e-3)
        dY, W = torch.randn(M, K, generator=g), torch.randn(K, N, generator=g) / math.sqrt(K)
        D = torch.zeros(M, round4(N), device=DEV)
        tc5s(padded(dY), True, padded(W), False, D, M, N, K)
        gemm_close(D[:, :N], dY, W.T.contiguous(), "tf32 single pass dX", tol=2.5e-3)
        dYt, X = torch.randn(2048, 69, generator=g), torch.randn(2048, 512, generator=g)
        G = torch.zeros(69, 512, device=DEV)
        tc5s(padded(dYt), False, padded(X), False, G, 69, 512, 2048, accumulate=True, k_splits=4)
        gemm_close(G, dYt.T.contiguous(), X.T.contiguous(), "tf32 single pass dW", tol=2.5e-3)
        assert r_fwd > 2e-5, "the single-pass mode must really skip the correction products"
    finally:
        _lib.check(lib.phc_gemm_set_precision(_lib.PHC_GEMM_FP32_3XTF32))
    tc5s(padded(A), True, padded(B), True, C3b, M, N, K, bias=bias.to(DEV))
    assert torch.equal(C3, C3b)


def _group(descs):
    lib = _lib.load()
    arr = (_lib.PhcGemmDesc * len(descs))(*descs)
    _lib.check(lib.phc_gemm_group(arr, len(descs), None), "phc_gemm_group")
    torch.cuda.synchronize()


def _desc(A, a_k, B, b_k, Cm, M, N, K, bias=None, act=0, aux=None, b_lo=None):
    return _lib.PhcGemmDesc(A.data_ptr(), A.stride(0), int(a_k), B.data_ptr(), B.stride(0), int(b_k), Cm.data_ptr(), Cm.stride(0), M, N, K, 1.0,
                            None if bias is None else bias.data_ptr(), act, None if aux is None else aux.data_ptr(),
                            0 if aux is None else aux.stride(0), 0, 1, None if b_lo is None else b_lo.data_ptr())


def test_presplit_weight_operand_is_bit_identical_to_the_in_kernel_split():
    """phc_split_lo computes exactly the low TF32 term the kernel makes from each staged tile (restated on the host), and a launch
    that is handed a pre-split PhcGemmDesc.B_lo (accepted, not read) gives bit-identical products -- K-major B (forward), MN-major B
    (input gradient), ragged edges, and one grouped launch that mixes problems with and without B_lo."""
    lib = _lib.load()
    g = torch.Generator().manual_seed(11)
    cases = []
    for (M, N, K, b_k) in [(300, 200, 934, True), (256, 936, 1024, False), (4096, 512, 1024, True), (130, 69, 100, False), (5, 3, 7, True)]:
        A = padded(torch.randn(M, K, generator=g))
        B = padded(torch.randn(N, K, generator=g) if b_k else torch.randn(K, N, generator=g))
        # lo over the whole padded allocation, like the parameter bucket
        flatB = B._base if B._base is not None else B
        lo_full = torch.empty_like(flatB)
        _lib.check(lib.phc_split_lo(flatB.data_ptr(), lo_full.data_ptr(), flatB.numel(), None), "phc_split_lo")
        lo = lo_full[:, :B.shape[1]] if lo_full.dim() == 2 else lo_full
        assert lo.stride(0) == B.stride(0)
        # phc_split_lo restated on the host: lo = rna_tf32(x - trunc_tf32(x))
        xb = flatB.cpu().view(torch.int32)
        hi = (xb & -8192).view(torch.float32)
        d = (flatB.cpu() - hi).view(torch.int32)
        ref = ((d + 0x1000) & -8192).view(torch.float32)
        assert torch.equal(lo_full.cpu(), ref)
        C0, C1 = torch.zeros(M, round4(N), device=DEV), torch.zeros(M, round4(N), device=DEV)
        cases.append((A, B, lo, C0, C1, M, N, K, b_k))
    for A, B, lo, C0, C1, M, N, K, b_k in cases:
        _group([_desc(A, True, B, b_k, C0, M, N, K)])
        _group([_desc(A, True, B, b_k, C1, M, N, K, b_lo=lo)])
        assert torch.equal(C0, C1), (M, N, K, b_k)
    # mixed group: problems 0, 2, 4 pre-split, 1 and 3 not
    for c in cases:
        c[4].zero_()
    _group([_desc(A, True, B, b_k, C1, M, N, K, b_lo=lo if i % 2 == 0 else None) for i, (A, B, lo, C0, C1, M, N, K, b_k) in enumerate(cases)])
    for A, B, lo, C0, C1, M, N, K, b_k in cases:
        assert torch.equal(C0, C1), ("group", M, N, K, b_k)


def test_dynamic_and_static_tile_order_give_the_same_products(ctas):
    """phc_gemm_tc5s_set_sched: tiles drawn from the global counter (default) vs static striding.  A tile's arithmetic does not depend
    on which CTA computes it, so plain stores are bit-identical; many more tiles than CTAs, tiles of very different length in one
    group, and repeated launches (the counters must be back at zero after every launch)."""
    lib = _lib.load()
    g = torch.Generator().manual_seed(21)
    probs = []
    for (M, N, K) in [(4096, 1024, 934), (3000, 512, 1960), (128, 69, 512), (700, 1, 64)]:
        A, B = padded(torch.randn(M, K, generator=g)), padded(torch.randn(N, K, generator=g))
        probs.append((A, B, M, N, K, torch.zeros(M, round4(N), device=DEV), torch.zeros(M, round4(N), device=DEV)))
    try:
        _lib.check(lib.phc_gemm_tc5s_set_sched(0))
        _group([_desc(A, True, B, True, C0, M, N, K) for A, B, M, N, K, C0, C1 in probs])
        _lib.check(lib.phc_gemm_tc5s_set_sched(1))
        for _ in range(70):                                     # more launches than counter slots
            _group([_desc(A, True, B, True, C1, M, N, K) for A, B, M, N, K, C0, C1 in probs])
        for A, B, M, N, K, C0, C1 in probs:
            assert torch.equal(C0, C1), (M, N, K)
    finally:
        lib.phc_gemm_tc5s_set_sched(-1)
