"""GPU parity of the wgmma GEMM with pre-split operands (phc_gemm_tc5, 3xTF32 with pre-split operands) in its three layer forms,
against an fp64 product with the fp32-equivalence criterion |err| <= tol * |A||B|^T."""
import math

import pytest
import torch

from phc_b200 import _lib
from phc_b200.learning.networks import round4
from tests.test_gpu_learner import gemm_close, padded

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


@pytest.fixture(params=["persistent", "one_tile_per_cta", "cta_pair", "cta_pair_persistent"], autouse=True)
def tc5_mode(request, monkeypatch):
    """The launch-variant environment variables of earlier builds: the kernel no longer reads them, and setting them must not
    change a result."""
    monkeypatch.delenv("PHC_TC5_PERSIST", raising=False)
    monkeypatch.delenv("PHC_TC5_PAIR", raising=False)
    monkeypatch.delenv("PHC_TC5_PAIRP", raising=False)
    if request.param == "one_tile_per_cta":
        monkeypatch.setenv("PHC_TC5_PERSIST", "0")
    elif request.param == "cta_pair":
        monkeypatch.setenv("PHC_TC5_PAIR", "1")
    elif request.param == "cta_pair_persistent":
        monkeypatch.setenv("PHC_TC5_PAIRP", "1")
    return request.param


def split(x):
    lib = _lib.load()
    hi, lo = torch.zeros_like(x), torch.zeros_like(x)
    _lib.check(lib.phc_split_tf32(x.data_ptr(), x.stride(0), x.shape[0], x.shape[1], hi.data_ptr(), lo.data_ptr(), x.stride(0), None))
    return hi, lo


def tc5(A, a_k, B, b_k, C, M, N, K, alpha=1.0, bias=None, relu=False, mask=None, accumulate=False, k_splits=1):
    lib = _lib.load()
    Ah, Al = split(A)
    Bh, Bl = split(B)
    rc = lib.phc_gemm_tc5(Ah.data_ptr(), Al.data_ptr(), A.stride(0), int(a_k), Bh.data_ptr(), Bl.data_ptr(), B.stride(0), int(b_k),
                          C.data_ptr(), None, None, C.stride(0), M, N, K, alpha, None if bias is None else bias.data_ptr(), int(relu),
                          None if mask is None else mask.data_ptr(), 0 if mask is None else mask.stride(0), int(accumulate), k_splits, None)
    _lib.check(rc, "phc_gemm_tc5")
    torch.cuda.synchronize()


def test_split_is_exact_to_2_pow_minus_21():
    x = torch.randn(300, 936, device=DEV) * 7
    hi, lo = split(x)
    assert float(((hi + lo) - x).abs().max() / x.abs().max()) < 2 ** -20
    assert int((hi.view(torch.int32) & 0x1FFF).abs().sum()) == 0 and int((lo.view(torch.int32) & 0x1FFF).abs().sum()) == 0


@pytest.mark.parametrize("M,N,K", [(128, 128, 32), (128, 128, 256), (300, 70, 934), (4096, 1024, 936), (130, 1, 512), (257, 69, 512),
                                   (260, 200, 100), (256, 256, 32), (1000, 520, 2048)])      # the last rows use CTA-pair tiles
def test_tc5_forward_form(M, N, K):
    g = torch.Generator().manual_seed(M + N + K)
    A, B, bias = torch.randn(M, K, generator=g), torch.randn(N, K, generator=g) / math.sqrt(K), torch.randn(N, generator=g)
    C = torch.zeros(M, round4(N), device=DEV)
    tc5(padded(A), True, padded(B), True, C, M, N, K, bias=bias.to(DEV), relu=True)
    gemm_close(C[:, :N], A, B, "tc5 fwd", extra=lambda e, b: (torch.relu(e + bias.double()), b + bias.double().abs()))
    assert float(C[:, N:].abs().sum()) == 0.0


@pytest.mark.parametrize("M,N,K", [(256, 936, 1024), (100, 72, 69), (64, 1960, 40)])
def test_tc5_input_grad_form(M, N, K):
    g = torch.Generator().manual_seed(1)
    dY, W, H = torch.randn(M, K, generator=g), torch.randn(K, N, generator=g) / math.sqrt(K), torch.randn(M, N, generator=g)
    C = torch.zeros(M, round4(N), device=DEV)
    tc5(padded(dY), True, padded(W), False, C, M, N, K, mask=padded(H))
    gemm_close(C[:, :N], dY, W.T.contiguous(), "tc5 dX", extra=lambda e, b: (e * (H > 0), b))


@pytest.mark.parametrize("M,N,K,splits", [(1024, 934, 4096, 4), (69, 512, 2048, 16), (1, 512, 1000, 1), (33, 17, 515, 2)])
def test_tc5_weight_grad_form(M, N, K, splits):
    g = torch.Generator().manual_seed(2)
    dY, X = torch.randn(K, M, generator=g), torch.randn(K, N, generator=g)
    C = torch.ones(M, round4(N), device=DEV)
    tc5(padded(dY), False, padded(X), False, C, M, N, K, alpha=0.5, accumulate=True, k_splits=splits)
    gemm_close(C[:, :N], dY.T.contiguous(), X.T.contiguous(), "tc5 dW", extra=lambda e, b: (1.0 + 0.5 * e, 1.0 + 0.5 * b))
