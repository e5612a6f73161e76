"""Ordered accumulation of the wgmma GEMM (gemm_wgmma.cu), bit for bit.

Split-K slices of an output tile add into C in slice order through a per-tile turnstile, and problems of one launch that accumulate
into the same C continue that order (the owner's slices, then each member's slices in problem order).  So a split-K result is exactly
the fp32 sum C0 + P_0 + P_1 + ... of its slice partials, added left to right -- which the tests restate with one plain launch per
slice.  alpha is 1 or 0.5: alpha * acc is then exact, and FMA contraction of alpha * acc + C cannot change a bit.  An ordering bug
(slices added out of order, two slices racing, unordered atomics) changes results at the 1e-7 level, far below the fp64 tolerances
of test_gpu_gemm_tc5s.py, so everything here compares with torch.equal."""
import pytest
import torch

from phc_b200 import _lib
from phc_b200.learning.networks import group_splits, round4

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
TURN_SLOTS, SCHED_SLOTS = 16, 64          # gemm_wgmma.cu: turnstile slots and scheduler counter pairs that launches rotate through


@pytest.fixture(params=[128, 256], ids=["tile128x128x32", "tile128x256x16"])
def tile(request):
    lib = _lib.load()
    _lib.check(lib.phc_gemm_tc5s_set_tile(request.param))
    yield request.param
    lib.phc_gemm_tc5s_set_tile(0)


def slices(K, ks, tile):
    """[k0, k1) of every split-K slice, cut as add_problem cuts them: BK = 32 (tile width 128) or 16 (256) rows of K per k-block,
    ks clamped to the k-block count, kb_per = ceil(kb_total / ks) k-blocks per slice, no empty slice."""
    bk = 32 if tile == 128 else 16
    kb_total = -(-K // bk)
    ks = max(1, min(ks, kb_total))
    kb_per = -(-kb_total // ks)
    return [(z * kb_per * bk, min(K, (z + 1) * kb_per * bk)) for z in range(-(-kb_total // kb_per))]


def test_slice_restatement_matches_the_documented_cuts():
    assert [k1 - k0 for k0, k1 in slices(288, 4, 128)] == [96, 96, 96]              # 9 k-blocks, ks 4 -> 3 per slice -> 3 slices
    assert [k1 - k0 for k0, k1 in slices(320, 4, 128)] == [96, 96, 96, 32]          # 10 k-blocks -> 3, 3, 3, 1
    assert [k1 - k0 for k0, k1 in slices(515, 3, 128)] == [192, 192, 131]
    assert len(slices(100, 64, 128)) == 4 and len(slices(100, 64, 256)) == 7        # ks > k-blocks: one k-block per slice
    assert len(slices(16384, group_splits(16384), 128)) == 16


def rnd(g, *shape):
    return torch.randn(*shape, device=DEV, generator=g)


class Prob:
    """One problem in one operand form.  form "dw": A(m, k) = A[k, m], B(n, k) = B[k, n] (weight gradient, both mn-major);
    "fwd": A(m, k) = A[m, k], B(n, k) = B[n, k] (both k-major)."""

    def __init__(self, g, M, N, K, form, alpha=1.0, bias=False, ks=1, C=None):
        self.M, self.N, self.K, self.alpha, self.ks = M, N, K, alpha, ks
        self.a_k = self.b_k = form == "fwd"
        self.A = torch.zeros(M, round4(K), device=DEV) if self.a_k else torch.zeros(K, round4(M), device=DEV)
        self.B = torch.zeros(N, round4(K), device=DEV) if self.b_k else torch.zeros(K, round4(N), device=DEV)
        self.A[:, :K if self.a_k else M] = rnd(g, *((M, K) if self.a_k else (K, M)))
        self.B[:, :K if self.b_k else N] = rnd(g, *((N, K) if self.b_k else (K, N)))
        self.bias = rnd(g, N) if bias else None
        self.C = C if C is not None else torch.zeros(M, round4(N), device=DEV)

    def desc(self, C=None, acc=True, ks=None, k0=0, k1=None, bias=True, M=None):
        """this problem (default: accumulating into self.C with its k_splits), or the k-range [k0, k1) of it as its own problem"""
        k1 = self.K if k1 is None else k1
        a_off = k0 if self.a_k else k0 * self.A.stride(0)
        b_off = k0 if self.b_k else k0 * self.B.stride(0)
        C = self.C if C is None else C
        return _lib.PhcGemmDesc(self.A.data_ptr() + 4 * a_off, self.A.stride(0), int(self.a_k), self.B.data_ptr() + 4 * b_off, self.B.stride(0),
                                int(self.b_k), C.data_ptr(), C.stride(0), self.M if M is None else M, self.N, k1 - k0, self.alpha,
                                self.bias.data_ptr() if (bias and self.bias is not None) else None, 0, None, 0, int(acc),
                                self.ks if ks is None else ks, None)

    def partials(self, tile):
        """P_z of every slice: a plain-store launch over the slice's k-range (k0 is a multiple of BK, so the operands stay aligned),
        the bias with slice 0 only"""
        out = []
        for z, (k0, k1) in enumerate(slices(self.K, self.ks, tile)):
            P = torch.zeros(self.M, round4(self.N), device=DEV)
            group([self.desc(C=P, acc=False, ks=1, k0=k0, k1=k1, bias=z == 0)])
            out.append(P)
        return out


def group(descs, stream=None):
    lib = _lib.load()
    arr = (_lib.PhcGemmDesc * len(descs))(*descs)
    _lib.check(lib.phc_gemm_group(arr, len(descs), stream), "phc_gemm_group")


def in_order(C0, parts):
    exp = C0.clone()
    for P in parts:
        exp = exp + P                 # one fp32 add per element and slice, in slice order
    return exp


CASES = {                                                   # M, N, K, k_splits, form, alpha, bias
    "dw_ragged_K1000": (300, 200, 1000, 4, "dw", 1.0, False),
    "fwd_ragged_K515_bias": (256, 136, 515, 3, "fwd", 0.5, True),
    "dw_splits_beyond_kblocks": (130, 70, 100, 64, "dw", 0.5, False),
    "dw_K288_ks4_normalised": (128, 128, 288, 4, "dw", 1.0, False),
    "fwd_K320_ks4": (200, 260, 320, 4, "fwd", 1.0, False),                  # 128-wide tiles: slices of 3, 3, 3, 1 k-blocks
    "dw_bench_16384_rows": (1024, 934, 16384, group_splits(16384), "dw", 1.0, False),
    "single_writer_atomic": (300, 200, 1000, 1, "dw", 0.5, False),       # accumulate without split-K: the atomic path
}


@pytest.mark.parametrize("case", list(CASES))
def test_split_k_equals_the_in_order_sum_of_its_slices(case, tile):
    M, N, K, ks, form, alpha, bias = CASES[case]
    g = torch.Generator(device=DEV).manual_seed(M * 7 + K)
    p = Prob(g, M, N, K, form, alpha=alpha, bias=bias, ks=ks)
    C0 = rnd(g, M, round4(N))
    parts = p.partials(tile)
    p.C.copy_(C0)
    group([p.desc()])
    torch.cuda.synchronize()
    exp = in_order(C0, parts)
    assert torch.equal(p.C, exp), f"{case}: {len(parts)} slices, max |diff| {float((p.C - exp).abs().max()):.3e}"


def shared_c_group(g):
    """three problems accumulating into one C (k_splits 4, 1, 8; different K and forms), an unrelated plain-store problem between
    them, and an empty problem on the same C"""
    M, N = 256, 200
    C = torch.zeros(M, round4(N), device=DEV)
    a = Prob(g, M, N, 1000, "dw", ks=4, C=C)
    b = Prob(g, M, N, 515, "fwd", bias=True, ks=1, C=C)
    c = Prob(g, M, N, 2048, "dw", alpha=0.5, ks=8, C=C)
    x = Prob(g, 300, 100, 64, "fwd", bias=True)
    descs = [a.desc(), x.desc(acc=False), b.desc(), a.desc(M=0), c.desc()]
    return C, (a, b, c), x, descs


def test_problems_accumulating_into_one_C_add_in_problem_order(tile):
    g = torch.Generator(device=DEV).manual_seed(5)
    C, members, x, descs = shared_c_group(g)
    C0 = rnd(g, *C.shape)
    parts = [P for p in members for P in p.partials(tile)]
    x_alone = torch.zeros_like(x.C)
    group([x.desc(C=x_alone, acc=False)])
    C.copy_(C0)
    group(descs)
    torch.cuda.synchronize()
    assert len(parts) == len(slices(1000, 4, tile)) + 1 + len(slices(2048, 8, tile))
    assert torch.equal(C, in_order(C0, parts))
    assert torch.equal(x.C, x_alone)


def test_accumulating_into_one_C_with_another_shape_is_refused():
    lib = _lib.load()
    g = torch.Generator(device=DEV).manual_seed(6)
    C, (a, b, c), x, _ = shared_c_group(g)
    other_ldc = _lib.PhcGemmDesc(b.A.data_ptr(), b.A.stride(0), 1, b.B.data_ptr(), b.B.stride(0), 1, C.data_ptr(), 400, 128, 200, 515, 1.0,
                                 None, 0, None, 0, 1, 1, None)
    for bad in (b.desc(M=255), Prob(g, 256, 196, 64, "fwd", C=C).desc(), other_ldc):
        arr = (_lib.PhcGemmDesc * 2)(a.desc(), bad)
        assert lib.phc_gemm_group(arr, 2, None) == -1, "PHC_ERR_INVALID_ARG expected"


def repeat(launch, C, C0, times, first=None):
    """run launch() `times` times from C0; every result must equal the first"""
    ref = first
    for i in range(times):
        C.copy_(C0)
        launch()
        if ref is None:
            ref = C.clone()
        elif not torch.equal(C, ref):
            torch.cuda.synchronize()
            raise AssertionError(f"launch {i} differs from the first: max |diff| {float((C - ref).abs().max()):.3e}")
    torch.cuda.synchronize()
    return ref


def test_ordered_launches_repeat_bit_for_bit_across_slot_reuse(tile):
    """more launches than turnstile slots (twice over) and scheduler counters: every slot is reused after a launch that had
    to put it back to zero"""
    g = torch.Generator(device=DEV).manual_seed(7)
    p = Prob(g, 512, 520, 4096, "dw", ks=8)
    C0 = rnd(g, *p.C.shape)
    d = [p.desc()]
    repeat(lambda: group(d), p.C, C0, 2 * TURN_SLOTS + 3)
    C, members, x, descs = shared_c_group(g)
    C0 = rnd(g, *C.shape)
    repeat(lambda: group(descs), C, C0, SCHED_SLOTS + 6)


def test_ordered_result_does_not_depend_on_a_busy_gpu(tile):
    """the same ordered launch while a large matmul occupies most SMs from another stream: its tiles start in another order"""
    g = torch.Generator(device=DEV).manual_seed(8)
    C, members, x, descs = shared_c_group(g)
    C0 = rnd(g, *C.shape)
    ref = repeat(lambda: group(descs), C, C0, 1)
    X, Y = rnd(g, 8192, 8192), rnd(g, 8192, 8192)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    C.copy_(C0)
    torch.cuda.synchronize()
    with torch.cuda.stream(side):
        Z = X @ Y
    group(descs)
    torch.cuda.synchronize()
    assert torch.isfinite(Z[:4, :4]).all()
    assert torch.equal(C, ref)


def split_tf32(x):
    lib = _lib.load()
    hi, lo = torch.zeros_like(x), torch.zeros_like(x)
    _lib.check(lib.phc_split_tf32(x.data_ptr(), x.stride(0), x.shape[0], x.shape[1], hi.data_ptr(), lo.data_ptr(), x.stride(0), None))
    return hi, lo


def test_presplit_split_k_repeats_bit_for_bit():
    """phc_gemm_tc5 (operands pre-split in global memory) takes the same turnstile"""
    lib = _lib.load()
    g = torch.Generator(device=DEV).manual_seed(9)
    p = Prob(g, 384, 300, 3000, "dw", ks=6)
    (Ah, Al), (Bh, Bl) = split_tf32(p.A), split_tf32(p.B)
    C0 = rnd(g, *p.C.shape)

    def launch():
        _lib.check(lib.phc_gemm_tc5(Ah.data_ptr(), Al.data_ptr(), p.A.stride(0), 0, Bh.data_ptr(), Bl.data_ptr(), p.B.stride(0), 0,
                                    p.C.data_ptr(), None, None, p.C.stride(0), p.M, p.N, p.K, 1.0, None, 0, None, 0, 1, 6, None), "phc_gemm_tc5")
    repeat(launch, p.C, C0, 2 * TURN_SLOTS + 3)
