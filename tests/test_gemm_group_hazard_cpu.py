"""phc_gemm_group refuses write hazards between the problems of one launch (gemm_wgmma.cu, validate_group).  Two problems may only
write overlapping C spans [C, C + (M-1)*ldc + N) when both accumulate into the same C with the same M, N and ldc: they then add in a
fixed order.  A plain store next to any other writer, or accumulating problems whose spans overlap without being identical, would
race.  The check runs before any CUDA call, so host buffers stand in for device memory here."""
import pytest
import torch

from phc_b200 import _lib

PHC_ERR_INVALID_ARG = -1
LD = 64


@pytest.fixture(scope="module")
def lib():
    from phc_b200 import build
    build.build()
    return _lib.load()


@pytest.fixture(scope="module")
def buf():
    t = torch.zeros(4096, LD)                        # 64-byte aligned host allocation: every row start is 16-byte aligned
    assert t.data_ptr() % 16 == 0
    return t


def desc(buf, row, col=0, M=64, N=32, ld=LD, acc=False, ks=1, K=64):
    c = buf.data_ptr() + (row * LD + col) * 4
    return _lib.PhcGemmDesc(buf.data_ptr(), LD, 1, buf.data_ptr(), LD, 1, c, ld, M, N, K, 1.0, None, 0, None, 0, int(acc), ks, None)


def run(lib, descs):
    arr = (_lib.PhcGemmDesc * len(descs))(*descs)
    return lib.phc_gemm_group(arr, len(descs), None)


def rejected(lib, descs):
    rc = run(lib, descs)
    assert rc == PHC_ERR_INVALID_ARG, rc
    msg = lib.phc_last_error().decode()
    assert "overlap" in msg, msg


def test_plain_store_next_to_any_writer_on_the_same_C_is_refused(lib, buf):
    rejected(lib, [desc(buf, 0), desc(buf, 0)])
    rejected(lib, [desc(buf, 0, acc=True), desc(buf, 0)])
    rejected(lib, [desc(buf, 0), desc(buf, 0, acc=True, ks=4)])
    rejected(lib, [desc(buf, 0, acc=True, ks=2), desc(buf, 1000), desc(buf, 0)])      # unrelated problem in between


def test_partially_overlapping_spans_are_refused(lib, buf):
    rejected(lib, [desc(buf, 0), desc(buf, 63)])                                        # last row of one, first row of the other
    rejected(lib, [desc(buf, 0, acc=True), desc(buf, 10, acc=True)])                    # accumulating, different C: unordered atomics
    rejected(lib, [desc(buf, 0, acc=True, ks=3), desc(buf, 0, col=4, acc=True, ks=3)])
    rejected(lib, [desc(buf, 63, col=28, M=1, N=1), desc(buf, 0)])                      # inside the last row of the span
    rejected(lib, [desc(buf, 0), desc(buf, 200), desc(buf, 100, M=101)])                # its last row is the first row of problem 1


def test_span_uses_the_leading_dimension_not_the_buffer(lib, buf):
    # a narrower ldc packs the rows: 64 rows of ldc 32 end at row 32 of the LD-64 buffer
    rejected(lib, [desc(buf, 0, N=32, ld=32), desc(buf, 31, col=32, M=1, N=4)])
    # a wider ldc spreads them: 10 rows of ldc 256 reach row 36 of the buffer
    rejected(lib, [desc(buf, 36, M=1, N=4), desc(buf, 0, M=10, N=32, ld=256)])


def test_same_C_accumulation_needs_the_same_shape(lib, buf):
    rejected(lib, [desc(buf, 0, acc=True, ks=2), desc(buf, 0, M=32, acc=True)])
    rejected(lib, [desc(buf, 0, acc=True, ks=2), desc(buf, 0, N=16, acc=True, ks=2)])
    rejected(lib, [desc(buf, 0, acc=True), desc(buf, 0, ld=128, acc=True)])


def test_empty_problems_take_no_part(lib, buf):
    # M == 0 / N == 0 problems are skipped before the hazard check; a launch of nothing but empty problems launches nothing
    assert run(lib, [desc(buf, 0, M=0), desc(buf, 0, N=0), desc(buf, 0, M=0, acc=True)]) == 0
    rejected(lib, [desc(buf, 0, M=0), desc(buf, 0, acc=True), desc(buf, 5)])
