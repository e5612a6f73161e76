"""Output images written by the GEMM epilogue (PhcGemmDesc.C_img): the image of the stored output equals phc_gemm_make_images of
that output bit for bit, for every epilogue and ragged shapes; a problem reading its A from such an image (the pair loop) gives
the same output as the image loop and the staged loop; the refusals; and MLPEngine's forward and backward chains, which feed
every hidden layer's forward and input-gradient GEMM from the image its producer wrote, against the chains without them,
eagerly and graph-replayed."""
import ctypes as C

import pytest
import torch

from phc_b200 import _lib
from phc_b200.learning.networks import AMPNetwork, MLPEngine, round4
from phc_b200.ops import _stream

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
PHC_ERR_INVALID_ARG, PHC_ERR_UNSUPPORTED = -1, -2
ACTS = {"none": _lib.PHC_ACT_NONE, "relu": _lib.PHC_ACT_RELU, "relu_bits": _lib.PHC_ACT_RELU_BITS, "mask_bits": _lib.PHC_ACT_MASK_BITS,
        "silu": _lib.PHC_ACT_SILU, "silu_bwd": _lib.PHC_ACT_SILU_BWD, "relu_bwd_saved": _lib.PHC_ACT_NONE}


@pytest.fixture
def lib():
    lib = _lib.load()
    yield lib
    lib.phc_gemm_tc5s_set_tile(0)
    lib.phc_gemm_set_precision(_lib.PHC_GEMM_FP32_3XTF32)
    MLPEngine._mode_set = None


def make_image(lib, T, rows, K, kmajor):
    img = torch.full((lib.phc_gemm_image_floats(rows, K),), float("nan"), device=DEV)
    d = _lib.PhcGemmImageDesc(T.data_ptr(), T.stride(0), int(kmajor), rows, K, img.data_ptr())
    _lib.check(lib.phc_gemm_make_images(C.byref(d), 1, _stream()), "phc_gemm_make_images")
    return img


class Fwd:
    """C[M, N] = epi(A[M, K] W[N, K]^T + bias) with the epilogue `act`, k-major A as in a forward or input-gradient layer"""

    def __init__(self, lib, g, M, N, K, act):
        rnd = lambda r, c: torch.nn.functional.pad(torch.randn(r, c, device=DEV, generator=g), (0, round4(c) - c))  # noqa: E731
        self.M, self.N, self.K, self.act = M, N, K, ACTS[act]
        self.A, self.W, self.bias = rnd(M, K), rnd(N, K) / K ** 0.5, torch.randn(N, device=DEV, generator=g)
        self.C = torch.zeros(M, round4(N), device=DEV)
        words = (N + 31) // 32
        self.aux = None
        if act in ("relu_bits", "mask_bits"):
            self.aux = torch.randint(-2**31, 2**31 - 1, (M, words), device=DEV, generator=g, dtype=torch.int64).to(torch.int32)
        elif act in ("silu", "silu_bwd", "relu_bwd_saved"):
            self.aux = rnd(M, N)
        self.aux0 = None if self.aux is None else self.aux.clone()
        self.w_img = make_image(lib, self.W, N, K, True)
        self.a_img = make_image(lib, self.A, M, K, True)
        self.c_img = torch.full((lib.phc_gemm_image_floats(M, N),), float("nan"), device=DEV)

    def desc(self, loop, c_img=True):
        """loop: 'staged' (no images), 'image' (B from its image, A from registers), 'pair' (both from images)"""
        b_img = None if loop == "staged" else self.w_img.data_ptr()
        a_img = self.a_img.data_ptr() if loop == "pair" else None
        aux = self.aux
        return _lib.PhcGemmDesc(self.A.data_ptr(), self.A.stride(0), 1, self.W.data_ptr(), self.W.stride(0), 1, self.C.data_ptr(),
                                self.C.stride(0), self.M, self.N, self.K, 1.0, self.bias.data_ptr(), self.act, None if aux is None else aux.data_ptr(),
                                0 if aux is None else aux.stride(0), 0, 1, None, b_img, a_img, self.c_img.data_ptr() if c_img else None)

    def run(self, lib, loop, c_img=True):
        self.C.fill_(float("nan"))
        self.c_img.fill_(float("nan"))
        if self.aux is not None:
            self.aux.copy_(self.aux0)
        d = self.desc(loop, c_img)
        _lib.check(lib.phc_gemm_group(C.byref(d), 1, _stream()), "phc_gemm_group")
        torch.cuda.synchronize()
        return self.C[:, :self.N].clone(), None if self.aux is None else self.aux.clone()


@pytest.mark.parametrize("act", list(ACTS))
@pytest.mark.parametrize("M,N,K", [(1000, 69, 512), (12288, 1960, 1024), (130, 1, 69), (257, 200, 934)])
def test_epilogue_image_equals_make_images(lib, M, N, K, act):
    g = torch.Generator(device=DEV).manual_seed(M + N + K + ACTS[act])
    p = Fwd(lib, g, M, N, K, act)
    base, base_aux = p.run(lib, "image", c_img=False)
    assert torch.isfinite(base).all() and base.abs().sum() > 0
    for loop in ("staged", "image", "pair"):
        out, aux = p.run(lib, loop)
        assert torch.equal(out, base), loop                          # the same products in the same order, on every loop
        if aux is not None:
            assert torch.equal(aux, base_aux), loop
        ref = make_image(lib, p.C, M, N, True)
        assert torch.equal(p.c_img, ref), f"{loop}: the epilogue's image differs from phc_gemm_make_images of C"


def test_output_image_feeds_the_next_layer(lib):
    """Two layers in two launches: the second takes its A from the image the first one's epilogue wrote (pair loop) and equals
    the second layer run from the fp32 activation (image loop)."""
    g = torch.Generator(device=DEV).manual_seed(11)
    p = Fwd(lib, g, 3000, 1000, 934, "relu")
    q = Fwd(lib, g, 3000, 300, 1000, "relu")
    q.A = p.C                                                        # q reads p's output
    _lib.check(lib.phc_gemm_group(C.byref(p.desc("image")), 1, _stream()))
    q.a_img = p.c_img
    ref, _ = q.run(lib, "image", c_img=False)
    got, _ = q.run(lib, "pair", c_img=False)
    assert torch.equal(got, ref) and ref.abs().sum() > 0


def test_output_image_refusals(lib):
    g = torch.Generator(device=DEV).manual_seed(12)
    p = Fwd(lib, g, 256, 128, 64, "none")
    go = lambda d: lib.phc_gemm_group(C.byref(d), 1, _stream())  # noqa: E731
    d = p.desc("image")
    d.accumulate = 1
    assert go(d) == PHC_ERR_INVALID_ARG                              # accumulating
    d.k_splits = 2
    assert go(d) == PHC_ERR_INVALID_ARG                              # split-K (accumulating too)
    d = p.desc("image")
    d.C_img = d.C_img + 4
    assert go(d) == PHC_ERR_INVALID_ARG                              # not 16-byte aligned
    _lib.check(lib.phc_gemm_tc5s_set_tile(256))
    assert go(p.desc("image")) == PHC_ERR_UNSUPPORTED                # 128 x 256 tiles
    assert go(p.desc("image", c_img=False)) == 0
    _lib.check(lib.phc_gemm_tc5s_set_tile(0))
    _lib.check(lib.phc_gemm_set_precision(_lib.PHC_GEMM_TF32_SINGLE_PASS))
    assert go(p.desc("image")) == PHC_ERR_UNSUPPORTED                # single-pass TF32
    _lib.check(lib.phc_gemm_set_precision(_lib.PHC_GEMM_FP32_3XTF32))
    assert go(p.desc("image")) == 0
    torch.cuda.synchronize()


@pytest.mark.parametrize("activation", ["relu", "silu"])
def test_engine_chains_with_and_without_images(lib, monkeypatch, activation):
    """Forward and backward of three-hidden-layer stacks through MLPEngine (every hidden layer's forward and dX on the pair loop,
    the first layer's input imaged by run_group) equal the chains with every activation image switched off; the graph-replayed
    forward equals the eager one."""
    B = 1000
    net = AMPNetwork(300, 28, 60, units=(256, 192, 130), disc_units=(128, 64), activation=activation, device=DEV, seed=0)
    eng = MLPEngine(net)
    assert eng.uses_images
    g = torch.Generator(device=DEV).manual_seed(13)
    x = torch.nn.functional.pad(torch.randn(B, 300, device=DEV, generator=g), (0, round4(300) - 300))
    xd = torch.nn.functional.pad(torch.randn(B, 60, device=DEV, generator=g), (0, round4(60) - 60))
    stacks = [(net.actor, x, eng.workspace("a", net.actor, B)), (net.critic, x, eng.workspace("c", net.critic, B)),
              (net.disc, xd, eng.workspace("d", net.disc, B))]
    douts = [torch.randn(ws["dout"].shape, device=DEV, generator=g) for _, _, ws in stacks]

    def chain():
        eng.forward_group(stacks)
        for (_, _, ws), d in zip(stacks, douts):
            ws["dout"].copy_(d)
        net.grads.zero_()
        depth = max(len(st.layers) for st, _, _ in stacks)
        for k in range(depth):
            descs = []
            for st, xin, ws in stacks:
                li = len(st.layers) - 1 - k
                if li >= 0:
                    descs += [d for d in eng.bwd_descs(st, li, xin, ws) if d is not None]
            eng.run_group(descs)
        torch.cuda.synchronize()
        return [t.clone() for _, _, ws in stacks for t in ws["h"] + ws["dh"] + [ws["out"]]] + [net.grads.clone()]

    d1 = eng.bwd_descs(net.actor, 2, x, stacks[0][2])[1]
    f1 = eng.fwd_desc(net.actor, 1, x, stacks[0][2])
    assert d1.A_img and d1.C_img and f1.A_img and f1.C_img            # the hidden layers do take and write images
    assert not eng.fwd_desc(net.actor, 3, x, stacks[0][2]).A_img      # the head does not
    with_images = chain()
    monkeypatch.setattr(MLPEngine, "_reads_image", lambda self, st, li: False)
    assert not eng.fwd_desc(net.actor, 1, x, stacks[0][2]).A_img
    without = chain()
    assert all(torch.equal(u, v) for u, v in zip(with_images, without))
    assert without[-1].abs().sum() > 0
    monkeypatch.undo()

    outs = [ws["out"][:, :st.out_dim] for st, _, ws in stacks]     # (the padding columns are no GEMM's output)
    eng.forward_group(stacks)                                         # eager once: every image buffer exists before the capture
    torch.cuda.synchronize()
    eager = [o.clone() for o in outs]
    graph = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        with torch.cuda.graph(graph, stream=s):
            eng.forward_group(stacks)
    torch.cuda.current_stream().wait_stream(s)
    for o in outs:
        o.fill_(float("nan"))
    for t in [ws["h"][0][:, :st.layers[0].out_dim] for st, _, ws in stacks]:
        t.fill_(float("nan"))                                         # the replay rewrites the activations and their images
    graph.replay()
    torch.cuda.synchronize()
    assert all(torch.equal(u, v) for u, v in zip(eager, outs))
