"""Activation images of the weight gradient (PhcGemmDesc.A_img with B_img): dW += dY^T X with both operands taken from their
images computes the same products in the same order as the staged path, so every result is compared with torch.equal -- over
ragged shapes, with and without split-K, inside mixed grouped launches, through MLPEngine.run_group (which makes the images),
and over one whole grouped minibatch backward with the gradient-penalty chain."""
import ctypes as C

import pytest
import torch

from phc_b200 import _lib
from phc_b200.learning.networks import MLPEngine, group_splits, round4
from phc_b200.ops import _stream

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
PHC_ERR_INVALID_ARG = -1


@pytest.fixture
def lib():
    lib = _lib.load()
    yield lib
    lib.phc_gemm_tc5s_set_tile(0)
    lib.phc_gemm_set_precision(_lib.PHC_GEMM_FP32_3XTF32)
    MLPEngine._mode_set = None


def image(lib, T, rows, K, fill=float("nan")):
    """image of the mn-major operand T[K, rows] (every float of it must be written)"""
    img = torch.full((lib.phc_gemm_image_floats(rows, K),), fill, device=DEV)
    d = _lib.PhcGemmImageDesc(T.data_ptr(), T.stride(0), 0, rows, K, img.data_ptr())
    _lib.check(lib.phc_gemm_make_images(C.byref(d), 1, _stream()), "phc_gemm_make_images")
    return img


class DW:
    """dW[M, N] += dY[K, M]^T X[K, N]: both operands mn-major, accumulating (split-K or not) into C"""

    def __init__(self, g, M, N, K, split=True, C_=None):
        rnd = lambda r, c: torch.nn.functional.pad(torch.randn(r, c, device=DEV, generator=g), (0, round4(c) - c))  # noqa: E731
        self.M, self.N, self.K = M, N, K
        self.dY, self.X = rnd(K, M), rnd(K, N)
        self.C = torch.zeros(M, round4(N), device=DEV) if C_ is None else C_
        self.ks = group_splits(K) if split else 1
        self.imgs = None

    def desc(self, use_img):
        if use_img and self.imgs is None:
            lib = _lib.load()
            self.imgs = (image(lib, self.dY, self.M, self.K), image(lib, self.X, self.N, self.K))
        a_img, b_img = (i.data_ptr() for i in self.imgs) if use_img else (None, None)
        return _lib.PhcGemmDesc(self.dY.data_ptr(), self.dY.stride(0), 0, self.X.data_ptr(), self.X.stride(0), 0, self.C.data_ptr(),
                                self.C.stride(0), self.M, self.N, self.K, 1.0, None, 0, None, 0, 1, self.ks, None, b_img, a_img)


def launch(lib, descs):
    _lib.check(lib.phc_gemm_group((_lib.PhcGemmDesc * len(descs))(*descs), len(descs), _stream()), "phc_gemm_group")
    torch.cuda.synchronize()


def run(lib, probs, use_img):
    for p in probs:
        p.C.zero_()
    launch(lib, [p.desc(u) for p, u in zip(probs, use_img)])
    return [p.C.clone() for p in probs]


@pytest.mark.parametrize("split", [True, False], ids=["splitk", "nosplit"])
@pytest.mark.parametrize("K", [5, 69, 4099, 16384])
def test_dw_images_equal_staged(lib, K, split):
    g = torch.Generator(device=DEV).manual_seed(K + split)
    for M in (1, 69, 300, 1024):
        for N in (1, 130, 934, 1960):
            p = DW(g, M, N, K, split)
            staged, imaged = run(lib, [p], [False]), run(lib, [p], [True])
            assert torch.equal(staged[0], imaged[0]), f"M={M} N={N} K={K} k_splits={p.ks}"
            assert staged[0].abs().sum() > 0


def test_mixed_group_with_same_c(lib):
    """One launch with image and staged dW problems, two of them adding into the same C (ordered), next to forward-form
    problems with and without a weight image: each equals the all-staged launch."""
    g = torch.Generator(device=DEV).manual_seed(3)
    a = DW(g, 300, 934, 4099)
    b = DW(g, 300, 934, 2000, C_=a.C)                                  # same C, M, N, ldc: adds after a, slice by slice
    c = DW(g, 1024, 130, 16384)
    d = DW(g, 69, 1960, 700, split=False)
    W = torch.randn(200, 936, device=DEV, generator=g)
    W[:, 934:] = 0
    x = torch.randn(1000, 936, device=DEV, generator=g)
    x[:, 934:] = 0
    y = torch.zeros(1000, 200, device=DEV)
    w_img = torch.full((lib.phc_gemm_image_floats(200, 934),), float("nan"), device=DEV)
    _lib.check(lib.phc_gemm_make_images(C.byref(_lib.PhcGemmImageDesc(W.data_ptr(), W.stride(0), 1, 200, 934, w_img.data_ptr())), 1, _stream()))

    def fwd(use_img):
        return _lib.PhcGemmDesc(x.data_ptr(), x.stride(0), 1, W.data_ptr(), W.stride(0), 1, y.data_ptr(), y.stride(0), 1000, 200, 934, 1.0,
                                None, _lib.PHC_ACT_RELU, None, 0, 0, 1, None, w_img.data_ptr() if use_img else None, None)

    def go(flags, fwd_img):
        for p in (a, c, d):
            p.C.zero_()
        launch(lib, [p.desc(u) for p, u in zip((a, b, c, d), flags)] + [fwd(fwd_img)])
        return [a.C.clone(), c.C.clone(), d.C.clone(), y.clone()]

    base = go([False] * 4, False)
    for flags, fwd_img in (([True] * 4, True), ([True, False, True, False], False), ([False, True, False, True], True)):
        got = go(flags, fwd_img)
        assert all(torch.equal(u, v) for u, v in zip(base, got)), (flags, fwd_img)


@pytest.mark.parametrize("mode", ["wide_tile", "single_pass"])
def test_wide_tile_and_single_pass_ignore_images(lib, mode):
    """128 x 256 tiles and single-pass TF32 stage from the fp32 arrays: images full of NaN change nothing."""
    if mode == "wide_tile":
        _lib.check(lib.phc_gemm_tc5s_set_tile(256))
    else:
        _lib.check(lib.phc_gemm_set_precision(_lib.PHC_GEMM_TF32_SINGLE_PASS))
    g = torch.Generator(device=DEV).manual_seed(4)
    probs = [DW(g, 300, 934, 4099), DW(g, 69, 130, 69, split=False)]
    for p in probs:
        p.imgs = (torch.full((lib.phc_gemm_image_floats(p.M, p.K),), float("nan"), device=DEV),
                  torch.full((lib.phc_gemm_image_floats(p.N, p.K),), float("nan"), device=DEV))
    staged, imaged = run(lib, probs, [False] * 2), run(lib, probs, [True] * 2)
    assert all(torch.equal(u, v) for u, v in zip(staged, imaged))
    assert all(torch.isfinite(u).all() for u in imaged)


def test_activation_image_refusals(lib):
    g = torch.Generator(device=DEV).manual_seed(5)
    p = DW(g, 64, 64, 64)
    d = p.desc(True)
    d.B_img = None                                                   # A_img without B_img
    assert lib.phc_gemm_group(C.byref(d), 1, _stream()) == PHC_ERR_INVALID_ARG
    d = p.desc(True)
    d.A_img = d.A_img + 4                                            # not 16-byte aligned
    assert lib.phc_gemm_group(C.byref(d), 1, _stream()) == PHC_ERR_INVALID_ARG
    d = p.desc(True)
    d.A_img = None                                                   # B_img with mn-major A and no A_img: still refused
    assert lib.phc_gemm_group(C.byref(d), 1, _stream()) == PHC_ERR_INVALID_ARG
    assert lib.phc_gemm_group(C.byref(p.desc(True)), 1, _stream()) == 0


def test_run_group_images_follow_the_activations(lib):
    """MLPEngine.run_group makes the images of a dw_desc right before the launch: a change to the activations between two
    launches is seen, and actor-and-critic-style problems that share an input share its image."""
    from phc_b200.learning.networks import AMPNetwork
    net = AMPNetwork(300, 28, 60, units=(256, 128), disc_units=(128, 64), device=DEV, seed=0)
    eng = MLPEngine(net)
    assert eng.uses_images
    g = torch.Generator(device=DEV).manual_seed(6)
    K, M1, M2, N = 3000, 1024, 1000, 1030                           # large enough for dw_desc to ask for images
    X = torch.randn(K, round4(N), device=DEV, generator=g)
    dY1, dY2 = torch.randn(K, M1, device=DEV, generator=g), torch.randn(K, M2, device=DEV, generator=g)
    C1, C2 = torch.zeros(M1, round4(N), device=DEV), torch.zeros(M2, round4(N), device=DEV)
    R1, R2 = torch.zeros_like(C1), torch.zeros_like(C2)
    for step in range(3):
        descs = [eng.dw_desc(dY1, X, C1, M1, N, K), eng.dw_desc(dY2, X, C2, M2, N, K)]
        jobs, n = eng.make_images(descs)
        assert n == 3 and descs[0].B_img == descs[1].B_img and descs[0].A_img
        for Cm in (C1, C2, R1, R2):
            Cm.zero_()
        eng.run_group(descs)
        ref = [eng.gdesc(dY1, False, X, False, R1, M1, N, K, accumulate=True, k_splits=group_splits(K)),
               eng.gdesc(dY2, False, X, False, R2, M2, N, K, accumulate=True, k_splits=group_splits(K))]
        eng.run_group(ref)
        torch.cuda.synchronize()
        assert torch.equal(C1, R1) and torch.equal(C2, R2), step
        assert C1.abs().sum() > 0
        X.mul_(-0.5).add_(1.0)                                       # the next launch must not read the old image
        dY1[step::7] += 1.0


def test_grouped_minibatch_backward_with_and_without_images(lib, monkeypatch):
    """One grouped minibatch (forward, loss gradients, backward of actor, critic and discriminator with the gradient-penalty
    chain merged in) gives the same gradient bucket bit for bit whether dW takes its activation images or stages."""
    from phc_b200 import synthetic as syn
    from phc_b200.env.humanoid_im import HumanoidIm, RLGPUEnv
    from phc_b200.learning.amp_agent import AMPAgent
    torch.manual_seed(0)
    motion = syn.make_motions(64, seed=0)
    task = HumanoidIm({"env": {"num_envs": 512}, "motion_data": motion, "seed": 0})
    agent = AMPAgent("dwimg", {"vec_env": RLGPUEnv(task), "seed": 0})
    eng, net = agent.engine, agent.model
    assert eng.backend == "tc5s" and eng.uses_images
    Bd, st = agent._amp_minibatch_size, _stream()
    g = torch.Generator(device=DEV).manual_seed(7)
    x, xa = agent._x_mb, agent._amp_mb
    x.copy_(torch.randn(x.shape, device=DEV, generator=g))
    xa.copy_(torch.randn(xa.shape, device=DEV, generator=g))
    douts = [torch.randn(ws["dout"].shape, device=DEV, generator=g) * 1e-2 for ws in (agent._ws_actor, agent._ws_critic, agent._ws_disc)]

    def loss_fn():
        for ws, d in zip((agent._ws_actor, agent._ws_critic, agent._ws_disc), douts):
            ws["dout"].copy_(d)

    made = []
    orig = MLPEngine.make_images

    def make_images(self, descs):
        jobs, n = orig(self, descs)
        made.append(n)
        return jobs, n

    def grads(use_img):
        monkeypatch.setattr(MLPEngine, "make_images", make_images if use_img else lambda self, descs: ((_lib.PhcGemmImageDesc * 0)(), 0))
        net.grads.zero_()
        agent._stats.zero_()
        agent._grouped_core(x, xa, Bd, st, loss_fn)
        torch.cuda.synchronize()
        return net.grads.clone()

    staged, imaged = grads(False), grads(True)
    assert sum(made) > 0
    assert staged.abs().sum() > 0
    assert torch.equal(staged, imaged)
