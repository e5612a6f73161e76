"""Weight images (PhcGemmDesc.B_img, phc_gemm_make_images): a problem whose B comes from its image computes the same products in
the same order as the staged path, so every result is compared with torch.equal -- per problem form, ragged shape, precision
mode and tile, inside mixed grouped launches, and through AMPNetwork after each way its parameters get written."""
import ctypes as C

import pytest
import torch

from phc_b200 import _lib
from phc_b200.learning.networks import AMPNetwork, MLPEngine, group_splits, round4
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


def image(lib, B, b_k, N, K):
    img = torch.full((lib.phc_gemm_image_floats(N, K),), float("nan"), device=DEV)     # every float must be written
    d = _lib.PhcGemmImageDesc(B.data_ptr(), B.stride(0), int(b_k), N, K, img.data_ptr())
    _lib.check(lib.phc_gemm_make_images(C.byref(d), 1, _stream()), "phc_gemm_make_images")
    return img


class Prob:
    """form "fwd": Y = X W^T + b, ReLU (B = W[N, K], k-major); "dx": dX = dY W (B = W[K, N], mn-major); "dw": dW += dY^T X
    (split-K, both operands mn-major, never an image)."""

    def __init__(self, g, form, M, N, K):
        self.form, self.M, self.N, self.K = form, M, N, K
        rnd = lambda r, c, ld: torch.nn.functional.pad(torch.randn(r, c, device=DEV, generator=g), (0, ld - c))  # noqa: E731
        self.a_k = form != "dw"
        self.b_k = form == "fwd"
        self.A = rnd(M, K, round4(K)) if self.a_k else rnd(K, M, round4(M))
        self.B = rnd(N, K, round4(K)) if self.b_k else rnd(K, N, round4(N))
        self.bias = torch.randn(N, device=DEV, generator=g) if form == "fwd" else None
        self.C = torch.zeros(M, round4(N), device=DEV)
        self.img = None

    def desc(self, use_img):
        if use_img and self.img is None:
            self.img = image(_lib.load(), self.B, self.b_k, self.N, self.K)
        dw = self.form == "dw"
        return _lib.PhcGemmDesc(self.A.data_ptr(), self.A.stride(0), int(self.a_k), self.B.data_ptr(), self.B.stride(0), int(self.b_k),
                                self.C.data_ptr(), self.C.stride(0), self.M, self.N, self.K, 1.0,
                                None if self.bias is None else self.bias.data_ptr(), _lib.PHC_ACT_RELU if self.form == "fwd" else 0,
                                None, 0, int(dw), group_splits(self.K) if dw else 1, None,
                                self.img.data_ptr() if use_img and self.img is not None else None)


def run(lib, probs, use_img):
    for p in probs:
        p.C.zero_()
    descs = [p.desc(use_img and p.form != "dw") for p in probs]
    arr = (_lib.PhcGemmDesc * len(descs))(*descs)
    _lib.check(lib.phc_gemm_group(arr, len(descs), _stream()), "phc_gemm_group")
    torch.cuda.synchronize()
    return [p.C.clone() for p in probs]


def same_both_ways(lib, probs):
    staged, imaged = run(lib, probs, False), run(lib, probs, True)
    for p, a, b in zip(probs, staged, imaged):
        assert torch.equal(a, b), f"{p.form} M={p.M} N={p.N} K={p.K}"
        assert a.abs().sum() > 0


@pytest.mark.parametrize("precision", [_lib.PHC_GEMM_FP32_3XTF32, _lib.PHC_GEMM_TF32_SINGLE_PASS], ids=["3xtf32", "single"])
@pytest.mark.parametrize("form", ["fwd", "dx"])
@pytest.mark.parametrize("M,N,K", [(300, 1, 934), (1000, 69, 1960), (4100, 512, 1024), (129, 1000, 69), (64, 130, 5)])
def test_image_problem_equals_staged(lib, precision, form, M, N, K):
    _lib.check(lib.phc_gemm_set_precision(precision))
    same_both_ways(lib, [Prob(torch.Generator(device=DEV).manual_seed(M + N + K), form, M, N, K)])


def test_image_layout_and_split():
    """The documented layout and split: element (n, k) of block (nt, kb), hi = trunc_tf32, lo = rna_tf32 of the remainder."""
    lib = _lib.load()
    N, K = 200, 70
    W = torch.zeros(N, round4(K), device=DEV)
    W[:, :K] = torch.randn(N, K, device=DEV)
    img = image(lib, W, True, N, K).view(2, 3, 2, 128, 32)          # [n-tile, k-block, hi|lo, 4096 floats as 128 x 32]
    w = W[:, :K].cpu()
    hi = (w.view(torch.int32) & ~0x1FFF).view(torch.float32)
    d = (w - hi).view(torch.int32)
    lo = ((d + 0x1000) & ~0x1FFF).view(torch.float32)
    got = torch.zeros(2, 2 * 128, 3 * 32)
    flat = img.cpu().reshape(2, 3, 2, 4096)
    n, k = torch.meshgrid(torch.arange(128), torch.arange(32), indexing="ij")
    pos = 256 * (n // 8) + 32 * (k // 4) + 4 * (n % 8) + k % 4
    for nt in range(2):
        for kb in range(3):
            for h in range(2):
                got[h, nt * 128:(nt + 1) * 128, kb * 32:(kb + 1) * 32] = flat[nt, kb, h][pos]
    assert torch.equal(got[0, :N, :K], hi) and torch.equal(got[1, :N, :K], lo)
    assert not got[:, N:].any() and not got[:, :, K:].any()


def test_mixed_group_and_wide_tile(lib):
    """One launch with image, staged (no image given) and split-K dW problems; with 128 x 256 tiles a given image is ignored."""
    g = torch.Generator(device=DEV).manual_seed(5)
    probs = [Prob(g, "fwd", 2000, 300, 934), Prob(g, "dx", 1500, 934, 512), Prob(g, "dw", 512, 300, 4096), Prob(g, "fwd", 700, 69, 200)]
    same_both_ways(lib, probs)

    staged = Prob(g, "fwd", 900, 100, 300)                            # same launch, one fwd problem without its image
    base = run(lib, probs + [staged], False)
    for p in probs + [staged]:
        p.C.zero_()
    descs = [p.desc(p is not staged and p.form != "dw") for p in probs + [staged]]
    _lib.check(lib.phc_gemm_group((_lib.PhcGemmDesc * len(descs))(*descs), len(descs), _stream()))
    torch.cuda.synchronize()
    mixed = [p.C.clone() for p in probs + [staged]]
    assert all(torch.equal(a, b) for a, b in zip(base, mixed))

    _lib.check(lib.phc_gemm_tc5s_set_tile(256))
    same_both_ways(lib, probs)


def test_image_refused_without_kmajor_a(lib):
    g = torch.Generator(device=DEV).manual_seed(1)
    p = Prob(g, "fwd", 64, 64, 64)
    d = p.desc(True)
    d.a_kmajor = 0
    assert lib.phc_gemm_group(C.byref(d), 1, _stream()) == PHC_ERR_INVALID_ARG
    d = p.desc(True)
    d.B_img = d.B_img + 4                                            # not 16-byte aligned
    assert lib.phc_gemm_group(C.byref(d), 1, _stream()) == PHC_ERR_INVALID_ARG


# ---- AMPNetwork: the images follow every writer of params -----------------------------------------------------------------------
def assert_images_current(eng, net, B=300, stacks=None, tag="img"):
    """the grouped forward through the images equals the one from the raw weights, bit for bit, for every stack"""
    g = torch.Generator(device=DEV).manual_seed(9)
    for k, st in enumerate(stacks or [*net.actor_stacks, net.critic, net.disc]):
        x = torch.zeros(B, round4(st.in_dim), device=DEV)
        x[:, :st.in_dim] = torch.randn(B, st.in_dim, device=DEV, generator=g)
        outs = []
        for use_img in (True, False):
            ws = eng.workspace(f"{tag}{k}{use_img}", st, B)
            for li in range(len(st.layers)):
                d = eng.fwd_desc(st, li, x, ws)
                assert d.B_img
                if not use_img:
                    d.B_img = None
                eng.run_group([d])
            outs.append(ws["out"].clone())
        torch.cuda.synchronize()
        assert torch.equal(outs[0], outs[1]) and outs[0].abs().sum() > 0


def test_images_follow_construction_and_load_state_dict(lib):
    net = AMPNetwork(934, 69, 110, units=(256, 128), disc_units=(128, 64), device=DEV, seed=0)
    eng = MLPEngine(net)
    assert_images_current(eng, net)
    other = AMPNetwork(934, 69, 110, units=(256, 128), disc_units=(128, 64), device=DEV, seed=1)
    net.load_state_dict(other.state_dict())
    assert_images_current(eng, net, tag="sd")
    net.weight(net.actor.head).mul_(0.5)                              # a write through torch: caught by the version counter
    assert_images_current(eng, net, tag="mul")


def test_images_follow_adam_and_restore(lib):
    from phc_b200 import synthetic as syn
    from phc_b200.env.humanoid_im import HumanoidIm, RLGPUEnv
    from phc_b200.learning.amp_agent import AMPAgent

    n = 64
    m = syn.make_motions(n, seed=2, min_frames=40, max_frames=90)
    task = HumanoidIm({"env": {"num_envs": n}, "motion_data": m, "seed": 2})
    agent = AMPAgent("t", {"vec_env": RLGPUEnv(task), "horizon_length": 8, "minibatch_size": 256, "amp_minibatch_size": 64,
                           "network": {"mlp": {"units": [128, 64], "activation": "relu"}, "disc": {"units": [128, 64], "activation": "relu"}}})
    net, eng = agent.model, agent.engine
    assert_images_current(eng, net)
    sd = agent.get_full_state_weights()
    p0 = net.params.clone()
    net.grads.copy_(torch.randn(net.num_floats, device=DEV, generator=torch.Generator(device=DEV).manual_seed(3)))
    agent._optimizer_step(1.0)                                       # Adam writes the bucket through a raw pointer
    torch.cuda.synchronize()
    assert not torch.equal(net.params, p0)
    assert_images_current(eng, net, tag="adam")
    agent.set_full_state_weights(sd)                                 # checkpoint restore
    assert all(torch.equal(v, sd["model"][k]) for k, v in net.state_dict().items())
    assert_images_current(eng, net, tag="restore")


def test_images_follow_pnn_loader(lib):
    from phc_b200.learning.network_loader import load_pnn

    src = AMPNetwork(934, 69, 8, units=(256, 128), disc_units=(8,), device=DEV, kind="amp_pnn", num_prim=2, seed=4)
    pnn = load_pnn({"model": src.state_dict()}, num_prim=2, device=DEV)
    assert_images_current(pnn.engine, pnn.net, stacks=pnn.net.pnn_actors)
