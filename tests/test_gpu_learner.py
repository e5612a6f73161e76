"""GPU parity of the learner path: tensor-core GEMM (3xTF32), running mean/std, loss-gradient kernels and one complete
PPO + AMP minibatch update (forward, hand-written backward incl. the discriminator gradient penalty, clip, Adam)
against torch-CPU oracles.  MLP math is fp32-equivalent (3xTF32): tolerances are rtol 1e-4 on gradients (sums over
16k-row batches re-associated by split-K / atomics) and rtol 2e-5 on forward activations."""
import math

import pytest
import torch

from oracle import phc_oracle as O
from oracle import ppo_oracle as PO
from phc_b200 import _lib
from phc_b200.learning.networks import AMPNetwork, MLPEngine, round4
from tests.helpers import close, load

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def gemm_close(got, A, B, what, extra=None, tol=4e-6):
    """fp32-equivalence criterion of a GEMM: |err[m,n]| <= tol * (|A| |B|^T)[m,n] (+tiny), against an fp64 product.
    (fp32 SGEMM's own bound is K*eps ~ 6e-5 at K=1000; typical sqrt(K)*eps ~ 2e-6.)  Prints the measured ratio."""
    exp = A.double() @ B.double().T
    bound = A.double().abs() @ B.double().abs().T
    if extra is not None:
        exp, bound = extra(exp, bound)
    err = (got.double().cpu() - exp).abs()
    ratio = float((err / (bound + 1e-30)).max())
    assert ratio <= tol and torch.isfinite(got).all(), f"{what}: max err/(|A||B|) = {ratio:.3e} > {tol}, max abs err {float(err.max()):.3e}"
    return ratio


def padded(t, ld=None):
    n, d = t.shape
    ld = round4(d) if ld is None else ld
    out = torch.zeros(n, ld, device=DEV)
    out[:, :d] = t.to(DEV)
    return out


@pytest.mark.parametrize("M,N,K", [(128, 128, 16), (300, 70, 934), (4096, 1024, 936), (130, 1, 512), (257, 69, 512), (5, 3, 7)])
def test_gemm_forward_form(M, N, K):
    g = torch.Generator().manual_seed(M + N + K)
    A, B, bias = torch.randn(M, K, generator=g), torch.randn(N, K, generator=g) / math.sqrt(K), torch.randn(N, generator=g)
    net = AMPNetwork(8, 2, 8, (4,), (4,), device=DEV)
    eng = MLPEngine(net, backend="mma")           # the pre-split tensor-core kernel has its own file (test_gpu_gemm_tc5.py)
    Ap, Bp = padded(A), padded(B)
    C = torch.zeros(M, round4(N), device=DEV)
    eng.gemm(Ap, True, Bp, True, C, M, N, K, bias=bias.to(DEV), relu=True)
    # relu only shrinks errors; compare post-activation against the fp64 value with the pre-activation bound
    gemm_close(C[:, :N], A, B, "gemm fwd", extra=lambda e, b: (torch.relu(e + bias.double()), b + bias.double().abs()))
    assert float(C[:, N:].abs().sum()) == 0.0


@pytest.mark.parametrize("M,N,K", [(256, 936, 1024), (100, 72, 69), (64, 1960, 40)])
def test_gemm_input_grad_form(M, N, K):
    g = torch.Generator().manual_seed(1)
    dY, W, H = torch.randn(M, K, generator=g), torch.randn(K, N, generator=g) / math.sqrt(K), torch.randn(M, N, generator=g)
    eng = MLPEngine(AMPNetwork(8, 2, 8, (4,), (4,), device=DEV), backend="mma")
    C = torch.zeros(M, round4(N), device=DEV)
    eng.gemm(padded(dY), True, padded(W), False, C, M, N, K, mask=padded(H))
    gemm_close(C[:, :N], dY, W.T.contiguous(), "gemm dX", extra=lambda e, b: (e * (H > 0), b))


@pytest.mark.parametrize("M,N,K,splits", [(1024, 934, 4096, 4), (69, 512, 2048, 16), (1, 512, 1000, 1), (33, 17, 515, 2)])
def test_gemm_weight_grad_form(M, N, K, splits):
    g = torch.Generator().manual_seed(2)
    dY, X = torch.randn(K, M, generator=g), torch.randn(K, N, generator=g)
    eng = MLPEngine(AMPNetwork(8, 2, 8, (4,), (4,), device=DEV), backend="mma")
    C = torch.ones(M, round4(N), device=DEV)            # accumulates on top of existing content
    eng.gemm(padded(dY), False, padded(X), False, C, M, N, K, alpha=0.5, accumulate=True, k_splits=splits)
    gemm_close(C[:, :N], dY.T.contiguous(), X.T.contiguous(), "gemm dW", extra=lambda e, b: (1.0 + 0.5 * e, 1.0 + 0.5 * b))
    out = torch.zeros(M, device=DEV)
    eng.colsum(padded(dY), K, M, out)
    cerr = (out.double().cpu() - dY.double().sum(0)).abs() / dY.double().abs().sum(0)
    assert float(cerr.max()) < 2e-6, f"colsum: {float(cerr.max()):.3e}"


def test_grouped_colsum_matches_fp64_column_sums():
    """phc_colsum_group: bias gradients of several stacks in one launch; ragged row / column counts, single columns, accumulation on
    top of existing content, the fp32 criterion |err| <= tol * sum |x|."""
    g = torch.Generator().manual_seed(5)
    eng = MLPEngine(AMPNetwork(8, 2, 8, (4,), (4,), device=DEV))
    shapes = [(16384, 1024), (16384, 69), (12288, 1), (300, 130), (7, 5), (257, 512), (1000, 934), (1, 1960), (33, 3)]     # > 8: two launches
    items, refs = [], []
    for M, N in shapes:
        X = torch.randn(M, N, generator=g) * 2 + 0.5
        Xp = padded(X)
        Xp[:, N:] = 7.0                                # pad columns must not leak into the sums
        out = torch.full((round4(N),), 0.25, device=DEV)
        items.append((Xp, M, N, out))
        refs.append((X.double().sum(0) + 0.25, X.double().abs().sum(0) + 0.25))
    eng.colsum_group(items)
    torch.cuda.synchronize()
    for (Xp, M, N, out), (e, b) in zip(items, refs):
        err = (out[:N].double().cpu() - e).abs() / b
        assert float(err.max()) < 2e-6, f"colsum_group {M}x{N}: {float(err.max()):.3e}"
        assert float((out[N:] - 0.25).abs().sum()) == 0.0


def test_running_mean_std_vs_reference_golden():
    from phc_b200.learning.amp_agent import RunningMeanStd
    g = load("learn.npz")
    rms = RunningMeanStd(12, DEV)
    rms.train()
    for i in range(3):
        y = rms(g[f"rms_x{i}"].to(DEV))
        close(y.cpu(), g[f"rms_y{i}"], what=f"rms_y{i}")
    close(rms.running_mean.cpu(), g["rms_mean"], rtol=1e-6, atol=1e-7, what="mean (fp64 batch moments vs torch's fp32)")
    close(rms.running_var.cpu(), g["rms_var"], rtol=1e-6, atol=1e-7, what="var")
    close(rms.count.cpu(), g["rms_count"], what="count")
    rms.eval()
    close(rms(g["rms_x0"].to(DEV) * 0.1, unnorm=True).cpu(), g["rms_unnorm"], what="unnorm")
    # gathered rows
    idx = torch.tensor([5, 1, 1, 30, 7], device=DEV)
    out = torch.zeros(5, 12, device=DEV)
    rms.apply(g["rms_x1"].to(DEV), out, row_idx=idx)
    close(out.cpu(), O.rms_normalize(g["rms_x1"][idx.cpu()], rms.running_mean.cpu(), rms.running_var.cpu()), what="gather")


def test_disc_reward_vs_reference_golden():
    g = load("learn.npz")
    lib = _lib.load()
    ws = [g["d_w1"], g["d_w2"], g["d_w3"]]
    bs = [g["d_b1"], g["d_b2"], g["d_b3"]]
    logits = O.mlp_forward(g["d_x_agent"], ws, bs).to(DEV).contiguous()
    n = logits.shape[0]
    dr, comb = torch.zeros(n, device=DEV), torch.zeros(n, device=DEV)
    task = torch.full((n,), 0.7, device=DEV)
    _lib.check(lib.phc_disc_reward(logits.data_ptr(), 1, task.data_ptr(), n, 2.0, 0.5, 0.5, dr.data_ptr(), comb.data_ptr(), None))
    torch.cuda.synchronize()
    close(dr.cpu(), g["d_reward"].reshape(-1), what="disc reward")
    close(comb.cpu(), g["d_combined"].reshape(-1), what="combined reward")


def _rand_batch(B, Bd, obs, act, amp, seed, mu_fn=None):
    """A PPO minibatch.  With mu_fn (obs_n -> current policy mean) the stored "old" policy sits close to the current one,
    like real PPO data: ratios are O(1) and both clip branches are hit; without it old_mu is random (stress case)."""
    g = torch.Generator().manual_seed(seed)
    r = lambda *s: torch.randn(*s, generator=g)
    logstd = torch.full((act,), -2.9)
    obs_n = torch.clamp(r(B, obs) * 1.5, -5, 5)
    old_sigma = torch.exp(logstd).expand(B, act).clone()
    old_mu = r(B, act) * 0.8 if mu_fn is None else (mu_fn(obs_n) + 0.03 * old_sigma * r(B, act)).float()
    actions = old_mu + old_sigma * r(B, act)
    old_nlp = O.gaussian_neglogp(actions, old_mu, old_sigma, logstd.expand(B, act))
    return dict(obs_n=obs_n, actions=actions, old_neglogp=old_nlp + 0.05 * r(B),
                advantages=r(B), old_mu=old_mu, old_sigma=old_sigma, returns=r(B, 1),
                amp_agent=torch.clamp(r(Bd, amp), -5, 5), amp_replay=torch.clamp(r(Bd, amp), -5, 5), amp_demo=torch.clamp(r(Bd, amp), -5, 5))


def make_lattice(net, seed=0):
    """Put the HIDDEN layers of all three MLPs on a dyadic lattice (weights in {-1,0,1}/8, biases an odd multiple of half the
    pre-activation granularity) so that, with inputs that are multiples of 1/4, every hidden pre-activation is computed
    EXACTLY by any arithmetic (fp64, fp32, 3xTF32) and is never zero: the ReLU masks are then identical on both sides and
    every remaining gradient difference is arithmetic error, not a flipped borderline unit (16.7 M pre-activations per
    minibatch otherwise contain a few |z| < 1e-6 whose mask legitimately differs between fp64 and fp32-class math)."""
    g = torch.Generator().manual_seed(seed)
    for st in (net.actor, net.critic, net.disc):
        if st.activation != "relu":      # SiLU is smooth: no borderline units, the default initialisation is kept
            continue
        gran = 1.0 / 4
        for l in st.hidden:
            w = torch.randint(-1, 2, (l.out_dim, l.in_dim), generator=g).float() / 8
            gran = gran / 8
            b = (torch.randint(0, 2, (l.out_dim,), generator=g).float() * 2 - 1) * gran / 2
            net.set_layer(l, w, b)


def lattice_inputs(t):
    return torch.round(t * 4) / 4


CFG = dict(e_clip=0.2, critic_coef=5.0, entropy_coef=0.0, bounds_loss_coef=10.0, disc_coef=5.0, disc_logit_reg=0.01,
           disc_grad_penalty=5.0, disc_weight_decay=0.0001, grad_norm=50.0, learning_rate=2e-5, truncate_grads=True)


@pytest.mark.parametrize("backend", ["tc5", "mma", "tc5s", "tc5s-1cta"])
@pytest.mark.parametrize("B,Bd,obs,act,amp,units,activation",
                         [(512, 128, 934, 69, 1960, (256, 128), "relu"), (16384, 4096, 934, 69, 1960, (1024, 512), "relu"),
                          (300, 100, 50, 7, 30, (64, 32), "relu"),
                          # nn.SiLU actor / critic of im_big.yaml, im_pnn_big.yaml, im_mcp_big.yaml (disc stays relu), 3 and 6 hidden layers
                          (512, 128, 934, 69, 1960, (256, 192, 128), "silu"), (300, 100, 50, 7, 30, (96, 80, 64, 64, 32, 32), "silu")])
def test_minibatch_update_vs_autograd_oracle(B, Bd, obs, act, amp, units, activation, backend):
    """forward values, every parameter gradient, the clipped Adam step: CUDA engine vs torch autograd on the CPU."""
    from tests.learner_harness import run_cuda_minibatch
    disc_units = units[-2:]
    net = AMPNetwork(obs, act, amp, units, disc_units, activation=activation, device=DEV, seed=3)
    make_lattice(net, seed=B)
    # rescale the mu head so that mu has unit spread: part of the batch sits beyond the +-1 soft bound (bound loss active)
    g0 = torch.Generator().manual_seed(99)
    x0 = lattice_inputs(torch.clamp(torch.randn(256, obs, generator=g0) * 1.5, -5, 5))
    sd0 = {k: v.cpu() for k, v in net.state_dict().items()}
    aw0, ab0 = PO.stack_params(sd0, "actor_mlp", "mu", len(units))
    spread = float(O.mlp_forward(x0.double(), [w.double() for w in aw0], [b.double() for b in ab0], act=activation).std())
    net.weight(net.actor.head).mul_(1.0 / spread)
    net.bias(net.actor.head).mul_(1.0 / spread)
    sd = {k: v.cpu() for k, v in net.state_dict().items()}
    aw, ab = PO.stack_params(sd, "actor_mlp", "mu", len(units))
    mu_fn = lambda x: O.mlp_forward(x.double(), [w.double() for w in aw], [b.double() for b in ab], act=activation)
    batch = _rand_batch(B, Bd, obs, act, amp, seed=B, mu_fn=lambda x: mu_fn(lattice_inputs(x)))
    for k in ("obs_n", "amp_agent", "amp_replay", "amp_demo"):
        batch[k] = lattice_inputs(batch[k])
    if backend.startswith("tc5s"):      # grouped launches (AMPAgent._grouped_core), CTA-pair tiles or one-CTA tiles
        _lib.check(_lib.load().phc_gemm_tc5s_set_ctas(1 if backend.endswith("1cta") else 2))
    try:
        got = run_cuda_minibatch(net, batch, CFG, backend=backend.split("-")[0])
    finally:
        _lib.load().phc_gemm_tc5s_set_ctas(0)
    # near-exact (fp64) reference; the loss is evaluated at OUR policy mean (see ppo_oracle.minibatch_update: sigma = e^-2.9
    # turns an fp32-level difference in mu into a 150x larger one in neglogp), the forward pass itself is compared below
    exp = PO.minibatch_update(sd, batch, CFG, n_hidden=len(units), dtype=torch.float64, mu_override=got["mu"].cpu().double(),
                              mlp_act=activation, n_hidden_disc=len(disc_units))

    def scaled(a, b, tol, what):       # error relative to the tensor's scale (entries are sums of large cancelling terms)
        err = float((a.double().cpu() - b.double()).abs().max())
        sc = float(b.double().abs().max()) + 1e-30
        assert err <= tol * sc, f"{what}: max abs err {err:.3e} vs scale {sc:.3e} -> {err / sc:.3e} > {tol}"

    scaled(got["mu"], exp["mu"], 2e-5, "mu")
    scaled(got["values"], exp["values"], 2e-5, "values")
    s = got["stats"]
    f32 = lambda t: t.float()
    close(torch.tensor(s["actor_loss"]), f32(exp["a_loss"]), rtol=2e-4, atol=1e-5, what="a_loss")
    close(torch.tensor(s["critic_loss"]), f32(exp["c_loss"]), rtol=1e-4, atol=1e-5, what="c_loss")
    close(torch.tensor(s["b_loss"]), f32(exp["b_loss"]), rtol=1e-4, atol=1e-5, what="b_loss")
    close(torch.tensor(s["kl"]), f32(exp["kl"]), rtol=1e-3, atol=1e-4, what="kl")
    close(torch.tensor(s["disc_grad_penalty"]), f32(exp["disc"]["disc_grad_penalty"]), rtol=1e-4, atol=1e-6, what="grad penalty")
    close(torch.tensor(s["disc_agent_acc"]), f32(exp["disc"]["disc_agent_acc"]), atol=2e-3, what="disc agent acc")
    assert 0.02 < s["actor_clip_frac"] < 0.98 and s["b_loss"] > 0, f"test batch must exercise both PPO branches and the bound loss: {s}"
    gsd = got["grads"]
    report = []
    for k, ge in exp["grads"].items():
        err = float((gsd[k].double().cpu() - ge.double()).abs().max())
        sc = float(ge.double().abs().max()) + 1e-30
        report.append((err / sc, k, err, sc))
    bad = [f"{k}: {e:.2e}/{sc:.2e}={r:.2e}" for r, k, e, sc in report if r > 1e-4]
    assert not bad, "gradient mismatches (max abs err / max abs value): " + "; ".join(bad) + " || ok: " + \
        "; ".join(f"{k.split('.', 1)[1]}={r:.1e}" for r, k, e, sc in report if r <= 1e-4)
    close(torch.tensor(got["total_norm"]), exp["total_norm"].float(), rtol=1e-4, atol=1e-6, what="grad norm")
    lr = CFG["learning_rate"]
    for k, pe in exp["new_params"].items():
        # Adam's first step is lr * g / (|g| + 1e-8 * sqrt(bias corr.)) ~ lr * sign(g): well determined only where |g| is well
        # above the gradient's own rounding error; compare those entries to 2 % of a step, bound the rest by one full step
        ge = exp["grads"][k].double()
        well = ge.abs() > 1e-3 * ge.abs().max()
        d = (got["new_params"][k].double().cpu() - pe.double()).abs()
        assert float(d[well].max()) <= 0.02 * lr + 1e-7 * float(pe.abs().max()), f"adam {k}: {float(d[well].max()):.3e}"
        assert float(d.max()) <= 2.1 * lr, f"adam (near-zero gradient entries) {k}: {float(d.max()):.3e}"


def test_fused_rms_apply_update_equals_apply_then_update():
    """phc_rms_apply_update (one pass: normalise with given statistics + fold the raw rows into the live ones) against phc_rms_apply
    followed by phc_rms_update, with a row gather and with a frozen copy as the apply statistics (AMPAgent._preproc_obs(use_temp=True))."""
    from phc_b200.learning.amp_agent import RunningMeanStd
    g = torch.Generator().manual_seed(3)
    n_src, n, d = 5000, 3001, 934
    x = (torch.randn(n_src, d, generator=g) * 3 + 1).to(DEV)
    idx = torch.randint(0, n_src, (n,), generator=g).to(DEV)
    a, b = RunningMeanStd(d, DEV), RunningMeanStd(d, DEV)
    mean0, var0 = torch.randn(d, generator=g).double(), (torch.rand(d, generator=g) + 0.5).double()
    for r in (a, b):
        r.running_mean.copy_(mean0)
        r.running_var.copy_(var0)
        r.count.fill_(777.0)
    frozen = a.frozen_copy()
    frozen.running_mean += 0.25                                  # the temp copy differs from the live statistics
    ya, yb = torch.zeros(n, round4(d), device=DEV), torch.zeros(n, round4(d), device=DEV)
    frozen.apply(x, ya, row_idx=idx)
    a.update(x, row_idx=idx)
    b.apply_update(x, yb, row_idx=idx, apply_stats=frozen)
    torch.cuda.synchronize()
    assert torch.equal(ya, yb)
    close(b.running_mean.cpu(), a.running_mean.cpu(), rtol=1e-12, atol=1e-12, what="running mean")
    close(b.running_var.cpu(), a.running_var.cpu(), rtol=1e-11, atol=1e-12, what="running var")
    assert float(b.count) == float(a.count) == 777.0 + n
    # and against the reference formula on the CPU
    rows = x[idx].cpu()
    exp = O.rms_normalize(rows, frozen.running_mean.cpu(), frozen.running_var.cpu())
    close(yb[:, :d].cpu(), exp, rtol=1e-6, atol=1e-6, what="normalised rows")
