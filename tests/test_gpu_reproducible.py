"""Run-to-run reproducibility outside the GEMM, bit for bit: every reduction whose partials meet in global memory adds them in a
fixed order -- the bias-gradient column sums (phc_colsum_group), the RunningMeanStd moments, the advantage normalisation, the
gradient norm for clipping and the loss statistics -- so the same inputs give the same bits on every launch, whatever the block
scheduling.  Then training end to end: two agents built from the same seeds, in one process and in two, end bit-identical."""
import math
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from phc_b200 import _lib
from phc_b200.learning.networks import round4

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CS_SLOTS, SUMSQ_SLOTS, STAT_SLOTS = 8, 8, 8          # slots that launches of these reductions rotate through


def lib():
    return _lib.load()


def rnd(g, *shape, mean=0.0):
    return torch.randn(*shape, device=DEV, generator=g) + mean


# ---------------------------------------------------------------------------------------------------------------------------
# phc_colsum_group
# ---------------------------------------------------------------------------------------------------------------------------
def colsum_in_order(X, M, N):
    """colsum_group_kernel's order restated in fp32 (alpha = 1): rows are cut into chunks of rows = max(256, round_up_64(ceil(M / 32)));
    in a chunk, row lane ry (0..7) adds rows ry, ry + 8, ... one after the other; the 8 lanes are added in order, then the chunks in
    order.  Zero rows pad the last chunk (x + 0 == x)."""
    rows = max(256, -(-(-(-M // 32)) // 64) * 64)
    chunks = -(-M // rows)
    Xp = torch.zeros(chunks * rows, N, device=DEV)
    Xp[:M] = X[:M, :N]
    total = torch.zeros(N, device=DEV)
    for rc in range(chunks):
        lanes = Xp[rc * rows:(rc + 1) * rows].view(rows // 8, 8, N)
        acc = torch.zeros(8, N, device=DEV)
        for i in range(rows // 8):
            acc = acc + lanes[i]
        t = torch.zeros(N, device=DEV)
        for ry in range(8):
            t = t + acc[ry]
        total = total + t
    return total


def colsum_group(items):
    """items: [(X, M, N, out)]: out[n] += sum_m X[m, n], one launch"""
    arr = (_lib.PhcColsumDesc * len(items))(*[_lib.PhcColsumDesc(X.data_ptr(), X.stride(0), M, N, 1.0, out.data_ptr()) for X, M, N, out in items])
    _lib.check(lib().phc_colsum_group(arr, len(items), None), "phc_colsum_group")


COLSUM_SHAPES = [(100, 1), (1000, 130), (8193, 934), (16384, 1024), (2047, 513)]


def test_colsum_group_is_the_fixed_order_fp32_sum():
    g = torch.Generator(device=DEV).manual_seed(1)
    items, exp = [], []
    for M, N in COLSUM_SHAPES:
        X = torch.zeros(M, round4(N), device=DEV)
        X[:, :N] = rnd(g, M, N, mean=0.3)
        out0 = rnd(g, N)
        items.append((X, M, N, out0.clone()))
        exp.append(out0 + colsum_in_order(X, M, N))
    colsum_group(items)
    torch.cuda.synchronize()
    for (X, M, N, out), e in zip(items, exp):
        assert torch.equal(out, e), (M, N, float((out - e).abs().max()))


def test_colsum_group_result_does_not_depend_on_group_mates_or_slot():
    g = torch.Generator(device=DEV).manual_seed(2)
    mats = []
    for M, N in COLSUM_SHAPES:
        X = torch.zeros(M, round4(N), device=DEV)
        X[:, :N] = rnd(g, M, N)
        mats.append((X, M, N))
    alone = []
    for X, M, N in mats:
        out = torch.zeros(N, device=DEV)
        colsum_group([(X, M, N, out)])
        alone.append(out)
    for rep in range(CS_SLOTS + 3):                          # every slot reused, group order rotated
        order = mats[rep % len(mats):] + mats[:rep % len(mats)]
        outs = [torch.zeros(N, device=DEV) for _, _, N in order]
        colsum_group([(X, M, N, o) for (X, M, N), o in zip(order, outs)])
        torch.cuda.synchronize()
        for (X, M, N), o in zip(order, outs):
            ref = alone[[id(m[0]) for m in mats].index(id(X))]
            assert torch.equal(o, ref), (rep, M, N)


# ---------------------------------------------------------------------------------------------------------------------------
# RunningMeanStd: phc_rms_update / phc_rms_apply_update, and phc_adv_norm
# ---------------------------------------------------------------------------------------------------------------------------
RMS_N = [2, 1023, 1024, 1025, 32 * 1024, 32 * 1024 + 1, 100000]


def rms_reference(x, mean, var, count):
    """running_mean_std.py:56-68 in fp64"""
    xd = x.double()
    n = xd.shape[0]
    bm, bv = xd.mean(0), xd.var(0, unbiased=True)
    delta, tot = bm - mean, count + n
    new_mean = mean + delta * n / tot
    m2 = var * count + bv * n + delta * delta * count * n / tot
    return new_mean, m2 / tot, tot


def nan_workspace(d):
    nbytes = int(lib().phc_rms_workspace_bytes(d))
    assert nbytes % 8 == 0
    return torch.full((nbytes // 8,), float("nan"), dtype=torch.float64, device=DEV)


@pytest.mark.parametrize("path", ["update_scalar", "apply_update_vec4", "apply_update_vec2", "apply_update_scalar"])
@pytest.mark.parametrize("n", RMS_N)
def test_running_mean_std_statistics_repeat_and_match_fp64(n, path):
    d = 37
    ld = {"apply_update_vec4": 40, "apply_update_vec2": 38, "apply_update_scalar": 37, "update_scalar": 37}[path]  # picks the kernel
    g = torch.Generator(device=DEV).manual_seed(n)
    x = torch.zeros(n, ld, device=DEV)
    x[:, :d] = rnd(g, n, d, mean=0.5) * 2.0
    y = torch.zeros(n, ld, device=DEV)
    mean0 = torch.rand(d, dtype=torch.float64, device=DEV, generator=g) * 0.1
    var0 = 1.0 + torch.rand(d, dtype=torch.float64, device=DEV, generator=g)
    runs = []
    for _ in range(3):
        mean, var, count = mean0.clone(), var0.clone(), torch.full((1,), 1e-4, dtype=torch.float64, device=DEV)
        ws = nan_workspace(d)
        if path == "update_scalar":
            rc = lib().phc_rms_update(x.data_ptr(), ld, n, d, mean.data_ptr(), var.data_ptr(), count.data_ptr(), ws.data_ptr(), None, None)
        else:
            rc = lib().phc_rms_apply_update(x.data_ptr(), ld, n, d, mean0.data_ptr(), var0.data_ptr(), 1e-5, y.data_ptr(), ld, None,
                                            mean.data_ptr(), var.data_ptr(), count.data_ptr(), ws.data_ptr(), None)
        _lib.check(rc, path)
        torch.cuda.synchronize()
        runs.append((mean, var, count, y.clone()))
    for m, v, c, yy in runs[1:]:
        assert torch.equal(m, runs[0][0]) and torch.equal(v, runs[0][1]) and torch.equal(c, runs[0][2]) and torch.equal(yy, runs[0][3])
    em, ev, ec = rms_reference(x[:, :d], mean0, var0, 1e-4)
    m, v, c, _ = runs[0]
    assert torch.isfinite(m).all() and torch.isfinite(v).all()
    assert float(c) == ec
    assert torch.allclose(m, em, rtol=1e-12, atol=1e-13), float((m - em).abs().max())
    assert torch.allclose(v, ev, rtol=1e-11, atol=0), float(((v - ev) / ev).abs().max())


@pytest.mark.parametrize("n", [2, 1023, 1025, 100000, 132 * 2 * 1024 + 7])
def test_advantage_normalisation_repeats_and_matches_fp64(n):
    g = torch.Generator(device=DEV).manual_seed(n)
    ret, val = rnd(g, n, mean=1.0), rnd(g, n)
    outs = []
    for _ in range(3):
        ws = torch.full((int(lib().phc_adv_norm_workspace_bytes(n)) // 8,), float("nan"), dtype=torch.float64, device=DEV)
        adv = torch.empty(n, device=DEV)
        _lib.check(lib().phc_adv_norm(ret.data_ptr(), val.data_ptr(), n, 1, adv.data_ptr(), ws.data_ptr(), None), "phc_adv_norm")
        torch.cuda.synchronize()
        outs.append(adv)
    assert all(torch.equal(o, outs[0]) for o in outs[1:])
    a = (ret - val).double()                                    # adv = ret - val is stored in fp32 first
    exp = (a - a.mean()) / (a.std() + 1e-8)
    assert torch.allclose(outs[0].double(), exp, rtol=2e-6, atol=2e-6), float((outs[0].double() - exp).abs().max())


# ---------------------------------------------------------------------------------------------------------------------------
# phc_grad_sumsq
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [0, 1, 255, 1056 * 256 + 1, 3_000_001])
def test_grad_sumsq_repeats_and_matches_fp64(n):
    g = torch.Generator(device=DEV).manual_seed(n + 1)
    buf = rnd(g, max(n, 1))                                     # (a valid pointer also for n = 0)
    x = buf[:n]
    outs = []
    for _ in range(SUMSQ_SLOTS + 3):
        out = torch.full((1,), float("nan"), dtype=torch.float64, device=DEV)
        _lib.check(lib().phc_grad_sumsq(buf.data_ptr(), n, out.data_ptr(), None), "phc_grad_sumsq")
        outs.append(out)
    torch.cuda.synchronize()
    assert all(torch.equal(o, outs[0]) for o in outs[1:])
    exp = float((x.double() ** 2).sum())
    got = float(outs[0])
    assert got == exp if n == 0 else abs(got - exp) <= 1e-12 * exp, (got, exp)


# ---------------------------------------------------------------------------------------------------------------------------
# loss statistics (ppo_update.cu): per-block partials added in block order by the last block
# ---------------------------------------------------------------------------------------------------------------------------
def loss_stat_launches(g):
    """every stat-producing entry point at bench-like sizes, each adding into its own slots of one caller-zeroed float[16]"""
    n, A, na, nd, d = 16384, 69, 8192, 4096, 1960
    mu = rnd(g, n, 72)
    t = dict(mu=mu, logstd=rnd(g, A) * 0.01, actions=mu[:, :A] + rnd(g, n, A), onlp=0.5 * A * (1.0 + math.log(2 * math.pi)) + 0.3 * rnd(g, n),
             adv=rnd(g, n), omu=mu[:, :A] + 0.1 * rnd(g, n, A), osig=1.0 + 0.1 * rnd(g, n, A).abs(), v=rnd(g, n), ret=rnd(g, n), logit=rnd(g, na + nd),
             gp=rnd(g, nd, d), w=rnd(g, 1024, d), idx=torch.randperm(n, device=DEV, generator=g))
    t["dmu"], t["dv"], t["dl"], t["y"] = torch.zeros(n, 72, device=DEV), torch.zeros(n, device=DEV), torch.zeros(na + nd, device=DEV), torch.zeros(1024, d, device=DEV)
    L = lib()

    def run(stats, gp):
        s = stats.data_ptr()
        _lib.check(L.phc_ppo_actor_grad(t["mu"].data_ptr(), 72, t["logstd"].data_ptr(), t["actions"].data_ptr(), t["onlp"].data_ptr(), t["adv"].data_ptr(),
                                        t["omu"].data_ptr(), t["osig"].data_ptr(), n, A, 0.2, 10.0, 1.0 / n, t["dmu"].data_ptr(), 72, s, None))
        _lib.check(L.phc_ppo_critic_grad(t["v"].data_ptr(), 1, t["ret"].data_ptr(), n, 5.0, 1.0 / n, t["dv"].data_ptr(), 1, s, None))
        _lib.check(L.phc_disc_logit_grad(t["logit"].data_ptr(), 1, na, nd, 5.0, t["dl"].data_ptr(), 1, s, None))
        _lib.check(L.phc_scale_sumsq(gp.data_ptr(), d, nd, d, 0.5, stats[10:].data_ptr(), None))
        _lib.check(L.phc_axpy2d(t["w"].data_ptr(), d, t["y"].data_ptr(), d, 1, d, 0.1, stats[11:].data_ptr(), None))
        _lib.check(L.phc_axpy2d(t["w"].data_ptr(), d, t["y"].data_ptr(), d, 1024, d, 0.1, stats[12:].data_ptr(), None))
        _lib.check(L.phc_ppo_grads_gather(t["mu"].data_ptr(), 72, t["logstd"].data_ptr(), t["actions"].data_ptr(), t["onlp"].data_ptr(), t["adv"].data_ptr(),
                                          t["omu"].data_ptr(), t["osig"].data_ptr(), t["v"].data_ptr(), 1, t["ret"].data_ptr(), t["idx"].data_ptr(), n, A,
                                          0.2, 10.0, 5.0, 1.0 / n, t["dmu"].data_ptr(), 72, t["dv"].data_ptr(), 1, stats[16:].data_ptr(), None))
    return t, run


def test_loss_statistics_repeat_bit_for_bit():
    """The same inputs launched again give the same statistics, bit for bit (they used to be float atomics in block order)."""
    g = torch.Generator(device=DEV).manual_seed(3)
    t, run = loss_stat_launches(g)
    results = []
    for _ in range(2 * STAT_SLOTS + 4):
        stats = torch.zeros(32, device=DEV)
        gp = t["gp"].clone()
        run(stats, gp)
        results.append(stats)
    torch.cuda.synchronize()
    for i, s in enumerate(results[1:]):
        diff = (s != results[0]).nonzero().flatten().tolist()
        assert not diff, f"launch {i + 1}: statistics {diff} differ from the first launch"
    s = results[0].double().cpu()
    # the sums themselves: plain fp64 restatements of what is summed
    d = t["v"].double() - t["ret"].double()
    assert math.isclose(s[5], float((d * d).sum()), rel_tol=1e-5)
    x = t["logit"].double()
    sp = torch.nn.functional.softplus(x)
    assert math.isclose(s[6], float(sp[:8192].sum()), rel_tol=1e-5) and math.isclose(s[7], float((sp[8192:] - x[8192:]).sum()), rel_tol=1e-5)
    assert s[8] == float((x[:8192] < 0).sum()) and s[9] == float((x[8192:] > 0).sum())
    assert math.isclose(s[10], float((t["gp"].double() ** 2).sum()), rel_tol=1e-5)
    assert math.isclose(s[11], float((t["w"][0].double() ** 2).sum()), rel_tol=1e-5)
    assert math.isclose(s[12], float((t["w"].double() ** 2).sum()), rel_tol=1e-5)
    dg = t["v"].double() - t["ret"][t["idx"]].double()       # phc_ppo_grads_gather: minibatch row i pairs with dataset row idx[i]
    assert math.isclose(s[21], float((dg * dg).sum()), rel_tol=1e-5)


def test_loss_statistics_accumulate_into_the_caller_buffer():
    """stats are caller-zeroed and accumulating: two launches into the same buffer give exactly twice one launch"""
    g = torch.Generator(device=DEV).manual_seed(4)
    t, run = loss_stat_launches(g)
    once, twice = torch.zeros(32, device=DEV), torch.zeros(32, device=DEV)
    run(once, t["gp"].clone())
    run(twice, t["gp"].clone())
    run(twice, t["gp"].clone())
    torch.cuda.synchronize()
    assert torch.equal(twice, 2 * once)


# ---------------------------------------------------------------------------------------------------------------------------
# training end to end
# ---------------------------------------------------------------------------------------------------------------------------
def train_snapshot(network, monkeypatch, record):
    """build an agent from fixed seeds at the default minibatch geometry (512 envs x horizon 32 = one 16384-row minibatch, 4096 AMP
    rows), train 2 epochs, and return every piece of state a run leaves behind"""
    from phc_b200 import synthetic as syn
    from phc_b200.env.humanoid_im import HumanoidIm, RLGPUEnv
    from phc_b200.learning.amp_agent import AMPAgent
    from phc_b200.learning.networks import MLPEngine
    orig = MLPEngine.run_group

    def run_group(self, descs):
        record.append([(d.C, d.M, d.N, d.ldc, d.accumulate, d.k_splits) for d in descs if d is not None])
        return orig(self, descs)
    monkeypatch.setattr(MLPEngine, "run_group", run_group)
    torch.manual_seed(0)
    motion = syn.make_motions(512, seed=0)
    task = HumanoidIm({"env": {"num_envs": 512}, "motion_data": motion, "seed": 0})
    agent = AMPAgent("repro", {"vec_env": RLGPUEnv(task), "seed": 0, "mini_epochs": 2, "network": network})
    agent.obs = agent.env_reset()
    agent._init_amp_demo_buf()
    for _ in range(2):
        result = agent.train_epoch()
    torch.cuda.synchronize()
    snap = {"params": agent.model.params, "exp_avg": agent.exp_avg, "exp_avg_sq": agent.exp_avg_sq}
    for name in ("running_mean_std", "value_mean_std", "_amp_input_mean_std"):
        rms = getattr(agent, name)
        if rms is not None:
            for k in ("running_mean", "running_var", "count"):
                snap[f"{name}.{k}"] = getattr(rms, k)
    for k, v in agent.experience_buffer.items():
        if torch.is_tensor(v):
            snap[f"experience.{k}"] = v
    for k, v in result.items():
        if torch.is_tensor(v):
            snap[f"result.{k}"] = v
    snap = {k: v.detach().clone() for k, v in snap.items()}
    losses = agent.train_result_dict()
    monkeypatch.undo()
    del agent, task
    torch.cuda.empty_cache()
    return snap, losses


@pytest.mark.parametrize("network", [
    {"mlp": {"units": [1024, 512], "activation": "relu"}, "disc": {"units": [1024, 512], "activation": "relu"}},
    {"mlp": {"units": [1024, 1024, 512], "activation": "silu"}, "disc": {"units": [1024, 512], "activation": "relu"}},
], ids=["relu", "silu3"])
def test_two_agents_with_the_same_seeds_train_bit_identically(network, monkeypatch):
    rec_a, rec_b = [], []
    a, la = train_snapshot(network, monkeypatch, rec_a)
    b, lb = train_snapshot(network, monkeypatch, rec_b)
    # the ordered paths were really taken: split-K, and two accumulating problems on one C (gradient penalty + regular dW)
    assert any(ks > 1 for launch in rec_a for (_, _, _, _, acc, ks) in launch)
    acc_cs = [[c for (c, m, n, ld, acc, ks) in launch if acc and m > 0 and n > 0] for launch in rec_a]
    assert any(len(cs) > len(set(cs)) for cs in acc_cs), "no launch had two accumulating problems on the same C"
    assert set(a) == set(b)
    differ = [k for k in sorted(a) if not torch.equal(a[k], b[k])]
    assert not differ, f"state differs between two identically seeded runs: {differ}"
    assert la == lb, {k: (la[k], lb[k]) for k in la if la[k] != lb[k]}


def test_two_bench_processes_dump_identical_outputs(tmp_path):
    """bench.py --dump-outputs in two processes: every array byte for byte the same"""
    dirs = []
    for i in range(2):
        out = tmp_path / f"run{i}"
        cmd = [sys.executable, os.path.join(ROOT, "bench.py"), "--gpus", "1", "--num-envs", "1024", "--steps", "1", "--warmup", "1", "--no-cpu-baseline",
               "--no-e2e", "--no-points", "--no-extras", "--dump-outputs", str(out)]
        r = subprocess.run(cmd, cwd=str(tmp_path), capture_output=True, text=True, timeout=1200)
        assert r.returncode == 0, r.stderr[-4000:]
        dirs.append(out)
    names = sorted(os.listdir(dirs[0]))
    assert names and names == sorted(os.listdir(dirs[1]))
    assert "losses.npy" in names and "params.npy" in names
    differ = [n for n in names if (dirs[0] / n).read_bytes() != (dirs[1] / n).read_bytes()]
    assert not differ, {n: float(np.abs(np.load(dirs[0] / n).astype(np.float64) - np.load(dirs[1] / n).astype(np.float64)).max()) for n in differ}
