"""Timing of the rollout's per-step episode statistics on the GPU, in one process: phc_episode_stats alone, and the torch sequence
it replaces in the rollout (`not_dones = 1 - dones.float()`, `cur_r.add_(r).mul_(not_dones)`, `cur_l.add_(1).mul_(not_dones)`),
at 4096 and 16384 envs with 5 % of the envs done per step.  Two CUDA-event timings of each:
  * `graph`: 100 steps captured into one CUDA graph and replayed, as the rollout runs them (device time per step);
  * `eager`: `iters` back-to-back launches from Python (bound by the host's launch rate, not by the kernel).
Prints the card name and power limit with the numbers as one JSON line.
    python tools/time_episode_stats.py [iters]"""
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from phc_b200 import ops  # noqa: E402

DEV = "cuda:0"


def timed(fn, iters):
    for _ in range(20):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1000.0 / iters


def timed_graph(fn, reps=20, per_graph=100):
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(3):
            fn()
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(per_graph):
            fn()
    g.replay()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        g.replay()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1000.0 / (reps * per_graph)


def main():
    if not torch.cuda.is_available():
        raise SystemExit("time_episode_stats: no CUDA device")
    iters = int(sys.argv[1]) if len(sys.argv) > 1 else 2000
    out = {}
    for n in (4096, 16384):
        g = torch.Generator(device=DEV).manual_seed(n)
        r = torch.randn(n, device=DEV, generator=g)
        dones = (torch.rand(n, device=DEV, generator=g) < 0.05).long()
        cur_r, cur_l = torch.zeros(n, device=DEV), torch.zeros(n, device=DEV)
        mean, size = torch.zeros(2, device=DEV), torch.zeros(2, dtype=torch.int32, device=DEV)

        def kernel():
            ops.episode_stats(r, dones, cur_r, cur_l, mean, size, 100)

        def torch_pair():
            not_dones = 1.0 - dones.float()
            cur_r.add_(r).mul_(not_dones)
            cur_l.add_(1).mul_(not_dones)
        out[str(n)] = {"graph": {"episode_stats_us": round(timed_graph(kernel), 2), "torch_add_mul_us": round(timed_graph(torch_pair), 2)},
                       "eager": {"episode_stats_us": round(timed(kernel, iters), 2), "torch_add_mul_us": round(timed(torch_pair, iters), 2)}}
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    print(json.dumps({"gpu": torch.cuda.get_device_name(0), "nvidia_smi": q.stdout.strip(), "iters": iters, "per_launch": out}))


if __name__ == "__main__":
    main()
