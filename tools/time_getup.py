"""CUDA-event timing of the get-up schedule on the GPU, in one process:
  * the fused env-step launch, L2 flushed before every launch (bench.env_kernel_roofline: CUDA events, flush-only batches subtracted),
    at 4096 and 16384 envs, three launches alternating twice per size:
      plain          HumanoidIm, specialised_step False: env_step_kernel<1, 24, false, false, false, false>, the instantiation the
                     get-up step would take without its template parameter;
      recovery_idle  HumanoidImGetup with every counter at 0: env_step_kernel<1, 24, true, false, false, true> (the flag selects this
                     instantiation; with no env recovering it does the plain step's work plus the counter read / write);
      recovery_half  the same launch with half of the envs recovering;
  * the whole reset() at 4096 envs with 10 % and with 0 % of the envs resetting (what every rollout step pays: argsort of N uniforms,
    the single-CTA selection, the state copy, the observation-only launch, the demo / ring-fill launches), HumanoidImGetup against
    HumanoidIm, median of CUDA-event pairs around the call (host launch overhead included).
Prints the card name and power limit with the numbers.
    python tools/time_getup.py [iters]"""
import json
import os
import statistics
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

import bench  # noqa: E402
from phc_b200 import synthetic as syn  # noqa: E402
from phc_b200.env.humanoid_im import HumanoidIm  # noqa: E402
from phc_b200.env.humanoid_im_getup import HumanoidImGetup  # noqa: E402

GETUP_ENV = {"recoveryEpisodeProb": 0.5, "recoverySteps": 90, "fallInitProb": 0.3, "getup_schedule": True}


def main():
    iters = int(sys.argv[1]) if len(sys.argv) > 1 else 60
    peak, src = bench.measured_peak_gbs()
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    out = {"gpu": torch.cuda.get_device_name(0), "nvidia_smi": q.stdout.strip().splitlines()[:1], "iters": iters, "step": [], "reset": [],
           "reset_timing": "CUDA events around reset(mask) (host launch overhead included), median of %d" % iters}
    for n in (4096, 16384):
        motion = syn.make_motions(n, seed=0)
        plain = HumanoidIm({"env": {"num_envs": n}, "motion_data": motion, "seed": 0, "specialised_step": False})
        getup = HumanoidImGetup({"env": dict(GETUP_ENV, num_envs=n), "motion_data": motion, "seed": 0, "specialised_step": False})
        for t in (plain, getup):
            t.reset()
        kernels = {"plain": "phc::env_step_kernel<1, 24, false, false, false, false>",
                   "recovery_idle": "phc::env_step_kernel<1, 24, true, false, false, true>",
                   "recovery_half": "phc::env_step_kernel<1, 24, true, false, false, true>"}
        for rep in range(2):
            for name in ("plain", "recovery_idle", "recovery_half"):
                if name != "plain":          # counters held for the whole measurement (each launch decrements them by one)
                    getup._recovery_counter.zero_()
                    if name == "recovery_half":
                        getup._recovery_counter[: n // 2] = 1 << 30
                t = plain if name == "plain" else getup
                r = bench.env_kernel_roofline(t, peak, src, iters=iters, kernel=kernels[name])
                out["step"].append({"num_envs": n, "launch": name, "rep": rep, "kernel": kernels[name],
                                    **{k: r[k] for k in ("kernel_us", "kernel_us_event_pair")}})
        if n == 4096:
            for frac in (0.1, 0.0):
                for name, t in (("HumanoidImGetup", getup), ("HumanoidIm", plain)):
                    g = torch.Generator(device=t.device).manual_seed(0)
                    times = []
                    for i in range(iters + 5):
                        mask = (torch.rand(n, generator=g, device=t.device) < frac).long()
                        t._terminate_buf.copy_((torch.rand(n, generator=g, device=t.device) < 0.5).long())
                        torch.cuda.synchronize()
                        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                        e0.record()
                        t.reset(mask)
                        e1.record()
                        torch.cuda.synchronize()
                        if i >= 5:
                            times.append(e0.elapsed_time(e1) * 1e3)
                    out["reset"].append({"task": name, "num_envs": n, "resetting": frac, "median_us": statistics.median(times),
                                         "min_us": min(times)})
        del plain, getup
        torch.cuda.empty_cache()
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
