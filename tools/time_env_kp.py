"""CUDA-event timing of the fused env-step launch with the keypoint-only task observation (env.obs_v: 7) against the v6 launch of
the same generic instantiation path, in one process (PHC_ENV_FAST=0 keeps the v6 launch off the steady-state specialisations,
which have no keypoint form).  bench.env_kernel_roofline times each; the two observation versions alternate, twice per size.
    python tools/time_env_kp.py [iters]

Algorithmic bytes per env step: v6 9384 (bench.ALGO_BYTES_PER_ENV_STEP, with a 3736 B observation row); the keypoint row is
358 + 216 = 574 floats = 2296 B, so 9384 - 3736 + 2296 = 7944 B."""
import json
import os
import subprocess
import sys

os.environ["PHC_ENV_FAST"] = "0"          # read once, at the first launch of the process
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

import bench  # noqa: E402
from phc_b200 import synthetic as syn  # noqa: E402
from phc_b200.env.humanoid_im import HumanoidIm  # noqa: E402

KP_ALGO_BYTES = bench.ALGO_BYTES_PER_ENV_STEP - 3736 + 2296


def main():
    iters = int(sys.argv[1]) if len(sys.argv) > 1 else 60
    peak, src = bench.measured_peak_gbs()
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    out = {"gpu": torch.cuda.get_device_name(0), "nvidia_smi": q.stdout.strip().splitlines()[:1], "iters": iters, "runs": []}
    for n in (4096, 16384):
        motion = syn.make_motions(n, seed=0)
        tasks = {}
        for v in (7, 6):
            t = HumanoidIm({"env": {"num_envs": n, "obs_v": v}, "motion_data": motion, "seed": 0})
            t.reset()
            tasks[v] = t
        assert tasks[7].get_obs_size() == 574 and tasks[6].get_obs_size() == 934
        for rep in range(2):
            for v in (7, 6):
                r = bench.env_kernel_roofline(tasks[v], peak, src, iters=iters,
                                              algo_bytes=KP_ALGO_BYTES if v == 7 else bench.ALGO_BYTES_PER_ENV_STEP,
                                              kernel="phc::env_step_kernel<1, 24, false, false, %s>" % ("true" if v == 7 else "false"))
                out["runs"].append({"num_envs": n, "obs_v": v, "rep": rep, "algo_bytes_per_env": KP_ALGO_BYTES if v == 7 else bench.ALGO_BYTES_PER_ENV_STEP,
                                    **{k: r[k] for k in ("kernel_us", "kernel_us_event_pair", "achieved", "frac", "differential_used")}})
        del tasks
        torch.cuda.empty_cache()
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
