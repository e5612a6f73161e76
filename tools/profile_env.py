"""Small driver for ncu: runs the fused env-step kernel (4096 envs, one clip per env, L2 flushed between launches),
one GAE pass and one PPO/AMP minibatch.  Used only for profiler captures (never for bench numbers)."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from phc_b200 import synthetic as syn
from phc_b200.env.humanoid_im import HumanoidIm, RLGPUEnv

n = int(sys.argv[1]) if len(sys.argv) > 1 else 4096
iters = int(sys.argv[2]) if len(sys.argv) > 2 else 12
with_update = len(sys.argv) > 3 and sys.argv[3] == "update"
task = HumanoidIm({"env": {"num_envs": n}, "motion_data": syn.make_motions(n, seed=0), "seed": 0})
task.reset()
flush = torch.empty(64 * 1024 * 1024, device="cuda")
for i in range(iters):
    task.sim.simulate(None)
    flush.fill_(float(i))
    task.post_physics_step()
torch.cuda.synchronize()
if with_update:
    from phc_b200.learning.amp_agent import AMPAgent
    agent = AMPAgent("prof", {"vec_env": RLGPUEnv(task), "seed": 0})
    agent.obs = agent.env_reset()
    agent._init_amp_demo_buf()
    agent.config["mini_epochs"] = 1
    agent.mini_epochs_num = 1
    agent.train_epoch()
    torch.cuda.synchronize()
print("done")
