"""The drop-in contract of SURVEY.md section 8(b): every method / buffer name the reference's callers use exists on the mirrors with a
compatible signature (against the reference's parameter lists, tests/golden/dropin_surface.json, make_golden.gen_dropin_surface), and
phc_b200.dropin rebinds the classes in modules with the reference's names (both import spellings run_hydra.py uses).  The rebinding
tests build a stand-in of the reference's package layout in a temporary directory: the hook looks only at module and class names.
CPU only: nothing is instantiated."""
import inspect
import json
import os
import sys

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))

TASK_METHODS = ["step", "reset", "_compute_observations", "_compute_task_obs", "_compute_reward", "_compute_reset", "_compute_humanoid_obs",
                "_compute_amp_observations", "fetch_amp_obs_demo", "get_obs_size", "get_task_obs_size", "get_self_obs_size", "get_num_amp_obs",
                "get_action_size", "resample_motions", "get_task_obs_size_detail", "get_running_mean_size", "post_physics_step"]
AGENT_METHODS = ["train", "train_epoch", "play_steps", "calc_gradients", "discount_values", "_calc_advs", "_preproc_obs", "_disc_loss",
                 "_calc_amp_rewards", "_combine_rewards", "get_stats_weights", "set_stats_weights", "get_full_state_weights",
                 "set_full_state_weights", "restore", "save", "env_reset", "env_step", "get_action_values", "_eval_critic", "prepare_dataset",
                 "pre_epoch", "_update_amp_demos", "_init_amp_demo_buf", "_store_replay_amp_obs", "set_eval", "set_train"]


def test_mirror_surface_is_complete():
    from phc_b200.env.humanoid_im import HumanoidIm
    from phc_b200.env.humanoid_im_mcp import HumanoidImMCP
    from phc_b200.learning.amp_agent import AMPAgent
    assert [m for m in TASK_METHODS if not callable(getattr(HumanoidIm, m, None))] == []
    assert [m for m in AGENT_METHODS if not callable(getattr(AMPAgent, m, None))] == []
    assert issubclass(HumanoidImMCP, HumanoidIm)
    assert list(inspect.signature(HumanoidIm.__init__).parameters)[1:] == ["cfg", "sim_params", "physics_engine", "device_type", "device_id", "headless"]
    assert list(inspect.signature(AMPAgent.__init__).parameters)[1:] == ["base_name", "config"]


# module files of the stand-in reference: the layout and class hierarchy of phc/env/tasks and phc/learning
STANDIN = {
    "phc/__init__.py": "",
    "phc/env/__init__.py": "",
    "phc/env/tasks/__init__.py": "",
    "phc/env/tasks/humanoid_im.py": "class HumanoidIm:\n    pass\n",
    "phc/env/tasks/humanoid_im_mcp.py": "import phc.env.tasks.humanoid_im as humanoid_im\n\nclass HumanoidImMCP(humanoid_im.HumanoidIm):\n    pass\n",
    "phc/learning/__init__.py": "",
    "phc/learning/amp_agent.py": "class AMPAgent:\n    pass\n",
    "phc/learning/im_amp.py": "import phc.learning.amp_agent as amp_agent\n\nclass IMAmpAgent(amp_agent.AMPAgent):\n    pass\n",
}


def _write_standin(root):
    for rel, body in STANDIN.items():
        path = os.path.join(root, rel)
        os.makedirs(os.path.dirname(path), exist_ok=True)
        with open(path, "w") as f:
            f.write(body)
    return [str(root), os.path.join(str(root), "phc")]         # `phc.x` and, as when run_hydra.py runs as a script, `x`


@pytest.fixture
def ref_modules(tmp_path):
    paths = _write_standin(tmp_path)
    saved_path, saved_mods = list(sys.path), set(sys.modules)
    sys.path[:0] = paths
    import importlib
    try:
        yield (importlib.import_module("phc.env.tasks.humanoid_im"), importlib.import_module("phc.learning.amp_agent"),
               importlib.import_module("learning.amp_agent"), importlib.import_module("phc.env.tasks.humanoid_im_mcp"))
    finally:
        sys.path[:] = saved_path
        for m in set(sys.modules) - saved_mods:
            if m.split(".")[0] in ("phc", "env", "learning"):     # the stand-in's modules only
                del sys.modules[m]


def test_signatures_match_the_reference():
    from phc_b200.env.humanoid_im import HumanoidIm
    from phc_b200.learning.amp_agent import AMPAgent
    with open(os.path.join(HERE, "golden", "dropin_surface.json")) as f:
        ref = json.load(f)                      # "Class.method" -> [[name, positional, has_default], ...] of the reference
    assert len(ref) == 18
    # the reference defines these itself (not only through rl_games / Isaac Gym bases): positional parameters must line up
    for key, rp in ref.items():
        cls_name, n = key.split(".")
        ours = {"HumanoidIm": HumanoidIm, "AMPAgent": AMPAgent}[cls_name]
        op = [p for p in inspect.signature(getattr(ours, n)).parameters.values()]
        r_req = [name for name, positional, has_default in rp if positional and not has_default]
        o_names = [p.name for p in op if p.kind in (p.POSITIONAL_ONLY, p.POSITIONAL_OR_KEYWORD)]
        assert o_names[:len(r_req)] == r_req or len(o_names) >= len(r_req), f"{cls_name}.{n}: reference {r_req} vs ours {o_names}"
        o_req = [p.name for p in op if p.default is p.empty and p.kind in (p.POSITIONAL_ONLY, p.POSITIONAL_OR_KEYWORD)]
        assert len(o_req) <= len([name for name, positional, _ in rp if positional]), \
            f"{cls_name}.{n}: ours requires {o_req}, the reference passes at most {[name for name, _, _ in rp]}"


def test_dropin_rebinds_both_import_spellings(ref_modules):
    from phc_b200 import dropin
    from phc_b200.env.humanoid_im import HumanoidIm
    from phc_b200.env.humanoid_im_mcp import HumanoidImMCP
    from phc_b200.learning.amp_agent import AMPAgent
    ref_env, ref_agent, ref_agent_short, ref_mcp = ref_modules
    saved = (ref_env.HumanoidIm, ref_agent.AMPAgent, ref_agent_short.AMPAgent, ref_mcp.HumanoidImMCP)
    try:
        assert dropin.install() >= 4
        assert ref_env.HumanoidIm is HumanoidIm and ref_mcp.HumanoidImMCP is HumanoidImMCP
        assert ref_agent.AMPAgent is AMPAgent and ref_agent_short.AMPAgent is AMPAgent
        assert eval("HumanoidIm", vars(ref_env)) is HumanoidIm          # what parse_task.py:60 does
    finally:
        ref_env.HumanoidIm, ref_agent.AMPAgent, ref_agent_short.AMPAgent, ref_mcp.HumanoidImMCP = saved


def test_install_on_import_rebinds_when_the_reference_modules_load_later(tmp_path):
    """The sitecustomize route: the hook is registered BEFORE the reference modules are imported (as when `python
    phc/run_hydra.py` starts) and rebinds the classes right after each module body ran -- checked in a fresh interpreter."""
    import subprocess
    code = r'''
import sys
sys.path[:0] = %r + [%r]
import phc_b200.dropin as d
d.install_on_import()                                     # what sitecustomize.py does
assert not any(m in sys.modules for m in ("phc.env.tasks.humanoid_im", "learning.amp_agent"))
import phc.env.tasks.humanoid_im as ref_env              # parse_task.py:29-38 spelling
import learning.amp_agent as ref_agent                   # run_hydra.py:57-64 spelling
import learning.im_amp as im_amp                          # class IMAmpAgent(amp_agent.AMPAgent)
from phc_b200.env.humanoid_im import HumanoidIm
from phc_b200.learning.amp_agent import AMPAgent
assert ref_env.HumanoidIm is HumanoidIm and eval("HumanoidIm", vars(ref_env)) is HumanoidIm
assert ref_agent.AMPAgent is AMPAgent
assert AMPAgent in im_amp.IMAmpAgent.__mro__, im_amp.IMAmpAgent.__mro__
print("OK")
''' % (_write_standin(tmp_path), os.path.dirname(HERE))
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and "OK" in r.stdout, r.stdout[-2000:] + r.stderr[-3000:]
