"""CPU checks of the get-up schedule's host side: the drop-in rebinds the reference's HumanoidImGetup / HumanoidImMCPGetup (both import
spellings, on a stand-in of the reference's package layout), IsaacGymBackend.generate_fall_states runs the reference procedure
(humanoid_im_getup.py:82-125) on a stub task that records its calls, SyntheticSim's bank is seeded and deterministic, and the C ABI
declares the flags and entry points."""
import os
import sys
import types

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

STANDIN = {
    "phc/__init__.py": "",
    "phc/env/__init__.py": "",
    "phc/env/tasks/__init__.py": "",
    "phc/env/tasks/humanoid_im.py": "class HumanoidIm:\n    pass\n",
    "phc/env/tasks/humanoid_im_mcp.py": "import phc.env.tasks.humanoid_im as humanoid_im\n\nclass HumanoidImMCP(humanoid_im.HumanoidIm):\n    pass\n",
    "phc/env/tasks/humanoid_im_getup.py": "import phc.env.tasks.humanoid_im as humanoid_im\n\nclass HumanoidImGetup(humanoid_im.HumanoidIm):\n    pass\n",
    "phc/env/tasks/humanoid_im_mcp_getup.py": ("from phc.env.tasks.humanoid_im_getup import HumanoidImGetup\n"
                                               "from phc.env.tasks.humanoid_im_mcp import HumanoidImMCP\n\n"
                                               "class HumanoidImMCPGetup(HumanoidImGetup, HumanoidImMCP):\n    pass\n"),
}


@pytest.fixture
def standin(tmp_path):
    for rel, body in STANDIN.items():
        p = tmp_path / rel
        p.parent.mkdir(parents=True, exist_ok=True)
        p.write_text(body)
    saved_path, saved_mods, saved_meta = list(sys.path), set(sys.modules), list(sys.meta_path)
    sys.path[:0] = [str(tmp_path), str(tmp_path / "phc")]
    yield
    sys.path[:] = saved_path
    sys.meta_path[:] = saved_meta
    for k in set(sys.modules) - saved_mods:
        del sys.modules[k]
    from phc_b200.env import backends
    backends.register_backend_factory(None)


@pytest.mark.parametrize("spelling", ["phc.env.tasks", "env.tasks"])
def test_dropin_rebinds_the_getup_tasks(standin, spelling):
    import importlib
    from phc_b200 import dropin
    from phc_b200.env.humanoid_im_getup import HumanoidImGetup, HumanoidImMCPGetup
    dropin.install_on_import()
    g = importlib.import_module(f"{spelling}.humanoid_im_getup")
    mg = importlib.import_module(f"{spelling}.humanoid_im_mcp_getup")
    assert g.HumanoidImGetup is HumanoidImGetup and mg.HumanoidImMCPGetup is HumanoidImMCPGetup
    assert g._RefHumanoidImGetup.__name__ == "HumanoidImGetup"      # the reference's class stays reachable
    assert eval("HumanoidImMCPGetup", vars(mg)) is HumanoidImMCPGetup   # parse_task.py:60 resolves `task:` with eval
    assert issubclass(HumanoidImMCPGetup, HumanoidImGetup)
    assert "HumanoidImMCPGetup" in dropin.__doc__ and "HumanoidImGetup" in dropin.__doc__


def test_getup_task_signatures_match_the_reference():
    import inspect
    from phc_b200.env.humanoid_im_getup import HumanoidImGetup, HumanoidImMCPGetup
    base = ["cfg", "sim_params", "physics_engine", "device_type", "device_id", "headless"]
    assert list(inspect.signature(HumanoidImGetup.__init__).parameters)[1:] == base
    assert list(inspect.signature(HumanoidImMCPGetup.__init__).parameters)[1:] == base + ["pnn_checkpoint"]
    for m in ("update_getup_schedule", "set_getup_probs", "resample_motions", "reset", "_generate_fall_states"):
        assert callable(getattr(HumanoidImGetup, m))


class _Gym:
    def __init__(self, log):
        self.log = log

    def set_actor_root_state_tensor_indexed(self, sim, root, ids, n):
        self.log.append(("set_root", n))

    def set_dof_state_tensor_indexed(self, sim, dof, ids, n):
        self.log.append(("set_dof", n, float(dof.abs().sum())))

    def simulate(self, sim):
        self.log.append(("simulate",))


class _StubTask:
    """What IsaacGymBackend reads from the reference task, recording every call."""

    def __init__(self, n=5, d=6):
        self.log = []
        self.num_envs, self.device = n, torch.device("cpu")
        self.gym, self.sim = _Gym(self.log), object()
        self._root_states = torch.randn(n, 13)
        self._humanoid_root_states = self._root_states            # a view in Isaac Gym; the same tensor here
        self._initial_humanoid_root_states = torch.randn(n, 13)
        self._humanoid_actor_ids = torch.arange(n, dtype=torch.int32)
        self._dof_state = torch.randn(n * d, 2)
        self._dof_pos = torch.randn(n, d)
        self._rigid_body_state_reshaped = torch.zeros(n, 24, 13)
        self.dof_force_tensor = torch.zeros(n, d)
        self._d = d

    def get_dof_action_size(self):
        return self._d

    def pre_physics_step(self, actions):
        self.log.append(("pre_physics_step", tuple(actions.shape), float(actions.abs().max())))

    def render(self):
        self.log.append(("render",))

    def _refresh_sim_tensors(self):
        self.log.append(("refresh",))
        self._humanoid_root_states[:, 7:13] = 5.0                  # the settled state still moves: the bank zeroes it


def test_isaacgym_backend_generate_fall_states_runs_the_reference_procedure(monkeypatch):
    gymtorch = types.SimpleNamespace(unwrap_tensor=lambda t: t)
    monkeypatch.setitem(sys.modules, "isaacgym", types.SimpleNamespace(gymtorch=gymtorch))
    monkeypatch.setitem(sys.modules, "isaacgym.gymtorch", gymtorch)
    from phc_b200.env.backends import IsaacGymBackend
    t = _StubTask()
    init = t._initial_humanoid_root_states.clone()
    root, dof_pos = IsaacGymBackend(t).generate_fall_states()
    kinds = [e[0] for e in t.log]
    assert kinds[:3] == ["set_root", "set_dof", "pre_physics_step"]
    assert t.log[1][2] == 0.0                                       # the dof state is zeroed
    assert t.log[2][1] == (5, 6) and t.log[2][2] <= 0.5
    assert kinds.count("simulate") == 150 and kinds.count("render") == 150 and kinds[-1] == "refresh"
    assert torch.allclose(root[:, 3:7].norm(dim=-1), torch.ones(5))   # random unit root rotations
    assert torch.equal(root[:, :3], init[:, :3])                    # at the initial root positions
    assert (root[:, 7:13] == 0).all()
    assert torch.equal(dof_pos, t._dof_pos)


def test_synthetic_fall_bank_is_seeded_and_deterministic():
    from phc_b200 import synthetic as syn
    from phc_b200.env.humanoid_im import SyntheticSim
    m = syn.make_motions(3, seed=0, min_frames=20, max_frames=40)
    a = SyntheticSim(m, 7, "cpu").generate_fall_states()
    b = SyntheticSim(m, 7, "cpu").generate_fall_states()
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
    root, dof = a
    assert root.shape == (7, 13) and dof.shape == (7, 69)
    assert torch.allclose(root[:, 3:7].norm(dim=-1), torch.ones(7)) and (root[:, 7:13] == 0).all()


def test_header_declares_the_getup_abi():
    from phc_b200 import _lib
    src = open(os.path.join(ROOT, "include", "phc_b200.h")).read()
    assert "#define PHC_FLAG_RECOVERY (1u << 14)" in src and _lib.PHC_FLAG_RECOVERY == 1 << 14
    assert "#define PHC_FLAG_AMP_CURRENT (1u << 15)" in src and _lib.PHC_FLAG_AMP_CURRENT == 1 << 15
    assert _lib.PhcStepArgs._fields_[-1][0] == "recovery_counter"      # appended: the earlier fields keep their offsets
    for name in ("phc_getup_reset", "phc_amp_ring_fill"):
        assert name in _lib.SIGNATURES and f"PHC_API int {name}(" in src
