"""Drop-in hook: make the reference's own entry point (`python phc/run_hydra.py ...`, unchanged) pick up the phc_b200 classes.

`run_hydra.py` runs as a script, so `phc/` is `sys.path[0]`: it imports `learning.amp_agent`, `learning.im_amp`, ... and
`env.tasks.*` by those short names (run_hydra.py:57-66), while `parse_task.py:29-38` imports `phc.env.tasks.*` and resolves the
task class with `eval(args.task)` (parse_task.py:60).  A plain PYTHONPATH override cannot shadow those modules (the script
directory wins), so the replacement is installed from a `sitecustomize.py` (or a `.pth` line `import phc_b200.dropin as d;
d.install_on_import()`) that runs before the script's imports:

    # sitecustomize.py, anywhere on PYTHONPATH
    import phc_b200.dropin
    phc_b200.dropin.install_on_import()

`install_on_import()` registers a meta-path hook that waits for the reference modules to be imported and then rebinds
  phc.env.tasks.humanoid_im.HumanoidIm / env.tasks.humanoid_im.HumanoidIm   -> phc_b200.env.humanoid_im.HumanoidIm
  phc.env.tasks.humanoid_im_mcp.HumanoidImMCP (+ short name)                 -> phc_b200.env.humanoid_im_mcp.HumanoidImMCP
  phc.env.tasks.humanoid_im_getup.HumanoidImGetup (+ short name)            -> phc_b200.env.humanoid_im_getup.HumanoidImGetup
  phc.env.tasks.humanoid_im_mcp_getup.HumanoidImMCPGetup (+ short name)      -> phc_b200.env.humanoid_im_getup.HumanoidImMCPGetup
  learning.amp_agent.AMPAgent / phc.learning.amp_agent.AMPAgent              -> phc_b200.learning.amp_agent.AMPAgent
  learning.im_amp.IMAmpAgent / phc.learning.im_amp.IMAmpAgent                -> phc_b200.learning.im_amp.IMAmpAgent
so `IMAmpAgent(AMPAgent)` (learning/im_amp.py) and `eval("HumanoidIm")` resolve to the phc_b200 implementations.  `install()` does
the same rebinding immediately for modules that are already imported (what the tests use).  Isaac Gym stays the reference's: the
rebinding keeps the original task class as `_RefHumanoidIm` and registers a backend factory that instantiates it as the owner of
gym / sim / assets (phc_b200/env/backends.py); a backend can also be handed over directly as cfg["sim_backend"] (INTEGRATION.md A).
"""
from __future__ import annotations

import importlib.abc
import sys
from typing import Dict, Tuple

# reference module (both spellings) -> {attribute: "our.module:Class"}
_TARGETS: Dict[Tuple[str, ...], Dict[str, str]] = {
    ("phc.env.tasks.humanoid_im", "env.tasks.humanoid_im"): {"HumanoidIm": "phc_b200.env.humanoid_im:HumanoidIm"},
    ("phc.env.tasks.humanoid_im_mcp", "env.tasks.humanoid_im_mcp"): {"HumanoidImMCP": "phc_b200.env.humanoid_im_mcp:HumanoidImMCP"},
    # the get-up schedule (env_im_getup_mcp.yaml, env_im_x_getup_mcp.yaml, env_im_x_pnn.yaml)
    ("phc.env.tasks.humanoid_im_getup", "env.tasks.humanoid_im_getup"): {"HumanoidImGetup": "phc_b200.env.humanoid_im_getup:HumanoidImGetup"},
    ("phc.env.tasks.humanoid_im_mcp_getup", "env.tasks.humanoid_im_mcp_getup"): {
        "HumanoidImMCPGetup": "phc_b200.env.humanoid_im_getup:HumanoidImMCPGetup"},
    ("phc.learning.amp_agent", "learning.amp_agent"): {"AMPAgent": "phc_b200.learning.amp_agent:AMPAgent"},
    # run_hydra.py:259 registers `im_amp.IMAmpAgent` as the 'im_amp' algorithm: the mirror keeps eval / _post_step_eval / get_action
    ("phc.learning.im_amp", "learning.im_amp"): {"IMAmpAgent": "phc_b200.learning.im_amp:IMAmpAgent"},
}


def _resolve(spec: str):
    mod, _, name = spec.partition(":")
    return getattr(importlib.import_module(mod), name)


def _rebind(module) -> int:
    n = 0
    for names, attrs in _TARGETS.items():
        if module.__name__ in names:
            for attr, spec in attrs.items():
                new = _resolve(spec)
                old = getattr(module, attr, None)
                if old is not None and old is not new:
                    setattr(module, "_Ref" + attr, old)          # the reference's own class stays reachable (physics owner, see below)
                setattr(module, attr, new)
                n += 1
            if "HumanoidIm" in attrs and getattr(module, "_RefHumanoidIm", None) is not None:
                _register_isaacgym_factory(module._RefHumanoidIm)
    return n


def _register_isaacgym_factory(ref_cls) -> None:
    """parse_task.py:60 constructs the task with `eval(args.task)(cfg=cfg, sim_params=..., physics_engine=..., device_type=...,
    device_id=..., headless=...)` and nothing else: the phc_b200 HumanoidIm then needs a simulator backend from somewhere.  This factory
    builds the reference's ORIGINAL task class with the same arguments -- it owns gym, sim, the actors and the asset data -- and wraps
    it as the backend (phc_b200.env.backends.IsaacGymBackend); its observation / reward / reset code is never called."""
    from .env import backends

    def factory(cfg, sim_params, physics_engine, device_type, device_id, headless):
        return backends.IsaacGymBackend(ref_cls(cfg=cfg, sim_params=sim_params, physics_engine=physics_engine, device_type=device_type,
                                                device_id=device_id, headless=headless))
    backends.register_backend_factory(factory)


def install() -> int:
    """Rebind the classes in every reference module that is already imported; returns the number of rebinds."""
    n = 0
    for names in _TARGETS:
        for name in names:
            m = sys.modules.get(name)
            if m is not None:
                n += _rebind(m)
    return n


class _Hook(importlib.abc.MetaPathFinder):
    """Wraps the loader of the watched modules so the rebinding happens right after the module body ran."""

    def find_spec(self, fullname, path, target=None):
        if not any(fullname in names for names in _TARGETS):
            return None
        for finder in sys.meta_path:
            if finder is self or not hasattr(finder, "find_spec"):
                continue
            spec = finder.find_spec(fullname, path, target)
            if spec is not None and spec.loader is not None and hasattr(spec.loader, "exec_module"):
                inner = spec.loader.exec_module

                def exec_module(module, _inner=inner):
                    _inner(module)
                    _rebind(module)
                spec.loader.exec_module = exec_module
                return spec
        return None


def install_on_import() -> None:
    if not any(isinstance(f, _Hook) for f in sys.meta_path):
        sys.meta_path.insert(0, _Hook())
    install()
