"""Import shim that lets the UNMODIFIED reference (ZhengyiLuo/PHC at /root/reference)
be imported in the build container, where isaacgym / rl_games / smpl_sim / hydra are absent.

Test infrastructure only: used by tests/golden/make_golden.py to generate the committed
golden vectors.  /root/reference does not exist on the GPU box, so nothing under the
`-m gpu` tests, smoke() or bench.py imports this module.

How: `isaacgym.torch_utils` is mapped to the reference's own isaacgym-free copy
(phc/utils/isaacgym_torch_utils.py); every other missing third-party module becomes a stub
whose attributes are MagicMocks (only class bodies/base classes touch them at import time).
"""
import importlib
import importlib.abc
import importlib.machinery
import sys
import types
from unittest.mock import MagicMock

REF_ROOT = "/root/reference"

_STUB_ROOTS = (
    "isaacgym", "rl_games", "smpl_sim", "easydict", "hydra", "omegaconf", "gym", "tensorboardX", "joblib",
    "open3d", "lxml", "skimage", "termcolor", "imageio", "matplotlib", "wandb", "ipdb", "mujoco",
    "cv2", "smplx", "torchgeometry", "vtk", "pyvista", "sklearn_extra", "gymnasium", "chumpy",
    "stl", "trimesh", "mujoco_py", "pytorch3d", "numpy_stl", "gdown", "autograd", "numba",
)


class _StubModule(types.ModuleType):
    def __getattr__(self, name):
        if name.startswith("__"):
            raise AttributeError(name)
        if name[:1].isupper():
            # CamelCase attributes are used as base classes (rl_games A2CAgent, PPODataset ...):
            # give them a real, empty class so the reference's subclasses keep their own methods.
            m = type(name, (object,), {"__init__": lambda self, *a, **k: None})
        else:
            # lower-case attributes may be sub-modules (`from rl_games.algos_torch import torch_ext`)
            # or functions; a callable stub module serves both.
            full = f"{self.__name__}.{name}"
            m = sys.modules.get(full)
            if m is None:
                m = _StubModule(full)
                m.__path__ = []
                sys.modules[full] = m
        setattr(self, name, m)
        return m

    def __call__(self, *a, **k):
        return MagicMock(name=self.__name__ + "()")


class ObjectFactory:
    """rl_games==1.1.4 rl_games/common/object_factory.py (third-party, absent here): a name -> builder registry.
    The reference's network_builder.BaseNetwork registers activations / initialisers in it and `create`s them by name."""

    def __init__(self):
        self._builders = {}

    def register_builder(self, name, builder):
        self._builders[name] = builder

    def set_builders(self, builders):
        self._builders = builders

    def create(self, name, **kwargs):
        builder = self._builders.get(name)
        if not builder:
            raise ValueError(name)
        return builder(**kwargs)


class _StubFinder(importlib.abc.MetaPathFinder, importlib.abc.Loader):
    def find_spec(self, fullname, path, target=None):
        root = fullname.split(".")[0]
        if root in _STUB_ROOTS and fullname != "isaacgym.torch_utils":
            return importlib.machinery.ModuleSpec(fullname, self, is_package=True)
        return None

    def create_module(self, spec):
        m = _StubModule(spec.name)
        m.__path__ = []
        return m

    def exec_module(self, module):
        pass


def install():
    if REF_ROOT not in sys.path:
        sys.path.insert(0, REF_ROOT)
        sys.path.insert(1, REF_ROOT + "/poselib")
        sys.path.insert(2, REF_ROOT + "/phc")  # run_hydra.py runs with phc/ as sys.path[0]
    if not any(isinstance(f, _StubFinder) for f in sys.meta_path):
        sys.meta_path.append(_StubFinder())
    import torch  # noqa
    real = importlib.import_module("phc.utils.isaacgym_torch_utils")
    sys.modules["isaacgym.torch_utils"] = real
    ig = importlib.import_module("isaacgym")
    ig.torch_utils = real
    of = importlib.import_module("rl_games.common.object_factory")
    of.ObjectFactory = ObjectFactory
    # the reference sets the legacy TorchScript executor (phc/env/tasks/base_task.py:95-96)
    torch._C._jit_set_profiling_mode(False)
    torch._C._jit_set_profiling_executor(False)
    return real
