"""CPU-side checks of the drop-in boundary: the C-ABI library builds, loads and exports every symbol that
include/phc_b200.h declares; the product package never touches the oracle; ops refuse CPU tensors (no fallback)."""
import os
import re

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def header_symbols():
    src = open(os.path.join(ROOT, "include", "phc_b200.h")).read()
    return sorted(set(re.findall(r"PHC_API\s+[\w\s\*]+?\b(phc_\w+)\s*\(", src)))


def test_library_exports_every_declared_symbol():
    from phc_b200 import _lib, build
    build.build()
    lib = _lib.load()
    syms = header_symbols()
    assert len(syms) >= 15
    for s in syms:
        assert hasattr(lib, s), f"{s} declared in include/phc_b200.h but not exported"
        assert s in _lib.SIGNATURES, f"{s} has no ctypes signature in phc_b200/_lib.py"
    assert set(_lib.SIGNATURES) == set(syms)
    assert lib.phc_compiled_sm() == 90
    assert lib.phc_self_obs_dim(24, _lib.PHC_FLAG_ROOT_HEIGHT_OBS) == 358
    assert lib.phc_task_obs_dim(24, 1) == 576
    assert lib.phc_amp_obs_dim(19, 4, _lib.PHC_FLAG_ROOT_HEIGHT_OBS) == 196
    assert lib.phc_self_obs_dim(20, _lib.PHC_FLAG_ROOT_HEIGHT_OBS) + lib.phc_task_obs_dim(20, 1) == 778   # H1 row of SURVEY.md


def test_ctypes_struct_layout_matches_header_order():
    """Field order of the ctypes mirrors follows the header (guards against silent ABI drift)."""
    from phc_b200 import _lib
    src = open(os.path.join(ROOT, "include", "phc_b200.h")).read()
    for cname, cls in (("PhcMotionLib", _lib.PhcMotionLib), ("PhcMotionStateOut", _lib.PhcMotionStateOut), ("PhcStepArgs", _lib.PhcStepArgs),
                       ("PhcGemmDesc", _lib.PhcGemmDesc)):
        body = re.search(r"typedef struct %s \{(.*?)\} %s;" % (cname, cname), src, re.S).group(1)
        body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
        names = []
        for decl in body.split(";"):
            decl = decl.strip()
            if not decl:
                continue
            for part in decl.split(","):
                m = re.search(r"(\w+)\s*(\[\w+\])*\s*$", part.strip())
                names.append(m.group(1))
        assert names == [f[0] for f in cls._fields_], cname


def test_product_never_imports_oracle():
    pkg = os.path.join(ROOT, "phc_b200")
    for dp, _, fs in os.walk(pkg):
        for f in fs:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                txt = open(os.path.join(dp, f)).read()
                assert not re.search(r"^\s*(from|import)\s+oracle\b", txt, re.M), f"{f} imports the oracle"
                assert "phc_oracle" not in txt, f"{f} references the oracle"
                assert "/root/reference" not in txt, f"{f} reads the reference checkout"


def test_ops_refuse_cpu_tensors():
    from phc_b200 import ops, synthetic as syn
    m = syn.make_motions(2, seed=0, min_frames=5, max_frames=6)
    with pytest.raises(ops.PhcError):
        ops.pack_motion_lib(m.gts, m.grs, m.gvs, m.gavs, m.lrs, m.dvs, m.lengths, m.num_frames, m.dts, m.length_starts)
    fd, v, r, nv = syn.make_rollout(4, 3)
    with pytest.raises(ops.PhcError):
        ops.gae(fd, v, r, nv, 0.99, 0.95)


def test_synthetic_generator_is_deterministic_and_unit():
    from phc_b200 import synthetic as syn
    a, b = syn.make_motions(3, seed=4), syn.make_motions(3, seed=4)
    assert torch.equal(a.gts, b.gts) and torch.equal(a.grs, b.grs)
    assert torch.allclose(a.grs.norm(dim=-1), torch.ones(a.grs.shape[:-1]), atol=1e-5)
    assert a.length_starts[0] == 0 and int(a.num_frames.sum()) == a.gts.shape[0]
    assert torch.allclose(a.lengths, a.dts * (a.num_frames - 1))
    assert len(syn.SMPL_DOF_SUBSET) == 57 and syn.SMPL_DOF_SUBSET[9] == 12


def test_header_is_plain_c_and_c_host_runs(tmp_path):
    """The boundary is a C ABI: the header compiles as pedantic C99, a C program (examples/c_host.c) links against the library and
    runs its no-device entry points, and the struct sizes the C compiler sees equal the ctypes mirrors'."""
    import ctypes as C
    import shutil
    import subprocess
    from phc_b200 import _lib, build
    gcc = shutil.which("gcc")
    if gcc is None:
        pytest.skip("gcc not available")
    lib_path = build.build()
    inc = os.path.join(ROOT, "include")
    r = subprocess.run([gcc, "-fsyntax-only", "-x", "c", "-std=c99", "-Wall", "-Wextra", "-pedantic", "-Werror", os.path.join(inc, "phc_b200.h")],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    exe = str(tmp_path / "c_host")
    r = subprocess.run([gcc, "-std=c99", "-Wall", "-I" + inc, os.path.join(ROOT, "examples", "c_host.c"), "-o", exe,
                        "-L" + os.path.dirname(lib_path), "-lphc_b200", "-Wl,-rpath," + os.path.dirname(lib_path)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    r = subprocess.run([exe], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    m = re.search(r"sizeof\(PhcStepArgs\) = (\d+), sizeof\(PhcMotionLib\) = (\d+)", r.stdout)
    assert (int(m.group(1)), int(m.group(2))) == (C.sizeof(_lib.PhcStepArgs), C.sizeof(_lib.PhcMotionLib))
    assert "phc_env_step(NULL) -> -1" in r.stdout
