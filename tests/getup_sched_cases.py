"""Test infrastructure: replay of tests/golden/getup_sched.npz (make_golden_getup_sched.py, the unmodified reference's get-up schedule)
through any implementation.  `step_cases` / `select_cases` yield the golden's inputs and expected outputs in order; the state each case
carries over (counters, bank, simulator tensors, AMP windows) is the caller's."""
import os

import numpy as np
import torch

from phc_b200 import synthetic as syn

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
STEPS, RESETS = 3, 4
CONFIGS = {"24": "getup.npz", "52": "getup_smplx.npz"}


def load(name):
    z = np.load(os.path.join(GOLDEN, name))
    return {k: torch.from_numpy(z[k]) for k in z.files}


def source(J):
    g = load(CONFIGS[J])
    m = syn.MotionData(**{k: g["tab_" + k] for k in syn.MotionData.__dataclass_fields__})
    st = syn.EnvState(**{k: g["in_" + k].clone() for k in syn.EnvState.__dataclass_fields__})
    return g, m, st


def prefixed(g, p):
    return {k[len(p):]: v for k, v in g.items() if k.startswith(p)}
