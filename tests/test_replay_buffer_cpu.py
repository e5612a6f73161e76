"""ReplayBuffer (row a18) against the reference's own class: circular store, the pre-fill `% head` rule, the permutation
refresh.  tests/golden/replay.npz holds what the reference ReplayBuffer (phc/learning/replay_buffer.py) stored and sampled for the
same seeded rows and the same generator state (make_golden.gen_replay)."""
import os

import numpy as np
import torch

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "replay.npz")
SIZE, WIDTH, STORES, SAMPLES = 50, 7, [8, 8, 8, 20, 13, 50, 3], (5, 17, 30)      # make_golden.REPLAY_*


def test_store_and_sample_match_the_reference():
    from phc_b200.learning.amp_agent import ReplayBuffer
    gold = np.load(GOLDEN)
    torch.manual_seed(5)                                             # the generator state the reference buffer was built with
    ours = ReplayBuffer(SIZE, WIDTH, "cpu")
    g = torch.Generator().manual_seed(1)
    for step, n in enumerate(STORES):                                # partial fill, wrap-around, a full-size store
        ours.store(torch.randn(n, WIDTH, generator=g))
        assert [ours.get_total_count(), ours.get_buffer_size()] == gold[f"count_{step}"].tolist()
        assert torch.equal(ours.data, torch.from_numpy(gold[f"data_{step}"])), f"store {step}"
        for k in SAMPLES:                                            # crosses the permutation refresh several times
            idx = ours.sample_indices(k)
            assert torch.equal(ours.data[idx], torch.from_numpy(gold[f"sample_{step}_{k}"])), f"sample after store {step}"
