"""Frozen-network loaders used on the env side of the hierarchical configs.

Mirrors phc/learning/network_loader.py:53-73 (`load_pnn`): build the K primitive columns from a PNN checkpoint's
`a2c_network.pnn.actors.K.*` entries and freeze them.  The primitives run through the same tensor-core GEMM engine as the
learner (MLPEngine); nothing here falls back to torch matmuls.
"""
from __future__ import annotations

from typing import Dict, Optional

import torch

from .networks import AMPNetwork, MLPEngine, round4


class FrozenPNN:
    """The K primitive actors of a trained PNN, evaluated together on a batch of normalised observations."""

    def __init__(self, net: AMPNetwork, engine: MLPEngine):
        self.net, self.engine = net, engine
        self.num_prim, self.action_dim = net.num_prim, net.action_dim
        self._x: Dict[int, torch.Tensor] = {}
        self._out: Dict[int, torch.Tensor] = {}

    def input_buffer(self, batch: int) -> torch.Tensor:
        """Zero-padded [batch, in_pad] buffer the caller writes the (normalised) observation into."""
        x = self._x.get(batch)
        if x is None:
            x = torch.zeros(batch, round4(self.net.pnn_actors[0].in_dim), dtype=torch.float32, device=self.net.device)
            self._x[batch] = x
        return x

    def forward_all(self, x: torch.Tensor) -> torch.Tensor:
        """PNN.forward(x, idx=-1) without laterals (pnn.py:99-107): every column's output, stacked [K, B, ld]."""
        B = x.shape[0]
        ws0 = self.engine.workspace("pnn0", self.net.pnn_actors[0], B)
        ld = ws0["out"].stride(0)
        out = self._out.get(B)
        if out is None:
            out = torch.zeros(self.num_prim, B, ld, dtype=torch.float32, device=self.net.device)
            self._out[B] = out
        for k, col in enumerate(self.net.pnn_actors):
            ws = self.engine.workspace(f"pnn{k}", col, B)
            ws["out"] = out[k]                       # the column writes straight into its slab of the stacked result
            self.engine.forward(col, x, ws)
        return out


def load_pnn(checkpoint: Dict, num_prim: int, has_lateral: bool = False, activation: str = "relu", device="cuda:0",
             backend: Optional[str] = None) -> FrozenPNN:
    if has_lateral:
        raise NotImplementedError("lateral PNN connections are not used by any shipped config (has_lateral: False)")
    sd = checkpoint["model"]
    biases = sorted((k for k in sd if k.startswith("a2c_network.pnn.actors.0.") and k.endswith("bias")),
                    key=lambda k: int(k.split(".")[-2]))
    widths = [sd[k].shape[0] for k in biases]
    obs_dim = sd["a2c_network.pnn.actors.0.0.weight"].shape[1]
    net = AMPNetwork(obs_dim, widths[-1], 4, units=widths[:-1], disc_units=(4,), activation=activation, device=device,
                     kind="amp_pnn", num_prim=num_prim, training_prim=0)
    for col in net.pnn_actors:
        for l in col.layers:
            net.set_layer(l, sd[f"a2c_network.{l.name}.weight"], sd[f"a2c_network.{l.name}.bias"])
    net.refresh_images()
    eng = MLPEngine(net, backend)
    if eng.backend == "tc5":
        net.refresh_split()
    return FrozenPNN(net, eng)
