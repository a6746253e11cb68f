"""ObsPointNet parameter container (same module tree / state_dict keys as
neupan/blocks/obs_point_net.py:25-49 so the reference's checkpoints load unchanged).

On the hot path the network is evaluated by the fused CUDA DUNE kernel
(neupan_b200/csrc/dune_tc_kernel.cuh) from these parameters; ``forward`` is the plain torch
definition of the same function, kept for API compatibility (e.g. DUNE training).
"""
import torch
import torch.nn as nn


class ObsPointNet(nn.Module):
    def __init__(self, input_dim: int = 2, output_dim: int = 4) -> None:
        super().__init__()
        hidden = 32
        layers = [nn.Linear(input_dim, hidden), nn.LayerNorm(hidden), nn.Tanh()]
        for _ in range(2):
            layers += [nn.Linear(hidden, hidden), nn.ReLU(), nn.Linear(hidden, hidden), nn.LayerNorm(hidden), nn.Tanh()]
        layers += [nn.Linear(hidden, output_dim), nn.ReLU()]
        self.MLP = nn.Sequential(*layers)

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        return self.MLP(x)
