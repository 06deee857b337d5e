"""2-layer MLP on MNIST-shaped inputs (BASELINE.json config 1: the CPU plumbing model)."""
from __future__ import annotations

import torch
import torch.nn as nn
import torch.nn.functional as F


class MLP(nn.Module):
    """``in → hidden → classes`` with ReLU.  ``first_linear`` can be swapped for the
    broadcast-fused wgmma GEMM (:class:`pytorch_ps_mpi_b200.ops.linear.BcastLinear`)."""

    def __init__(self, in_features: int = 784, hidden: int = 512, classes: int = 10, bias: bool = True):
        super().__init__()
        self.fc1 = nn.Linear(in_features, hidden, bias=bias)
        self.fc2 = nn.Linear(hidden, classes, bias=bias)

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        x = x.flatten(1)
        return self.fc2(F.relu(self.fc1(x)))


def mnist_mlp(hidden: int = 512, **kw) -> MLP:
    return MLP(784, hidden, 10, **kw)
