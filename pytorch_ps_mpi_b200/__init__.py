"""pytorch_ps_mpi_b200 — a Hopper-native parameter-server data-parallel engine.

Public surface of the reference (``/root/reference/__init__.py:1``: ``MPI_PS, Adam, SGD``) plus
``AdamW``, the coding plug-ins, the comm façade and the SPMD launcher.
"""
from . import runtime
from . import codings
from . import mpi_comms
from . import mpi_comms as comms
from . import serialization
from .codings import Coding, Identity, Cast, Scale, TopK, QSGD, Sign, SVD
from .ps import MPI_PS, Adam, AdamW, SGD, _bytes_of, find_param

__version__ = "0.1.0"
__all__ = ["MPI_PS", "Adam", "AdamW", "SGD", "Coding", "Identity", "Cast", "Scale", "TopK", "QSGD", "Sign", "SVD", "codings",
           "mpi_comms", "comms", "serialization", "runtime", "find_param", "_bytes_of"]
