"""mpi_operator_b200 — a Hopper-native (H100, sm_90a) MPIJob launcher + collective runtime.

Same user-facing API as kubeflow/mpi-operator (MPIJob ``kubeflow.org/v2beta1``,
Python SDK, status/conditions, metrics), rebuilt for one 8-GPU NVSwitch box:
a local controller/daemon instead of a Kubernetes operator, processes instead
of pods, and a first-party collective runtime (``libb200mpi.so``: hand-written
sm_90a peer-memory / NVLS kernels) instead of the NCCL+Horovod stack the
reference merely launches.  See DESIGN.md and SURVEY.md.
"""
from .version import __version__  # noqa: F401
