"""Hand-written sm_90a ops with autograd wrappers (kernels in csrc/kernels)."""
from .fused_bn import bn_act, fused_bn_available  # noqa: F401
