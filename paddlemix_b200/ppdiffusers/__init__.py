"""Host-side mirrors of the ppdiffusers classes on the hot path (same names, signatures and error behaviour)."""
from .schedulers import EulerAncestralDiscreteScheduler, UniPCMultistepScheduler  # noqa: F401
