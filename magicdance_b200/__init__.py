"""magicdance_b200 — H100 (sm_90a) kernels and host schedule for MagicPose's DDIM denoising hot path.

`ops` binds the C ABI (include/magicdance_b200.h); `engine` schedules the reference's three
networks over it.  Importing the package does not touch CUDA; using it without the compiled
library or without an sm_90 GPU raises (there is no fallback path).
"""
from . import ops  # noqa: F401

__all__ = ["ops"]
