"""model_lib.ControlNet.cldm.cldm — the dotted path the reference's YAML `target:` strings name
(models/cldm_v15_reference_only_pose.yaml:2,22,40,57; models/cldm_v15_reference_only.yaml for stage 1).  The
classes are the H100 drop-ins."""
from magicdance_b200.dropin.cldm import (  # noqa: F401
    ControlLDMReferenceOnly, ControlLDMReferenceOnlyPose, ControlNet, ControlNetReferenceOnly, ControlledUnetModelAttn,
    ControlledUnetModelAttnPose)
from magicdance_b200.dropin.ddpm import LatentDiffusionReferenceOnly  # noqa: F401
from magicdance_b200.dropin.ddim import DDIMSampler_ReferenceOnly  # noqa: F401
