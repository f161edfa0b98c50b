from .controlmodel import ControlledUNetModel3D, ControlNet3D  # noqa: F401
from .denoiser import DiscreteDenoiser  # noqa: F401
from .discretizer import LegacyDDPMDiscretization  # noqa: F401
from .guiders import IdentityGuider, VanillaCFG  # noqa: F401
from .sampling import (AncestralSampler, BaseDiffusionSampler, DPMPP2MSampler, DPMPP2SAncestralSampler,  # noqa: F401
                       EDMSampler, EulerAncestralSampler, EulerEDMSampler, HeunEDMSampler, LinearMultistepSampler,
                       SingleStepDiffusionSampler)
from .wrappers import OpenAIWrapperControlLDM3D  # noqa: F401
