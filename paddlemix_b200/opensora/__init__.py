"""Host-side mirror of Open-Sora's STDiT2 (ppdiffusers/examples/Open-Sora/models/stdit/stdit2.py) and its
text-to-video sampling: the IDDPM scheduler, the video VAE decode and the pipeline around them."""
from .iddpm import IDDPM, space_timesteps  # noqa: F401
from .pipeline import OpenSoraPipeline  # noqa: F401
from .stdit2 import STDiT2, STDiT2Config  # noqa: F401
from .vae import VideoAutoencoderKL  # noqa: F401
