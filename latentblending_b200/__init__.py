"""latentblending_b200: H100-native (sm_90a) backend of latentblending's branch-tree
denoising hot path (BlendingEngine.run_transition -> DiffusersHolder.run_diffusion_sd_xl).
Same public names as the reference package (latentblending/__init__.py:1-3)."""
from .utils import add_frames_linear_interp, interpolate_linear, interpolate_spherical  # noqa: F401
from .blending_engine import BlendingEngine  # noqa: F401
from .diffusers_holder import DiffusersHolder  # noqa: F401
from .pipe import SyntheticSDXLPipe  # noqa: F401
