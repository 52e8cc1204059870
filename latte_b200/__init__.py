"""latte_b200 — H100-native (sm_90a) implementation of the Latte denoising hot path behind the
reference's own module surface.  See DESIGN.md / INTEGRATION.md."""
from .latte import Latte, Latte_models  # noqa: F401
from .latte_img import LatteIMG, LatteIMG_models  # noqa: F401
from .latte_t2v import LatteT2V  # noqa: F401
from .vae import AutoencoderKL, AutoencoderKLTemporalDecoder  # noqa: F401
from .t5 import T5EncoderModel  # noqa: F401
from . import ops  # noqa: F401

__all__ = ["Latte", "LatteIMG", "LatteT2V", "AutoencoderKL", "AutoencoderKLTemporalDecoder", "T5EncoderModel", "Latte_models", "LatteIMG_models", "ops"]
