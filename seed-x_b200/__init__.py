"""seedx-b200: H100-native (sm_90a) inference kernels + host for the SEED-X ViT -> LLaMA -> SDXL pipeline."""
from ._version import __version__  # noqa: F401
