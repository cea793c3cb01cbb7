"""q / k / v quantization hooks on attention modules (the reference's modeling/ package); transformers is imported on use"""
from .kvcache import *  # noqa: F401,F403
from .attention import *  # noqa: F401,F403
