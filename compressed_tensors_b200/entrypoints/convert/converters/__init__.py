from .base import *  # noqa: F401,F403
from .autoawq import *  # noqa: F401,F403
from .ct_dequantizer import *  # noqa: F401,F403
from .fp8block_dequantizer import *  # noqa: F401,F403
from .modelopt_nvfp4 import *  # noqa: F401,F403
from .quantizer import *  # noqa: F401,F403
