"""adanerf_b200 -- H100-native (sm_90a) AdaNeRF inference renderer: hand-written CUDA kernels behind a
C ABI (include/adanerf_b200.h), driven from Python through ctypes.  No CPU fallback."""
from ._lib import AdnError, LIB_PATH, load_library  # noqa: F401
from .renderer import Renderer, make_scene, render  # noqa: F401
from .onnx_weights import read_onnx_initializers  # noqa: F401
from .adapter import B200Inference  # noqa: F401
from .tiling import gather_bands, render_frame_distributed, row_bands  # noqa: F401
